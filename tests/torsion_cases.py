"""Cases off ed25519's prime-order subgroup (test helper, no GPU): the 8-torsion, mixed-order points Q + T, their SEC1
encodings, curve25519 u-coordinates of small and mixed order (canonical and + p) and on the twist, and scalars around
n and 8n.

The ed25519 group is cyclic of order 8n, so k P == (k mod 8n) P for every point, while k P == (k mod n) P holds only
inside the prime-order subgroup: a kernel that reduces the scalar mod n agrees with the reference on every multiple of
G and disagrees on these points.  The arithmetic here is plain affine twisted-Edwards arithmetic on Python integers,
independent of the oracle that the tests compare against."""
import random

P = 2**255 - 19
N = 0x1000000000000000000000000000000014DEF9DEA2F79CD65812631A5CF5D3ED
D = -121665 * pow(121666, -1, P) % P
G = (0x216936D3CD6E53FEC0A4E231FDD6DC5C692CC7609525A7B2C9562D608F25D51A,
     0x6666666666666666666666666666666666666666666666666666666666666658)
O = (0, 1)
A_MONT = 486662
SQRT_M1 = pow(2, (P - 1) // 4, P)


def add(a, b):
    """a + b on -x^2 + y^2 = 1 + d x^2 y^2 (the unified affine law; complete on ed25519)."""
    (x1, y1), (x2, y2) = a, b
    t = D * x1 * x2 * y1 * y2 % P
    return ((x1 * y2 + y1 * x2) * pow(1 + t, -1, P) % P, (y1 * y2 + x1 * x2) * pow(1 - t, -1, P) % P)


def mul(k, pt):
    """k pt for any k >= 0: double-and-add over every bit of k, no reduction."""
    acc = O
    for bit in bin(k)[2:] if k else "":
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, pt)
    return acc


def small_order(pt):
    """The order of pt if it divides 8, else None."""
    for m in (1, 2, 4, 8):
        if mul(m, pt) == O:
            return m
    return None


def on_curve(pt):
    x, y = pt
    return (y * y - x * x - 1 - D * x * x * y * y) % P == 0


def sqrt(a):
    """A square root mod p (p = 5 mod 8), or None for a non-residue."""
    r = pow(a, (P + 3) // 8, P)
    if r * r % P != a % P:
        r = r * SQRT_M1 % P
    return r if r * r % P == a % P else None


def point_from_y(y):
    x = sqrt((y * y - 1) * pow(D * y * y + 1, -1, P) % P)
    return None if x is None else (x, y)


def torsion():
    """The 8 points of the 8-torsion as [(order, (x, y))]: i T8 for i = 0..7, T8 = n R for a point R whose n R has
    order 8 (8n R = O always; 4n R != O picks an R with a full torsion component)."""
    rnd = random.Random(8)
    while True:
        R = point_from_y(rnd.randrange(P))
        if R is None:
            continue
        t8 = mul(N, R)
        if mul(4, t8) != O:
            break
    pts, acc = [], O
    for i in range(8):
        pts.append(({0: 1, 4: 2, 2: 4, 6: 4}.get(i, 8), acc))
        acc = add(acc, t8)
    return pts


def mixed(seed=1):
    """[(d, order of T, d G + T)] for every torsion point T (T = O gives a prime-order point), d seeded in [1, n)."""
    rnd = random.Random(seed)
    out = []
    for order, T in torsion():
        d = rnd.randrange(1, N)
        out.append((d, order, add(mul(d, G), T)))
    return out


def points(seed=1):
    """[(order of the torsion component, point)]: the torsion itself, then the mixed-order points."""
    return torsion() + [(order, pt) for _, order, pt in mixed(seed)]


def sec1(pt, compressed):
    """BaseCurve.encode-style public keys that decodePoint takes back: 04 || x || y, or 02 / 03 (y's parity) || x."""
    x, y = pt
    if compressed:
        return bytes([3 if y & 1 else 2]) + x.to_bytes(32, "big")
    return b"\x04" + x.to_bytes(32, "big") + y.to_bytes(32, "big")


def u_of(pt):
    """The curve25519 u of an Edwards point other than O: u = (1 + y) / (1 - y)."""
    return (1 + pt[1]) * pow(1 - pt[1], -1, P) % P


def x25519_us(seed=3):
    """curve25519 u inputs as [(kind, u)]: small order (0, 1, p - 1 and the two order-8 u), mixed order, each of those
    + p (a non-canonical encoding below 2^256), and u on the twist (u^3 + A u^2 + u a non-residue)."""
    small = [0, 1, P - 1]
    for order, T in torsion():
        if order == 8 and u_of(T) not in small:
            small.append(u_of(T))
    mix = [u_of(pt) for _, _, pt in mixed(seed)]
    rnd = random.Random(seed)
    twist = []
    while len(twist) < 4:
        u = rnd.randrange(P)
        if pow((u * u * u + A_MONT * u * u + u) % P, (P - 1) // 2, P) == P - 1:
            twist.append(u)
    return ([("small", u) for u in small] + [("mixed", u) for u in mix] +
            [("plus_p", u + P) for u in small + mix] + [("twist", u) for u in twist])


def scalars(seed=4, randoms=4):
    """Scalars below 2^256 at the edges of n, 8n and the bit widths a 4-bit window schedule has to cover, plus seeded
    random values in [n, 2^256)."""
    ks = [0, 1, 7, 8, N - 1, N, N + 1, N + 7, 2 * N, 5 * N, 8 * N - 1, 8 * N, 8 * N + 1,
          2**252, 2**253 - 1, 2**253, 2**255, 2**256 - 1]
    rnd = random.Random(seed)
    return ks + [rnd.randrange(N, 2**256) for _ in range(randoms)]


def wide_scalars(seed=5):
    """Scalars of 2^256 and above, which only the host-side batch wrappers see (they reduce them before the call)."""
    rnd = random.Random(seed)
    return [2**256, 2**256 + 1, 2**256 + 8 * N - 1, 3 * 2**256 + 5 * N + 3, rnd.randrange(2**256, 2**300)]


def mul_cases():
    """(order of the point's torsion component, point, k) over every point and every scalar below 2^256."""
    return [(order, pt, k) for order, pt in points() for k in scalars()]


def verify_items(seed=6):
    """EC.verify items (e, r, s, key, u2 T == O) against the mixed-order keys d G + T.  The signature is minted from a
    nonce k with u2 = r / s chosen: u1 G + u2 (d G + T) = k G + u2 T, so it verifies exactly when u2 T = O, i.e. when
    the order of T divides u2.  Both outcomes are minted for every T of order > 1."""
    rnd = random.Random(seed)
    items = []
    for d, order, Q in mixed():
        for want in (True, False):
            if order == 1 and not want:
                continue
            k = rnd.randrange(2, N - 1)
            r = mul(k, G)[0] % N
            if want:
                u2 = order * rnd.randrange(1, N // order)
            else:
                u2 = rnd.randrange(1, N)
                u2 += 1 if u2 % order == 0 else 0
            s = r * pow(u2, -1, N) % N
            items.append(((s * k - r * d) % N, r, s, Q, u2 % order == 0))
    return items


def be(vals, ln=32):
    return b"".join(v.to_bytes(ln, "big") for v in vals)
