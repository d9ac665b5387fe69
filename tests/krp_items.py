"""getKeyRecoveryParam cases and the oracle's answers for them (test helper)."""
import random

from oracle.ref_py.bn import RefError
from oracle.ref_py.signature import Signature

NO_RECOVERY = 11
CURVES = [("secp256k1", 1, 32), ("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)]
# test/ecdsa-test.js:477-489: r = n - 1 is no x coordinate on secp256k1, and r + n >= p
NO_SQRT = (0xf75c6b18a72fabc0f0b888c3da58e004f0af1fe14f7ca5d8c897fe164925d5e9,
           0xfffffffffffffffffffffffffffffffebaaedce6af48a03bbfd25e8cd0364140,
           0x8887321be575c8095f789dd4c743dfe42c1820f9231f98a962b210e3ac2452a3)


def get_key_recovery_param(ec, e, signature, Q, enc=None):
    """EC.prototype.getKeyRecoveryParam (ec/index.js:261-278), line by line over the oracle's recoverPubKey."""
    signature = Signature(signature, enc)
    if signature.recovery_param is not None:
        return signature.recovery_param
    for i in range(4):
        try:
            q_prime = ec.recover_pub_key(e, signature, i)
        except RefError:
            continue
        if q_prime.eq(Q):
            return i
    raise RefError("Unable to find valid recovery factor")


def krp_expected(ec, item):
    """The reference's answer for one (e, r, s, qx, qy) item: j, or NO_RECOVERY where it throws."""
    e, r, s, qx, qy = item
    sg = Signature.__new__(Signature)          # r = 0 / s = 0 do not pass the {r, s} constructor
    sg.r, sg.s, sg.recovery_param = r, s, None
    try:
        return get_key_recovery_param(ec, e, sg, ec.curve.point(qx, qy))
    except RefError as ex:
        assert ex.args[0] == "Unable to find valid recovery factor"
        return NO_RECOVERY


def _has_point(ec, x):
    try:
        ec.curve.point_from_x(x, 0)
        return True
    except RefError:
        return False


def _points_from(ec, x, count):
    """The first `count` points with x coordinate >= x, parities alternating."""
    out = []
    while len(out) < count:
        try:
            out.append(ec.curve.point_from_x(x, len(out) & 1))
        except RefError:
            pass
        x += 1
    return out


def _forge(ec, R, r, e, s):
    """Q = (r mod n)^-1 (s R - e G): the key for which candidate R recovers (needs r, s != 0 mod n)."""
    n = ec.n
    ri = pow(r % n, -1, n)
    return ec.g.mul_add((n - e) * ri % n, R, s * ri % n)


def krp_items(ec, ln, seed=5, count=4):
    """(e, r, s, qx, qy) items: e as `new BN(msg)` (not reduced), r, s below 2^(8 ln), Q's coordinates below 2^(8 ln).
    Returns (items, truth): truth maps an item index to the recoveryParam the signer reported."""
    rnd = random.Random(seed)
    n, p = ec.n, ec.curve.p
    top = 1 << (8 * ln)
    mbits = min(n.bit_length() - 1, 512)             # messages _truncateToN leaves alone
    items, truth = [], {}

    def add(e, r, s, Q, dx=0, dy=0):
        if Q.is_infinity():
            return
        items.append((e, r, s, Q.x + dx, Q.y + dy))

    for t in range(count):                           # signatures from the signer, with their key and without it
        d = rnd.randrange(1, n)
        m = rnd.randrange(2**mbits)
        sig = ec.sign(m, d, canonical=bool(t & 1))
        Q = ec.g.mul(d)
        truth[len(items)] = sig.recovery_param
        add(m, sig.r, sig.s, Q)
        add(m, sig.r, sig.s, ec.g.mul(d + 1))             # the wrong key
        add(m + 1, sig.r, sig.s, Q)                       # a forged e
        add(m, sig.r, sig.s, Q, dy=1)                     # Q off the curve
        add(m, sig.r, 0, ec.g.mul((n - m) * pow(sig.r, -1, n) % n))     # s = 0 with Q = ((n - e) / r) G
        add(m, sig.r, n, ec.g.mul((n - m) * pow(sig.r, -1, n) % n))     # s = n, the same Q
        add(m, sig.r, 0, Q)                               # s = 0, another Q
        add(m, sig.r, n, Q)
        add(m, 0, sig.s, Q)                               # r = 0 and r = n: rInv = 0
        add(m, n, sig.s, Q)
        add(0, sig.r, 0, Q)                               # s = 0 and e = 0: every Q' is infinity

    # candidates with x in [n, p): r = x - n recovers through j = 2 / 3; r = x (>= n) through j = 0 / 1
    for R in _points_from(ec, n + 1, 3):
        e, s = rnd.randrange(n), rnd.randrange(1, n)
        add(e, R.x - n, s, _forge(ec, R, R.x - n, e, s))
        add(e, R.x, s, _forge(ec, R, R.x, e, s))
    # r >= p (x = r mod p) where the wire width allows it, and Q with an x coordinate >= p
    for R in _points_from(ec, 1, 2):
        e, s = rnd.randrange(n), rnd.randrange(1, n)
        if R.x + p < top:
            add(e, R.x + p, s, _forge(ec, R, R.x + p, e, s))
            u1, u2 = rnd.randrange(n), rnd.randrange(1, n)      # a signature for the key R: P = u1 G + u2 R
            P = ec.g.mul_add(u1, R, u2)
            rr = P.x
            ss = rr * pow(u2, -1, n) % n
            add(u1 * ss % n, rr, ss, R, dx=p)
    # e = 0 (mod n)
    for e in (0, n):
        R = ec.g.mul(rnd.randrange(1, n))
        s = rnd.randrange(1, n)
        add(e, R.x, s, _forge(ec, R, R.x, e, s))
    # small r: no x coordinate (on p224 a non-residue, where bn.js's Tonelli-Shanks asserts), and r + n one or not
    found = {}
    r = 1
    while len(found) < 2 and r < 4000:
        if not _has_point(ec, r):
            found.setdefault(_has_point(ec, r + n), r)
        r += 1
    Q = ec.g.mul(rnd.randrange(1, n))
    for r in found.values():
        e = rnd.randrange(1, n)
        add(e, r, 0, ec.g.mul((n - e) * pow(r, -1, n) % n))
        add(e, r, rnd.randrange(1, n), Q)
    if p == 2**256 - 2**32 - 977:                        # secp256k1
        add(NO_SQRT[0], NO_SQRT[1], NO_SQRT[2], Q)
    return items, truth
