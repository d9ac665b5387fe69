"""Key sets and keyed verify items, with the oracle's answers for them (test helper)."""
import random

import numpy as np

CURVES = [("secp256k1", 1, 32), ("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)]
MBITS = {1: 131, 2: 255, 3: 383, 6: 520, 7: 191, 8: 223}       # bits covered by a key's windows (keyset_plan.h)
LIMBS = {1: 8, 2: 8, 3: 12, 6: 18, 7: 6, 8: 8}


def windows(cid, W):
    return MBITS[cid] // W + 1


def first_g_digit(ec, u1, gw):
    """The signed multiple of G the main loop adds first from the fixed-base table (window 0 of the odd-ified u1)."""
    n = ec.n
    sgn = 1
    if u1 % 2 == 0:
        u1, sgn = n - u1, -1
    m = (u1 - 1) // 2
    return sgn * (2 * (m & ((1 << gw) - 1)) + 1 - (1 << gw))


def minted(ec, u1, u2, Q):
    """(e, r, s) whose verify recomputes exactly (u1, u2) and is TRUE when the group law is exact; None if degenerate."""
    n = ec.n
    R = ec.g.mul(u1).add(Q.mul(u2))
    if R.is_infinity():
        return None
    r = R.x % n
    if r == 0:
        return None
    s = r * pow(u2, -1, n) % n
    return (u1 * s % n, r, s)


def adversarial_keys(ec, cid, widths):
    """[(d, Q)]: G, -G, 2G, 2^20 G and a few (2i+1) 2^(W j) G, i.e. keys whose tables share entries with G's."""
    n = ec.n
    ds = [1, n - 1, 2, 1 << 20]
    for W in widths:
        for i, j in ((0, 1), (3, 2), ((1 << (W - 1)) - 1, windows(cid, W) - 1)):
            ds.append((2 * i + 1) << (W * j))
    ds = list(dict.fromkeys(d % n for d in ds))
    return [(d, ec.g.mul(d)) for d in ds]


def adversarial_items(ec, cid, keys_d, gw, seed=11):
    """Items on keys Q = d G chosen so that the keyed main loop meets every exceptional addition: the sum is the point
    at infinity (e = -r d), u1 G = u2 Q (e = r d), and u2 Q equal to plus / minus the first fixed-base entry it adds
    (a doubling, and a cancellation followed by O + P).  The minted ones verify TRUE only if those additions are exact."""
    rnd = random.Random(seed)
    n = ec.n
    lim = 1 << (n.bit_length() - 1)
    items = []
    for k, (d, Q) in enumerate(keys_d):
        for sign in (-1, 1):
            while True:
                r, s = rnd.randrange(1, n), rnd.randrange(1, n)
                if (sign * r * d) % n < lim:
                    break
            items.append(((sign * r * d) % n, r, s, k))
        made = 0
        while made < 4:
            u1 = rnd.randrange(1, n)
            u2 = (1 if made % 2 else -1) * first_g_digit(ec, u1, gw) * pow(d, -1, n) % n
            sig = minted(ec, u1, u2, Q) if u2 else None
            if sig and sig[0] < lim:
                items.append(sig + (k,))
                made += 1
        sig = ec.sign(7 + k, d)
        items.append((7 + k, sig.r, sig.s, k))
    return items


def seeded_set(ec, ln, nkeys, nitems, seed=3, corrupt=8):
    """nkeys honest keys and nitems signatures spread over them; one item in `corrupt` is damaged in turn in e, r, s,
    the key index, or by r / s out of range."""
    rnd = random.Random(seed)
    n = ec.n
    lim = 1 << (n.bit_length() - 1)
    ds = [rnd.randrange(1, n) for _ in range(nkeys)]
    keys = [ec.g.mul(d) for d in ds]
    items = []
    for t in range(nitems):
        k = rnd.randrange(nkeys)
        e = rnd.randrange(lim)
        sig = ec.sign(e, ds[k])
        r, s = sig.r, sig.s
        if t % corrupt == 1:
            kind = (t // corrupt) % 6
            if kind == 0: e ^= 1 << rnd.randrange(lim.bit_length() - 1)
            if kind == 1: r = rnd.randrange(1, n)
            if kind == 2: s = n - s
            if kind == 3: k = (k + 1) % nkeys
            if kind == 4: r = 0
            if kind == 5: s = n
        items.append((e, r, s, k))
    return [(Q.x, Q.y) for Q in keys], items


def expected(ec, keys_xy, items):
    n = ec.n
    out = []
    for e, r, s, k in items:
        if not (1 <= r < n and 1 <= s < n):
            out.append(0)
            continue
        x, y = keys_xy[k]
        out.append(int(ec.verify(e, {"r": r, "s": s}, {"x": x, "y": y})))
    return out


def pack(ln, keys_xy, items):
    """(xy (m, 2 ln), e, r, s (n, ln), key_idx (n,)) as the C ABI takes them."""
    col = lambda vals: np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in vals), np.uint8).reshape(len(vals), ln).copy()
    xy = np.concatenate([col([k[0] for k in keys_xy]), col([k[1] for k in keys_xy])], axis=1)
    e, r, s = (col([it[j] for it in items]) for j in range(3))
    return np.ascontiguousarray(xy), e, r, s, np.array([it[3] for it in items], np.uint32)
