"""EdDSA key-set cases (test helper): keys and items for the keyed bodies and entry points, and the oracle's answer for
each item.  An item is (R, S, key index, h, msg): h is hashInt(R, key bytes, msg) when msg is given, else a chosen h < n
with R minted so that the answer depends on it."""
import gzip
import json
import os
import random

import numpy as np

N = 0x1000000000000000000000000000000014DEF9DEA2F79CD65812631A5CF5D3ED
P = 2**255 - 19
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ed25519_sign_input.json.gz")
ORDER8 = "26e8958fc2b227b045c3f489f2ef98f0d5dfac05d3c63339b13802886d53fc05"
THROW = {"invalid point": 2, "Assertion failed": 5}


def windows(W):
    return -(-253 // W)


def expected(ed, R, S, A, h):
    """EDDSA.verify (eddsa/index.js:52-63) with the given h in place of hashInt, in the reference's order."""
    from oracle.ref_py.bn import RefError
    s = int.from_bytes(S, "little")
    if s >= N:
        return 0
    try:
        Rp = ed.decode_point(R)
        Ap = ed.decode_point(A)
    except RefError as ex:
        return THROW[ex.args[0]]
    return int(Rp.add(Ap.mul(h)).eq(ed.g.mul(s)))


def le(v):
    return v.to_bytes(32, "little")


def mint(ed, A, h, s):
    """R = S G - h A: the item verifies only if h A is formed exactly, torsion included."""
    Ap = ed.decode_point(A)
    return ed.encode_point(ed.g.mul(s).add(Ap.mul(h).neg()))


def throwing(ed, code, start=2):
    """The first encoding y = start, start + 1, ... whose decoding throws `code`."""
    from oracle.ref_py.bn import RefError
    y = start
    while True:
        try:
            ed.decode_point(le(y))
        except RefError as ex:
            if THROW[ex.args[0]] == code:
                return le(y)
        y += 1


def digit_patterns(W, rnd, count=3):
    """h < n whose every signed digit below the top is 0 or -2^(W-1), top digit 1."""
    K, half = windows(W), 1 << (W - 1)
    out = []
    for t in range(count):
        ds = [0 if (t == 0 or rnd.random() < 0.5) and t != 1 else -half for _ in range(K - 1)]
        out.append(sum(d << (W * j) for j, d in enumerate(ds)) + (1 << (W * (K - 1))))
    return out


def cases(ed, vectors=None, seed=7):
    """(keys, items) over every class of key the set must answer for; vectors: how many sign.input vectors (all 1024 by
    default), each valid and forged."""
    rnd = random.Random(seed)
    data = json.load(gzip.open(GOLD, "rt"))["vectors"]
    data = data if vectors is None else data[:vectors]
    keys, at = [], {}

    def key(A):
        if A not in at:
            at[A] = len(keys)
            keys.append(A)
        return at[A]

    items = []

    def signed(R, S, A, msg):
        items.append((R, S, key(A), ed.hash_int(R, A, msg), msg))

    for v in data:
        sig, pk, msg = bytes.fromhex(v["sig"]), bytes.fromhex(v["pk"]), bytes.fromhex(v["msg"])
        signed(sig[:32], sig[32:], pk, msg)
        signed(sig[:32], sig[32:], pk, msg + b"!")                     # forged
    sig, pk, msg = bytes.fromhex(data[3]["sig"]), bytes.fromhex(data[3]["pk"]), bytes.fromhex(data[3]["msg"])
    R0, S0 = sig[:32], sig[32:]
    # S >= n, also where R or the key would throw
    R2 = bytes([1] + [0] * 30 + [0x80])                                # x = 0 with the sign bit: 'invalid point'
    R5 = throwing(ed, 5)                                               # y^2 - 1 / (d y^2 + 1) not a square
    for S in (le(N), le(int.from_bytes(S0, "little") + N), le(2**256 - 1)):
        signed(R0, S, pk, msg)
        signed(R2, S, R5, msg)
    # throws: R's first, then the key's
    for R, A in ((R0, R2), (R0, R5), (R2, R5), (R5, R2), (R2, pk), (R5, pk)):
        signed(R, S0, A, msg)
    # the eight small-order keys, and full-order keys plus a torsion point of order 2, 4 or 8
    T8 = ed.decode_point(bytes.fromhex(ORDER8))
    small = [ed.encode_point(T8.mul(k)) for k in range(8)]
    mixed = [ed.encode_point(ed.g.mul(rnd.randrange(1, N)).add(T8.mul(k))) for k in (4, 2, 1, 3)]
    # non-canonical encodings y + p (y < 19): the identity, the order-4 point (0 -> p) and whichever others decode
    noncanon = [le(y + P) for y in range(19)]
    noncanon = [A for A in noncanon if expected(ed, ed.encode_point(ed.g), le(1), A, 0) in (0, 1)]
    plain = ed.encode_point(ed.g.mul(rnd.randrange(1, N)))
    for A in small + mixed + noncanon + [plain]:
        for _ in range(2):
            h, s = rnd.randrange(N), rnd.randrange(N)
            R = mint(ed, A, h, s)
            items.append((R, le(s), key(A), h, None))
            Rt = ed.encode_point(ed.decode_point(R).add(T8.mul(4)))    # R + T (order 2): FALSE
            items.append((Rt, le(s), key(A), h, None))
    # h = 0, 1, n - 1 and digits at the edges of every width
    hs = [0, 1, N - 1, N - 2, 1 << 252] + [h for W in range(4, 9) for h in digit_patterns(W, rnd)]
    for A in (plain, mixed[2], small[3]):
        for h in hs:
            s = rnd.randrange(N)
            items.append((mint(ed, A, h, s), le(s), key(A), h, None))
    # raw messages against non-canonical keys: hashInt reads the key's bytes as given.  With the order-4 key, R = r G
    # verifies only when 4 | h, which a hash over a re-encoded key breaks in 3 of 4 items.
    T4raw = le(P)
    for t in range(8):
        while True:
            r = rnd.randrange(1, N)
            R, m = ed.encode_point(ed.g.mul(r)), b"noncanonical %d" % t
            h = ed.hash_int(R, T4raw, m)
            if h % 4 == 0:
                items.append((R, le(r), key(T4raw), h, m))
                break
        R = ed.encode_point(ed.g.mul(r + 1))
        items.append((R, le(r + 1), key(le(1 + P)), ed.hash_int(R, le(1 + P), m), m))    # the identity: any h
    return keys, items


def answers(ed, keys, items):
    return [expected(ed, R, S, keys[k], h) for R, S, k, h, _ in items]


def pack(keys, items):
    """A (m, 32), R, S, h (n, 32), key_idx (n,) uint32 as the C ABI takes them."""
    rows = lambda col: np.frombuffer(b"".join(col), np.uint8).reshape(-1, 32).copy()
    A = rows(keys)
    R, S = rows([it[0] for it in items]), rows([it[1] for it in items])
    h = rows([le(it[3]) for it in items])
    idx = np.array([it[2] for it in items], np.uint32)
    return A, R, S, h, idx


def msg_items(items):
    """The indices of the items that carry a message, and their messages as (blob, n + 1 offsets)."""
    sel = [i for i, it in enumerate(items) if it[4] is not None]
    ms = [items[i][4] for i in sel]
    off = np.zeros(len(ms) + 1, np.uint64)
    off[1:] = np.cumsum([len(m) for m in ms])
    return np.array(sel, np.int64), np.frombuffer(b"".join(ms) + b"\x00", np.uint8), off
