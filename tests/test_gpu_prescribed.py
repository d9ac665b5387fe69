"""ECDSA with prescribed scalars u1 = e / s and u2 = r / s (mod n), end to end, and the 32-item prep of the
secp256k1 device-pointer call at the bench's shape.

A valid signature with chosen (u1, u2): take a nonce k, r = x(kG) mod n, d = (k - u1) / u2, Q = d G, s = r / u2,
e = u1 s; then u1 G + u2 Q = k G.  Its twin with e + 1 must come back FALSE.  The scalars sit where the recodings go
wrong: 2^k +- 1 at every window edge (the fixed-base window, the 4-bit Q windows and the keyed widths 4..8), all-ones
windows, the signed-digit carries (digit patterns 0x77..7 and 0x88..8), the odd-ification of an even u1, u1 = 0, the
largest GLV halves, and e = 2^256 - 1 with s = n - 1.  Every item goes through the batch verify, the keyed verify
at W = 4..8 with a set of the minted keys, recoverPubKey, getKeyRecoveryParam and G.mulAdd(u1, Q, u2)."""
import random

import numpy as np
import pytest

import arith_cases as ac

pytestmark = pytest.mark.gpu

CURVES = {"secp256k1": 32, "p256": 32, "p384": 48, "p521": 66, "p192": 24, "p224": 28}
SW_GW = 13               # EB_SW_GW's default: fixed-base window of the short curves
K256_GW = 20             # fixed-base window of the secp256k1 verify (GTAB_W)
KEYED_W = (4, 5, 6, 7, 8)


def scalar_values(name, rnd):
    """The u values of one curve (all in [0, n))."""
    from oracle.ref_py import curves
    n = curves.get(name).n
    bits = n.bit_length()
    vals = {1, 2, n - 1, n - 2, (n - 1) // 2, (n + 1) // 2}
    widths = ((K256_GW if name == "secp256k1" else SW_GW),) + KEYED_W
    for k in {w * j for w in widths for j in range(1, bits // w + 1) if w * j < bits}:
        vals |= {(1 << k) - 1, (1 << k) + 1}
    for w in widths:
        vals |= {((1 << (w * j)) - 1) % n for j in range(1, bits // w + 2)}
    for d in (7, 8):
        vals.add(int(("%x" % d) * ((bits + 3) // 4), 16) % n)
    if name == "secp256k1":
        vals |= set(ac.glv_cases(rnd, n_random=4000, keep=16))
    return sorted(v % n for v in vals)


class Minted:
    """Items (e, r, s, qx, qy) with e as the packed calls take it (the truncated hash), and per item the scalars
    (u1, u2), the point kG = u1 G + u2 Q and the recovery parameter of the signature."""

    def __init__(self, name):
        self.name, self.ln = name, CURVES[name]
        self.items, self.u, self.kg, self.recid = [], [], [], []

    def add(self, e, r, s, Q, u1, u2, kG, n):
        self.items.append((e, r, s, Q.get_x(), Q.get_y()))
        self.u.append((u1, u2))
        self.kg.append((kG.get_x(), kG.get_y()))
        self.recid.append((kG.get_y() & 1) | (2 if kG.get_x() != r else 0))


def mint(name, pairs, rnd, out):
    """Appends to `out` a signature for each prescribed (u1, u2), and the same signature with e + n where the wire
    width holds it."""
    from oracle.ref_py.ec import EC
    ec = EC(name)
    n, g = ec.n, ec.g
    k = rnd.randrange(2, n - 1)
    kG = g.mul(k)
    r = kG.get_x() % n
    for u1, u2 in pairs:
        if u2 == 0 or (k - u1) % n == 0:
            continue
        s = r * pow(u2, -1, n) % n
        if (2 * k + pow(s, -1, n)) % n == 0:   # the twin would land on -kG, same x
            continue
        Q = g.mul((k - u1) * pow(u2, -1, n) % n)
        e = u1 * s % n
        out.add(e, r, s, Q, u1, u2, kG, n)
        if e + n < 1 << (8 * out.ln):
            out.add(e + n, r, s, Q, u1, u2, kG, n)


def special_k256(rnd, out):
    """e = 2^256 - 1 (e mod n = 2^256 - 1 - n) with s = n - 1, i.e. s^-1 = n - 1: the prep's raw e times s^-1 at
    the top of the Montgomery multiplier's range."""
    from oracle.ref_py.ec import EC
    ec = EC("secp256k1")
    n, g = ec.n, ec.g
    for _ in range(4):
        k = rnd.randrange(2, n - 1)
        kG = g.mul(k)
        r = kG.get_x() % n
        s = n - 1
        u1, u2 = ((1 << 256) - 1 - n) * (n - 1) % n, r * (n - 1) % n
        Q = g.mul((k - u1) * pow(u2, -1, n) % n)
        out.add((1 << 256) - 1, r, s, Q, u1, u2, kG, n)


def pack(items, ln):
    e = np.frombuffer(b"".join(it[0].to_bytes(ln, "big") for it in items), np.uint8).reshape(-1, ln)
    r = np.frombuffer(b"".join(it[1].to_bytes(ln, "big") for it in items), np.uint8).reshape(-1, ln)
    s = np.frombuffer(b"".join(it[2].to_bytes(ln, "big") for it in items), np.uint8).reshape(-1, ln)
    pub = np.frombuffer(b"".join(it[3].to_bytes(ln, "big") + it[4].to_bytes(ln, "big") for it in items),
                        np.uint8).reshape(-1, 2 * ln)
    return e.copy(), r.copy(), s.copy(), pub.copy()


def minted(name, seed):
    """Every value as u1 against a random u2 and as u2 against a random u1, and u1 = 0."""
    from oracle.ref_py import curves
    rnd = random.Random(seed)
    n = curves.get(name).n
    vals = scalar_values(name, rnd)
    pairs = [(v, rnd.randrange(1, n)) for v in vals] + [(rnd.randrange(n), v) for v in vals if v]
    pairs += [(0, rnd.randrange(1, n)) for _ in range(4)]
    out = Minted(name)
    mint(name, pairs, rnd, out)
    if name == "secp256k1":
        special_k256(rnd, out)
    return out


def prescribed_items(name, seed):
    """(items, expected statuses): the minted items, then each item's twin with e + 1."""
    m = minted(name, seed)
    twins = [(it[0] + 1,) + it[1:] for it in m.items if it[0] + 1 < 1 << (8 * m.ln)]
    return m.items + twins, [1] * len(m.items) + [0] * len(twins)


_CACHE = {}


def _minted(name):
    if name not in _CACHE:
        _CACHE[name] = minted(name, 0x5CA1 + CURVES[name])
    return _CACHE[name]


@pytest.mark.parametrize("name", list(CURVES))
def test_verify_with_prescribed_scalars(native, name):
    from elliptic_b200.ec import EC
    from oracle.ref_py.ec import EC as RefEC
    m = _minted(name)
    twins = [(it[0] + 1,) + it[1:] for it in m.items if it[0] + 1 < 1 << (8 * m.ln)]
    items, expected = m.items + twins, [1] * len(m.items) + [0] * len(twins)
    st = EC(name).verify_batch_packed(*pack(items, m.ln))
    assert st.tolist() == expected, [i for i, (a, b) in enumerate(zip(st, expected)) if a != b][:20]
    # the construction agrees with the oracle (a sample: the Python verify is slow on the larger curves).  The packed
    # e is the already truncated hash, so the oracle takes it as an n-bit message
    ref = RefEC(name)
    for i in list(range(0, len(items), max(1, len(items) // 12))):
        e, r, s, qx, qy = items[i]
        got = ref.verify(e, {"r": r, "s": s}, {"x": qx, "y": qy}, msg_bit_length=ref.n.bit_length())
        assert got == bool(expected[i]), (name, i)


def test_p521_message_in_its_66_byte_encoding(native):
    """EC.verify with 66-byte messages on p521: the host keeps the top 521 of the 528 bits (ec/index.js:81-108), so
    e << 7 with junk in the 7 dropped bits must verify, and (e + 1) << 7 must not."""
    from elliptic_b200.ec import EC
    from oracle.ref_py.ec import EC as RefEC
    m = _minted("p521")
    n = ac.ORDERS["p521"]
    items = [it for it in m.items if it[0] < n]
    msgs = [((e << 7) | 0x5A).to_bytes(66, "big") for e, *_ in items] + \
           [((e + 1) << 7).to_bytes(66, "big") for e, *_ in items]
    sigs = [{"r": r, "s": s} for _, r, s, _, _ in items] * 2
    keys = [{"x": qx, "y": qy} for *_, qx, qy in items] * 2
    st = EC("p521").verify_batch(msgs, sigs, keys)
    assert st.tolist() == [1] * len(items) + [0] * len(items)
    ref = RefEC("p521")
    for i in range(0, len(msgs), len(msgs) // 8):
        assert ref.verify(msgs[i], sigs[i], keys[i]) == bool(st[i]), i


@pytest.mark.parametrize("name", list(CURVES))
def test_keyed_verify_with_prescribed_scalars(native, name):
    """The same items against a key set of the minted keys at every table width W = 4..8: the keyed windows read
    the GLV halves (secp256k1, budgeted 131 bits) or m = (u2' - 1) / 2 directly, so the window-edge scalars and the
    largest halves meet the top digits of each width."""
    from elliptic_b200.ec import EC
    m = _minted(name)
    keys = sorted({(qx, qy) for *_, qx, qy in m.items})
    where = {q: i for i, q in enumerate(keys)}
    twins = [(it[0] + 1,) + it[1:] for it in m.items if it[0] + 1 < 1 << (8 * m.ln)]
    items = m.items + twins
    expected = [1] * len(m.items) + [0] * len(twins)
    e, r, s, _ = pack(items, m.ln)
    idx = np.array([where[(it[3], it[4])] for it in items], np.uint32)
    ec = EC(name)
    for W in KEYED_W:
        with ec.key_set([{"x": x, "y": y} for x, y in keys], table_bits=W) as ks:
            assert ks.table_bits == W and (ks.status == 1).all()
            st = ks.verify_batch_packed(e, r, s, idx)
        assert st.tolist() == expected, (W, [i for i, (a, b) in enumerate(zip(st, expected)) if a != b][:20])


@pytest.mark.parametrize("name", list(CURVES))
def test_recover_and_recovery_param_with_prescribed_scalars(native, name):
    """recoverPubKey(e, (r, s), j) returns the minted Q; getKeyRecoveryParam finds j, and finds none for the e + 1
    twin.  Both run the same prep (u1 = -e / r, u2 = s / r) over the prescribed scalars' signatures."""
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    m = _minted(name)
    ec = EC(name)
    msgs = [it[0] for it in m.items]
    sigs = [{"r": it[1], "s": it[2]} for it in m.items]
    pts, st = ec.recover_pub_key_batch(msgs, sigs, m.recid)
    assert (st == nat.ST_TRUE).all()
    assert pts == [(it[3], it[4]) for it in m.items]
    qs = [(it[3], it[4]) for it in m.items]
    js, st = ec.get_key_recovery_param_batch(msgs + [e + 1 for e in msgs], sigs * 2, qs * 2)
    assert js[:len(msgs)] == m.recid and (st[:len(msgs)] == nat.ST_TRUE).all()
    assert js[len(msgs):] == [None] * len(msgs) and (st[len(msgs):] == nat.ST_THROW_NO_RECOVERY).all()


@pytest.mark.parametrize("name", list(CURVES))
def test_mul_add_with_prescribed_scalars(native, name):
    """G.mulAdd(u1, Q, u2) = kG for every prescribed pair."""
    from elliptic_b200.ec import EC
    m = _minted(name)
    got = EC(name).mul_add_batch([u1 for u1, _ in m.u], [(it[3], it[4]) for it in m.items], [u2 for _, u2 in m.u])
    assert got == m.kg


def _poison_plan(n, T):
    """{item: (r, s) override} for the 32-item prep's strided batches: thread tid owns tid, tid + T, ..."""
    N = ac.ORDERS["secp256k1"]
    bad = [(0, 1), (1, 0), (1, N), (N, 1), (1, (1 << 256) - 1), (N + 5, 1)]
    plan = {}
    k = 0
    last = T - 1 if (T - 1) < n else n - 1
    for tid in (0, 1, 12345, T // 2 + 3, last):
        for j in (0, 1, 31):
            i = tid + j * T
            if i < n:
                plan[i] = bad[k % len(bad)]
                k += 1
    for tid in (777, last):                          # every member of one full thread and of the last one
        for j in range(32):
            i = tid + j * T
            if i < n:
                plan[i] = bad[k % len(bad)]
                k += 1
    return plan


@pytest.mark.parametrize("n", [1 << 20, (1 << 20) + 3])
def test_bench_shape_device_call_with_poisoned_batches(native, n):
    """eb200_ecdsa_verify_batch_dev at 2^20 (+3) items runs the 32-item prep (k256_prep_batch); the host-buffer
    call on the same data is chunked and runs the 16-item prep.  Items with r or s out of [1, n - 1] at members 0, 1
    and 31 of chosen threads, at every member of one thread and of the last thread must return 0, every other
    item its own verdict, and the two calls must agree byte for byte."""
    import torch
    import benchdata
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    ds = benchdata.gen_secp256k1_verify(1 << 20, seed=0xE1110002, cache_dir=benchdata.cache_dir())
    e, r, s, pub = (ds[k].copy() for k in ("e", "r", "s", "pub"))
    expected = ds["expected"].copy()
    items, exp_p = prescribed_items("secp256k1", 0xBE7C)
    pe, pr, ps, pp = pack(items, 32)
    if n > 1 << 20:
        e, r, s, pub = (np.concatenate([a, b[:n - (1 << 20)]]) for a, b in ((e, pe), (r, pr), (s, ps), (pub, pp)))
        expected = np.concatenate([expected, np.array(exp_p[:n - (1 << 20)], np.uint8)])
    T = ((n + 31) // 32 + 127) // 128 * 128          # threads of the prep grid: batch_blocks(n, 32) x 128
    # prescribed items at every member of thread 4242 and spread over the rest
    rnd = random.Random(n)
    slots = [4242 + j * T for j in range(32) if 4242 + j * T < n] + rnd.sample(range(n - 8), len(items) - 32)
    for i, it in zip(slots, range(len(items))):
        e[i], r[i], s[i], pub[i], expected[i] = pe[it], pr[it], ps[it], pp[it], exp_p[it]
    for i, (rv, sv) in _poison_plan(n, T).items():
        r[i] = np.frombuffer(rv.to_bytes(32, "big"), np.uint8)
        s[i] = np.frombuffer(sv.to_bytes(32, "big"), np.uint8)
        expected[i] = 0
    lib = native
    dev = torch.device("cuda", 0)
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in (("e", e), ("r", r), ("s", s), ("pub", pub))}
    st = torch.empty(n, dtype=torch.uint8, device=dev)
    ws = torch.empty(lib.eb200_ecdsa_verify_workspace_bytes(nat.CURVE_SECP256K1, n), dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev)
    nat.check(lib.eb200_ecdsa_verify_batch_dev(nat.CURVE_SECP256K1, n, d["e"].data_ptr(), d["r"].data_ptr(),
                                               d["s"].data_ptr(), d["pub"].data_ptr(), 0, st.data_ptr(), ws.data_ptr(),
                                               stream.cuda_stream))
    torch.cuda.synchronize(dev)
    got = st.cpu().numpy()
    bad = np.nonzero(got != expected)[0]
    assert bad.size == 0, [(int(i), int(got[i]), int(expected[i])) for i in bad[:20]]
    host = EC("secp256k1").verify_batch_packed(e, r, s, pub)
    assert np.array_equal(host, got)
