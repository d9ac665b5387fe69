"""Keyed getKeyRecoveryParam on the GPU: eb200_ecdsa_recovery_param_batch_keyed must write exactly the recid and status
bytes of eb200_ecdsa_recovery_param_batch for the same e, r, s with each item's key gathered, on every short preset, for
on-curve, off-curve and throwing keys and adversarial items; plus a sample against the oracle, the argument, lifetime
and timing contract, sharding over two GPUs where there are two, and the Python KeySet methods."""
import ctypes
import random

import numpy as np
import pytest

from krp_items import NO_RECOVERY, krp_expected
from ks_items import CURVES, adversarial_keys, minted

pytestmark = pytest.mark.gpu
NKEYS = {1: 4096, 2: 4096, 3: 512, 6: 256, 7: 1024, 8: 1024}


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


def col(vals, ln):
    return np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in vals), np.uint8).reshape(len(vals), ln).copy()


def create(lib, cid, pub, fmt=0, bits=0):
    from elliptic_b200 import _native as nat
    pub = np.ascontiguousarray(pub, np.uint8)
    kst, h = np.zeros(len(pub), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_keyset_create(cid, len(pub), pub.ctypes.data, fmt, bits, kst.ctypes.data, ctypes.byref(h)))
    return h, kst


def unkeyed(lib, cid, e, r, s, q):
    from elliptic_b200 import _native as nat
    n = len(e)
    rid, st = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    nat.call(lib.eb200_ecdsa_recovery_param_batch, cid, n, e, r, s, np.ascontiguousarray(q), rid, st)
    return rid, st


def keyed(lib, h, e, r, s, idx):
    from elliptic_b200 import _native as nat
    n = len(e)
    rid, st = np.full(n, 0xA5, np.uint8), np.full(n, 0xEE, np.uint8)
    nat.call(lib.eb200_ecdsa_recovery_param_batch_keyed, h, n, e, r, s, np.ascontiguousarray(idx, np.uint32), rid, st)
    return rid, st


def assert_same(got, want, what):
    bad = np.nonzero((got[0] != want[0]) | (got[1] != want[1]))[0]
    assert len(bad) == 0, (what, bad[:8], got[0][bad[:8]], want[0][bad[:8]], got[1][bad[:8]], want[1][bad[:8]])


def signed_items(lib, ec, cid, ln, m, n, seed):
    """m keys d G (computed on the GPU) and n GPU signatures by them, one item in eight damaged in turn: the wrong key,
    r = 0, s = 0, s = n, r = n, a flipped e, r + 1, r + p.  Returns (d, xy, e, r, s, idx, recid of the signer)."""
    from elliptic_b200 import _native as nat
    rnd = random.Random(seed)
    rng = np.random.default_rng(seed)
    d = [rnd.randrange(1, ec.n) for _ in range(m)]
    dk = col(d, ln)
    xy, st = np.zeros((m, 2 * ln), np.uint8), np.zeros(m, np.uint8)
    nat.call(lib.eb200_scalar_mul_batch, cid, m, dk, None, xy, st)
    assert (st == nat.ST_TRUE).all()
    idx = rng.integers(0, m, size=n).astype(np.uint32)
    e = rng.integers(0, 256, size=(n, ln), dtype=np.uint8)
    e[:, 0] = 0                                           # e < 2^(8 (len - 1)) < n
    r, s, rec, st = np.zeros((n, ln), np.uint8), np.zeros((n, ln), np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    nat.call(lib.eb200_ecdsa_sign_batch, cid, n, e, np.ascontiguousarray(dk[idx]), 0, r, s, rec, st)
    assert (st == nat.ST_TRUE).all()
    nb, pb = col([ec.n], ln)[0], ec.curve.p
    for t in range(1, n, 8):
        kind = (t // 8) % 8
        if kind == 0: idx[t] = (idx[t] + 1) % m
        if kind == 1: r[t] = 0
        if kind == 2: s[t] = 0
        if kind == 3: s[t] = nb
        if kind == 4: r[t] = nb
        if kind == 5: e[t, -1] ^= 1
        if kind in (6, 7):
            rv = int.from_bytes(r[t].tobytes(), "big") + (1 if kind == 6 else pb)
            if rv < 1 << (8 * ln):
                r[t] = col([rv], ln)[0]
    return d, xy, e, r, s, idx, rec


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_keyed_equals_unkeyed_on_every_preset(lib, name, cid, ln):
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    ec = EC(name)
    n = (1 << 18) + 333                                    # five chunks, the first one short
    d, xy, e, r, s, idx, rec = signed_items(lib, ec, cid, ln, NKEYS[cid], n, cid)
    want = unkeyed(lib, cid, e, r, s, xy[idx])
    honest = np.ones(n, bool)
    honest[1::8] = False
    assert (want[1][honest] == nat.ST_TRUE).all() and (want[0][honest] == rec[honest]).all()
    assert NO_RECOVERY in want[1] and set(want[0][honest].tolist()) >= {0, 1}
    for bits in (4, 8, 0):
        h, kst = create(lib, cid, xy, 0, bits)
        assert (kst == 1).all()
        assert_same(keyed(lib, h, e, r, s, idx), want, (name, bits))
        t = nat.last_timing()
        assert t["launches"] % 4 == 0 and t["launches"] >= 20 and t["main_kernel_ms"] > 0
        m = 4099                                           # one chunk, an odd tail
        assert_same(keyed(lib, h, e[:m], r[:m], s[:m], idx[:m]), (want[0][:m], want[1][:m]), (name, bits, m))
        assert nat.last_timing()["launches"] == 4
        nat.check(lib.eb200_keyset_destroy(h))
    sample = np.random.default_rng(7).choice(n, 12, replace=False)
    for i in sample:
        x, y = int.from_bytes(xy[idx[i], :ln].tobytes(), "big"), int.from_bytes(xy[idx[i], ln:].tobytes(), "big")
        it = tuple(int.from_bytes(a[i].tobytes(), "big") for a in (e, r, s)) + (x, y)
        assert krp_expected(ec, it) == (want[0][i] if want[1][i] == nat.ST_TRUE else want[1][i]), (name, i)


def adversarial(ec, cid, ln, rnd):
    """Keys G, -G, 2^j G and entries of G's tables, with (u1, u2) pairs meeting the exceptional additions of the keyed
    accumulation, signed when P has an x (else e = u1 s, r = u2 s); s = 0 items whose cold answer is found."""
    n = ec.n
    keys = adversarial_keys(ec, cid, (4, 6, 8))
    items = []
    for k, (d, Q) in enumerate(keys):
        for _ in range(3):
            u1 = rnd.randrange(1, n)
            for u2 in ((-u1 * pow(d, -1, n)) % n, (u1 * pow(d, -1, n)) % n, rnd.randrange(1, n)):
                sig = minted(ec, u1, u2, Q)
                if sig is None:
                    s = rnd.randrange(1, n)
                    sig = (u1 * s % n, u2 * s % n, s)
                items.append(sig + (k,))
        e = rnd.randrange(1, n)
        for rr in (Q.x % n, rnd.randrange(1, n)):         # s = 0: Q = ((n - e) / r) G found for the matching e only
            items.append(((n - d * rr) % n, rr, 0, k))
            items.append((e, rr, 0, k))
    return [(Q.x, Q.y) for _, Q in keys], items


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_throwing_off_curve_and_adversarial_keys(lib, name, cid, ln):
    """An {x, y} set with the adversarial keys and an off-curve one (THROW_NO_RECOVERY for every item on it), and a
    compressed set with a bad prefix and an x without a square root (the key's throw, recid 0)."""
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    ec = EC(name)
    rnd = random.Random(300 + cid)
    keys, items = adversarial(ec, cid, ln, rnd)
    keys.append((keys[3][0], (keys[3][1] + 1) % ec.curve.p))                  # off the curve
    off = len(keys) - 1
    items += [(it[0], it[1], it[2], off) for it in items[:24]]
    reps = -(-4099 // len(items))
    items = (items * reps)[:4099]
    xy = np.concatenate([col([k[0] for k in keys], ln), col([k[1] for k in keys], ln)], axis=1)
    e, r, s = (col([it[j] for it in items], ln) for j in range(3))
    idx = np.array([it[3] for it in items], np.uint32)
    h, kst = create(lib, cid, xy)
    assert list(kst) == [1] * off + [0]
    want = unkeyed(lib, cid, e, r, s, xy[idx])
    got = keyed(lib, h, e, r, s, idx)
    assert_same(got, want, name)
    assert (got[1][idx == off] == nat.ST_THROW_NO_RECOVERY).all()
    assert nat.ST_TRUE in got[1] and {0, 1} <= set(got[0][got[1] == nat.ST_TRUE].tolist())
    for i in range(0, len(keys) * 12, 7):                 # against the oracle, once per distinct item
        it = items[i]
        assert krp_expected(ec, it[:3] + keys[it[3]]) == (got[0][i] if got[1][i] == nat.ST_TRUE else got[1][i]), (name, i)
    nat.check(lib.eb200_keyset_destroy(h))

    comp = np.concatenate([(2 + (xy[:off, -1:] & 1)).astype(np.uint8), xy[:off, :ln]], axis=1)
    comp[1, 0] = 5                                        # 'Unknown point format'
    x = 1
    while True:                                           # an x with no point
        try:
            ec.curve.point_from_x(x, 0)
            x += 1
        except Exception:
            break
    comp[2, 1:] = col([x], ln)[0]
    h, kst = create(lib, cid, comp, 2)
    assert kst[1] == nat.ST_THROW_POINT_FORMAT and kst[2] in (nat.ST_THROW_INVALID_POINT, nat.ST_THROW_ASSERT)
    sel = idx < off
    gr, gs = keyed(lib, h, e[sel], r[sel], s[sel], idx[sel])
    thrown = kst[idx[sel]] != 1
    assert (gs[thrown] == kst[idx[sel]][thrown]).all() and not gr[thrown].any()
    assert (gs[~thrown] == want[1][sel][~thrown]).all() and (gr[~thrown] == want[0][sel][~thrown]).all(), name
    nat.check(lib.eb200_keyset_destroy(h))


def test_argument_and_lifetime_contract(lib):
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    ec = EC("secp256k1")
    n = 1000
    d, xy, e, r, s, idx, rec = signed_items(lib, ec, 1, 32, 16, n, 9)
    rid, st = np.full(n, 0xA5, np.uint8), np.full(n, 0xEE, np.uint8)
    p = lambda a: a.ctypes.data
    f = lib.eb200_ecdsa_recovery_param_batch_keyed
    h, _ = create(lib, 1, xy)
    bad = idx.copy(); bad[500] = 16
    assert f(h, n, p(e), p(r), p(s), p(bad), p(rid), p(st)) == nat.ERR_ARG
    for k in range(6):
        args = [p(e), p(r), p(s), p(idx), p(rid), p(st)]
        args[k] = None
        assert f(h, n, *args) == nat.ERR_ARG, k
    assert f(h, 0, None, None, None, None, None, None) == nat.OK
    assert (st == 0xEE).all() and (rid == 0xA5).all()
    ed, est = ctypes.c_void_p(), np.zeros(4, np.uint8)
    nat.check(lib.eb200_eddsa_keyset_create(4, p(np.full((4, 32), 0x11, np.uint8)), 4, p(est), ctypes.byref(ed)))
    assert f(ed, n, p(e), p(r), p(s), p(np.zeros(n, np.uint32)), p(rid), p(st)) == nat.ERR_ARG
    nat.check(lib.eb200_keyset_destroy(ed))
    sg, pub = ctypes.c_void_p(), np.zeros((4, 32), np.uint8)
    nat.check(lib.eb200_eddsa_signing_set_create(4, p(np.full((4, 32), 0x22, np.uint8)), p(pub), ctypes.byref(sg)))
    assert f(sg, n, p(e), p(r), p(s), p(np.zeros(n, np.uint32)), p(rid), p(st)) == nat.ERR_ARG
    nat.check(lib.eb200_keyset_destroy(sg))
    assert (st == 0xEE).all() and (rid == 0xA5).all()
    got = keyed(lib, h, e, r, s, idx)
    assert nat.last_timing()["launches"] == 4
    assert_same(got, unkeyed(lib, 1, e, r, s, xy[idx]), "secp256k1")
    nat.shutdown()
    try:
        assert f(h, n, p(e), p(r), p(s), p(idx), p(rid), p(st)) == nat.ERR_NOT_INIT
        assert (st == 0xEE).all() and (rid == 0xA5).all()
    finally:
        nat.check(lib.eb200_keyset_destroy(h))
        nat.init(0)


def test_sharding_over_two_gpus_gives_the_same_bytes():
    import torch
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    lib = nat.init(0)
    for name, cid, ln in (CURVES[0], CURVES[3]):
        n = (1 << 16) + 77
        d, xy, e, r, s, idx, rec = signed_items(lib, EC(name), cid, ln, 256, n, 50 + cid)
        h, _ = create(lib, cid, xy)
        one = keyed(lib, h, e, r, s, idx)
        nat.check(lib.eb200_keyset_destroy(h))
        nat.init_devices([0, 1])
        try:
            h, _ = create(lib, cid, xy)
            assert_same(keyed(lib, h, e, r, s, idx), one, (name, "2 GPUs"))
            nat.check(lib.eb200_keyset_destroy(h))
        finally:
            nat.shutdown()
            nat.init(0)


def test_python_key_set_methods_match_ec():
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC, EllipticError, NeedsReferencePath
    from oracle.ref_py.ec import EC as RefEC
    ref, ec = RefEC("secp256k1"), EC("secp256k1")
    ds = (11, 22, 33)
    pts = [ref.g.mul(d) for d in ds]
    keys = [{"x": pts[0].x, "y": pts[0].y}, "04%064x%064x" % (pts[1].x, pts[1].y), "%02x%064x" % (2 + (pts[2].y & 1), pts[2].x),
            {"x": pts[0].x, "y": pts[0].y + 1}]
    xy = [(pts[0].x, pts[0].y), (pts[1].x, pts[1].y), (pts[2].x, pts[2].y), (pts[0].x, pts[0].y + 1)]
    rnd = random.Random(4)
    kidx = [t % 4 for t in range(40)]
    msgs, sigs = [], []
    for t, k in enumerate(kidx):
        m = rnd.randrange(1 << 255)
        sg = ref.sign(m, ds[k % 3], canonical=bool(t & 1))
        msgs.append(m)
        if t % 5 == 2:
            sigs.append({"r": sg.r, "s": sg.s, "recoveryParam": 3})          # answered without a call
        elif t % 7 == 3:
            sigs.append({"r": sg.r, "s": (sg.s + 1) % ref.n})
        else:
            sigs.append({"r": sg.r, "s": sg.s})
    with ec.key_set(keys, "hex") as ks:
        assert list(ks.status) == [1, 1, 1, 0]
        got, st = ks.get_key_recovery_param_batch(msgs, sigs, kidx)
        want, wst = ec.get_key_recovery_param_batch(msgs, sigs, [xy[k] for k in kidx])
        assert got == want and (st == wst).all()
        assert {0, 1, 3, None} <= set(got) and nat.ST_THROW_NO_RECOVERY in st.tolist()
        rid, pst = ks.recovery_param_batch_packed(*ec._recover_args(msgs[:4], [(s["r"], s["s"]) for s in sigs[:4]]), kidx[:4])
        assert pst.shape == (4,) and rid.dtype == np.uint8
        with pytest.raises(NeedsReferencePath):
            ks.get_key_recovery_param_batch(msgs[:1], [{"r": 1 << 256, "s": 5}], [0])
    comp = ec.key_set(["02" + "00" * 31 + "05", "%02x%064x" % (2 + (pts[2].y & 1), pts[2].x)], "hex")    # no point has x = 5
    assert comp.status[0] == 2 and comp.status[1] == 1
    sg = ref.sign(123, 33)
    bare = {"r": sg.r, "s": sg.s}
    got, st = comp.get_key_recovery_param_batch([123, 123], [sg, bare], [1, 1])
    want, wst = ec.get_key_recovery_param_batch([123, 123], [sg, bare], [xy[2], xy[2]])
    assert got == want == [sg.recovery_param] * 2 and (st == wst).all()
    with pytest.raises(EllipticError):
        comp.get_key_recovery_param_batch([123, 123], [sg, sg], [1, 0])
    comp.close()
