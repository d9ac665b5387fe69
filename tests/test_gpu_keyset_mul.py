"""Keyed Point.mul / mulAdd / derive on the GPU: eb200_scalar_mul_batch_keyed, eb200_mul_add_batch_keyed and
eb200_ecdh_derive_batch_keyed must write exactly the bytes of eb200_scalar_mul_batch / eb200_mul_add_batch /
eb200_ecdh_derive_batch for the same scalars with the keys gathered, on every short preset and width, for on-curve,
throwing and off-curve keys; plus their argument, lifetime and timing contract and the Python KeySet methods."""
import ctypes

import numpy as np
import pytest

from ks_items import CURVES

pytestmark = pytest.mark.gpu
OPS = ("mul", "mul_add", "derive")


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


def create(lib, cid, pub, fmt=0, bits=0):
    from elliptic_b200 import _native as nat
    pub = np.ascontiguousarray(pub, np.uint8)
    kst, h = np.zeros(len(pub), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_keyset_create(cid, len(pub), pub.ctypes.data, fmt, bits, kst.ctypes.data, ctypes.byref(h)))
    return h, kst


def scalars(rng, cid, n, ln):
    """n scalars of ln bytes, any value below 2^(8 ln), the edge values 0, 1, n - 1, n, n + 1 and 2^(8 ln) - 1 among them."""
    from oracle.ref_py.ec import EC
    name = next(nm for nm, c, _ in CURVES if c == cid)
    order = EC(name).n
    k = rng.integers(0, 256, size=(n, ln), dtype=np.uint8)
    for j, v in enumerate((0, 1, order - 1, order, order + 1, (1 << (8 * ln)) - 1)):
        k[7 * j + 3] = np.frombuffer(v.to_bytes(ln, "big"), np.uint8)
    return k


def unkeyed(lib, cid, op, k1, k2, pts):
    from elliptic_b200 import _native as nat
    n, ln = k2.shape
    out, st = np.zeros((n, ln if op == "derive" else 2 * ln), np.uint8), np.zeros(n, np.uint8)
    pts = np.ascontiguousarray(pts)
    if op == "mul":
        nat.call(lib.eb200_scalar_mul_batch, cid, n, k2, pts, out, st)
    elif op == "mul_add":
        nat.call(lib.eb200_mul_add_batch, cid, n, k1, k2, pts, out, st)
    else:
        nat.call(lib.eb200_ecdh_derive_batch, cid, n, k2, pts, out, st)
    return out, st


def keyed(lib, h, op, k1, k2, idx):
    from elliptic_b200 import _native as nat
    n, ln = k2.shape
    out = np.full((n, ln if op == "derive" else 2 * ln), 0xA5, np.uint8)
    st = np.full(n, 0xEE, np.uint8)
    idx = np.ascontiguousarray(idx, np.uint32)
    if op == "mul":
        nat.call(lib.eb200_scalar_mul_batch_keyed, h, n, k2, idx, out, st)
    elif op == "mul_add":
        nat.call(lib.eb200_mul_add_batch_keyed, h, n, k1, k2, idx, out, st)
    else:
        nat.call(lib.eb200_ecdh_derive_batch_keyed, h, n, k2, idx, out, st)
    return out, st


def keys_on_gpu(lib, cid, ln, m, rng):
    from elliptic_b200 import _native as nat
    d = rng.integers(0, 256, size=(m, ln), dtype=np.uint8)
    xy, st = np.zeros((m, 2 * ln), np.uint8), np.zeros(m, np.uint8)
    nat.call(lib.eb200_scalar_mul_batch, cid, m, d, None, xy, st)
    assert (st == nat.ST_TRUE).all()
    return xy


def assert_same(got, want, what):
    (go, gs), (wo, ws) = got, want
    bad = np.nonzero((gs != ws) | (go != wo).any(axis=1))[0]
    assert len(bad) == 0, (what, bad[:8], gs[bad[:8]], ws[bad[:8]])


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_keyed_equals_unkeyed_on_every_preset(lib, name, cid, ln):
    from elliptic_b200 import _native as nat
    rng = np.random.default_rng(cid)
    xy = keys_on_gpu(lib, cid, ln, 64, rng)
    for n in (1 << 16, (1 << 18) + 333):                   # the second spans four chunks with a short first one
        idx = rng.integers(0, 64, size=n).astype(np.uint32)
        k1, k2 = scalars(rng, cid, n, ln), scalars(rng, cid, n, ln)
        want = {op: unkeyed(lib, cid, op, k1, k2, xy[idx]) for op in OPS}
        for op in OPS:
            assert (want[op][1] == nat.ST_TRUE).sum() > n - 16 and nat.ST_INFINITY in want[op][1]
        for bits in ((4, 8, 0) if n == 1 << 16 else (8,)):
            h, kst = create(lib, cid, xy, 0, bits)
            assert (kst == 1).all()
            for op in OPS:
                assert_same(keyed(lib, h, op, k1, k2, idx), want[op], (name, bits, op, n))
                launches = nat.last_timing()["launches"]
                assert launches == 4 if n == 1 << 16 else (launches % 4 == 0 and launches >= 16)
            nat.check(lib.eb200_keyset_destroy(h))


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_throwing_and_off_curve_keys(lib, name, cid, ln):
    """A compressed set with a bad prefix and an x without a square root (the key's throw, output zeroed), and an {x, y}
    set with an off-curve key (mul / mulAdd: the unkeyed call's replay; derive: THROW_NOT_VALIDATED); G, -G and 2G
    among the keys, with mulAdd pairs that sum to the point at infinity."""
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    ec = EC(name)
    rng = np.random.default_rng(100 + cid)
    col = lambda v: np.frombuffer(v.to_bytes(ln, "big"), np.uint8)
    xy = keys_on_gpu(lib, cid, ln, 8, rng)
    for j, d in enumerate((1, ec.n - 1, 2)):
        P = ec.g.mul(d)
        xy[j] = np.concatenate([col(P.x), col(P.y)])
    xy[7, ln:] = col((int.from_bytes(xy[7, ln:].tobytes(), "big") + 1) % ec.curve.p)       # off the curve
    n = 4096
    idx = (np.arange(n) % 8).astype(np.uint32)
    k1, k2 = scalars(rng, cid, n, ln), scalars(rng, cid, n, ln)
    k2[8:16] = np.frombuffer((12345).to_bytes(ln, "big"), np.uint8)
    k1[8:11] = [col(12345 * d % ec.n) for d in (ec.n - 1, 1, ec.n - 2)]       # k1 G + k2 Q = O on keys G, -G, 2G
    h, kst = create(lib, cid, xy)
    assert list(kst) == [1] * 7 + [0]
    for op in OPS:
        want = unkeyed(lib, cid, op, k1, k2, xy[idx])
        got = keyed(lib, h, op, k1, k2, idx)
        assert_same(got, want, (name, op))
        sts = set(got[1].tolist())
        assert (nat.ST_THROW_NOT_VALIDATED in sts) == (op == "derive") and nat.ST_INFINITY in sts
    nat.check(lib.eb200_keyset_destroy(h))

    comp = np.concatenate([(2 + (xy[:, -1:] & 1)).astype(np.uint8), xy[:, :ln]], axis=1)
    comp[1, 0] = 5                                        # 'Unknown point format'
    x = 1
    while True:                                           # an x with no point: 'invalid point' (p224: the Tonelli-Shanks assertion)
        try:
            ec.curve.point_from_x(x, 0)
            x += 1
        except Exception:
            break
    comp[2, 1:] = col(x)
    h, kst = create(lib, cid, comp[:7], 2)
    assert kst[1] == nat.ST_THROW_POINT_FORMAT and kst[2] in (nat.ST_THROW_INVALID_POINT, nat.ST_THROW_ASSERT)
    dec = np.zeros((7, 2 * ln), np.uint8)                 # the decoded keys, as the unkeyed call gets them
    for j in range(7):
        if kst[j] == 1:
            P = ec.curve.point_from_x(int.from_bytes(comp[j, 1:].tobytes(), "big"), comp[j, 0] == 3)
            dec[j] = np.concatenate([col(P.x), col(P.y)])
    idx7 = (np.arange(n) % 7).astype(np.uint32)
    for op in OPS:
        go, gs = keyed(lib, h, op, k1, k2, idx7)
        thrown = kst[idx7] != 1
        assert (gs[thrown] == kst[idx7][thrown]).all() and not go[thrown].any()
        wo, ws = unkeyed(lib, cid, op, k1[~thrown], k2[~thrown], dec[idx7[~thrown]])
        assert (gs[~thrown] == ws).all() and (go[~thrown] == wo).all(), (name, op)
    nat.check(lib.eb200_keyset_destroy(h))


def test_argument_and_lifetime_contract(lib):
    from elliptic_b200 import _native as nat
    rng = np.random.default_rng(9)
    xy = keys_on_gpu(lib, 1, 32, 16, rng)
    n = 1000
    idx = rng.integers(0, 16, size=n).astype(np.uint32)
    k = scalars(rng, 1, n, 32)
    out, st = np.zeros((n, 64), np.uint8), np.full(n, 0xEE, np.uint8)
    p = lambda a: a.ctypes.data
    h, _ = create(lib, 1, xy)
    bad = idx.copy(); bad[500] = 16
    assert lib.eb200_scalar_mul_batch_keyed(h, n, p(k), p(bad), p(out), p(st)) == nat.ERR_ARG
    assert lib.eb200_mul_add_batch_keyed(h, n, p(k), p(k), p(bad), p(out), p(st)) == nat.ERR_ARG
    assert lib.eb200_ecdh_derive_batch_keyed(h, n, p(k), p(bad), p(out), p(st)) == nat.ERR_ARG
    assert lib.eb200_mul_add_batch_keyed(h, n, None, p(k), p(idx), p(out), p(st)) == nat.ERR_ARG
    assert lib.eb200_scalar_mul_batch_keyed(h, n, p(k), p(idx), None, p(st)) == nat.ERR_ARG
    assert lib.eb200_scalar_mul_batch_keyed(h, 0, None, None, None, None) == nat.OK
    assert (st == 0xEE).all() and not out.any()
    ed, est = ctypes.c_void_p(), np.zeros(4, np.uint8)
    nat.check(lib.eb200_eddsa_keyset_create(4, p(np.full((4, 32), 0x11, np.uint8)), 4, p(est), ctypes.byref(ed)))
    assert lib.eb200_scalar_mul_batch_keyed(ed, n, p(k), p(np.zeros(n, np.uint32)), p(out), p(st)) == nat.ERR_ARG
    assert lib.eb200_ecdh_derive_batch_keyed(ed, n, p(k), p(np.zeros(n, np.uint32)), p(out), p(st)) == nat.ERR_ARG
    assert (st == 0xEE).all()
    nat.check(lib.eb200_keyset_destroy(ed))
    got = keyed(lib, h, "derive", None, k, idx)
    assert nat.last_timing()["launches"] == 4
    assert_same(got, unkeyed(lib, 1, "derive", None, k, xy[idx]), "derive")
    nat.shutdown()
    try:
        assert lib.eb200_scalar_mul_batch_keyed(h, n, p(k), p(idx), p(out), p(st)) == nat.ERR_NOT_INIT
        assert lib.eb200_ecdh_derive_batch_keyed(h, n, p(k), p(idx), p(out), p(st)) == nat.ERR_NOT_INIT
        assert (st == 0xEE).all()
    finally:
        nat.check(lib.eb200_keyset_destroy(h))
        nat.init(0)


def test_python_key_set_methods_match_ec():
    from elliptic_b200.ec import EC, EllipticError
    from oracle.ref_py.ec import EC as RefEC
    ref, ec = RefEC("secp256k1"), EC("secp256k1")
    pts = [ref.g.mul(d) for d in (11, 22, 33)]
    keys = [{"x": pts[0].x, "y": pts[0].y}, "04%064x%064x" % (pts[1].x, pts[1].y), "%02x%064x" % (2 + (pts[2].y & 1), pts[2].x),
            {"x": pts[0].x, "y": pts[0].y + 1}]
    xy = [(pts[0].x, pts[0].y), (pts[1].x, pts[1].y), (pts[2].x, pts[2].y), (pts[0].x, pts[0].y + 1)]
    kidx = [t % 4 for t in range(40)]
    ks1 = [t * 0x1234567 + (t == 3) * ref.n for t in range(40)]
    ks2 = [(t + 5) * 0x7654321 if t != 6 else 0 for t in range(40)]
    with ec.key_set(keys, "hex") as ks:
        assert list(ks.status) == [1, 1, 1, 0]
        assert ks.mul_batch(kidx, ks2) == ec.mul_batch([xy[k] for k in kidx], ks2)
        assert ks.mul_add_batch(ks1, kidx, ks2) == ec.mul_add_batch(ks1, [xy[k] for k in kidx], ks2)
        got, st = ks.derive_batch(ks2, kidx)
        want, wst = ec.derive_batch(ks2, [xy[k] for k in kidx])
        assert got == want and (st == wst).all() and 3 in st.tolist()
        out, st = ks.mul_batch_packed(ec._scalars(ks2), kidx)
        assert (st[:3] == 1).all() and out.shape == (40, 64)
    comp = ec.key_set(["02" + "00" * 31 + "05", "%02x%064x" % (2 + (pts[2].y & 1), pts[2].x)], "hex")    # no point has x = 5
    assert comp.status[0] == 2 and comp.status[1] == 1
    assert comp.mul_batch([1, 1], [3, 4]) == ec.mul_batch([xy[2], xy[2]], [3, 4])
    with pytest.raises(EllipticError):
        comp.mul_batch([1, 0], [3, 4])
    with pytest.raises(EllipticError):
        comp.derive_batch([3], [0])
    comp.close()
