"""The cases of torsion_cases.py through the C ABI on the GPU: ed25519 Point.mul / mulAdd / ECDH derive / EC.verify and
the curve25519 ladder on points with a torsion component, small-order and twist inputs.  Each base case list is tiled to
at least 4099 items (32 full blocks of 128 threads and a partial one) and every item is compared with the oracle."""
import numpy as np
import pytest

import torsion_cases as tc
from torsion_cases import mul_cases, verify_items

pytestmark = pytest.mark.gpu
TILE = 4099


def _tiled(rows):
    return rows * -(-TILE // len(rows))


def _be(vals, ln=32):
    return np.frombuffer(tc.be(vals, ln), np.uint8).reshape(-1, ln).copy()


def _ints(a):
    return [int.from_bytes(row.tobytes(), "big") for row in a]


def _xy_rows(a):
    return list(zip(_ints(a[:, :32]), _ints(a[:, 32:])))


def _pts(pts):
    return np.concatenate([_be([p[0] for p in pts]), _be([p[1] for p in pts])], axis=1)


@pytest.fixture(scope="module")
def ec():
    from oracle.ref_py.ec import EC
    return EC("ed25519")


def test_ed25519_mul_and_mul_add_exact(native, ec):
    from elliptic_b200 import _native as nat
    base = mul_cases()
    k1_base = [k for _, _, k in base][7:] + [k for _, _, k in base][:7]
    want_mul = [(lambda w: (w.get_x(), w.get_y()))(ec.curve.point(*pt).mul(k)) for _, pt, k in base]
    want_add = [(lambda w: (w.get_x(), w.get_y()))(ec.g.mul_add(k1, ec.curve.point(*pt), k))
                for k1, (_, pt, k) in zip(k1_base, base)]
    cases, k1s = _tiled(base), _tiled(k1_base)
    n = len(cases)
    k2, k1, pts = _be([k for _, _, k in cases]), _be(k1s), _pts([pt for _, pt, _ in cases])
    out, st = np.zeros((n, 64), np.uint8), np.zeros(n, np.uint8)
    nat.call(native.eb200_scalar_mul_batch, nat.CURVE_ED25519, n, k2, pts, out, st)
    assert (st == nat.ST_TRUE).all()
    assert _xy_rows(out) == _tiled(want_mul)
    out[:] = 0
    nat.call(native.eb200_mul_add_batch, nat.CURVE_ED25519, n, k1, k2, pts, out, st)
    assert (st == nat.ST_TRUE).all()
    assert _xy_rows(out) == _tiled(want_add)


def test_ed25519_ecdh_derive_small_and_mixed_order_peers(native, ec):
    """KeyPair.derive against peers of every torsion order, alone and added to d G: priv reduced mod n as
    _importPrivate does, and shared points that are the neutral point (0, 1) or the order-2 point (0, -1) among them."""
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import KeyPair
    base = mul_cases()
    privs = [k % ec.n for _, _, k in base]
    shared = [ec.curve.point(*pt).mul(d) for d, (_, pt, _) in zip(privs, base)]
    want = [KeyPair(ec, priv=d).derive(ec.curve.point(*pt)) for d, (_, pt, _) in zip(privs, base)]
    assert [s.get_x() for s in shared] == want
    assert any((s.get_x(), s.get_y()) == tc.O for s in shared) and any((s.get_x(), s.get_y()) == (0, tc.P - 1) for s in shared)
    cases = _tiled(list(zip(privs, [pt for _, pt, _ in base])))
    n = len(cases)
    out, st = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    nat.call(native.eb200_ecdh_derive_batch, nat.CURVE_ED25519, n, _be([d for d, _ in cases]), _pts([pt for _, pt in cases]), out, st)
    assert (st == nat.ST_TRUE).all()
    assert _ints(out) == _tiled(want)


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_ed25519_verify_mixed_order_keys(native, ec, fmt):
    """EC.verify against d G + T with {x, y}, 04 || x || y and 02/03 || x keys: true exactly when u2 T = O."""
    from elliptic_b200 import _native as nat
    base = verify_items()
    enc = {0: lambda q: q[0].to_bytes(32, "big") + q[1].to_bytes(32, "big"),
           1: lambda q: tc.sec1(q, False), 2: lambda q: tc.sec1(q, True)}[fmt]
    want = [int(ec.verify(e, {"r": r, "s": s}, {"x": q[0], "y": q[1]} if fmt == 0 else enc(q), msg_bit_length=253))
            for e, r, s, q, _ in base]
    assert want == [int(passes) for *_, passes in base] and 0 in want and 1 in want
    cases = _tiled(base)
    n = len(cases)
    pub = np.frombuffer(b"".join(enc(it[3]) for it in cases), np.uint8).copy()
    st = np.zeros(n, np.uint8)
    nat.call(native.eb200_ecdsa_verify_batch, nat.CURVE_ED25519, n, _be([it[0] for it in cases]), _be([it[1] for it in cases]),
             _be([it[2] for it in cases]), pub, fmt, st)
    assert [int(v) for v in st] == _tiled(want)


def test_x25519_mul_and_derive_on_small_mixed_noncanonical_and_twist_u(native):
    import torch
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    from oracle.ref_py import curves
    from ed_items import x_expected
    ec25, c25 = EC("curve25519"), curves.get("curve25519").curve
    base = [(u, k) for _, u in tc.x25519_us() for k in tc.scalars(randoms=1)]
    want_mul = [c25.point(u, 1).mul(k).get_x() for u, k in base]
    want_derive = [x_expected(ec25, c25, k % ec25.n, u) for u, k in base]
    assert {s for s, _ in want_derive} == {nat.ST_TRUE, nat.ST_THROW_ASSERT}
    cases = _tiled(base)
    n = len(cases)
    ks, us, privs = _be([k for _, k in cases]), _be([u for u, _ in cases]), _be([k % ec25.n for _, k in cases])
    out, st = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    nat.call(native.eb200_x25519_mul_batch, n, ks, us, out, st)
    assert (st == nat.ST_TRUE).all() and _ints(out) == _tiled(want_mul)
    nat.call(native.eb200_x25519_derive_batch, n, privs, us, out, st)
    assert list(zip([int(v) for v in st], _ints(out))) == _tiled(want_derive)
    d_priv, d_u = torch.from_numpy(privs).cuda(), torch.from_numpy(us).cuda()
    d_out, d_st = torch.zeros((n, 32), dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda")
    nat.check(native.eb200_x25519_derive_batch_dev(n, d_priv.data_ptr(), d_u.data_ptr(), d_out.data_ptr(), d_st.data_ptr(),
                                                   torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert list(zip([int(v) for v in d_st.cpu().numpy()], _ints(d_out.cpu().numpy()))) == _tiled(want_derive)


def test_python_mirror_mul_and_mul_add_with_wide_scalars(native, ec):
    """EC('ed25519').mul_batch / mul_add_batch: scalars of 2^256 and more are reduced on the host before the call, by 8n
    (the group order), so the answer stays P.mul(k) for points with a torsion component."""
    from elliptic_b200.ec import EC as GpuEC
    gec = GpuEC("ed25519")
    ks = tc.wide_scalars() + [tc.N, 8 * tc.N - 1, 2**256 - 1]
    cases = [(pt, k) for _, pt in tc.points() for k in ks]
    k1s = [k + 2**256 * (i % 3) for i, (_, k) in enumerate(cases)]
    pts = [pt for pt, _ in cases]
    got = gec.mul_batch(pts, [k for _, k in cases])
    assert got == [(lambda w: (w.get_x(), w.get_y()))(ec.curve.point(*pt).mul(k)) for pt, k in cases]
    got = gec.mul_add_batch(k1s, pts, [k for _, k in cases])
    assert got == [(lambda w: (w.get_x(), w.get_y()))(ec.g.mul_add(k1, ec.curve.point(*pt), k)) for k1, (pt, k) in zip(k1s, cases)]
