"""ed25519 and curve25519 off the prime-order subgroup, on the CPU.  First facts about the cases of torsion_cases.py
(the torsion orders, the reference's period 8n, and cases that tell a reduction mod n from one mod 8n), then the
host-emulation builds of the `.curve` / `ec` kernel bodies -- Point.mul, mulAdd, KeyPair.derive, EC.verify, and the
curve25519 ladder -- against the oracle on every case."""
import ctypes

import pytest

import torsion_cases as tc
from test_hostemu_k256 import he  # noqa: F401  (the host-emulation library fixture)
from torsion_cases import mul_cases, verify_items

N8 = 8 * tc.N


@pytest.fixture(scope="module")
def ec():
    from oracle.ref_py.ec import EC
    return EC("ed25519")


def _xy(pt):
    return pt.get_x(), pt.get_y()


def _pts(pts):
    return b"".join(x.to_bytes(32, "big") + y.to_bytes(32, "big") for x, y in pts)


def _rows(buf, width, n):
    return [int.from_bytes(bytes(buf[width * i:width * (i + 1)]), "big") for i in range(n)]


def test_torsion_orders(ec):
    tors = tc.torsion()
    assert sorted(o for o, _ in tors) == [1, 2, 4, 4, 8, 8, 8, 8] and len({pt for _, pt in tors}) == 8
    for order, T in tors:
        assert tc.on_curve(T) and tc.small_order(T) == order
        Tp = ec.curve.point(*T)
        assert Tp.validate() and _xy(Tp.mul(order)) == tc.O
        assert order == 1 or _xy(Tp.mul(order // 2)) != tc.O
    for d, order, Q in tc.mixed():
        assert tc.on_curve(Q) and tc.small_order(tc.mul(tc.N, Q)) == order
        assert (tc.mul(tc.N, Q) == tc.O) == (order == 1)
    for kind, u in tc.x25519_us():
        if kind == "small":
            assert u in (0, 1, tc.P - 1) or tc.small_order(tc.point_from_y((u - 1) * pow(u + 1, -1, tc.P) % tc.P)) == 8
        if kind == "plus_p":
            assert tc.P <= u < 2**256


def test_oracle_mul_has_period_8n_and_the_cases_split_mod_n(ec):
    """P.mul(k) == P.mul(k mod 8n) everywhere; for each torsion order 2, 4, 8 some case has P.mul(k) != P.mul(k mod n),
    so a body that reduces mod n cannot pass the comparisons below."""
    split = {1: 0, 2: 0, 4: 0, 8: 0}
    for order, pt in tc.points():
        Pp = ec.curve.point(*pt)
        for k in tc.scalars() + tc.wide_scalars():
            w = _xy(Pp.mul(k))
            assert w == _xy(Pp.mul(k % N8)) == tc.mul(k % N8, pt), (order, k)
            if w != _xy(Pp.mul(k % tc.N)):
                split[order] += 1
    assert split[1] == 0 and split[2] and split[4] and split[8], split


def test_ed_ec_mul_and_mul_add_bodies(he, ec):
    cases = mul_cases()
    m = len(cases)
    ks = [k for _, _, k in cases]
    k1s = ks[7:] + ks[:7]
    pts = _pts([pt for _, pt, _ in cases])
    out, st = (ctypes.c_uint8 * (64 * m))(), (ctypes.c_uint8 * m)()
    he.he_ed_ec_mul_add(ctypes.c_size_t(m), None, tc.be(ks), pts, 0, out, st)
    got = list(zip(_rows(out, 32, 2 * m)[0::2], _rows(out, 32, 2 * m)[1::2]))
    for i, (order, pt, k) in enumerate(cases):
        assert st[i] == 1 and got[i] == _xy(ec.curve.point(*pt).mul(k)), ("mul", order, k)
    he.he_ed_ec_mul_add(ctypes.c_size_t(m), tc.be(k1s), tc.be(ks), pts, 0, out, st)
    got = list(zip(_rows(out, 32, 2 * m)[0::2], _rows(out, 32, 2 * m)[1::2]))
    for i, (order, pt, k) in enumerate(cases):
        assert st[i] == 1 and got[i] == _xy(ec.g.mul_add(k1s[i], ec.curve.point(*pt), k)), ("mulAdd", order, k1s[i], k)


def test_ed_ec_derive_body(he, ec):
    """KeyPair.derive: the private key is reduced mod n at import (ec/key.js:76-82), then pub.mul(priv).getX()."""
    from oracle.ref_py.ec import KeyPair
    cases = mul_cases()
    m = len(cases)
    out, st = (ctypes.c_uint8 * (64 * m))(), (ctypes.c_uint8 * m)()
    he.he_ed_ec_mul_add(ctypes.c_size_t(m), None, tc.be([k for _, _, k in cases]), _pts([pt for _, pt, _ in cases]), 1, out, st)
    xs = _rows(out, 32, 2 * m)[0::2]
    for i, (order, pt, k) in enumerate(cases):
        assert st[i] == 1 and xs[i] == KeyPair(ec, priv=k).derive(ec.curve.point(*pt)), (order, k)


def test_ed_ec_verify_body_on_mixed_order_keys(he, ec):
    items = verify_items()
    m = len(items)
    e, r, s = (tc.be([it[j] for it in items]) for j in range(3))
    outcomes = []
    for fmt, key in ((0, lambda q: q[0].to_bytes(32, "big") + q[1].to_bytes(32, "big")),
                     (1, lambda q: tc.sec1(q, False)), (2, lambda q: tc.sec1(q, True))):
        keys = [key(it[3]) for it in items]
        st = (ctypes.c_uint8 * m)()
        he.he_ed_ec_verify(ctypes.c_size_t(m), e, r, s, b"".join(keys), fmt, st)
        for i, (ev, rv, sv, q, passes) in enumerate(items):
            ref = {"x": q[0], "y": q[1]} if fmt == 0 else keys[i]
            want = ec.verify(ev, {"r": rv, "s": sv}, ref, msg_bit_length=253)
            assert want == passes and st[i] == int(want), (fmt, i)
            outcomes.append(want)
    assert True in outcomes and False in outcomes


def test_x25519_bodies_on_small_mixed_noncanonical_and_twist_u(he):
    from oracle.ref_py.ec import EC
    from oracle.ref_py import curves
    from ed_items import x_expected
    ec25, c25 = EC("curve25519"), curves.get("curve25519").curve
    cases = [(kind, u, k) for kind, u in tc.x25519_us() for k in tc.scalars(randoms=1)]
    m = len(cases)
    ks, us = tc.be([k for _, _, k in cases]), tc.be([u for _, u, _ in cases])
    out, st = (ctypes.c_uint8 * (32 * m))(), (ctypes.c_uint8 * m)()
    he.he_x25519_mul(ctypes.c_size_t(m), ks, us, out, st)
    got = _rows(out, 32, m)
    for i, (kind, u, k) in enumerate(cases):
        assert st[i] == 1 and got[i] == c25.point(u, 1).mul(k).get_x(), ("mul", kind, u, k)
    privs = [k % ec25.n for _, _, k in cases]
    he.he_x25519_derive(ctypes.c_size_t(m), tc.be(privs), us, out, st)
    got = _rows(out, 32, m)
    for i, (kind, u, k) in enumerate(cases):
        assert (st[i], got[i]) == x_expected(ec25, c25, privs[i], u), ("derive", kind, u, k)
    assert {st[i] for i in range(m)} == {1, 5}
