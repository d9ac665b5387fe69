"""Kernel-body logic (recoding, tables, exceptional cases, status codes) run through the portable
C++ fallbacks of the .cuh headers on the CPU (tests/hostemu) and compared with the oracle.
The PTX paths themselves are covered by the -m gpu tests."""
import ctypes
import os
import sys
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**256 - 2**32 - 977
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
LAM = 0x5363ad4cc05c30e0a5261c028812645a122e22ea20816678df02967c1b23bd72


@pytest.fixture(scope="module")
def he():
    out = os.path.join(ROOT, "tests", "_hostemu")
    os.makedirs(out, exist_ok=True)
    lib = os.path.join(out, "libhostemu.so")
    src = os.path.join(ROOT, "tests", "hostemu", "hostemu.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", "-shared", "-fPIC", "-o", lib, src], check=True)
    return ctypes.CDLL(lib)


def L(x, k=8):
    return (ctypes.c_uint32 * k)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(k)])


def I(a, k=8):
    return sum(int(a[i]) << (32 * i) for i in range(k))


def test_field_ops(he):
    rnd = random.Random(1)
    edge = [0, 1, P - 1, P, P + 1, 2**256 - 1, 2**32 + 977, 2**256 - 2**32 - 978, 2**255]
    vals = edge + [rnd.randrange(2**256) for _ in range(60)]

    def op(o, a, b=0):
        out = (ctypes.c_uint32 * 8)()
        he.he_fe_op(o, L(a), L(b), out)
        return I(out)
    for a in vals:
        for b in vals[:12]:
            assert op(0, a, b) % P == a * b % P
            assert op(2, a, b) % P == (a + b) % P
            assert op(3, a, b) % P == (a - b) % P
        assert op(1, a) % P == a * a % P and op(4, a) % P == -a % P and op(6, a) == a % P
    for a in vals[:12]:
        assert op(7, a) % P == pow(a % P, P - 2, P)


def test_glv_split_is_odd_and_bounded(he):
    rnd = random.Random(2)
    for k in [0, 1, 2, N - 1, LAM, LAM + 1] + [rnd.randrange(N) for _ in range(500)]:
        m1, m2 = (ctypes.c_uint32 * 5)(), (ctypes.c_uint32 * 5)()
        n1, n2 = ctypes.c_int(), ctypes.c_int()
        he.he_glv(L(k), m1, ctypes.byref(n1), m2, ctypes.byref(n2))
        k1 = (2 * I(m1, 5) + 1) * (-1 if n1.value else 1)
        k2 = (2 * I(m2, 5) + 1) * (-1 if n2.value else 1)
        assert (k1 + k2 * LAM - k) % N == 0 and abs(k1) < 2**131 and abs(k2) < 2**131


def test_verify_pipeline_against_oracle(he):
    from oracle.ref_py.ec import EC
    from test_gpu_k256 import _edge_items, _expected
    ec = EC("secp256k1")
    W, E, B = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    he.he_gtab_dims(ctypes.byref(W), ctypes.byref(E), ctypes.byref(B))
    gtab = np.zeros(W.value * E.value * 16, np.uint32)
    he.he_gtab_fast(gtab.ctypes.data_as(ctypes.c_void_p))
    items = _edge_items(ec, random.Random(77))[::3] + _edge_items(ec, random.Random(78))[-9:]
    n = len(items)
    col = lambda k: b"".join(it[k].to_bytes(32, "big") for it in items)
    pub = b"".join(it[3].to_bytes(32, "big") + it[4].to_bytes(32, "big") for it in items)
    st = (ctypes.c_uint8 * n)()
    he.he_verify(ctypes.c_size_t(n), col(0), col(1), col(2), pub, gtab.ctypes.data_as(ctypes.c_void_p), st)
    assert [int(v) for v in st] == [_expected(ec, it) for it in items]


@pytest.mark.parametrize("name,cid,ln", [("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)])
def test_sw_verify_pipeline_against_oracle(he, name, cid, ln):
    from oracle.ref_py.ec import EC
    from sw_items import sw_edge_items, sw_expected
    ec = EC(name)
    items = sw_edge_items(ec, ln, seed=21, count=30 if ln < 66 else 12, ebits=520 if ln == 66 else None)
    n = len(items)
    col = lambda k: b"".join(it[k].to_bytes(ln, "big") for it in items)
    pub = b"".join(it[3].to_bytes(ln, "big") + it[4].to_bytes(ln, "big") for it in items)
    st = (ctypes.c_uint8 * n)()
    he.he_sw_verify(cid, ctypes.c_size_t(n), col(0), col(1), col(2), pub, st)
    assert [int(v) for v in st] == [sw_expected(ec, ln, it, replay=False) for it in items]


def test_ed25519_and_x25519_bodies_against_oracle(he):
    from oracle.ref_py.eddsa import EDDSA
    from oracle.ref_py.ec import EC
    from oracle.ref_py import curves
    from ed_items import ed_items, ed_expected, x_items, x_expected
    ed = EDDSA()
    items = ed_items(limit=20)
    n = len(items)
    cat = lambda k: b"".join(it[k] for it in items)
    h = b"".join(ed.hash_int(it[0], it[2], it[3]).to_bytes(32, "little") for it in items)
    st = (ctypes.c_uint8 * n)()
    he.he_ed25519_verify(ctypes.c_size_t(n), cat(0), cat(1), cat(2), h, st)
    assert [int(v) for v in st] == [ed_expected(ed, it) for it in items]
    ec, c = EC("curve25519"), curves.get("curve25519").curve
    its = x_items(ec.n, count=24)
    m = len(its)
    out, st = (ctypes.c_uint8 * (32 * m))(), (ctypes.c_uint8 * m)()
    he.he_x25519_derive(ctypes.c_size_t(m), b"".join(k.to_bytes(32, "big") for k, _ in its),
                        b"".join(x.to_bytes(32, "big") for _, x in its), out, st)
    for i, (k, x) in enumerate(its):
        assert (st[i], int.from_bytes(bytes(out[32 * i:32 * i + 32]), "big")) == x_expected(ec, c, k, x)


def test_recover_pub_key_body_against_oracle(he):
    from oracle.ref_py.ec import EC
    from rec_items import rec_items, rec_expected
    ec = EC("secp256k1")
    W, E, B = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    he.he_gtab_dims(ctypes.byref(W), ctypes.byref(E), ctypes.byref(B))
    gtab = np.zeros(W.value * E.value * 16, np.uint32)
    he.he_gtab_fast(gtab.ctypes.data_as(ctypes.c_void_p))
    items, truth = rec_items(ec, count=12)
    n = len(items)
    e = b"".join((it[0] % ec.n).to_bytes(32, "big") for it in items)
    r = b"".join((it[1] % 2**256).to_bytes(32, "big") for it in items)
    s = b"".join((it[2] % ec.n).to_bytes(32, "big") for it in items)
    out, st = (ctypes.c_uint8 * (64 * n))(), (ctypes.c_uint8 * n)()
    he.he_recover(ctypes.c_size_t(n), e, r, s, bytes(it[3] for it in items), gtab.ctypes.data_as(ctypes.c_void_p), out, st)
    for i, it in enumerate(items):
        pt = (int.from_bytes(bytes(out[64 * i:64 * i + 32]), "big"), int.from_bytes(bytes(out[64 * i + 32:64 * i + 64]), "big"))
        assert (st[i], pt if st[i] == 1 else None) == rec_expected(ec, it), i
        if i in truth:
            assert st[i] == 1 and pt == truth[i]


def test_sign_and_hash_bodies_against_oracle(he):
    """RFC 6979 signing body (HMAC-DRBG/SHA-256, fixed-base k*G, inversion chain) and EdDSA hashInt body."""
    import hashlib
    from oracle.ref_py.ec import EC
    from oracle.ref_py.eddsa import EDDSA
    from ed_items import ed_items
    ec = EC("secp256k1")
    W, E, B = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    he.he_gtab_dims(ctypes.byref(W), ctypes.byref(E), ctypes.byref(B))
    gtab = np.zeros(W.value * E.value * 16, np.uint32)
    he.he_gtab_fast(gtab.ctypes.data_as(ctypes.c_void_p))
    rnd = random.Random(5)
    items = [(rnd.randrange(ec.n), rnd.randrange(1, ec.n)) for _ in range(10)] + [(0, 1), (ec.n - 1, ec.n - 1)]
    n = len(items)
    e = b"".join(x.to_bytes(32, "big") for x, _ in items)
    d = b"".join(y.to_bytes(32, "big") for _, y in items)
    for canon in (0, 1):
        r, s = (ctypes.c_uint8 * (32 * n))(), (ctypes.c_uint8 * (32 * n))()
        rec, st = (ctypes.c_uint8 * n)(), (ctypes.c_uint8 * n)()
        he.he_sign(ctypes.c_size_t(n), e, d, canon, gtab.ctypes.data_as(ctypes.c_void_p), r, s, rec, st)
        for i, (ev, dv) in enumerate(items):
            sig = ec.sign(ev.to_bytes(32, "big"), dv, canonical=bool(canon))
            assert (int.from_bytes(bytes(r[32 * i:32 * i + 32]), "big"), int.from_bytes(bytes(s[32 * i:32 * i + 32]), "big"),
                    rec[i], st[i]) == (sig.r, sig.s, sig.recovery_param, 1)
    # the two-kernel pipeline (word-oriented DRBG, batched inversions) must give the same bytes, with and
    # without items routed through the literal retry loop
    items = items + [(rnd.randrange(ec.n), rnd.randrange(1, ec.n)) for _ in range(25)]
    n = len(items)
    e = b"".join(x.to_bytes(32, "big") for x, _ in items)
    d = b"".join(y.to_bytes(32, "big") for _, y in items)
    for canon, every in ((0, 0), (1, 0), (1, 5)):
        r, s = (ctypes.c_uint8 * (32 * n))(), (ctypes.c_uint8 * (32 * n))()
        rec, st = (ctypes.c_uint8 * n)(), (ctypes.c_uint8 * n)()
        he.he_sign_fast(ctypes.c_size_t(n), e, d, canon, gtab.ctypes.data_as(ctypes.c_void_p), r, s, rec, st, every)
        for i, (ev, dv) in enumerate(items):
            sig = ec.sign(ev.to_bytes(32, "big"), dv, canonical=bool(canon))
            assert (int.from_bytes(bytes(r[32 * i:32 * i + 32]), "big"), int.from_bytes(bytes(s[32 * i:32 * i + 32]), "big"),
                    rec[i], st[i]) == (sig.r, sig.s, sig.recovery_param, 1), (i, canon, every)
    ed = EDDSA()
    eit = ed_items(limit=16)
    m = len(eit)
    off = np.zeros(m + 1, np.uint64)
    off[1:] = np.cumsum([len(it[3]) for it in eit])
    h = (ctypes.c_uint8 * (32 * m))()
    he.he_ed25519_hash(ctypes.c_size_t(m), b"".join(it[0] for it in eit), b"".join(it[2] for it in eit),
                       b"".join(it[3] for it in eit), off.ctypes.data_as(ctypes.c_void_p), h)
    assert bytes(h) == b"".join(ed.hash_int(it[0], it[2], it[3]).to_bytes(32, "little") for it in eit)
    for nbytes in (0, 1, 55, 56, 63, 64, 111, 112, 127, 128, 129, 1000):
        msg = rnd.randbytes(nbytes)
        o = (ctypes.c_uint8 * 64)(); he.he_sha512(msg, ctypes.c_size_t(nbytes), o)
        assert bytes(o) == hashlib.sha512(msg).digest()
        o = (ctypes.c_uint8 * 32)(); he.he_sha256(msg, ctypes.c_size_t(nbytes), o)
        assert bytes(o) == hashlib.sha256(msg).digest()


@pytest.mark.parametrize("name,cid,ln", [("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)])
def test_sw_replay_matches_reference_schedule_point_for_point(he, name, cid, ln):
    """The off-curve replay (ecdsa_sw_replay.cuh) must land on the same Jacobian triple as the
    oracle's _wnaf_mul_add, not just the same verdict: the coordinates are compared exactly."""
    from oracle.ref_py.ec import EC
    ec = EC(name)
    n, p, k = ec.n, ec.curve.p, {32: 8, 48: 12, 66: 18, 24: 6, 28: 8}[ln]
    rnd = random.Random(9 + cid)
    cases = []
    for t in range(10):
        u1, u2 = rnd.randrange(n), rnd.randrange(n)
        x, y = rnd.randrange(p), rnd.randrange(p)
        if t == 0: u1 = 0
        if t == 1: u2 = 0
        if t == 2: y = 0
        if t == 3: x = 0
        if t == 4: x, y = ec.g.x, ec.g.y
        if t == 5: u1, u2 = 255, 3
        if t == 6: x, y, u1, u2 = ec.g.x, p - ec.g.y, 1, 1       # G + (-G)
        if t == 7: x, y, u1, u2 = ec.g.x, ec.g.y, 1, 1           # G + G through mixedAdd's dbl branch
        cases.append((u1, u2, x, y))
    for u1, u2, x, y in cases:
        ref = ec.g.jmul_add(u1, ec.curve.point(x, y), u2)
        out = (ctypes.c_uint32 * (3 * k))()
        he.he_sw_replay_jmuladd(cid, L(u1, k), L(u2, k), L(x, k), L(y, k), out)
        got = tuple(sum(int(out[c * k + i]) << (32 * i) for i in range(k)) for c in range(3))
        if ref.z % p == 0:
            assert got[2] == 0
        else:
            assert got == (ref.x % p, ref.y % p, ref.z % p), (u1, u2, x, y)


@pytest.mark.parametrize("name,cid,ln", [("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)])
def test_sw_replay_verdicts_for_off_curve_keys(he, name, cid, ln):
    from oracle.ref_py.ec import EC
    from sw_items import sw_off_curve_items
    ec = EC(name)
    items = sw_off_curve_items(ec, ln, seed=4, count=12 if ln < 66 else 6, ebits=520 if ln == 66 else None)
    n = len(items)
    col = lambda k: b"".join(it[k].to_bytes(ln, "big") for it in items)
    pub = b"".join(it[3].to_bytes(ln, "big") + it[4].to_bytes(ln, "big") for it in items)
    st = (ctypes.c_uint8 * n)()
    he.he_sw_replay_verify(cid, ctypes.c_size_t(n), col(0), col(1), col(2), pub, st)
    exp = [int(ec.verify(it[0], {"r": it[1], "s": it[2]}, {"x": it[3], "y": it[4]})) for it in items]
    assert [int(v) for v in st] == exp
    assert 1 in exp and 0 in exp


def mul_cases(ec, seed=3, bits=256):
    """(k1, k2, x, y) for Point.mul / mulAdd: ordinary, oversize, zero and cancelling scalars, P = +-G,
    off-curve points (short.js:251-271 never validates)."""
    rnd = random.Random(seed)
    n, p, G = ec.n, ec.curve.p, ec.g
    P1 = G.mul(rnd.randrange(1, n))
    cases = []
    for t in range(8):
        cases.append((rnd.randrange(n), rnd.randrange(n), P1.x, P1.y))
    d = rnd.randrange(1, n)
    Pd = G.mul(d)
    cases += [
        (0, 5, P1.x, P1.y), (7, 0, P1.x, P1.y), (0, 0, P1.x, P1.y),
        (n + 3 if n + 3 < 2**bits else 3, 2**bits - 1, P1.x, P1.y),                       # not reduced by the reference
        ((n - d * 9 % n) % n, 9, Pd.x, Pd.y),                  # k1*G + k2*P = O
        (5, 1, G.x, G.y), (5, n - 5, G.x, G.y), (1, 1, G.x, p - G.y),
        (rnd.randrange(n), rnd.randrange(n), rnd.randrange(p), rnd.randrange(p)),     # off-curve
        (rnd.randrange(n), rnd.randrange(n), 0, 0),
        (3, 2**bits - 5, rnd.randrange(p), rnd.randrange(p)),
    ]
    return cases


@pytest.mark.parametrize("name,cid,ln", [("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)])
def test_sw_mul_and_mul_add_bodies_against_oracle(he, name, cid, ln):
    from oracle.ref_py.ec import EC
    ec = EC(name)
    cases = mul_cases(ec, seed=6, bits=8 * ln)
    n = len(cases)
    k1 = b"".join(c[0].to_bytes(ln, "big") for c in cases)
    k2 = b"".join(c[1].to_bytes(ln, "big") for c in cases)
    pts = b"".join(c[2].to_bytes(ln, "big") + c[3].to_bytes(ln, "big") for c in cases)

    def unpack(out, st):
        return [(int.from_bytes(bytes(out[2 * ln * i:2 * ln * i + ln]), "big"), int.from_bytes(bytes(out[2 * ln * i + ln:2 * ln * (i + 1)]), "big"))
                if st[i] == 1 else None for i in range(n)]

    ref = lambda pt: None if pt.is_infinity() else (pt.get_x(), pt.get_y())
    out = (ctypes.c_uint8 * (2 * ln * n))(); st = (ctypes.c_uint8 * n)()
    he.he_sw_mul_add(cid, ctypes.c_size_t(n), k1, k2, pts, out, st)
    assert unpack(out, st) == [ref(ec.g.mul_add(c[0], ec.curve.point(c[2], c[3]), c[1])) for c in cases]
    assert set(st) == {1, 7}
    he.he_sw_mul_add(cid, ctypes.c_size_t(n), None, k2, pts, out, st)
    assert unpack(out, st) == [ref(ec.curve.point(c[2], c[3]).mul(c[1])) for c in cases]
    he.he_sw_mul_add(cid, ctypes.c_size_t(n), None, k2, None, out, st)
    assert unpack(out, st) == [ref(ec.g.mul(c[1])) for c in cases]


def test_mul_and_mul_add_bodies_against_oracle(he):
    from oracle.ref_py.ec import EC
    ec = EC("secp256k1")
    W, E, B = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    he.he_gtab_dims(ctypes.byref(W), ctypes.byref(E), ctypes.byref(B))
    gtab = np.zeros(W.value * E.value * 16, np.uint32)
    he.he_gtab_fast(gtab.ctypes.data_as(ctypes.c_void_p))
    gp = gtab.ctypes.data_as(ctypes.c_void_p)
    cases = mul_cases(ec)
    n = len(cases)
    k1 = b"".join(c[0].to_bytes(32, "big") for c in cases)
    k2 = b"".join(c[1].to_bytes(32, "big") for c in cases)
    pts = b"".join(c[2].to_bytes(32, "big") + c[3].to_bytes(32, "big") for c in cases)

    def unpack(out, st):
        return [(int.from_bytes(bytes(out[64 * i:64 * i + 32]), "big"), int.from_bytes(bytes(out[64 * i + 32:64 * i + 64]), "big"))
                if st[i] == 1 else None for i in range(n)]

    def ref(pt):
        return None if pt.is_infinity() else (pt.get_x(), pt.get_y())

    out = (ctypes.c_uint8 * (64 * n))(); st = (ctypes.c_uint8 * n)()
    he.he_mul_add(ctypes.c_size_t(n), k1, k2, pts, gp, out, st)
    assert unpack(out, st) == [ref(ec.g.mul_add(c[0], ec.curve.point(c[2], c[3]), c[1])) for c in cases]
    assert set(st) == {1, 7}
    he.he_mul_add(ctypes.c_size_t(n), None, k2, pts, gp, out, st)
    assert unpack(out, st) == [ref(ec.curve.point(c[2], c[3]).mul(c[1])) for c in cases]
    he.he_mul_g(ctypes.c_size_t(n), k2, gp, out, st)
    assert unpack(out, st) == [ref(ec.g.mul(c[1])) for c in cases]


def der_corpus(seed=4, count=400):
    """Valid DER signatures, single-bit corruptions, truncations, long-form lengths, oversize integers."""
    from oracle.ref_py.signature import Signature
    rnd = random.Random(seed)
    out = []
    for t in range(count):
        r = rnd.randrange(1, 2 ** rnd.choice([1, 8, 64, 255, 256, 257, 384, 520]))
        s = rnd.randrange(1, 2 ** rnd.choice([8, 128, 256, 300]))
        der = bytearray(Signature({"r": r, "s": s}).to_der())
        k = t % 8
        if k == 1: der[rnd.randrange(len(der))] ^= 1 << rnd.randrange(8)
        if k == 2: der = der[:rnd.randrange(len(der))]
        if k == 3: der += bytes([rnd.randrange(256)])
        if k == 4: der[1:2] = bytes([0x81, der[1]])                        # long form where short is required
        if k == 5: der = bytearray(b"\x30\x06\x02\x01\x00\x02\x01\x01")     # r = 0
        if k == 6: der = bytearray(rnd.randbytes(rnd.randrange(0, 12)))
        out.append(bytes(der))
    out += [b"", b"\x30", b"\x30\x00", b"\x30\x02\x02\x00", b"\x30\x04\x02\x00\x02\x00",
            b"\x30\x84\x00\x00\x00\x08\x02\x02\x00\x80\x02\x02\x00\x81", b"\x30\x81\x88" + b"\x02\x41\x00" + b"\xff" * 64 + b"\x02\x41\x00" + b"\x80" * 64]
    return out


def ref_der(der):
    from oracle.ref_py.signature import Signature
    chk = Signature.__new__(Signature)
    return (chk.r, chk.s) if chk._import_der(der, None) else None


def test_der_import_body_matches_reference(he):
    corpus = der_corpus()
    kinds = set()
    for der in corpus:
        want = ref_der(der)
        for ln in (32, 48):
            r, s = (ctypes.c_uint8 * ln)(), (ctypes.c_uint8 * ln)()
            ok = he.he_der_import(der, ctypes.c_size_t(len(der)), ctypes.c_size_t(ln), r, s)
            assert bool(ok) == (want is not None), der.hex()
            if want:
                fit = lambda v: v if v < 2 ** (8 * ln) else 0
                assert (int.from_bytes(bytes(r), "big"), int.from_bytes(bytes(s), "big")) == (fit(want[0]), fit(want[1])), der.hex()
        kinds.add(want is not None)
    assert kinds == {True, False}


@pytest.mark.parametrize("name,cid,ln", [("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)])
def test_sw_sign_pipeline_against_oracle(he, name, cid, ln):
    """EC.sign on p256 (HMAC-DRBG/SHA-256) and p384 (SHA-384): r, s, recoveryParam equal the oracle's, with and
    without `canonical`, and with items routed through the literal retry loop."""
    from oracle.ref_py.ec import EC
    ec = EC(name)
    rnd = random.Random(15 + cid)
    cnt = 18 if ln < 66 else 8
    # e is what _truncateToN hands to sign(): below n; kept below 2^(bits(n) - 1) so that passing it back to the
    # oracle as a BN is not shortened a second time (p521)
    lim = min(ec.n, 2 ** (ec.n.bit_length() - 1))
    items = [(rnd.randrange(lim), rnd.randrange(1, ec.n)) for _ in range(cnt)] + [(0, 1), (lim - 1, ec.n - 1)]
    n = len(items)
    e = b"".join(x.to_bytes(ln, "big") for x, _ in items)
    d = b"".join(y.to_bytes(ln, "big") for _, y in items)
    for canon, every in ((0, 0), (1, 0), (1, 4)):
        r, s = (ctypes.c_uint8 * (ln * n))(), (ctypes.c_uint8 * (ln * n))()
        rec, st = (ctypes.c_uint8 * n)(), (ctypes.c_uint8 * n)()
        he.he_sw_sign(cid, ctypes.c_size_t(n), e, d, canon, r, s, rec, st, every)
        for i, (ev, dv) in enumerate(items):
            sig = ec.sign(ev, dv, canonical=bool(canon))
            assert (int.from_bytes(bytes(r[ln * i:ln * i + ln]), "big"), int.from_bytes(bytes(s[ln * i:ln * i + ln]), "big"),
                    rec[i], st[i]) == (sig.r, sig.s, sig.recovery_param, 1), (i, canon, every)


@pytest.mark.parametrize("name,cid,ln", [("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)])
def test_sw_recover_pub_key_body_against_oracle(he, name, cid, ln):
    from oracle.ref_py.ec import EC
    from rec_items import rec_items, rec_expected
    ec = EC(name)
    items, truth = rec_items(ec, count=6 if ln < 66 else 3)
    n = len(items)
    e = b"".join((it[0] % ec.n).to_bytes(ln, "big") for it in items)
    r = b"".join(it[1].to_bytes(ln, "big") for it in items)
    s = b"".join((it[2] % ec.n).to_bytes(ln, "big") for it in items)
    out, st = (ctypes.c_uint8 * (2 * ln * n))(), (ctypes.c_uint8 * n)()
    he.he_sw_recover(cid, ctypes.c_size_t(n), e, r, s, bytes(it[3] for it in items), out, st)
    seen = set()
    for i, it in enumerate(items):
        pt = (int.from_bytes(bytes(out[2 * ln * i:2 * ln * i + ln]), "big"), int.from_bytes(bytes(out[2 * ln * i + ln:2 * ln * (i + 1)]), "big"))
        assert (st[i], pt if st[i] == 1 else None) == rec_expected(ec, it), i
        if i in truth:
            assert st[i] == 1 and pt == truth[i]
        seen.add(int(st[i]))
    assert {1, 8} <= seen and (7 in seen or name == "p224") and (2 in seen or 5 in seen)      # p224: bn.js's Tonelli-Shanks asserts on a non-residue


@pytest.mark.parametrize("name,cid,k", [("p256", 2, 8), ("p224", 8, 8), ("p192", 7, 6)])
def test_sw_sqrt_matches_bn_js_red_sqrt(he, name, cid, k):
    """Red.prototype.sqrt (dist:7177-7232) as pointFromX uses it: the same candidate root for residues, and for
    non-residues garbage (p = 3 mod 4) or the 'Assertion failed' throw (p224, Tonelli-Shanks)."""
    from oracle.ref_py import curves
    from oracle.ref_py.bn import RefError
    red = curves.get(name).curve.red
    p = curves.get(name).curve.p
    rnd = random.Random(40 + cid)
    vals = [0, 1, 4, p - 1] + [rnd.randrange(p) for _ in range(24)] + [pow(rnd.randrange(1, p), 2, p) for _ in range(8)]
    seen = set()
    for a in vals:
        out = (ctypes.c_uint32 * k)()
        st = he.he_sw_sqrt(cid, L(a, k), out)
        try:
            want = (0, red.sqrt(a))
        except RefError as ex:
            assert str(ex) == "Assertion failed"
            want = (5, None)
        got = (st, I(out, k) if st == 0 else None)
        assert got == want, (name, hex(a))
        seen.add(st)
    assert 0 in seen and (name != "p224" or 5 in seen)


def test_der_import_fuzz_with_hypothesis(he):
    """Structured fuzzing of the DER importer against the oracle: arbitrary byte strings, and valid encodings with a
    slice replaced, must be accepted / rejected identically and yield the same integers."""
    from hypothesis import given, settings, strategies as st
    from oracle.ref_py.signature import Signature

    def check(der):
        want = ref_der(der)
        r, s = (ctypes.c_uint8 * 32)(), (ctypes.c_uint8 * 32)()
        ok = he.he_der_import(der, ctypes.c_size_t(len(der)), ctypes.c_size_t(32), r, s)
        assert bool(ok) == (want is not None), der.hex()
        if want:
            fit = lambda v: v if v < 2 ** 256 else 0
            assert (int.from_bytes(bytes(r), "big"), int.from_bytes(bytes(s), "big")) == (fit(want[0]), fit(want[1])), der.hex()

    @settings(max_examples=400, deadline=None)
    @given(st.binary(max_size=80))
    def arbitrary(der):
        check(der)

    @settings(max_examples=400, deadline=None)
    @given(st.integers(1, 2 ** 264), st.integers(1, 2 ** 256), st.integers(0, 79), st.binary(max_size=4))
    def spliced(r, s, pos, patch):
        der = bytearray(Signature({"r": r, "s": s}).to_der())
        pos %= len(der)
        der[pos:pos + len(patch)] = patch
        check(bytes(der))

    arbitrary()
    spliced()


# ---------------------------------------------------------------------------------------------
# carry-free 9 x 29-bit field (fq_pm.cuh) and the group law on it (gq_k256.cuh)
P25 = 2**255 - 19


def _fq(he, which, o, a, b=0):
    out = (ctypes.c_uint32 * 8)()
    he.he_fq_op(which, o, L(a), L(b), out)
    return I(out)


@pytest.mark.parametrize("which,p", [(0, P), (1, P25)])
def test_fq_field_ops(he, which, p):
    rnd = random.Random(11 + which)
    top = 2**256 - 1
    edge = [0, 1, 2, p - 1, p, p + 1, top, top - 1, 2**255, 2**255 - 1, 2**232, 2**232 - 1, 2**261 % p,
            (1 << 256) - (1 << 29), sum((2**29 - 1) << (29 * i) for i in range(0, 9, 2)) % 2**256,
            sum(1 << (29 * i) for i in range(9)) % 2**256, 2**32 + 977, p - (2**32 + 977), 19, p - 19]
    vals = edge + [rnd.randrange(2**256) for _ in range(80)]
    for a in vals:
        for b in vals[:24]:
            assert _fq(he, which, 0, a, b) == a * b % p
            assert _fq(he, which, 2, a, b) == (a + b) % p
            assert _fq(he, which, 3, a, b) == (a - b) % p
            assert _fq(he, which, 9, a, b) == (3 * a - 2 * b) % p
            assert _fq(he, which, 11, a, b) == 6 * a * b % p         # lazy operands of magnitude 3 and 2
            assert _fq(he, which, 12, a, b) == (a + b) ** 2 % p
            assert _fq(he, which, 10, a, b) == int((a - b) % p == 0)
        assert _fq(he, which, 1, a) == a * a % p
        assert _fq(he, which, 4, a) == -a % p
        assert _fq(he, which, 6, a) == a % p
        assert _fq(he, which, 13, a, 1) == -a % p and _fq(he, which, 13, a, 0) == a % p
    # values congruent mod p compare equal
    for a in vals[:20]:
        if a + p < 2**256:
            assert _fq(he, which, 10, a + p, a) == 1


def test_gq_group_law_matches_packed_field(he):
    """gq_dbl / gq_madd (carry-free field) against plain integer formulas, incl. the exceptional cases."""
    from oracle.ref_py.ec import EC
    ec = EC("secp256k1")
    rnd = random.Random(5)

    def to_aff(X, Y, Z):
        if Z % P == 0:
            return None
        zi = pow(Z, -1, P)
        return X * zi * zi % P, Y * zi ** 3 % P

    def run(op, jac, aff):
        j = (ctypes.c_uint32 * 24)(*[(c >> (32 * i)) & 0xFFFFFFFF for c in jac for i in range(8)])
        a = (ctypes.c_uint32 * 16)(*[(c >> (32 * i)) & 0xFFFFFFFF for c in aff for i in range(8)])
        out = (ctypes.c_uint32 * 24)()
        he.he_gq_op(op, j, a, out)
        return [sum(int(out[8 * k + i]) << (32 * i) for i in range(8)) for k in range(3)]

    for _ in range(40):
        k1, k2, z = rnd.randrange(1, N), rnd.randrange(1, N), rnd.randrange(1, P)
        p1, p2 = ec.g.mul(k1), ec.g.mul(k2)
        jac = (p1.x * z * z % P, p1.y * z ** 3 % P, z)
        d = p1.dbl()
        assert to_aff(*run(0, jac, (p2.x, p2.y))) == (d.x, d.y)
        s = p1.add(p2)
        assert to_aff(*run(1, jac, (p2.x, p2.y))) == (s.x, s.y)
        # P + P, P + (-P), O + P through the cold path
        assert to_aff(*run(1, jac, (p1.x, p1.y))) == (d.x, d.y)
        assert to_aff(*run(1, jac, (p1.x, P - p1.y))) is None
        assert to_aff(*run(1, (1, 1, 0), (p2.x, p2.y))) == (p2.x, p2.y)
        assert to_aff(*run(0, (1, 1, 0), (p2.x, p2.y))) is None


@pytest.mark.parametrize("cid,nl,p", [
    (2, 8, 2**256 - 2**224 + 2**192 + 2**96 - 1), (3, 12, 2**384 - 2**128 - 2**96 + 2**32 - 1), (6, 18, 2**521 - 1),
    (7, 6, 2**192 - 2**64 - 1), (8, 8, 2**224 - 2**96 + 1)])
def test_sw_coordinate_field_ops(he, cid, nl, p):
    """F::{mul, sqr, add, sub, neg, inv, toRed} of every short preset on values that stress the word-level
    reductions of fp_special.cuh (all-ones / all-zero word patterns, p - small, values >= p)."""
    rnd = random.Random(100 + cid)
    bits = 32 * nl if cid != 6 else 528          # p521: what a 66-byte wire value can hold
    top = 2**bits - 1
    words = [0, 0xFFFFFFFF, 1, 0xFFFFFFFE, 0x80000000]
    pats = [sum(rnd.choice(words) << (32 * i) for i in range(nl)) & top for _ in range(60)]
    edge = [0, 1, 2, p - 1, p - 2, p, p + 1, top, top - 1, 2**(p.bit_length() - 1), (p + 1) // 2, 2**32, 2**96 - 1, 2**224, p - 2**96]
    vals = [v & top for v in edge] + pats + [rnd.randrange(2**bits) for _ in range(60)]

    def op(o, a, b=0):
        out = (ctypes.c_uint32 * nl)()
        he.he_sw_fe_op(cid, o, L(a, nl), L(b, nl), out)
        return I(out, nl)
    for a in vals:
        for b in vals[:20] + pats[:8]:
            assert op(0, a, b) == a * b % p, (hex(a), hex(b))
            assert op(2, a, b) == (a + b) % p
            assert op(3, a, b) == (a - b) % p
        assert op(1, a) == a * a % p, hex(a)
        assert op(10, a) == 8 * a * a % p, hex(a)
        for b in vals[:6]:
            assert op(8, a, b) == 3 * a * b % p and op(9, a, b) == 4 * a * b % p, (hex(a), hex(b))
        assert op(4, a) == -a % p and op(6, a) == a % p
    for a in vals[:10]:
        assert op(7, a) == pow(a % p, p - 2, p)


@pytest.mark.parametrize("cid,name", [(2, "P256"), (3, "P384")])
def test_solinas_reduction_rare_branches(he, cid, name):
    """The column-wise reductions (tools/gen_solinas.py) keep two steps in branches that random products almost never
    take: the second fold (the first fold wrapped 2^(32N), in either direction) and the final subtraction (result's top
    limb all ones).  Inputs are built with the generator's integer model to land in each of them and checked against
    integer arithmetic; the model also counts how often each branch was really taken."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_solinas as g
    cfg = getattr(g, name)
    nl = cfg["N"]
    p = {"P256": 2**256 - 2**224 + 2**192 + 2**96 - 1, "P384": 2**384 - 2**128 - 2**96 + 2**32 - 1}[name]
    R = 2**(32 * nl)
    K = sum(d << (32 * j) for j, d in cfg["K"].items())
    cols = g.columns(cfg)
    rnd = random.Random(7 + cid)

    def model(c):                      # (top, top2) of the generated code's two folds
        tot = sum(coef * c[i] << (32 * j) for j, col in enumerate(cols) for i, coef in col.items())
        top, w = tot >> (32 * nl), tot & (R - 1)
        return top, (w + top * K) >> (32 * nl)

    cases = []
    for _ in range(400):
        hi = [rnd.choice([0, 0xFFFFFFFF, rnd.randrange(2**32)]) for _ in range(nl)]
        F = sum(coef * hi[i - nl] << (32 * j) for j, col in enumerate(cols) for i, coef in col.items() if i >= nl)
        for w in (rnd.randrange(3 * K), R - 1 - rnd.randrange(3 * K), rnd.randrange(K), R - 1 - rnd.randrange(K), p + rnd.randrange(-4, 4) if True else 0):
            lo = (w - F) % R           # the low half enters every column with coefficient 1: w = (lo + F) mod R
            cases.append([(lo >> (32 * i)) & 0xFFFFFFFF for i in range(nl)] + hi)
    for v in (0, R - 1, R * R - 1, (p - 1) ** 2, p * p - 1, (R - 1) * R, R, p, p - 1, R + p, (R - 1) * (R - 1)):
        cases.append([(v >> (32 * i)) & 0xFFFFFFFF for i in range(2 * nl)])
    cases += [[rnd.randrange(2**32) for _ in range(2 * nl)] for _ in range(300)]
    seen = {-1: 0, 0: 0, 1: 0}
    hit_top = 0
    for c in cases:
        v = sum(x << (32 * i) for i, x in enumerate(c))
        out = (ctypes.c_uint32 * nl)()
        he.he_solinas_reduce(cid, (ctypes.c_uint32 * (2 * nl))(*c), 1, out)
        got = I(out, nl)
        assert got == v % p, hex(v)
        seen[model(c)[1]] += 1
        hit_top += got >> (32 * (nl - 1)) == 0xFFFFFFFF
    # the scaled forms (3 a b, 4 a b, 8 a^2 of the doubling): same inputs, the factor applied inside the column sums
    for k in (3, 4, 8):
        for c in cases[::3]:
            v = sum(x << (32 * i) for i, x in enumerate(c))
            out = (ctypes.c_uint32 * nl)()
            he.he_solinas_reduce(cid, (ctypes.c_uint32 * (2 * nl))(*c), k, out)
            assert I(out, nl) == k * v % p, (k, hex(v))
    # p384: the word sums leave the top in [-1, 3] and a negative top cannot coincide with a low part below K, so
    # the downward wrap exists only for p256 (top in [-4, 4])
    assert seen[1] > 50 and seen[0] > 300 and (seen[-1] > 50 if name == "P256" else seen[-1] == 0), seen
    assert hit_top > 20            # the final-subtraction branch was exercised (and not taken blindly)


def test_eddsa_sign_body_reproduces_sign_input(he):
    """EDDSA.sign (eddsa/index.js:34-44) through the kernel body: byte-identical signatures and public keys for the
    reference's own test/fixtures/sign.input vectors (message lengths 0..1023)."""
    import gzip
    import json
    data = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "ed25519_sign_input.json.gz"), "rt"))
    vecs = data["vectors"][:40] + data["vectors"][-12:]
    n = len(vecs)
    sec = b"".join(bytes.fromhex(v["secret"]) for v in vecs)
    msgs = [bytes.fromhex(v["msg"]) for v in vecs]
    off = (ctypes.c_uint64 * (n + 1))(*np.concatenate([[0], np.cumsum([len(m) for m in msgs])]).astype(np.uint64))
    sig, pub = (ctypes.c_uint8 * (64 * n))(), (ctypes.c_uint8 * (32 * n))()
    he.he_ed25519_sign(ctypes.c_size_t(n), sec, b"".join(msgs) + b"\x00", off, sig, pub)
    for i, v in enumerate(vecs):
        assert bytes(sig[64 * i:64 * i + 64]).hex() == v["sig"], v["i"]
        assert bytes(pub[32 * i:32 * i + 32]).hex() == v["pk"], v["i"]


@pytest.mark.parametrize("name,cid,ln", [("secp256k1", 1, 32), ("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)])
def test_sign_options_and_keygen_bodies_against_oracle(he, name, cid, ln):
    """EC.sign with options.k / options.pers (ec/index.js:143-157) and EC.genKeyPair({entropy, pers}) (:55-79)
    through the kernel bodies, against the oracle."""
    from oracle.ref_py.ec import EC
    ec = EC(name)
    n_ord = ec.n
    rnd = random.Random(300 + cid)
    W, E, B = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    he.he_gtab_dims(ctypes.byref(W), ctypes.byref(E), ctypes.byref(B))
    gtab = np.zeros(W.value * E.value * 16, np.uint32)
    if cid == 1:
        he.he_gtab_fast(gtab.ctypes.data_as(ctypes.c_void_p))
    cnt = 10 if ln < 66 else 5
    privs = [rnd.randrange(1, n_ord) for _ in range(cnt)]
    es = [rnd.randrange(min(n_ord, 1 << (8 * ln - 8))) for _ in range(cnt)]     # not shortened by _truncateToN (p521)
    col = lambda vals: b"".join(v.to_bytes(ln, "big") for v in vals)
    outs = lambda: ((ctypes.c_uint8 * (ln * cnt))(), (ctypes.c_uint8 * (ln * cnt))(), (ctypes.c_uint8 * cnt)(), (ctypes.c_uint8 * cnt)())
    # ---- pers
    for pers in (b"", b"my.pers", bytes(range(200))):
        for canon in (0, 1):
            r, s, rec, st = outs()
            he.he_sign_opt(cid, 1, ctypes.c_size_t(cnt), col(es), col(privs), None, pers + b"\x00", len(pers), canon,
                           gtab.ctypes.data_as(ctypes.c_void_p), r, s, rec, st)
            for i in range(cnt):
                sig = ec.sign(es[i], privs[i], canonical=bool(canon), pers=pers)
                assert st[i] == 1
                assert int.from_bytes(bytes(r[ln * i:ln * i + ln]), "big") == sig.r, (name, i)
                assert int.from_bytes(bytes(s[ln * i:ln * i + ln]), "big") == sig.s and rec[i] == sig.recovery_param
    # ---- caller nonces: a good k, then the loop's reject cases (k <= 1, k >= n - 1) which come back as RETRY (10)
    ks = [rnd.randrange(2, n_ord - 1) for _ in range(cnt)]
    ks[1], ks[2], ks[3] = 1, n_ord - 1, 0
    if ln == 66:
        ks[4] = (rnd.randrange(2, n_ord - 1) << 7) | 0x55           # 528-bit value: _truncateToN(k, true) shifts it by 7
    r, s, rec, st = outs()
    he.he_sign_opt(cid, 0, ctypes.c_size_t(cnt), col(es), col(privs), col(ks), None, 0, 0, gtab.ctypes.data_as(ctypes.c_void_p), r, s, rec, st)
    for i in range(cnt):
        calls = []

        def kf(it, i=i, calls=calls):
            calls.append(it)
            return ks[i] if it == 0 else ec.n - 5 - i
        sig = ec.sign(es[i], privs[i], k_fn=kf)
        if len(calls) == 1:
            assert st[i] == 1 and int.from_bytes(bytes(r[ln * i:ln * i + ln]), "big") == sig.r
            assert int.from_bytes(bytes(s[ln * i:ln * i + ln]), "big") == sig.s and rec[i] == sig.recovery_param
        else:
            assert st[i] == 10, (name, i, st[i])
    # (p521: n - 1 is a 521-bit value, so _truncateToN(k, true) shifts it by 7 and the reference accepts it)
    assert st[1] == 10 and (st[2] == 10 or ln == 66) and st[3] == 10 and st[0] == 1
    # ---- genKeyPair({entropy, pers})
    for ne, pers in ((24, b""), (32, b""), (48, b"key-pers")):
        ents = [bytes(rnd.randrange(256) for _ in range(ne)) for _ in range(cnt)]
        out, st8 = (ctypes.c_uint8 * (ln * cnt))(), (ctypes.c_uint8 * cnt)()
        he.he_keygen(cid, ctypes.c_size_t(cnt), b"".join(ents), ne, pers + b"\x00", len(pers), out, st8)
        for i in range(cnt):
            assert st8[i] == 1
            assert int.from_bytes(bytes(out[ln * i:ln * i + ln]), "big") == ec.gen_key_pair(ents[i], pers).priv, (name, ne, i)


def test_ec_api_over_ed25519_bodies_against_oracle(he):
    """new elliptic.ec('ed25519') (test/ecdsa-test.js:130, test/ecdh-test.js:26): verify (eqXToP with up to eight
    candidates), SEC1 keys incl. EdwardsCurve.pointFromX, sign (default / canonical / pers / k), genKeyPair, Point.mul /
    mulAdd and KeyPair.derive through the kernel bodies, against the oracle."""
    from oracle.ref_py.bn import RefError
    from oracle.ref_py.ec import EC, KeyPair
    ec = EC("ed25519")
    n_ord, p = ec.n, ec.curve.p
    rnd = random.Random(900)
    cnt = 24
    privs = [rnd.randrange(1, n_ord) for _ in range(cnt)]
    pubs = [ec.g.mul(d) for d in privs]
    es = [rnd.randrange(1 << 248) for _ in range(cnt)]
    col = lambda vals: b"".join(v.to_bytes(32, "big") for v in vals)
    # ---- sign: default, canonical, pers; then caller nonces
    sigs = []
    for pers in (b"", b"1234"):
        for canon in (0, 1):
            r, s = (ctypes.c_uint8 * (32 * cnt))(), (ctypes.c_uint8 * (32 * cnt))()
            rec, st = (ctypes.c_uint8 * cnt)(), (ctypes.c_uint8 * cnt)()
            he.he_ed_ec_sign(ctypes.c_size_t(cnt), col(es), col(privs), None, pers + b"\x00", len(pers), canon, r, s, rec, st)
            for i in range(cnt):
                sig = ec.sign(es[i], privs[i], canonical=bool(canon), pers=pers)
                got = (int.from_bytes(bytes(r[32 * i:32 * i + 32]), "big"), int.from_bytes(bytes(s[32 * i:32 * i + 32]), "big"), rec[i])
                assert st[i] == 1 and got == (sig.r, sig.s, sig.recovery_param), i
                if not pers and not canon:
                    sigs.append(sig)
    ks = [rnd.randrange(2, n_ord - 1) for _ in range(cnt)]
    ks[0], ks[1], ks[2], ks[3] = 1358, 1, n_ord - 1, (rnd.randrange(2, n_ord - 1) << 3) | 5      # 256-bit value: shifted by 3
    r, s = (ctypes.c_uint8 * (32 * cnt))(), (ctypes.c_uint8 * (32 * cnt))()
    rec, st = (ctypes.c_uint8 * cnt)(), (ctypes.c_uint8 * cnt)()
    he.he_ed_ec_sign(ctypes.c_size_t(cnt), col(es), col(privs), col(ks), None, 0, 0, r, s, rec, st)
    for i in range(cnt):
        calls = []
        sig = ec.sign(es[i], privs[i], k_fn=lambda it, i=i, calls=calls: (calls.append(it), ks[i] if it == 0 else 77 + i)[1])
        if len(calls) == 1:
            assert st[i] == 1 and int.from_bytes(bytes(r[32 * i:32 * i + 32]), "big") == sig.r and int.from_bytes(bytes(s[32 * i:32 * i + 32]), "big") == sig.s
        else:
            assert st[i] == 10
    assert st[1] == 10 and st[0] == 1          # (n - 1 is a 32-byte value: _truncateToN(k, true) shifts it by 3 and the loop accepts it)
    # ---- verify: valid, wrong key, flipped bits, range failures, off-curve key, SEC1 forms
    items = []
    for i in range(cnt):
        e, rr, ss, q = es[i], sigs[i].r, sigs[i].s, pubs[i]
        k = i % 8
        if k == 1: e ^= 1 << rnd.randrange(240)
        if k == 2: rr ^= 1 << rnd.randrange(250)
        if k == 3: ss = n_ord - ss
        if k == 4: q = pubs[(i + 1) % cnt]
        if k == 5: rr = 0
        if k == 6: ss = n_ord
        items.append((e, rr, ss, q.get_x(), q.get_y()))
    items.append((es[0], sigs[0].r, sigs[0].s, pubs[0].get_x(), (pubs[0].get_y() + 1) % p))       # off the curve
    m = len(items)
    stv = (ctypes.c_uint8 * m)()
    he.he_ed_ec_verify(ctypes.c_size_t(m), col([t[0] for t in items]), col([t[1] for t in items]), col([t[2] for t in items]),
                       b"".join(t[3].to_bytes(32, "big") + t[4].to_bytes(32, "big") for t in items), 0, stv)
    for j, (e, rr, ss, x, y) in enumerate(items[:-1]):
        want = int(ec.verify(e, {"r": rr, "s": ss}, {"x": x, "y": y})) if 1 <= rr < n_ord and 1 <= ss < n_ord else 0
        assert stv[j] == want, j
    assert stv[m - 1] == 4 and 1 in list(stv) and 0 in list(stv)
    assert sum(1 for sg in sigs if sg.recovery_param & 2) > cnt // 2       # x(R) >= n: the multi-candidate loop is live
    # compressed / uncompressed / hybrid keys through decodePoint + pointFromX
    for fmt, size in ((2, 33), (1, 65)):
        keys, exp = [], []
        for i in range(cnt):
            x, y = pubs[i].get_x(), pubs[i].get_y()
            if fmt == 2:
                tag = 3 if y & 1 else 2
                if i % 6 == 5: tag ^= 1                                     # other root: a different (valid) point
                if i % 6 == 4: tag = 5
                kb = bytes([tag]) + (x if i % 6 != 3 else (x + 1) % p).to_bytes(32, "big")
            else:
                tag = [4, 6 if y % 2 == 0 else 7, 7 if y % 2 == 0 else 6, 9][i % 4]
                kb = bytes([tag]) + x.to_bytes(32, "big") + y.to_bytes(32, "big")
            keys.append(kb)
            try:
                exp.append(int(ec.verify(es[i], sigs[i], kb)))
            except RefError as ex:
                exp.append({"invalid point": 2, "Assertion failed": 5, "Unknown point format": 6}[ex.args[0]])
        stv = (ctypes.c_uint8 * cnt)()
        he.he_ed_ec_verify(ctypes.c_size_t(cnt), col(es), col([sg.r for sg in sigs]), col([sg.s for sg in sigs]), b"".join(keys), fmt, stv)
        assert list(stv) == exp, (fmt, list(stv), exp)
    # ---- genKeyPair
    ents = [bytes(rnd.randrange(256) for _ in range(25)) for _ in range(cnt)]
    out, st8 = (ctypes.c_uint8 * (32 * cnt))(), (ctypes.c_uint8 * cnt)()
    he.he_ed_ec_keygen(ctypes.c_size_t(cnt), b"".join(ents), 25, b"\x00", 0, out, st8)
    assert [int.from_bytes(bytes(out[32 * i:32 * i + 32]), "big") for i in range(cnt)] == [ec.gen_key_pair(x).priv for x in ents]
    assert ec.gen_key_pair(bytes(range(1, 26))).priv == 0x5f305137244598fbe2e7bfe14ff6c3537fa37c392973908fc7820e2b24d4ea1
    # ---- Point.mul / mulAdd / G.mul, KeyPair.derive
    k1 = [rnd.randrange(2**256) for _ in range(cnt)]
    k2 = [rnd.randrange(2**256) for _ in range(cnt)]
    k2[0], k2[1], k1[2] = 0, n_ord, 0
    pts = b"".join(q.get_x().to_bytes(32, "big") + q.get_y().to_bytes(32, "big") for q in pubs)
    out, st8 = (ctypes.c_uint8 * (64 * cnt))(), (ctypes.c_uint8 * cnt)()
    xy = lambda i: (int.from_bytes(bytes(out[64 * i:64 * i + 32]), "big"), int.from_bytes(bytes(out[64 * i + 32:64 * i + 64]), "big"))
    he.he_ed_ec_mul_add(ctypes.c_size_t(cnt), col(k1), col(k2), pts, 0, out, st8)
    for i in range(cnt):
        w = ec.g.mul_add(k1[i], pubs[i], k2[i])
        assert st8[i] == 1 and xy(i) == (w.get_x(), w.get_y()), i
    he.he_ed_ec_mul_add(ctypes.c_size_t(cnt), None, col(k2), pts, 0, out, st8)
    for i in range(cnt):
        w = pubs[i].mul(k2[i])
        assert xy(i) == (w.get_x(), w.get_y()), i
    he.he_ed_ec_mul_add(ctypes.c_size_t(cnt), None, col(k2), None, 0, out, st8)
    for i in range(cnt):
        w = ec.g.mul(k2[i] % n_ord)
        assert xy(i) == (w.get_x(), w.get_y()), i
    he.he_ed_ec_mul_add(ctypes.c_size_t(cnt), None, col(privs), pts[64:] + pts[:64], 1, out, st8)
    for i in range(cnt):
        assert st8[i] == 1 and xy(i)[0] == KeyPair(ec, priv=privs[i]).derive(pubs[(i + 1) % cnt]), i
    bad = bytearray(pts); bad[63] ^= 1
    he.he_ed_ec_mul_add(ctypes.c_size_t(1), None, col(privs[:1]), bytes(bad[:64]), 1, out, st8)
    assert st8[0] == 3
    # ---- Montgomery-curve Point.mul (x only, no validation)
    from oracle.ref_py import curves
    c25 = curves.get("curve25519").curve
    xs = [9, 9, 5] + [rnd.randrange(2**255 - 19) for _ in range(9)]
    kk = [6, 0, 1] + [rnd.randrange(2**256) for _ in range(9)]
    o2, s2 = (ctypes.c_uint8 * (32 * 12))(), (ctypes.c_uint8 * 12)()
    he.he_x25519_mul(ctypes.c_size_t(12), col(kk), col(xs), o2, s2)
    for i in range(12):
        assert int.from_bytes(bytes(o2[32 * i:32 * i + 32]), "big") == c25.point(xs[i], 1).mul(kk[i]).get_x(), i


def test_runtime_short_curve_bodies(he):
    """sw_runtime.cuh (run-time p, a, b): add / dbl / mul / mulAdd / validate on the reference's toy curve
    (test/curve-test.js:9-22: p = 0x1d, a = 4, b = 0x14) exhaustively, and on random prime fields, against
    plain affine arithmetic."""
    def params(p, a, b):
        R = 1 << 256
        return (L(p), L(R % p), L(R * R % p), L(a * R % p), L(b * R % p), (-pow(p, -1, 1 << 32)) % (1 << 32))

    def aff_add(P, Q, p, a):
        if P is None: return Q
        if Q is None: return P
        if P[0] == Q[0] and (P[1] + Q[1]) % p == 0: return None
        lam = ((3 * P[0] * P[0] + a) * pow(2 * P[1], -1, p) if P == Q else (Q[1] - P[1]) * pow(Q[0] - P[0], -1, p)) % p
        x = (lam * lam - P[0] - Q[0]) % p
        return x, (lam * (P[0] - x) - P[1]) % p

    def aff_mul(k, P, p, a):
        R = None
        for bit in bin(k)[2:] if k else "":
            R = aff_add(R, R, p, a)
            if bit == "1": R = aff_add(R, P, p, a)
        return R

    def run(prm, ln, op, P1, k1=0, P2=None, k2=None, klen=1):
        pw, r1, r2, am, bm, n0 = prm
        enc = lambda P: P[0].to_bytes(ln, "big") + P[1].to_bytes(ln, "big")
        out, st = (ctypes.c_uint8 * (2 * ln))(), (ctypes.c_uint8 * 1)()
        he.he_rt_item(op, pw, r1, r2, am, bm, ctypes.c_uint32(n0), ctypes.c_uint32(ln), k1.to_bytes(klen, "big"), enc(P1),
                      k2.to_bytes(klen, "big") if k2 is not None else None, enc(P2) if P2 else None, ctypes.c_uint32(klen), out, st)
        if st[0] == 1:
            return int.from_bytes(bytes(out[:ln]), "big"), int.from_bytes(bytes(out[ln:]), "big")
        return {7: None, 4: "off", 0: False}[st[0]]

    p, a, b = 0x1d, 4, 0x14
    prm = params(p, a, b)
    pts = [(x, y) for x in range(p) for y in range(p) if (y * y - x ** 3 - a * x - b) % p == 0]
    assert (0x18, 0x16) in pts                                             # the point the reference's test uses
    for P in pts:
        assert run(prm, 1, 2, P) == aff_add(P, P, p, a)
        for Q in pts:
            assert run(prm, 1, 1, P, P2=Q) == aff_add(P, Q, p, a)
        for k in (0, 1, 2, 5, 36, 37, 255):
            assert run(prm, 1, 0, P, k) == aff_mul(k, P, p, a)
    assert run(prm, 1, 0, pts[3], 9, pts[7], 200) == aff_add(aff_mul(9, pts[3], p, a), aff_mul(200, pts[7], p, a), p, a)
    assert run(prm, 1, 3, (3, 3)) is False and run(prm, 1, 0, (3, 3), 5) == "off"
    rnd = random.Random(12)
    for pp in (2**61 - 1, 2**127 - 1, 2**256 - 2**32 - 977, 2**256 - 2**224 + 2**192 + 2**96 - 1):      # all = 3 mod 4
        ln = (pp.bit_length() + 7) // 8
        aa, bb = rnd.randrange(pp), rnd.randrange(pp)
        prm = params(pp, aa, bb)
        found = []
        while len(found) < 3:
            x = rnd.randrange(pp)
            rhs = (x ** 3 + aa * x + bb) % pp
            if pow(rhs, (pp - 1) // 2, pp) == 1:
                found.append((x, pow(rhs, (pp + 1) // 4, pp)))
        P, Q, S = found
        k1, k2 = rnd.randrange(2**200), rnd.randrange(2**64)
        assert run(prm, ln, 1, P, P2=Q) == aff_add(P, Q, pp, aa)
        assert run(prm, ln, 2, S) == aff_add(S, S, pp, aa)
        assert run(prm, ln, 0, P, k1, klen=25) == aff_mul(k1, P, pp, aa)
        assert run(prm, ln, 0, P, k1, Q, k2, klen=25) == aff_add(aff_mul(k1, P, pp, aa), aff_mul(k2, Q, pp, aa), pp, aa)


def test_chunk_plan_of_the_pipelined_host_calls(he, monkeypatch):
    """make_plan (csrc/chunk_plan.h): the chunks tile [0, n) in order, every boundary except the last is a multiple
    of 128 items (the kernels' block size), there are never more chunks than the context has events for, the lead
    chunk is the short one, and the tuning knobs do what INTEGRATION.md says."""
    def plan(n):
        lo = (ctypes.c_ulonglong * 18)()
        mx = ctypes.c_ulonglong()
        k = he.he_chunk_plan(ctypes.c_size_t(n), lo, ctypes.byref(mx))
        b = [int(lo[i]) for i in range(k + 1)]
        assert b[0] == 0 and b[-1] == n and all(x < y for x, y in zip(b, b[1:])), (n, b)
        assert all(x % 128 == 0 for x in b[:-1]) and 1 <= k <= 16
        assert int(mx.value) == max(y - x for x, y in zip(b, b[1:]))
        return b
    monkeypatch.delenv("EB200_CHUNKS", raising=False)
    monkeypatch.delenv("EB200_LEAD", raising=False)
    for n in (1, 127, 128, 129, 4099, (1 << 18) - 1):
        assert plan(n) == [0, n]                                   # below 2^18 items: one chunk
    b = plan(1 << 20)
    assert len(b) == 6 and b[1] == 1 << 16 and max(y - x for x, y in zip(b[1:], b[2:])) <= (1 << 18)   # 1/4 lead + 4
    assert len(plan(1 << 22)) == 17 and len(plan((1 << 23) + 12345)) == 17                            # 16 equal chunks
    rnd = random.Random(5)
    for _ in range(300):
        plan(rnd.randrange(1, 1 << 24))
    monkeypatch.setenv("EB200_LEAD", "0")
    assert plan(1 << 20) == [0, 1 << 18, 2 << 18, 3 << 18, 1 << 20]
    monkeypatch.setenv("EB200_CHUNKS", "15")
    monkeypatch.delenv("EB200_LEAD", raising=False)
    assert len(plan(1 << 20)) == 17                                # 15 + the lead chunk: the most the event arrays hold
    monkeypatch.setenv("EB200_CHUNKS", "99")                       # out of range: ignored
    assert len(plan(1 << 20)) == 6
