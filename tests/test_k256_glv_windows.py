"""The secp256k1 double-scalar core's per-item windows (ecdsa_k256_body.cuh, k256_dsm): the bound on the GLV halves
that sizes them, derived from glv_split_odd's rounding and parity fix; the 16-entry co-Z table, split between the\nworkspace and thread-local memory; and scalars whose halves
reach that bound, through verify, recoverPubKey and mulAdd, in both field forms (packed 8 x 32 and -DEB_K256_FQ=1)."""
import ctypes
import itertools
import os
import random
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import arith_cases as ac

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**256 - 2**32 - 977
N = ac.ORDERS["secp256k1"]
BETA = 0x7ae96a2b657c07106e64479eac3434e99cf0497512f58995c1396c28719501ee
V1, V2 = (ac.A1, ac.B1), (ac.A2, ac.B2)


def _compile(src, name, flags=()):
    out = os.path.join(ROOT, "tests", "_hostemu")
    os.makedirs(out, exist_ok=True)
    lib = os.path.join(out, name)
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", *flags, "-shared", "-fPIC", "-o", lib,
                    os.path.join(ROOT, "tests", "hostemu", src)], check=True)
    return ctypes.CDLL(lib)


@pytest.fixture(scope="module", params=[0, 1], ids=["packed", "fq"])
def he(request):
    fq = request.param
    return _compile("k256_window_emu.cpp", "libk256_window%d.so" % fq, ["-DEB_K256_FQ=%d" % fq])


@pytest.fixture(scope="module")
def ec():
    from oracle.ref_py.ec import EC
    return EC("secp256k1")


def windows(lib):
    v = [ctypes.c_int() for _ in range(4)]
    lib.fx_glv_windows(*[ctypes.byref(x) for x in v])
    return tuple(x.value for x in v)        # W, windows, entries, GLV_M_BITS


# ---- the bound ---------------------------------------------------------------------------------------------------
# Before the parity fix, (k1, k2) = -(d1 v1 + d2 v2) with |d1|, |d2| <= 1/2: c1, c2 are k b2 / n and -k b1 / n rounded
# (through 2^384-scaled constants, off by at most k / 2^385, which moves k1, k2 by less than 2).  The fix subtracts
# e1 v1 when k1 is even (e1 = +1 if k1 >= 0, else -1), then e2 v2 when k2 is even (the sign of k1 after the first
# step).  Each (e1, e2) holds on a convex piece of the square, so |k1| and |k2| peak at its vertices.
HALF = Fraction(1, 2)


def _pieces():
    """(e1, e2, constraints a d1 + b d2 <= c) for every way the parity fix can go."""
    box = [(1, 0, HALF), (-1, 0, HALF), (0, 1, HALF), (0, -1, HALF)]
    for e1, e2 in itertools.product((-1, 0, 1), repeat=2):
        cons = list(box)
        if e1:                                       # k1 = -(d1 a1 + d2 a2) >= 0 for e1 = +1, < 0 for e1 = -1
            cons.append((e1 * ac.A1, e1 * ac.A2, 0))
        if e2:                                       # the same test on -((d1 + e1) a1 + d2 a2)
            cons.append((e2 * ac.A1, e2 * ac.A2, -e2 * e1 * ac.A1))
        yield e1, e2, cons


def _vertices(cons):
    out = set()
    for (a1, b1, c1), (a2, b2, c2) in itertools.combinations(cons, 2):
        det = a1 * b2 - a2 * b1
        if det:
            x, y = Fraction(c1 * b2 - c2 * b1, det), Fraction(a1 * c2 - a2 * c1, det)
            if all(a * x + b * y <= c for a, b, c in cons):
                out.add((x, y))
    return sorted(out)


def _halves(e1, e2, d1, d2):
    t1, t2 = d1 + e1, d2 + e2
    return -(t1 * V1[0] + t2 * V2[0]), -(t1 * V1[1] + t2 * V2[1])


def glv_bound():
    """max |k1|, max |k2| over every piece, exact (before the < 2 of the scaled constants)."""
    b1 = b2 = 0
    for e1, e2, cons in _pieces():
        for d1, d2 in _vertices(cons):
            k1, k2 = _halves(e1, e2, d1, d2)
            b1, b2 = max(b1, abs(k1)), max(b2, abs(k2))
    return b1, b2


def extreme_scalars():
    """k whose halves sit at every vertex of every piece, moved 2^-40 of the way to the piece's centre so that rounding
    and the sign tests fall the same way, with the parities that make glv_split_odd take that piece's fix.
    Returns [(k, (k1, k2))] with the halves glv_split_odd must return."""
    out = []
    for e1, e2, cons in _pieces():
        vs = _vertices(cons)
        if len(vs) < 3:
            continue
        cx, cy = sum(v[0] for v in vs) / len(vs), sum(v[1] for v in vs) / len(vs)
        for d1, d2 in vs:
            d1, d2 = d1 + (cx - d1) / 2**40, d2 + (cy - d2) / 2**40
            x, y = (round(-(d1 * V1[0] + d2 * V2[0])), round(-(d1 * V1[1] + d2 * V2[1])))
            if (x % 2 == 0) != (e1 != 0):
                x += 1
            if ((y - e1 * V1[1]) % 2 == 0) != (e2 != 0):
                y += 1
            k = (x + y * ac.LAMBDA) % N
            out.append((k, (x - e1 * V1[0] - e2 * V2[0], y - e1 * V1[1] - e2 * V2[1])))
    return out


def test_glv_half_bound_fits_the_windows(he):
    """The derived bound gives m = (|k| - 1) / 2 < 2^GLV_M_BITS (with the < 2 the scaled constants add), and the
    windows of k256_dsm cover those bits with a top digit 2m + 1 that has a table entry."""
    W, nwin, entries, mbits = windows(he)
    b1, b2 = glv_bound()
    assert 2**128 < max(b1, b2) < 2**128.7
    assert ((int(max(b1, b2)) + 2 - 1) // 2).bit_length() == mbits == 128
    assert entries == 1 << (W - 1) and (W, nwin) == (5, 26)
    top_bits = mbits - W * (nwin - 1)
    assert 2 * (2**top_bits - 1) + 1 <= 2 * entries - 1


def test_extreme_halves_reach_the_bound(he):
    """The constructed scalars take every piece's fix, split (on the host body and in Python) to the expected halves,
    and come within 2^-30 of the bound for both |k1| and |k2|: m then has its top bit, 127, set."""
    b1, b2 = glv_bound()
    cases = extreme_scalars()
    assert len(cases) >= 30
    top1 = top2 = 0
    for k, (k1, k2) in cases:
        assert ac.glv_split_odd(k) == (k1, k2), hex(k)
        m1, m2 = (ctypes.c_uint32 * 5)(), (ctypes.c_uint32 * 5)()
        n1, n2 = ctypes.c_int(), ctypes.c_int()
        he.he_glv((ctypes.c_uint32 * 8)(*[(k >> (32 * i)) & 0xFFFFFFFF for i in range(8)]), m1, ctypes.byref(n1), m2,
                  ctypes.byref(n2))
        got = [(2 * sum(int(m[i]) << (32 * i) for i in range(5)) + 1) * (-1 if s.value else 1) for m, s in ((m1, n1), (m2, n2))]
        assert tuple(got) == (k1, k2), hex(k)
        assert abs(k1) <= b1 + 2 and abs(k2) <= b2 + 2
        top1, top2 = max(top1, abs(k1)), max(top2, abs(k2))
    assert top1 > b1 * (1 - Fraction(1, 2**30)) and top2 > b2 * (1 - Fraction(1, 2**30))
    assert ((top2 - 1) // 2) >> 127 == 1


def _gtab(lib):
    W, E, B = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    lib.he_gtab_dims(ctypes.byref(W), ctypes.byref(E), ctypes.byref(B))
    gtab = np.zeros(W.value * E.value * 16, np.uint32)
    lib.he_gtab_fast(gtab.ctypes.data_as(ctypes.c_void_p))
    return gtab


def _col(vals):
    return b"".join(v.to_bytes(32, "big") for v in vals)


def test_extreme_halves_through_verify_recover_and_mul_add(he, ec):
    """u2 = k for every extreme scalar k, and its negation: verify (valid and altered signatures), recoverPubKey and
    mulAdd / mul give the oracle's answers."""
    from rec_items import rec_expected
    rnd = random.Random(55)
    ks = [k for k, _ in extreme_scalars()]
    ks += [N - k for k in ks]
    gtab = _gtab(he)
    gp = gtab.ctypes.data_as(ctypes.c_void_p)
    # verify: Q = d G, R = u1 G + k Q, r = x(R), s = r / k, e = u1 s, so that r / s = k
    items = []
    for t, k in enumerate(ks):
        d, u1 = rnd.randrange(1, N), rnd.randrange(1, N)
        Q = ec.g.mul(d)
        r = ec.g.mul_add(u1, Q, k).get_x() % N
        s = r * pow(k, -1, N) % N
        e = u1 * s % N
        if t % 3 == 2:
            e = (e + 1) % N
        items.append((e, r, s, Q.get_x(), Q.get_y()))
    st = (ctypes.c_uint8 * len(items))()
    he.he_verify(ctypes.c_size_t(len(items)), _col([i[0] for i in items]), _col([i[1] for i in items]),
                 _col([i[2] for i in items]), b"".join(i[3].to_bytes(32, "big") + i[4].to_bytes(32, "big") for i in items), gp, st)
    want = [int(ec.verify(e, {"r": r, "s": s}, {"x": x, "y": y})) for e, r, s, x, y in items]
    assert [int(v) for v in st] == want
    assert want.count(1) >= len(ks) // 2
    # recoverPubKey: u2 = s / r = k
    rec = []
    for t, k in enumerate(ks):
        R = ec.g.mul(rnd.randrange(1, N))
        r = R.get_x() % N
        rec.append((rnd.randrange(N), r, k * r % N, (R.get_y() & 1) ^ (t & 1)))
    out, st = (ctypes.c_uint8 * (64 * len(rec)))(), (ctypes.c_uint8 * len(rec))()
    he.he_recover(ctypes.c_size_t(len(rec)), _col([i[0] for i in rec]), _col([i[1] for i in rec]), _col([i[2] for i in rec]),
                  bytes(i[3] for i in rec), gp, out, st)
    for i, it in enumerate(rec):
        pt = (int.from_bytes(bytes(out[64 * i:64 * i + 32]), "big"), int.from_bytes(bytes(out[64 * i + 32:64 * i + 64]), "big"))
        assert (st[i], pt if st[i] == 1 else None) == rec_expected(ec, it), i
    # mulAdd and mul
    k1 = [rnd.randrange(N) for _ in ks]
    pts = [ec.g.mul(rnd.randrange(1, N)) for _ in ks]
    enc = b"".join(p.get_x().to_bytes(32, "big") + p.get_y().to_bytes(32, "big") for p in pts)
    out, st = (ctypes.c_uint8 * (64 * len(ks)))(), (ctypes.c_uint8 * len(ks))()
    xy = lambda i: (int.from_bytes(bytes(out[64 * i:64 * i + 32]), "big"), int.from_bytes(bytes(out[64 * i + 32:64 * i + 64]), "big"))
    he.he_mul_add(ctypes.c_size_t(len(ks)), _col(k1), _col(ks), enc, gp, out, st)
    for i in range(len(ks)):
        w = ec.g.mul_add(k1[i], pts[i], ks[i])
        assert st[i] == 1 and xy(i) == (w.get_x(), w.get_y()), i
    he.he_mul_add(ctypes.c_size_t(len(ks)), None, _col(ks), enc, gp, out, st)
    for i in range(len(ks)):
        w = pts[i].mul(ks[i])
        assert st[i] == 1 and xy(i) == (w.get_x(), w.get_y()), i


def affine(X, Y, Z):
    zi = pow(Z, -1, P)
    return X * zi * zi % P, Y * zi ** 3 % P


def test_split_table_holds_the_odd_multiples(ec):
    """The table k256_dsm builds: (2k + 1) Q for k < 16, the first 8 in the item's workspace table and the other 8 in
    thread-local memory, all on the isomorphic curve scaled by the one returned Z, with beta x beside each x."""
    lib = _compile("k256_window_emu.cpp", "libk256_window_split.so")
    entries = windows(lib)[2]
    nw = 8 * 24
    rnd = random.Random(33)
    n = ec.n
    keys = [ec.g.mul(d) for d in (1, n - 1, 2, n - 2, 3, 1 << 20, 1 << 255)] + [ec.g.mul(rnd.randrange(1, n)) for _ in range(24)]
    for Q in keys:
        q = (ctypes.c_uint32 * 16)(*[(v >> (32 * i)) & 0xFFFFFFFF for v in (Q.x, Q.y) for i in range(8)])
        tab, hi, zg = (ctypes.c_uint32 * nw)(), (ctypes.c_uint32 * (24 * (entries - 8)))(), (ctypes.c_uint32 * 8)()
        lib.fx_qtab_split(q, tab, hi, zg)
        words = list(tab) + list(hi)
        vals = [sum(int(words[8 * k + i]) << (32 * i) for i in range(8)) for k in range(len(words) // 8)]
        z = sum(int(zg[i]) << (32 * i) for i in range(8))
        assert len(vals) == 3 * entries == 48 and z % P
        for k in range(entries):
            x, y, bx = vals[3 * k:3 * k + 3]
            m = Q.mul(2 * k + 1)
            assert affine(x, y, z) == (m.x, m.y), k
            assert bx % P == x * BETA % P


@pytest.mark.gpu
def test_extreme_halves_on_the_device(ec):
    """The same scalars through the device's k256_dsm: verify with u2 = k and mulAdd with k2 = k, against the oracle."""
    from elliptic_b200 import _native
    from elliptic_b200.ec import EC as GpuEC
    _native.init(0)
    rnd = random.Random(56)
    ks = [k for k, _ in extreme_scalars()]
    ks += [N - k for k in ks]
    items = []
    for t, k in enumerate(ks):
        Q = ec.g.mul(rnd.randrange(1, N))
        u1 = rnd.randrange(1, N)
        r = ec.g.mul_add(u1, Q, k).get_x() % N
        s = r * pow(k, -1, N) % N
        items.append(((u1 * s + (t % 3 == 2)) % N, r, s, Q.get_x(), Q.get_y()))
    pack = lambda idx: np.frombuffer(_col([it[idx] for it in items]), np.uint8).reshape(-1, 32)
    st = GpuEC("secp256k1").verify_batch_packed(pack(0), pack(1), pack(2), np.concatenate([pack(3), pack(4)], axis=1))
    assert [int(v) for v in st] == [int(ec.verify(e, {"r": r, "s": s}, {"x": x, "y": y})) for e, r, s, x, y in items]
    k1 = [rnd.randrange(N) for _ in ks]
    pts = [ec.g.mul(rnd.randrange(1, N)) for _ in ks]
    got = GpuEC("secp256k1").mul_add_batch(k1, [(p.get_x(), p.get_y()) for p in pts], ks)
    assert got == [(w.get_x(), w.get_y()) for w in (ec.g.mul_add(a, p, b) for a, p, b in zip(k1, pts, ks))]

