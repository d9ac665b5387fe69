"""The secp256k1 verify kernel's per-item table, built with co-Z additions, against the table built by mixed additions
that it replaced (tests/hostemu/k256_qtab_emu.cpp) and against the oracle's odd multiples; then whole verifies on
keys G, -G and 2^k G whose answers depend on exact exceptional additions after that table."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**256 - 2**32 - 977
BETA = 0x7ae96a2b657c07106e64479eac3434e99cf0497512f58995c1396c28719501ee


@pytest.fixture(scope="module")
def fx():
    out = os.path.join(ROOT, "tests", "_hostemu")
    os.makedirs(out, exist_ok=True)
    lib = os.path.join(out, "libk256_qtab.so")
    src = os.path.join(ROOT, "tests", "hostemu", "k256_qtab_emu.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", "-shared", "-fPIC", "-o", lib, src], check=True)
    return ctypes.CDLL(lib)


@pytest.fixture(scope="module")
def ec():
    from oracle.ref_py.ec import EC
    return EC("secp256k1")


def affine(X, Y, Z):
    zi = pow(Z, -1, P)
    return X * zi * zi % P, Y * zi ** 3 % P


def qtab(fx, which, Q):
    nw = fx.fx_qtab_words()
    q = (ctypes.c_uint32 * 16)(*[(v >> (32 * i)) & 0xFFFFFFFF for v in (Q.x, Q.y) for i in range(8)])
    tab, zg = (ctypes.c_uint32 * nw)(), (ctypes.c_uint32 * 8)()
    fx.fx_qtab(which, q, tab, zg)
    vals = [sum(int(tab[8 * k + i]) << (32 * i) for i in range(8)) for k in range(nw // 8)]
    return [tuple(vals[3 * k:3 * k + 3]) for k in range(nw // 24)], sum(int(zg[i]) << (32 * i) for i in range(8))


def test_coz_table_matches_previous_table_and_oracle(fx, ec):
    rnd = random.Random(33)
    n = ec.n
    keys = [ec.g.mul(d) for d in (1, n - 1, 2, n - 2, 3, 1 << 20, 1 << 255)] + [ec.g.mul(rnd.randrange(1, n)) for _ in range(24)]
    for Q in keys:
        new, zn = qtab(fx, 0, Q)
        old, zo = qtab(fx, 1, Q)
        assert len(new) == 8 and zn % P and zo % P
        for k, ((xn, yn, bn), (xo, yo, bo)) in enumerate(zip(new, old)):
            m = Q.mul(2 * k + 1)
            assert affine(xn, yn, zn) == affine(xo, yo, zo) == (m.x, m.y), k
            assert bn % P == xn * BETA % P and bo % P == xo * BETA % P


def test_verify_meets_exceptional_additions(fx, ec):
    """Signatures minted (ks_items) so that the fixed-base adds after the Q half meet P + P, P - P and O + P, on keys
    G, -G, 2^k G: TRUE only if the whole pipeline (prep, co-Z table, main loop, cold path, eqXToP) is exact."""
    from ks_items import adversarial_keys, adversarial_items
    W, E, B = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    fx.he_gtab_dims(ctypes.byref(W), ctypes.byref(E), ctypes.byref(B))
    gtab = np.zeros(W.value * E.value * 16, np.uint32)
    fx.he_gtab_fast(gtab.ctypes.data_as(ctypes.c_void_p))
    keys = adversarial_keys(ec, 1, [4, 8])
    items = adversarial_items(ec, 1, keys, B.value)
    col = lambda k: b"".join(it[k].to_bytes(32, "big") for it in items)
    pub = b"".join(keys[it[3]][1].x.to_bytes(32, "big") + keys[it[3]][1].y.to_bytes(32, "big") for it in items)
    st = (ctypes.c_uint8 * len(items))()
    fx.he_verify(ctypes.c_size_t(len(items)), col(0), col(1), col(2), pub, gtab.ctypes.data_as(ctypes.c_void_p), st)
    want = [int(ec.verify(e, {"r": r, "s": s}, {"x": keys[k][1].x, "y": keys[k][1].y})) for e, r, s, k in items]
    assert [int(v) for v in st] == want
    assert sum(want) >= 4 * len(keys)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 4099, (1 << 16) + 3])
def test_prep_batches_give_the_same_workspace(fx, ec, n):
    """The verify prep at 32 and 64 items per thread writes the same workspace as at 16 (which the verify tests check
    against the oracle), with r and s out of range scattered and at the batch boundaries; on the exact grid and on the
    128-thread-rounded grid the launches use."""
    rnd = random.Random(n)
    N_ = ec.n
    e = [rnd.randrange(2**256) for _ in range(n)]
    r = [rnd.randrange(1, N_) for _ in range(n)]
    s = [rnd.randrange(1, N_) for _ in range(n)]
    for i in list(range(0, n, 7)) + [j for j in (0, 15, 16, 31, 32, 63, 64, n - 1) if j < n]:
        k = rnd.randrange(4)
        if k == 0: r[i] = 0
        if k == 1: s[i] = N_
        if k == 2: s[i] = 2**256 - 1
        if k == 3: r[i] = N_ + 1
    col = lambda v: b"".join(x.to_bytes(32, "big") for x in v)
    E, R, S = col(e), col(r), col(s)

    def ws(mode, batch, T):
        out = np.zeros(19 * n, np.uint32)
        fx.fx_prep(ctypes.c_size_t(n), E, R, S, mode, batch, ctypes.c_size_t(T), out.ctypes.data_as(ctypes.c_void_p))
        return out
    for mode in (0, 1, 2):
        want = ws(mode, 16, -(-n // 16))
        if mode == 0:
            assert (want[18 * n:] & 1).any()      # r or s out of range flags the item
        for batch in (32, 64):
            exact = -(-n // batch)
            for T in (exact, -(-exact // 128) * 128):
                assert np.array_equal(ws(mode, batch, T), want), (mode, batch, T)
