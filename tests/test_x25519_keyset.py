"""curve25519 key sets without a GPU: the classify, table-build, keyed-derive and normalisation bodies run through the
host emulation at every width against the oracle's MontCurve ladder and against the unkeyed ladder body, on small-order,
mixed-order, non-canonical, twist and random keys and on scalars at the edges of n and of the keys' orders; then the C
entry points' return codes without a device and X25519KeySet's argument checks."""
import ctypes
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import torsion_cases as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_hostemu(root, out_dir):
    lib = os.path.join(out_dir, "libx25519_keyset_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", lib,
                    os.path.join(root, "tests", "hostemu", "x25519_keyset_emu.cpp")], check=True)
    he = ctypes.CDLL(lib)
    he.he_x25519_keyset_derive.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 6
    he.he_x25519_unkeyed_derive.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 4
    return he


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    return build_hostemu(ROOT, str(tmp_path_factory.mktemp("hostemu")))


def keys():
    """u values: small order (0, 1, the order-8 u), p - 1, mixed order, each + p, twist points, u >= p up to 2^256 - 1
    and random keys on the curve."""
    us = [u for _, u in tc.x25519_us()] + [tc.P, tc.P + 1, 2**256 - 1]
    rnd = random.Random(25519)
    while len(us) < 40:
        u = rnd.randrange(tc.P)
        if pow((u ** 3 + tc.A_MONT * u * u + u) % tc.P, (tc.P - 1) // 2, tc.P) == 1:
            us.append(u)
    return us


def scalars():
    """0, 1, 2, 8, n - 1, n - 8, multiples of the small orders 2, 4 and 8, and random scalars below n."""
    rnd = random.Random(2)
    return [0, 1, 2, 4, 8, 16, 24, tc.N - 1, tc.N - 8, 8 * rnd.randrange(1, tc.N // 8), 4 * rnd.randrange(1, tc.N // 4)] + \
        [rnd.randrange(tc.N) for _ in range(3)]


_CASES = {}


def cases():
    """Every key against every scalar, and the oracle's (status, x) for each: KeyPair(priv).derive(point(u, 1))."""
    if not _CASES:
        from oracle.ref_py.ec import EC
        from oracle.ref_py import curves
        from ed_items import x_expected
        ec25, c25 = EC("curve25519"), curves.get("curve25519").curve
        us, ks = keys(), scalars()
        items = [(j, k) for j in range(len(us)) for k in ks]
        _CASES.update(us=us, items=items, want=[x_expected(ec25, c25, k, us[j] % tc.P) for j, k in items])
    return _CASES


def _rows(buf, n):
    b = buf.tobytes()
    return [int.from_bytes(b[32 * i:32 * (i + 1)], "big") for i in range(n)]


def run_keyed(he, W, us, items):
    """(key statuses, Edwards images, [(status, x)]) of the keyed pipeline."""
    m, n = len(us), len(items)
    pubx = np.frombuffer(tc.be(us), np.uint8).copy()
    priv = np.frombuffer(tc.be([k for _, k in items]), np.uint8).copy()
    idx = np.array([j for j, _ in items], np.uint32)
    kst, A = np.zeros(m, np.uint8), np.zeros((m, 32), np.uint8)
    out, st = np.full((n, 32), 0xAA, np.uint8), np.zeros(n, np.uint8)
    he.he_x25519_keyset_derive(W, m, pubx.ctypes.data, n, priv.ctypes.data, idx.ctypes.data, kst.ctypes.data, A.ctypes.data,
                               out.ctypes.data, st.ctypes.data)
    return [int(v) for v in kst], A, list(zip([int(v) for v in st], _rows(out, n)))


@pytest.mark.parametrize("W", [4, 5, 6, 7, 8])
def test_bodies_against_oracle(he, W):
    c = cases()
    us, items, want = c["us"], c["items"], c["want"]
    kst, A, got = run_keyed(he, W, us, items)
    bad = [(hex(us[items[i][0]]), items[i][1], got[i], want[i]) for i in range(len(items)) if got[i] != want[i]]
    assert not bad, bad[:5]
    nk = len(scalars())
    assert kst == [want[nk * j][0] for j in range(len(us))]
    assert {5, 1} == set(kst)
    assert tc.P - 1 in us and kst[us.index(tc.P - 1)] == 5                 # the one u without an Edwards image
    # a key's image is y = (u - 1) / (u + 1) with x's sign bit clear, or zeros for a twist key
    for j, u in enumerate(us):
        y = (u - 1) * pow(u + 1, -1, tc.P) % tc.P if kst[j] == 1 else 0
        assert bytes(A[j]) == y.to_bytes(32, "little"), hex(u)
    # the special results are all reached: the point at infinity (x = 0) from priv = 0 and from small-order keys
    assert sum(1 for s, x in got if s == 1 and x == 0) > len(scalars())


def test_unkeyed_body_gives_the_same_bytes(he):
    c = cases()
    us, items = c["us"], c["items"]
    n = len(items)
    priv = np.frombuffer(tc.be([k for _, k in items]), np.uint8).copy()
    pubx = np.frombuffer(tc.be([us[j] for j, _ in items]), np.uint8).copy()
    out, st = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    he.he_x25519_unkeyed_derive(n, priv.ctypes.data, pubx.ctypes.data, out.ctypes.data, st.ctypes.data)
    assert list(zip([int(v) for v in st], _rows(out, n))) == run_keyed(he, 7, us, items)[2] == c["want"]


def test_partial_normalisation_batches(he):
    """Item counts around the 16-item batch, so that the strided batches are uneven and some threads hold one item."""
    c = cases()
    us, items, want = c["us"], c["items"], c["want"]
    for n in (1, 15, 16, 17, 33, 255):
        assert run_keyed(he, 6, us, items[:n])[2] == want[:n], n


MUTATIONS = {
    "digit sign": ("acc = ed_add_niels(acc, ed_niels_neg_if(q, neg));\n  }\n  x25519_ks_ws_store",
                   "acc = ed_add_niels(acc, q);\n  }\n  x25519_ks_ws_store"),
    "Z - Y read for Z + Y": ("r = f25_normalize(f25_mul(x25519_ks_ws_load(ws, X25519_KS_WS_ZPY, ld, i), zi));",
                             "r = f25_normalize(f25_mul(x25519_ks_ws_load(ws, X25519_KS_WS_ZMY, ld, i), zi));"),
    "twist accepted": ("if (!(one || is_zero_n<8>(leg.v))) {", "if (false) {"),
    "zero Z - Y kept": ("      if (!f25_is_zero(d)) prod = f25_mul(prod, d);", "      prod = f25_mul(prod, d);"),
}


@pytest.mark.parametrize("kind", sorted(MUTATIONS))
def test_oracle_comparison_catches_a_broken_body(tmp_path, kind):
    root = str(tmp_path)
    shutil.copytree(os.path.join(ROOT, "elliptic_b200", "csrc"), os.path.join(root, "elliptic_b200", "csrc"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(root, "include"))
    shutil.copytree(os.path.join(ROOT, "tests", "hostemu"), os.path.join(root, "tests", "hostemu"))
    path = os.path.join(root, "elliptic_b200", "csrc", "x25519_keyset_body.cuh")
    old, new = MUTATIONS[kind]
    src = open(path).read()
    assert src.count(old) == 1, old
    open(path, "w").write(src.replace(old, new))
    bad = build_hostemu(root, root)
    c = cases()
    assert run_keyed(bad, 7, c["us"], c["items"])[2] != c["want"]


def test_return_codes_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    buf = np.zeros(1 << 12, np.uint8)
    p = buf.ctypes.data
    out = ctypes.c_void_p(1)
    create = lambda *a: lib.eb200_x25519_keyset_create(*a, ctypes.byref(out))
    assert create(4, p, 0, p) == _native.ERR_NOT_INIT and out.value is None
    assert create(4, None, 0, p) == _native.ERR_ARG and create(4, p, 0, None) == _native.ERR_ARG
    assert lib.eb200_x25519_keyset_create(4, p, 0, p, None) == _native.ERR_ARG
    assert create(0, p, 0, p) == _native.ERR_ARG and create(1 << 32, p, 0, p) == _native.ERR_ARG
    assert create(4, p, 3, p) == _native.ERR_ARG and create(4, p, 9, p) == _native.ERR_ARG
    assert create(1 << 16, p, 0, p) == _native.ERR_ARG                  # no width fits the default budget
    assert create(1 << 16, p, 4, p) == _native.ERR_NOT_INIT             # an explicit width is not held to it
    assert lib.eb200_x25519_derive_batch_keyed(None, 4, p, p, p, p) == _native.ERR_ARG
    # the short-curve entry point still refuses the 25519 curves
    assert lib.eb200_keyset_create(_native.CURVE_CURVE25519, 4, p, 0, 0, p, ctypes.byref(out)) == _native.ERR_UNSUPPORTED


def test_x25519_key_set_argument_errors():
    from elliptic_b200.ec import EC, EllipticError, X25519KeySet
    with pytest.raises(EllipticError):
        EC("ed25519").key_set([{"x": 1, "y": 2}])                        # still the short curves' message, before any device
    ks = X25519KeySet.__new__(X25519KeySet)                              # a set as built, without its native handle
    ks._ec, ks.status, ks._sets = EC("curve25519"), np.ones(3, np.uint8), []
    z = np.zeros((2, 32), np.uint8)
    with pytest.raises(ValueError):
        ks.derive_batch_packed(np.zeros((2, 31), np.uint8), [0, 1])
    with pytest.raises(ValueError):
        ks.derive_batch_packed(z, [0])
    with pytest.raises(ValueError):
        ks.derive_batch_packed(z, [0, 3])
    with pytest.raises(ValueError):
        ks.derive_batch_packed(z, [-1, 0])
    with pytest.raises(ValueError):
        ks.derive_batch_packed(z, [0, 1], out=np.zeros((2, 31), np.uint8))
    with pytest.raises(ValueError):
        ks.derive_batch_packed(z, [0, 1], status=np.zeros(3, np.uint8))
    with pytest.raises(ValueError):
        ks.derive_batch([1, 2], [0])
    with pytest.raises(EllipticError):
        ks.derive_batch_packed(z, [0, 1])                                # closed
