"""Keyed Point.mul / mulAdd / derive without a GPU: the build, scalar-prep, keyed main, normalisation and replay bodies
run through the host emulation in kernel order against the oracle's Point.mul, G.mulAdd and KeyPair.derive on all six
presets, with mutation checks, and the C entry points' return codes without a device."""
import ctypes
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

from ks_items import CURVES, adversarial_keys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BY_NAME = {nm: (cid, ln) for nm, cid, ln in CURVES}
OPS = {"mul": 0, "mul_add": 1, "derive": 2}
ST_TRUE, ST_THROW_NOT_VALIDATED, ST_INFINITY = 1, 3, 7


def build_hostemu(root, out_dir):
    lib = os.path.join(out_dir, "libkeyset_mul_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", "-shared", "-fPIC", "-o", lib,
                    os.path.join(root, "tests", "hostemu", "keyset_mul_emu.cpp")], check=True)
    he = ctypes.CDLL(lib)
    he.he_keyset_mul.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                 ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3
    return he


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    return build_hostemu(ROOT, str(tmp_path_factory.mktemp("hostemu_mul")))


def col(vals, ln):
    return np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in vals), np.uint8).reshape(len(vals), ln).copy()


def run_bodies(he, cid, ln, W, op, keys_xy, items, batch=16):
    """items: (k1, k2, key index).  Returns (key statuses, [(status, output bytes)])."""
    xy = np.ascontiguousarray(np.concatenate([col([k[0] for k in keys_xy], ln), col([k[1] for k in keys_xy], ln)], axis=1))
    k1, k2 = col([it[0] for it in items], ln), col([it[1] for it in items], ln)
    idx = np.array([it[2] for it in items], np.uint32)
    n = len(items)
    ol = ln if op == 2 else 2 * ln
    kst, st, out = np.zeros(len(keys_xy), np.uint8), np.zeros(n, np.uint8), np.full((n, ol), 0xA5, np.uint8)
    he.he_keyset_mul(cid, W, op, len(keys_xy), xy.ctypes.data, n, k1.ctypes.data, k2.ctypes.data, idx.ctypes.data, batch,
                     kst.ctypes.data, out.ctypes.data, st.ctypes.data)
    return list(kst), [(int(st[i]), out[i].tobytes()) for i in range(n)]


def expected(ec, ln, op, keys_xy, items):
    """What eb200_scalar_mul_batch / eb200_mul_add_batch / eb200_ecdh_derive_batch give: the oracle's Point.mul and
    G.mulAdd on the point as given (not precomputed), KeyPair.derive's validation, affine x || y or INFINITY."""
    out = []
    for k1, k2, ki in items:
        P = ec.curve.point(*keys_xy[ki])
        if op == 2:
            if not P.validate():
                out.append((ST_THROW_NOT_VALIDATED, bytes(ln)))
                continue
            R = P.mul(k2 % ec.n)
        elif op == 0:
            R = P.mul(k2)
        else:
            R = ec.g.mul_add(k1, P, k2)
        if R.is_infinity():
            out.append((ST_INFINITY, bytes(ln if op == 2 else 2 * ln)))
        else:
            out.append((ST_TRUE, R.x.to_bytes(ln, "big") + (b"" if op == 2 else R.y.to_bytes(ln, "big"))))
    return out


_CASES = {}


def cases(name):
    """Keys (seeded, G, -G, 2^j G, table entries of G, one off the curve) and items: edge scalars on every key, pairs
    with k1 G + k2 Q = O and k1 G = k2 Q, seeded scalars, and items on the off-curve key."""
    if name not in _CASES:
        from oracle.ref_py.ec import EC
        cid, ln = BY_NAME[name]
        ec = EC(name)
        n, top = ec.n, (1 << (8 * ln)) - 1
        rnd = random.Random(cid)
        ds = [rnd.randrange(1, n) for _ in range(2)] + [d for d, _ in adversarial_keys(ec, cid, (4, 8))]
        if ln >= 48:
            ds = ds[:6]
        keys = [(Q.x, Q.y) for Q in (ec.g.mul(d) for d in ds)]
        keys.append((keys[0][0], (keys[0][1] + 1) % ec.curve.p))          # imported, not validated, off the curve
        edges = [0, 1, n - 1, n, n + 1, top]
        items = []
        for ki, d in enumerate(ds):
            for j, k in enumerate(edges if ki < 3 or ln < 48 else edges[::2]):
                items.append((edges[(j + ki) % len(edges)] if ki % 2 else rnd.randrange(top), k, ki))
            k2 = rnd.randrange(1, n)
            items.append(((-k2 * d) % n, k2, ki))                         # k1 G + k2 Q = O
            items.append(((k2 * d) % n, k2, ki))                          # k1 G = k2 Q: a doubling
        off = len(keys) - 1
        items += [(rnd.randrange(top), k, off) for k in (1, n - 1, rnd.randrange(top))]
        rnd.shuffle(items)
        _CASES[name] = (ec, keys, items, {op: expected(ec, ln, op, keys, items) for op in OPS.values()})
    return _CASES[name]


@pytest.mark.parametrize("name,W", [("secp256k1", W) for W in (4, 5, 6, 7, 8)] +
                         [(nm, W) for nm in ("p256", "p384", "p521", "p192", "p224") for W in (4, 8)])
@pytest.mark.parametrize("op", sorted(OPS))
def test_bodies_against_oracle(he, name, W, op):
    """Mutation checks (test_oracle_comparison_catches_a_broken_body): dropping the sign of a digit, skipping the
    exceptional-addition path, or letting an infinity into the normalisation's product chain each make this fail."""
    cid, ln = BY_NAME[name]
    ec, keys, items, want = cases(name)
    kst, got = run_bodies(he, cid, ln, W, OPS[op], keys, items)
    assert kst == [1] * (len(keys) - 1) + [0]
    assert got == want[OPS[op]], [i for i in range(len(items)) if got[i] != want[OPS[op]][i]]
    sts = [s for s, _ in got]
    assert ST_INFINITY in sts and sts.count(ST_TRUE) > len(sts) // 2
    assert (ST_THROW_NOT_VALIDATED in sts) == (op == "derive")


def norm_items(ec, B, T, rnd):
    """B T items of pub.mul(k) on one key, so that normalisation thread t (items t, t + T, ...) sees: t = 0 only
    infinities, t = 1 an infinity in its first slot only, t = 2 in its last slot only, the others none."""
    items = []
    for i in range(B * T):
        t, j = i % T, i // T
        inf = t == 0 or (t == 1 and j == 0) or (t == 2 and j == B - 1)
        items.append((0, (ec.n if i % 2 else 0) if inf else rnd.randrange(1, ec.n), 0))
    return items


@pytest.mark.parametrize("name,B", [("secp256k1", 16), ("secp256k1", 32), ("p256", 16), ("p521", 16)])
def test_normalisation_batches(he, name, B):
    from oracle.ref_py.ec import EC
    cid, ln = BY_NAME[name]
    ec = EC(name)
    Q = ec.g.mul(0xC0FFEE)
    items = norm_items(ec, B, 4, random.Random(B))
    want = expected(ec, ln, 0, [(Q.x, Q.y)], items)
    for op in (0, 2):
        got = run_bodies(he, cid, ln, 4, op, [(Q.x, Q.y)], items, batch=B)[1]
        assert got == (want if op == 0 else [(s, o[:ln]) for s, o in want]), op
    assert [s for s, _ in want[::4]] == [ST_INFINITY] * B


# Each mutation breaks one decision of both keyed multiplication bodies (or of the additions they call).
MUTATIONS = {
    "digit sign": [("ecdsa_keyset_body.cuh", "const bool neg = ((flags & (h ? FL_NEG2 : FL_NEG1)) != 0) != dneg;",
                    "const bool neg = (flags & (h ? FL_NEG2 : FL_NEG1)) != 0;"),
                   ("ecdsa_keyset_body.cuh", "const bool neg = ((flags & W_::FL_NEG2) != 0) != dneg;",
                    "const bool neg = (flags & W_::FL_NEG2) != 0;")],
    "cold path": [("ge_k256.cuh", "if (fe_is_zero(r.z)) {                       // cold: a == inf, or h == 0", "if (false) {"),
                  ("ecdsa_sw_body.cuh", "    r.z = F::mul(a.z, h);\n    if (F::is_zero(r.z)) {", "    r.z = F::mul(a.z, h);\n    if (false) {")],
    "infinity in chain": [("ecdsa_keyset_body.cuh", "if (status[i] != ST_TRUE || fe_is_zero(z)) continue;",
                           "if (status[i] != ST_TRUE) continue;"),
                          ("ecdsa_keyset_body.cuh", "if (status[i] != 1 || F::is_zero(z)) continue;", "if (status[i] != 1) continue;")],
}


@pytest.mark.parametrize("kind", sorted(MUTATIONS))
def test_oracle_comparison_catches_a_broken_body(he, tmp_path, kind):
    root = str(tmp_path)
    shutil.copytree(os.path.join(ROOT, "elliptic_b200", "csrc"), os.path.join(root, "elliptic_b200", "csrc"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(root, "include"))
    shutil.copytree(os.path.join(ROOT, "tests", "hostemu"), os.path.join(root, "tests", "hostemu"))
    for fname, old, new in MUTATIONS[kind]:
        path = os.path.join(root, "elliptic_b200", "csrc", fname)
        src = open(path).read()
        assert src.count(old) == 1, (fname, old)
        open(path, "w").write(src.replace(old, new))
    bad = build_hostemu(root, root)
    for name in ("secp256k1", "p256"):
        cid, ln = BY_NAME[name]
        ec, keys, items, want = cases(name)
        assert any(run_bodies(bad, cid, ln, 8, OPS[op], keys, items)[1] != want[OPS[op]] for op in ("mul", "mul_add")), (kind, name)


def test_return_codes_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    p = np.zeros(1 << 12, np.uint8).ctypes.data
    for fn, nargs in ((lib.eb200_scalar_mul_batch_keyed, 4), (lib.eb200_mul_add_batch_keyed, 5), (lib.eb200_ecdh_derive_batch_keyed, 4)):
        assert fn(None, 4, *[p] * nargs) == _native.ERR_ARG              # no set
        assert fn(None, 0, *[p] * nargs) == _native.ERR_ARG
