"""Key sets without a GPU: the build and keyed-verify bodies run through the host emulation against the oracle's
EC.verify, the table geometry against the oracle's point arithmetic, the automatic width choice, and the C entry
points' return codes without a device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from ks_items import CURVES, LIMBS, adversarial_items, adversarial_keys, expected, pack, seeded_set, windows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BY_NAME = {nm: (cid, ln) for nm, cid, ln in CURVES}
EMU_GW = {"secp256k1": 8}          # fixed-base window of the emulation build (-DEB_GW=8 -DEB_SW_GW=6)


def build_hostemu(root, out_dir):
    lib = os.path.join(out_dir, "libkeyset_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", "-shared", "-fPIC", "-o", lib,
                    os.path.join(root, "tests", "hostemu", "keyset_emu.cpp")], check=True)
    he = ctypes.CDLL(lib)
    he.he_keyset_key_bytes.restype = ctypes.c_size_t
    he.he_keyset_choose_bits.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t]
    he.he_keyset_verify.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 6
    he.he_keyset_table.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    he.he_k256_beta_x.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    return he


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    return build_hostemu(ROOT, str(tmp_path_factory.mktemp("hostemu")))


def run_bodies(he, cid, ln, W, keys_xy, items):
    xy, e, r, s, idx = pack(ln, keys_xy, items)
    kst, st = np.zeros(len(keys_xy), np.uint8), np.zeros(len(items), np.uint8)
    he.he_keyset_verify(cid, W, len(keys_xy), xy.ctypes.data, len(items), e.ctypes.data,
                        r.ctypes.data, s.ctypes.data, idx.ctypes.data, kst.ctypes.data, st.ctypes.data)
    return list(kst), [int(v) for v in st]


_CASES = {}


def cases(name):
    """Keys and items of one curve: seeded honest traffic, the adversarial keys, and an off-curve key."""
    if name not in _CASES:
        from oracle.ref_py.ec import EC
        cid, ln = BY_NAME[name]
        ec = EC(name)
        keys, items = seeded_set(ec, ln, 3, 24 if ln < 66 else 12)
        adv = adversarial_keys(ec, cid, (4, 8))
        if ln >= 48:
            adv = adv[:4] + adv[-2:]
        base = len(keys)
        keys += [(Q.x, Q.y) for _, Q in adv]
        items += [it[:3] + (it[3] + base,) for it in adversarial_items(ec, cid, adv, EMU_GW.get(name, 6))]
        keys.append((keys[0][0], (keys[0][1] + 1) % ec.curve.p))             # imported, not validated, off the curve
        items += [(e, r, s, len(keys) - 1) for e, r, s, _ in items[:3]]
        _CASES[name] = (ec, keys, items, expected(ec, keys, items))
    return _CASES[name]


@pytest.mark.parametrize("name,W", [("secp256k1", W) for W in (4, 5, 6, 7, 8)] + [("p256", 4), ("p256", 7), ("p384", 5), ("p384", 8),
                                    ("p224", 4), ("p224", 8), ("p192", 6), ("p521", 8)])
def test_bodies_against_oracle(he, name, W):
    """Mutation checks (test_oracle_comparison_catches_a_broken_body): dropping the sign of a digit, skipping the
    exceptional-addition path, or dropping the second eqXToP candidate each make this comparison fail."""
    cid, ln = BY_NAME[name]
    ec, keys, items, want = cases(name)
    kst, got = run_bodies(he, cid, ln, W, keys, items)
    assert kst == [1] * (len(keys) - 1) + [0]
    assert got == want, [i for i in range(len(items)) if got[i] != want[i]]
    assert sum(want) > len(want) // 2 and 0 in want


def test_second_candidate_is_reached(he):
    """r + n < p: the fixture-free way to reach eqXToP's second candidate is a key forged for a chosen R, as
    recoverPubKey does: Q = r^-1 (s R - e G)."""
    from oracle.ref_py.ec import EC
    ec = EC("secp256k1")
    n = ec.n
    keys, items = [], []
    x = n
    while len(items) < 3:
        x += 1
        try:
            R = ec.curve.point_from_x(x, len(items) & 1)
        except Exception:
            continue
        r, e, s = x - n, 0x1111 * (len(items) + 1), 0x2222 * (len(items) + 3)
        ri = pow(r, -1, n)
        Q = ec.g.mul_add((n - e) * ri % n, R, s * ri % n)
        keys.append((Q.x, Q.y))
        items.append((e, r, s, len(keys) - 1))
    want = expected(ec, keys, items)
    assert want == [1, 1, 1]
    for W in (4, 8):
        assert run_bodies(he, 1, 32, W, keys, items)[1] == want
    _CASES["second"] = (ec, keys, items, want)


@pytest.mark.parametrize("name,W", [("secp256k1", 4), ("secp256k1", 8), ("p256", 5), ("p384", 4), ("p521", 4), ("p192", 8), ("p224", 6)])
def test_table_geometry(he, name, W):
    """Entry (j, i) of a key's table is (2i+1) 2^(W j) Q; on secp256k1 the second GLV half reads (beta x, y) = lambda times it."""
    from oracle.ref_py.ec import EC
    cid, ln = BY_NAME[name]
    ec = EC(name)
    Q = ec.g.mul(0xC0FFEE)
    nw, E, L = windows(cid, W), 1 << (W - 1), LIMBS[cid]
    assert he.he_keyset_windows(cid, W) == nw and he.he_keyset_key_bytes(cid, W) == nw * E * 2 * L * 4
    out = np.zeros(nw * E * 2 * L, np.uint32)
    xy = pack(ln, [(Q.x, Q.y)], [])[0]
    he.he_keyset_table(cid, W, xy.ctypes.data, out.ctypes.data)
    val = lambda w: sum(int(v) << (32 * k) for k, v in enumerate(w))
    for j, i in {(0, 0), (0, E - 1), (1, 1), (nw // 2, E // 2), (nw - 1, 0), (nw - 1, E - 1)}:
        P = Q.mul(((2 * i + 1) << (W * j)) % ec.n)
        ent = out[(j * E + i) * 2 * L:(j * E + i + 1) * 2 * L]
        assert (val(ent[:L]), val(ent[L:])) == (P.x, P.y), (j, i)
        if cid == 1:
            bx = np.zeros(8, np.uint32)
            he.he_k256_beta_x(ent[:8].copy().ctypes.data, bx.ctypes.data)
            lam = 0x5363ad4cc05c30e0a5261c028812645a122e22ea20816678df02967c1b23bd72
            lP = P.mul(lam)
            assert (val(bx), val(ent[L:])) == (lP.x, lP.y), (j, i)


# Each mutation breaks one decision of both keyed bodies (or of the additions they call).
MUTATIONS = {
    "digit sign": [("ecdsa_keyset_body.cuh", "bool neg = dneg != ((flags & (h ? FL_NEG2 : FL_NEG1)) != 0);",
                    "bool neg = (flags & (h ? FL_NEG2 : FL_NEG1)) != 0;"),
                   ("ecdsa_keyset_body.cuh", "bool neg = dneg != ((flags & W_::FL_NEG2) != 0);", "bool neg = (flags & W_::FL_NEG2) != 0;")],
    "cold path": [("ge_k256.cuh", "if (fe_is_zero(r.z)) {                       // cold: a == inf, or h == 0", "if (false) {"),
                  ("ecdsa_sw_body.cuh", "    r.z = F::mul(a.z, h);\n    if (F::is_zero(r.z)) {", "    r.z = F::mul(a.z, h);\n    if (false) {")],
    "second candidate": [("ecdsa_keyset_body.cuh", "if (!geq_n<8>(rf.v, pmn)) {      // r + n < p: second candidate",
                          "if (false) {")],
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
    if kind == "second candidate":
        test_second_candidate_is_reached(he)
        ec, keys, items, want = _CASES["second"]
        assert run_bodies(bad, 1, 32, 8, keys, items)[1] != want
        return
    for name in ("secp256k1", "p256"):
        cid, ln = BY_NAME[name]
        ec, keys, items, want = cases(name)
        assert run_bodies(bad, cid, ln, 8, keys, items)[1] != want, (kind, name)


def test_width_chooser(he):
    """The widest W in 4..8 whose m tables fit the budget; 0 (the entry point then answers ERR_ARG) when W = 4 does not."""
    G = 1 << 30
    per = lambda cid, W: windows(cid, W) * (1 << (W - 1)) * 2 * LIMBS[cid] * 4
    for cid in (1, 2, 3, 6, 7, 8):
        for m in (1, 64, 4096, 1 << 16, 1 << 20):
            want = next((W for W in (8, 7, 6, 5, 4) if m * per(cid, W) <= G), 0)
            assert he.he_keyset_choose_bits(cid, m, G) == want, (cid, m)
    assert he.he_keyset_choose_bits(1, 4096, G) == 8                 # 4096 keys x 139264 B = 544 MiB
    assert he.he_keyset_choose_bits(1, 1 << 16, G) == 0              # 2^16 keys x 16896 B at W = 4 is over 1 GiB
    assert he.he_keyset_choose_bits(1, 1 << 16, 2 * G) == 5             # 27 windows x 16 entries x 64 B = 27648 B a key
    assert he.he_keyset_choose_bits(4, 1, G) == 0 and he.he_keyset_choose_bits(5, 1, G) == 0     # the 25519 curves


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
    create = lambda *a: lib.eb200_keyset_create(*a, ctypes.byref(out))
    assert create(1, 4, p, 0, 0, p) == _native.ERR_NOT_INIT and out.value is None
    assert create(1, 4, None, 0, 0, p) == _native.ERR_ARG
    assert create(1, 4, p, 0, 0, None) == _native.ERR_ARG
    assert lib.eb200_keyset_create(1, 4, p, 0, 0, p, None) == _native.ERR_ARG
    assert create(1, 4, p, 3, 0, p) == _native.ERR_ARG               # pub_fmt
    assert create(1, 4, p, 0, 3, p) == _native.ERR_ARG and create(1, 4, p, 0, 9, p) == _native.ERR_ARG
    assert create(1, 0, p, 0, 0, p) == _native.ERR_ARG
    assert create(1, 1 << 16, p, 0, 0, p) == _native.ERR_ARG         # no width fits the default budget
    assert create(1, 1 << 16, p, 0, 4, p) == _native.ERR_NOT_INIT    # an explicit width is not held to it
    assert create(4, 4, p, 0, 0, p) == _native.ERR_UNSUPPORTED and create(5, 4, p, 0, 0, p) == _native.ERR_UNSUPPORTED
    assert create(77, 4, p, 0, 0, p) == _native.ERR_UNSUPPORTED
    assert lib.eb200_keyset_destroy(None) == _native.OK
    assert lib.eb200_keyset_info(None, None, None, None, None) == _native.ERR_ARG
    assert lib.eb200_ecdsa_verify_batch_keyed(None, 4, p, p, p, p, p) == _native.ERR_ARG
