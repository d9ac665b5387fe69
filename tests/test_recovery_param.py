"""EC.getKeyRecoveryParam without a GPU: the kernel bodies (prep, main and cold) run through the host emulation
against the oracle's restatement of the reference, the C entry point's return codes without a device, and the
host mirror's recoveryParam shortcut."""
import ctypes
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

from krp_items import CURVES, NO_RECOVERY, get_key_recovery_param, krp_expected, krp_items

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_hostemu(root, out_dir):
    lib = os.path.join(out_dir, "librecovery_param_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", "-shared", "-fPIC", "-o", lib,
                    os.path.join(root, "tests", "hostemu", "recovery_param_emu.cpp")], check=True)
    return ctypes.CDLL(lib)


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    return build_hostemu(ROOT, str(tmp_path_factory.mktemp("hostemu")))


def run_bodies(he, cid, ln, items):
    """The three bodies on `items`: (recid list, status list)."""
    from oracle.ref_py import curves
    n = len(items)
    nmod = curves.get(dict((c, nm) for nm, c, _ in CURVES)[cid]).curve.n
    col = lambda k, mod=None: b"".join(((it[k] % mod) if mod else it[k]).to_bytes(ln, "big") for it in items)
    q = b"".join(it[3].to_bytes(ln, "big") + it[4].to_bytes(ln, "big") for it in items)
    rid, st = (ctypes.c_uint8 * n)(), (ctypes.c_uint8 * n)()
    he.he_recovery_param(cid, ctypes.c_size_t(n), col(0, nmod), col(1), col(2), q, rid, st)
    return [int(v) for v in rid], [int(v) for v in st]


def answers(rid, st):
    for j, s in zip(rid, st):
        assert s in (1, NO_RECOVERY) and (s == 1 or j == 0)
    return [j if s == 1 else s for j, s in zip(rid, st)]


_ITEMS = {}


def cases(name, ln):
    if name not in _ITEMS:
        from oracle.ref_py.ec import EC
        ec = EC(name)
        items, truth = krp_items(ec, ln, count=4 if ln < 66 else 2)
        _ITEMS[name] = (ec, items, truth, [krp_expected(ec, it) for it in items])
    return _ITEMS[name]


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_bodies_against_oracle(he, name, cid, ln):
    ec, items, truth, want = cases(name, ln)
    got = answers(*run_bodies(he, cid, ln, items))
    for i, t in truth.items():
        assert want[i] == t and got[i] == t, i
    assert got == want
    assert {0, 1, 2, 3, NO_RECOVERY} <= set(want), set(want)


# Each mutation breaks one decision of both bodies; the oracle comparison must notice it on every curve kind.
MUTATIONS = {
    "parity": [("ecdsa_k256_body.cuh", "zi))) j |= 1;", "zi))) j |= 0;"),
               ("ecdsa_sw_body.cuh", "recid[i] = (uint8_t)(j | (y.v[0] & 1));", "recid[i] = (uint8_t)j;")],
    "second candidate": [("ecdsa_k256_body.cuh", "if (geq_n<8>(rv, pmn)) return ST_THROW_NO_RECOVERY;    // no second",
                          "if (true) return ST_THROW_NO_RECOVERY;    // no second"),
                         ("ecdsa_sw_body.cuh", "if (geq_n<N>(rp.v, pmn)) return 11;                // no second",
                          "if (true) return 11;                // no second")],
}


@pytest.mark.parametrize("kind", sorted(MUTATIONS))
def test_oracle_comparison_catches_a_broken_body(tmp_path, kind):
    root = str(tmp_path)
    shutil.copytree(os.path.join(ROOT, "elliptic_b200", "csrc"), os.path.join(root, "elliptic_b200", "csrc"))
    shutil.copytree(os.path.join(ROOT, "tests", "hostemu"), os.path.join(root, "tests", "hostemu"))
    for fname, old, new in MUTATIONS[kind]:
        path = os.path.join(root, "elliptic_b200", "csrc", fname)
        src = open(path).read()
        assert src.count(old) == 1, (fname, old)
        open(path, "w").write(src.replace(old, new))
    bad = build_hostemu(root, root)
    for name, cid, ln in (CURVES[0], CURVES[1], CURVES[5]):
        ec, items, truth, want = cases(name, ln)
        assert answers(*run_bodies(bad, cid, ln, items)) != want, (kind, name)


# Return codes of the new entry point without a device (-3 ERR_ARG, -4 ERR_NOT_INIT, -5 ERR_UNSUPPORTED), beside what
# eb200_ecdsa_recover_batch returns for the same cases: without a device both answer ERR_NOT_INIT first.
RECOVER_NO_DEVICE = {"curve77": -4, "ed25519": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4,
                     "null6": -4, "null7": -4}
RECOVERY_PARAM_NO_DEVICE = {"curve77": -4, "ed25519": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4,
                            "null6": -4, "null7": -4}


def abi_cases():
    """(tag, args) for calls of the shape (curve, n, e, r, s, x, out, status): four secp256k1 items, then an empty
    batch, a NULL in each pointer, an unknown curve and ed25519."""
    buf = np.zeros(1 << 12, np.uint8)
    base = [1, 4] + [buf.ctypes.data] * 6
    out = []
    for tag, pos, val in [("curve77", 0, 77), ("ed25519", 0, 4), ("n0", 1, 0)] + [("null%d" % k, k, None) for k in range(2, 8)]:
        args = list(base)
        args[pos] = val
        out.append((tag, args))
    return out, buf


def test_return_codes_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    cases_, _keep = abi_cases()
    assert {t: lib.eb200_ecdsa_recover_batch(*a) for t, a in cases_} == RECOVER_NO_DEVICE
    assert {t: lib.eb200_ecdsa_recovery_param_batch(*a) for t, a in cases_} == RECOVERY_PARAM_NO_DEVICE


def test_mirror_answers_a_carried_recovery_param_without_a_device():
    """ec/index.js:263-264, and the reference's own round trip (test/ecdsa-test.js:467-475) through the mirror."""
    from elliptic_b200.ec import EC, EllipticError
    from oracle.ref_py.ec import EC as RefEC
    ref, ec = RefEC("secp256k1"), EC("secp256k1")
    rnd = random.Random(9)
    d = rnd.randrange(1, ref.n)
    key = ref.g.mul(d)
    msg = list(range(11))
    signature = ref.sign(msg, d)
    recid = ec.get_key_recovery_param(msg, signature, (key.x, key.y))
    assert recid == signature.recovery_param == get_key_recovery_param(ref, msg, signature, key)
    assert key.eq(ref.recover_pub_key(msg, signature, recid))
    sig = {"r": signature.r, "s": signature.s, "recoveryParam": 3}
    assert ec.get_key_recovery_param(msg, sig, None) == 3          # returned before Q is looked at, as the reference
    js, st = ec.get_key_recovery_param_batch([msg, msg], [sig, signature], [None, (key.x, key.y)])
    assert js == [3, signature.recovery_param] and list(st) == [1, 1]
    with pytest.raises(EllipticError, match="Signature without r or s"):
        ec.get_key_recovery_param(msg, {"r": 0, "s": 5, "recoveryParam": 1}, None)
    with pytest.raises(EllipticError, match="short curves only"):
        EC("ed25519").get_key_recovery_param_batch([msg], [sig], [None])
