"""Keyed getKeyRecoveryParam without a GPU: the build, recovery-parameter prep, keyed main, recid normalisation and cold
bodies run through the host emulation in kernel order against the oracle's getKeyRecoveryParam on all six presets,
with mutation checks, and the C entry point's return codes without a device."""
import ctypes
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

from krp_items import CURVES, NO_RECOVERY, krp_expected, krp_items
from ks_items import adversarial_keys, first_g_digit, minted

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BY_NAME = {nm: (cid, ln) for nm, cid, ln in CURVES}
ST_TRUE, THROW = 1, 2                  # THROW: the decoder's 'invalid point', standing for any import throw


def build_hostemu(root, out_dir):
    lib = os.path.join(out_dir, "libkeyset_rp_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", "-shared", "-fPIC", "-o", lib,
                    os.path.join(root, "tests", "hostemu", "keyset_rp_emu.cpp")], check=True)
    he = ctypes.CDLL(lib)
    he.he_keyset_recovery_param.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_size_t] + [ctypes.c_void_p] * 4 + [ctypes.c_int] + [ctypes.c_void_p] * 3
    return he


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    return build_hostemu(ROOT, str(tmp_path_factory.mktemp("hostemu_krp")))


def col(vals, ln):
    return np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in vals), np.uint8).reshape(len(vals), ln).copy()


def run_bodies(he, cid, ln, n_mod, W, keys_xy, pre, items, batch=16):
    """items: (e, r, s, key index), e below n.  Returns (key statuses, [j or the status where it is not TRUE])."""
    xy = np.ascontiguousarray(np.concatenate([col([k[0] for k in keys_xy], ln), col([k[1] for k in keys_xy], ln)], axis=1))
    pre = np.array(pre, np.uint8)
    e, r, s = (col([it[j] for it in items], ln) for j in range(3))
    idx = np.array([it[3] for it in items], np.uint32)
    n = len(items)
    kst, rid, st = np.zeros(len(keys_xy), np.uint8), np.full(n, 0xA5, np.uint8), np.zeros(n, np.uint8)
    he.he_keyset_recovery_param(cid, W, len(keys_xy), xy.ctypes.data, pre.ctypes.data, n, e.ctypes.data, r.ctypes.data,
                                s.ctypes.data, idx.ctypes.data, batch, kst.ctypes.data, rid.ctypes.data, st.ctypes.data)
    for j, v in zip(rid, st):
        assert v == ST_TRUE or j == 0, (j, v)
    return list(kst), [int(j) if v == ST_TRUE else int(v) for j, v in zip(rid, st)]


def expected(ec, keys_xy, pre, items):
    """eb200_ecdsa_recovery_param_batch's answer with q = the key's x || y (the oracle's getKeyRecoveryParam on
    curve.point(x, y)), or the key's throw."""
    return [pre[k] if pre[k] else krp_expected(ec, (e, r, s) + tuple(keys_xy[k])) for e, r, s, k in items]


_CASES = {}


def cases(name):
    """Keys: every point krp_items uses (the signer's, wrong and forged keys, off-curve ones, x >= p), seeded keys, the
    adversarial keys (G, -G, 2^j G, entries of G's tables) and two keys whose import threw.  Items: krp_items' own
    (signatures, j = 2 / 3 forgeries, r = 0 / n, s = 0 / n found and not, r >= p, r without a square root), signatures by
    the seeded keys, and on each adversarial key (u1, u2) pairs that meet the exceptional additions (u1 G + u2 Q = O,
    u1 G = u2 Q, u2 Q = +- the first fixed-base entry), signed when P has an x, else with e = u1 s, r = u2 s."""
    if name not in _CASES:
        from oracle.ref_py.ec import EC
        cid, ln = BY_NAME[name]
        ec = EC(name)
        n = ec.n
        rnd = random.Random(cid + 40)
        big = ln >= 48
        kitems, _ = krp_items(ec, ln, count=2 if big else 4)
        keys, where = [], {}

        def key(xy):
            if xy not in where:
                where[xy] = len(keys)
                keys.append(xy)
            return where[xy]
        items = [(e % n, r, s, key((qx, qy))) for e, r, s, qx, qy in kitems]
        for _ in range(4 if big else 8):                    # j = 0 / 1 (and 2 / 3 where x(R) >= n happens)
            d = rnd.randrange(1, n)
            Q = ec.g.mul(d)
            k = key((Q.x, Q.y))
            for t in range(2):
                m = rnd.randrange(n)
                sig = ec.sign(m, d, canonical=bool(t))
                items.append((m, sig.r, sig.s, k))
        adv = adversarial_keys(ec, cid, (4, 8))
        for d, Q in adv[:5] if big else adv:
            k = key((Q.x, Q.y))
            u1 = rnd.randrange(1, n)
            u2s = [(-u1 * pow(d, -1, n)) % n, (u1 * pow(d, -1, n)) % n]
            u2s += [sg * first_g_digit(ec, u1, 6 if cid > 1 else 8) * pow(d, -1, n) % n for sg in (1, -1)]
            for u2 in u2s:
                sig = minted(ec, u1, u2, Q)
                if sig is None:
                    s = rnd.randrange(1, n)
                    sig = (u1 * s % n, u2 * s % n, s)
                items.append(sig + (k,))
        thrown = [key((ec.g.x, ec.g.y + t)) for t in (3, 5)]   # coordinates stored, never read
        pre = [THROW if k in thrown else 0 for k in range(len(keys))]
        items += [(rnd.randrange(n), rnd.randrange(1, n), rnd.randrange(1, n), k) for k in thrown]
        items += [(rnd.randrange(n), rnd.randrange(1, n), 0, thrown[0])]
        rnd.shuffle(items)
        _CASES[name] = (ec, keys, pre, items, expected(ec, keys, pre, items))
    return _CASES[name]


@pytest.mark.parametrize("name,W", [(nm, W) for nm, _, _ in CURVES for W in (4, 8)])
def test_bodies_against_oracle(he, name, W):
    cid, ln = BY_NAME[name]
    ec, keys, pre, items, want = cases(name)
    kst, got = run_bodies(he, cid, ln, ec.n, W, keys, pre, items)
    assert THROW in kst and 0 in kst and ST_TRUE in kst            # thrown, off the curve, on the curve
    assert got == want, [i for i in range(len(items)) if got[i] != want[i]]
    assert {0, 1, 2, 3, NO_RECOVERY, THROW} <= set(want), set(want)


def norm_items(ec, d, B, T, rnd):
    """B T items on key d G, so that normalisation thread t (items t, t + T, ...) sees: t = 0 no live item (r = 0),
    t = 1 a dead first slot only, t = 2 a dead last slot only, the others none."""
    items = []
    for i in range(B * T):
        t, j = i % T, i // T
        m = rnd.randrange(ec.n)
        sig = ec.sign(m, d)
        dead = t == 0 or (t == 1 and j == 0) or (t == 2 and j == B - 1)
        items.append((m, 0 if dead else sig.r, sig.s, 0))
    return items


@pytest.mark.parametrize("name,B", [("secp256k1", 16), ("secp256k1", 32), ("p256", 16), ("p521", 16)])
def test_normalisation_batches(he, name, B):
    from oracle.ref_py.ec import EC
    cid, ln = BY_NAME[name]
    ec = EC(name)
    d = 0xC0FFEE
    Q = ec.g.mul(d)
    items = norm_items(ec, d, B, 4, random.Random(B))
    items.append(items[5])                                  # one more item: the last thread's batch is partial
    want = expected(ec, [(Q.x, Q.y)], [0], items)
    assert run_bodies(he, cid, ln, ec.n, 4, [(Q.x, Q.y)], [0], items, batch=B)[1] == want
    assert want[:B * 4:4] == [NO_RECOVERY] * B and {0, 1} <= set(want)


# Each mutation breaks one decision of both keyed bodies.
MUTATIONS = {
    "parity": [("ecdsa_keyset_rp_body.cuh", "zi))) recid[i] |= 1;", "zi))) recid[i] |= 0;"),
               ("ecdsa_keyset_rp_body.cuh", "recid[i] |= (uint8_t)(y.v[0] & 1);", "recid[i] |= 0;")],
    "second candidate": [("ecdsa_keyset_rp_body.cuh", "j = 2;\n  }", "j = 0;\n  }"),
                         ("ecdsa_keyset_rp_body.cuh", "j = 2;\n    }", "j = 0;\n    }")],
    "live chain": [("ecdsa_keyset_rp_body.cuh", "if (status[i] != ST_TRUE) continue;\n    cnt", "cnt"),
                   ("ecdsa_keyset_rp_body.cuh", "if (status[i] != 1) continue;\n      cnt", "cnt")],
}


@pytest.mark.parametrize("kind", sorted(MUTATIONS))
def test_oracle_comparison_catches_a_broken_body(tmp_path, kind):
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
        ec, keys, pre, items, want = cases(name)
        assert run_bodies(bad, cid, ln, ec.n, 8, keys, pre, items)[1] != want, (kind, name)


def test_return_codes_without_device():
    """As tests/test_keyset_mul.py checks the keyed mul calls: no set is ERR_ARG before the device count is looked at."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    p = np.zeros(1 << 12, np.uint8).ctypes.data
    assert lib.eb200_ecdsa_recovery_param_batch_keyed(None, 4, *[p] * 6) == _native.ERR_ARG
    assert lib.eb200_ecdsa_recovery_param_batch_keyed(None, 0, *[p] * 6) == _native.ERR_ARG
