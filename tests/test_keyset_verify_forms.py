"""The DER and device-pointer forms of the keyed ECDSA verify without a GPU: the keyed DER decode, index screen and
verdict merge bodies run through the host emulation, alone on hand-built cases and on bit-flipped DER, and framed around
the keyed verify bodies in kernel order against the oracle's key.verify with DER signatures on all six presets; and the
C entry points' return codes without a device."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import ks_der_items as kd
from ks_items import CURVES, pack, seeded_set

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BY_NAME = {nm: (cid, ln) for nm, cid, ln in CURVES}
ST_FALSE, ST_TRUE, ST_INVALID_POINT, ST_ASSERT, ST_POINT_FORMAT, ST_SIG_FORMAT, ST_BAD_KEY_INDEX = 0, 1, 2, 5, 6, 9, 12
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostemu")), "libkeyset_forms_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-DEB_GW=8", "-DEB_SW_GW=6", "-shared", "-fPIC", "-o", lib,
                    os.path.join(ROOT, "tests", "hostemu", "keyset_forms_emu.cpp")], check=True)
    h = ctypes.CDLL(lib)
    h.he_keyset_verify.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, P, ctypes.c_size_t] + [P] * 6
    h.he_ks_der_decode.argtypes = [ctypes.c_size_t, ctypes.c_uint32] + [P] * 7
    h.he_ks_index_screen.argtypes = [ctypes.c_size_t, P, ctypes.c_size_t, P, P]
    h.he_ks_verdict_merge.argtypes = [ctypes.c_size_t, P, P]
    return h


def decode(he, ln, ders, key_idx, kst):
    data, off = kd.blob(ders)
    n = len(ders)
    r, s = np.full((n, ln), 0xAA, np.uint8), np.full((n, ln), 0xAA, np.uint8)     # stale bytes the decode must clear
    vd = np.zeros(n, np.uint8)
    idx = np.ascontiguousarray(key_idx, np.uint32)
    kst = np.ascontiguousarray(kst, np.uint8)
    he.he_ks_der_decode(n, ln, data.ctypes.data, off.ctypes.data, idx.ctypes.data, kst.ctypes.data, r.ctypes.data,
                        s.ctypes.data, vd.ctypes.data)
    return r, s, vd


def merge(he, vd, status):
    st = np.array(status, np.uint8)
    he.he_ks_verdict_merge(len(st), np.ascontiguousarray(vd, np.uint8).ctypes.data, st.ctypes.data)
    return st


def test_der_decode_verdicts_hand_built(he):
    """Key throw first, then the DER rejection, else 0; a rejected encoding leaves r = s = 0."""
    good = kd.canonical(0x1234, 0x5678)
    bad = good[:-1]
    kst = [ST_TRUE, ST_FALSE, ST_INVALID_POINT, ST_POINT_FORMAT, ST_ASSERT]
    ders = [good, bad] * len(kst)
    key_idx = [k for k in range(len(kst)) for _ in range(2)]
    r, s, vd = decode(he, 32, ders, key_idx, kst)
    want = []
    for k in kst:
        want += [k if k > ST_TRUE else 0, k if k > ST_TRUE else ST_SIG_FORMAT]
    assert list(vd) == want
    for i in range(0, len(ders), 2):
        assert int.from_bytes(r[i].tobytes(), "big") == 0x1234 and int.from_bytes(s[i].tobytes(), "big") == 0x5678
        assert not r[i + 1].any() and not s[i + 1].any()


def test_index_screen_and_merge_precedence(he):
    """An index >= m is replaced by 0 and gets BAD_KEY_INDEX, which the merge writes over any keyed status; a zero
    verdict leaves the keyed status alone."""
    m = 5
    key_idx = np.array([0, m - 1, m, 1 << 31, (1 << 32) - 1, 2], np.uint32)
    out, vd = np.full(len(key_idx), 7, np.uint32), np.full(len(key_idx), 0xEE, np.uint8)
    he.he_ks_index_screen(len(key_idx), key_idx.ctypes.data, m, out.ctypes.data, vd.ctypes.data)
    assert list(out) == [0, m - 1, 0, 0, 0, 2]
    assert list(vd) == [0, 0, ST_BAD_KEY_INDEX, ST_BAD_KEY_INDEX, ST_BAD_KEY_INDEX, 0]
    assert list(merge(he, vd, [ST_TRUE, ST_FALSE, ST_TRUE, ST_INVALID_POINT, ST_SIG_FORMAT, ST_TRUE])) == \
        [ST_TRUE, ST_FALSE, ST_BAD_KEY_INDEX, ST_BAD_KEY_INDEX, ST_BAD_KEY_INDEX, ST_TRUE]
    assert list(merge(he, [0, ST_SIG_FORMAT, ST_POINT_FORMAT, 0], [ST_FALSE, ST_TRUE, ST_TRUE, 4])) == \
        [ST_FALSE, ST_SIG_FORMAT, ST_POINT_FORMAT, 4]


@pytest.mark.parametrize("ln", [24, 28, 32, 48, 66])
def test_bit_flipped_der_decode(he, ln):
    """The keyed decode reads each DER exactly as the oracle's _importDER: accept / reject, and the value it writes
    (0 where the integer does not fit len bytes, which the range test then rejects as the reference does)."""
    rnd = random.Random(ln)
    ders = []
    for _ in range(300):
        r, s = rnd.randrange(1, 1 << (8 * ln)), rnd.randrange(1, 1 << rnd.choice([8, 8 * ln - 1, 8 * ln]))
        ders += kd.variants(r, s, rnd)
    r, s, vd = decode(he, ln, ders, [0] * len(ders), [ST_TRUE])
    accepted = 0
    for i, der in enumerate(ders):
        rs = kd.parse(der)
        if rs is None:
            assert vd[i] == ST_SIG_FORMAT and not r[i].any() and not s[i].any(), der.hex()
            continue
        accepted += 1
        assert vd[i] == 0, der.hex()
        for got, v in ((r[i], rs[0]), (s[i], rs[1])):
            assert int.from_bytes(got.tobytes(), "big") == (v if v < 1 << (8 * ln) else 0), der.hex()
    assert 0 < accepted < len(ders)


def keyed_der_pipeline(he, cid, ln, W, keys_xy, es, ders, key_idx, kst):
    """Keyed DER decode -> prep -> keyed main -> keyed replay -> verdict merge, as one chunk of the GPU call runs them.
    kst: the set's verdicts as the decode reads them (import throws included)."""
    n = len(ders)
    xy = pack(ln, keys_xy, [])[0]
    idx = np.ascontiguousarray(key_idx, np.uint32)
    e = np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in es), np.uint8).reshape(n, ln).copy()
    r, s, vd = decode(he, ln, ders, idx, kst)
    st = np.zeros(n, np.uint8)
    he.he_keyset_verify(cid, W, len(keys_xy), xy.ctypes.data, n, e.ctypes.data, r.ctypes.data, s.ctypes.data,
                        idx.ctypes.data, np.zeros(len(keys_xy), np.uint8).ctypes.data, st.ctypes.data)
    return merge(he, vd, st)


@pytest.mark.parametrize("name,W", [("secp256k1", 4), ("secp256k1", 8), ("p256", 5), ("p384", 6), ("p521", 4), ("p192", 8),
                                    ("p224", 7)])
def test_keyed_der_pipeline_against_oracle(he, name, W):
    """Every DER form of honest and damaged signatures, on on-curve keys and an imported off-curve key, equals the
    oracle's key.verify(msg, der); with import throws put into the set's verdicts, those keys' items take the throw."""
    from oracle.ref_py.ec import EC
    cid, ln = BY_NAME[name]
    ec = EC(name)
    rnd = random.Random(cid * 10 + W)
    keys, items = seeded_set(ec, ln, 3, 6 if ln < 66 else 4, seed=cid)
    keys.append((keys[0][0], (keys[0][1] + 1) % ec.curve.p))             # imported, not validated, off the curve
    items += [(e, r, s, len(keys) - 1) for e, r, s, _ in items[:2]]
    es, ders, key_idx = [], [], []
    for e, r, s, k in items:
        for der in kd.variants(r, s, rnd):
            es.append(e); ders.append(der); key_idx.append(k)
    got = keyed_der_pipeline(he, cid, ln, W, keys, es, ders, key_idx, [ST_TRUE] * 3 + [ST_FALSE])
    want = [kd.status(ec, es[i], ders[i], keys[key_idx[i]]) for i in range(len(ders))]
    assert list(got) == want, [i for i in range(len(want)) if got[i] != want[i]]
    assert ST_TRUE in want and ST_FALSE in want and ST_SIG_FORMAT in want
    kst = [ST_TRUE, ST_POINT_FORMAT, ST_TRUE, ST_INVALID_POINT]       # keys 1 and 3 threw at import
    got = keyed_der_pipeline(he, cid, ln, W, keys, es, ders, key_idx, kst)
    want = [kd.status(ec, es[i], ders[i], keys[key_idx[i]], kst[key_idx[i]] if kst[key_idx[i]] > ST_TRUE else 0)
            for i in range(len(ders))]
    assert list(got) == want, [i for i in range(len(want)) if got[i] != want[i]]


def test_return_codes_without_device():
    """No set is ERR_ARG before the device count is looked at, for every n and pointer; its workspace is 0 bytes."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    p = np.zeros(1 << 12, np.uint8).ctypes.data
    for n in (0, 4):
        for ptr in (p, None):
            assert lib.eb200_ecdsa_verify_batch_keyed_der(None, n, *[ptr] * 5) == _native.ERR_ARG
            assert lib.eb200_ecdsa_verify_batch_keyed_dev(None, n, *[ptr] * 7) == _native.ERR_ARG
        assert lib.eb200_ecdsa_verify_keyed_workspace_bytes(None, n) == 0
    assert _native.ST_BAD_KEY_INDEX == 12
