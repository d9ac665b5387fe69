"""The device-pointer forms of the keyed calls without a GPU: the index / scalar / range screens, the merge that zeroes
outputs and the screened hash, nonce and challenge bodies run through the host emulation on boundary cases, each
compared with a small Python model (and the model's mutants, which the cases must tell apart); and the C entry points'
return codes without a device."""
import ctypes
import hashlib
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N25519 = 2**252 + 27742317777372353535851937790883648493
ST_TRUE, ST_BAD_KEY_INDEX, ST_BAD_ITEM = 1, 12, 13
P = ctypes.c_void_p
M = 5                                                          # keys in the set
INDICES = [0, M - 1, M, 1 << 31, (1 << 32) - 1]
SCALARS = [0, 1, N25519 - 1, N25519, N25519 + 1, 2**252, 2**253, 2**256 - 1]


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostemu")), "libkeyset_dev_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", lib,
                    os.path.join(ROOT, "tests", "hostemu", "keyset_dev_emu.cpp")], check=True)
    h = ctypes.CDLL(lib)
    h.he_ks_index_scalar_screen.argtypes = [ctypes.c_size_t, P, ctypes.c_size_t, P, ctypes.c_int, P, P, P]
    h.he_ks_index_range_screen.argtypes = [ctypes.c_size_t, P, ctypes.c_size_t, P, ctypes.c_uint64, P, P]
    h.he_ks_verdict_merge_out.argtypes = [ctypes.c_size_t, P, P, P, ctypes.c_uint32]
    h.he_ks_ed_hash_screened.argtypes = [ctypes.c_size_t] + [P] * 6
    h.he_ed_signset_create.argtypes = [ctypes.c_size_t] + [P] * 3
    h.he_ed_signset_sign.argtypes = [P, P, ctypes.c_size_t] + [P] * 4
    h.he_ks_sign_screened.argtypes = [P, P, ctypes.c_size_t, ctypes.c_size_t, P, ctypes.c_uint64] + [P] * 4
    return h


def verdict_model(idx, m, bad_item, mut=None):
    """BAD_KEY_INDEX for idx >= m, else BAD_ITEM when the host form refuses the item's other argument, else 0."""
    bad_idx = idx > m if mut == "idx_le" else idx >= m
    if mut == "item_first" and bad_item:
        return ST_BAD_ITEM
    return ST_BAD_KEY_INDEX if bad_idx else ST_BAD_ITEM if bad_item else 0


def scalar_bad(k, mut=None):
    return k > N25519 if mut == "n_le" else k >= N25519


def aligned_bytes(nbytes, shift):
    """nbytes of 0xA5 starting `shift` bytes past a 16-byte boundary."""
    raw = np.full(nbytes + 32, 0xA5, np.uint8)
    at = (-raw.ctypes.data) % 16 + shift
    return raw[at:at + nbytes]


def scalar_screen(he, key_idx, ks, big_endian, shift=0):
    """The screen over the cases, with the scalars `shift` bytes past a 16-byte boundary (the body moves words only when
    both the scalars and their copies are 16-byte aligned)."""
    n = len(key_idx)
    idx = np.ascontiguousarray(key_idx, np.uint32)
    k = aligned_bytes(32 * n, shift)
    k[:] = np.frombuffer(b"".join(v.to_bytes(32, "big" if big_endian else "little") for v in ks), np.uint8)
    idx_out, k_out, vd = np.full(n, 0xA5A5A5A5, np.uint32), aligned_bytes(32 * n, 0), np.full(n, 0xA5, np.uint8)
    he.he_ks_index_scalar_screen(n, idx.ctypes.data, M, k.ctypes.data, int(big_endian), idx_out.ctypes.data, k_out.ctypes.data,
                                 vd.ctypes.data)
    return list(idx_out), k_out.reshape(n, 32), list(vd), k.reshape(n, 32)


@pytest.mark.parametrize("shift", [0, 1, 4])
@pytest.mark.parametrize("big_endian", [False, True])
def test_index_scalar_screen(he, big_endian, shift):
    """Every index beside every boundary scalar: verdict, screened index and scalar copy; the mutants (n accepted,
    index m accepted, BAD_ITEM before BAD_KEY_INDEX, the other byte order) each disagree somewhere."""
    cases = [(i, k) for i in INDICES for k in SCALARS]
    key_idx, ks = [c[0] for c in cases], [c[1] for c in cases]
    idx_out, k_out, vd, k_in = scalar_screen(he, key_idx, ks, big_endian, shift)
    want = [verdict_model(i, M, scalar_bad(k)) for i, k in cases]
    assert vd == want
    for j, (i, k) in enumerate(cases):
        assert idx_out[j] == (0 if want[j] else i)
        assert (k_out[j] == (0 if want[j] else k_in[j])).all()
    assert ST_BAD_KEY_INDEX in want and ST_BAD_ITEM in want and 0 in want
    for mut in ("n_le", "idx_le", "item_first"):
        assert vd != [verdict_model(i, M, scalar_bad(k, mut), mut) for i, k in cases], mut
    swapped = [int.from_bytes(k.to_bytes(32, "big")[::-1], "big") for k in ks]
    assert vd != [verdict_model(i, M, scalar_bad(k)) for i, k in zip(key_idx, swapped)]


def test_range_screen(he):
    """Equal, increasing, decreasing offsets and ranges that end at msgs_len or one past it, beside every index."""
    L = 40
    ranges = [(0, 0), (3, 3), (0, L), (L, L), (10, 9), (L, L + 1), (L - 1, L + 1), (L + 1, L + 1), (5, 20)]
    key_idx, off_pairs = [], []
    for i in INDICES:
        for r in ranges:
            key_idx.append(i)
            off_pairs.append(r)
    # offsets are n + 1 consecutive values: lay each item out as its own [a, b) by interleaving a spacer item
    items_idx, off = [], [off_pairs[0][0]]
    for j, (a, b) in enumerate(off_pairs):
        if off[-1] != a:
            items_idx.append(0)
            off.append(a)
        items_idx.append(key_idx[j])
        off.append(b)
    n = len(items_idx)
    idx = np.array(items_idx, np.uint32)
    offs = np.array(off, np.uint64)
    idx_out, vd = np.full(n, 0xA5A5A5A5, np.uint32), np.full(n, 0xA5, np.uint8)
    he.he_ks_index_range_screen(n, idx.ctypes.data, M, offs.ctypes.data, L, idx_out.ctypes.data, vd.ctypes.data)

    def model(mut=None):
        out = []
        for i in range(n):
            a, b = off[i], off[i + 1]
            bad = b > L if mut == "no_decrease" else b < a or (b >= L if mut == "end_ge" else b > L)
            out.append(verdict_model(items_idx[i], M, bad, mut))
        return out

    want = model()
    assert list(vd) == want
    assert list(idx_out) == [0 if want[i] else items_idx[i] for i in range(n)]
    assert ST_BAD_KEY_INDEX in want and ST_BAD_ITEM in want and 0 in want
    for mut in ("end_ge", "no_decrease", "idx_le", "item_first"):
        assert list(vd) != model(mut), mut


@pytest.mark.parametrize("ol", [1, 32, 64, 132])
def test_merge_out_zeroes_rows(he, ol):
    """A non-zero verdict replaces the status and zeroes exactly the item's ol-byte row; a zero verdict touches nothing."""
    rnd = random.Random(ol)
    n = 50
    vd = np.array([rnd.choice([0, 0, ST_BAD_KEY_INDEX, ST_BAD_ITEM]) for _ in range(n)], np.uint8)
    st = np.array([rnd.randrange(12) for _ in range(n)], np.uint8)
    out = np.frombuffer(rnd.randbytes(n * ol + 16), np.uint8).copy()
    st0, out0 = st.copy(), out.copy()
    he.he_ks_verdict_merge_out(n, vd.ctypes.data, st.ctypes.data, out.ctypes.data, ol)
    for i in range(n):
        assert st[i] == (vd[i] or st0[i])
        row = out[ol * i: ol * (i + 1)]
        assert (row == 0).all() if vd[i] else (row == out0[ol * i: ol * (i + 1)]).all()
    assert (out[n * ol:] == out0[n * ol:]).all()


def test_hash_screened(he):
    """h = SHA512(R || A || M) mod n (little-endian) for a zero verdict, 0 for the others."""
    rnd = random.Random(7)
    n = 12
    R, A = rnd.randbytes(32 * n), rnd.randbytes(32 * n)
    msgs = [rnd.randbytes(rnd.choice([0, 1, 111, 112, 200])) for _ in range(n)]
    off = [0]
    for mm in msgs:
        off.append(off[-1] + len(mm))
    blob = np.frombuffer(b"".join(msgs) + b"\0", np.uint8).copy()
    vd = np.array([0, ST_BAD_ITEM, 0, ST_BAD_KEY_INDEX] * 3, np.uint8)
    h = np.full(32 * n, 0xA5, np.uint8)
    Rb, Ab = np.frombuffer(R, np.uint8).copy(), np.frombuffer(A, np.uint8).copy()
    he.he_ks_ed_hash_screened(n, vd.ctypes.data, Rb.ctypes.data, Ab.ctypes.data, blob.ctypes.data,
                              np.array(off, np.uint64).ctypes.data, h.ctypes.data)
    for i in range(n):
        got = int.from_bytes(h[32 * i: 32 * i + 32].tobytes(), "little")
        d = hashlib.sha512(R[32 * i: 32 * i + 32] + A[32 * i: 32 * i + 32] + msgs[i]).digest()
        assert got == (0 if vd[i] else int.from_bytes(d, "little") % N25519), i


def test_sign_screened_batch(he):
    """Screened items scattered through the normalisation batches (one of them in the first) leave every other item's
    signature exactly the unscreened body's (the items whose ranges the bad offsets widened included, against a
    one-item batch of their own); a screened item gets its verdict and a zeroed signature."""
    rnd = random.Random(3)
    m, n = 3, 40
    secrets = np.frombuffer(rnd.randbytes(32 * m), np.uint8).copy()
    keys, pub = np.zeros(16 * m, np.uint32), np.zeros(32 * m, np.uint8)
    he.he_ed_signset_create(m, secrets.ctypes.data, keys.ctypes.data, pub.ctypes.data)
    msgs = [rnd.randbytes(rnd.choice([0, 5, 64, 130])) for _ in range(n)]
    msgs[0] = rnd.randbytes(7)                                  # item 2 starts past 0, so its range can decrease
    off = [0]
    for mm in msgs:
        off.append(off[-1] + len(mm))
    msgs_len = off[-1]
    key_idx = [rnd.randrange(m) for _ in range(n)]
    bad_idx = {1: m, 17: (1 << 32) - 1}
    idx_bad = list(key_idx)
    for i, v in bad_idx.items():
        idx_bad[i] = v
    off_bad = list(off)
    assert off[2] > 0
    off_bad[2 + 1] = off_bad[2] - 1                          # item 2 decreases; item 3 starts one byte earlier
    off_bad[33 + 1] = msgs_len + 1                           # past the end; msgs_len + 1 stays in the buffer below
    blob = np.frombuffer(b"".join(msgs) + b"\0" * 8, np.uint8).copy()

    def run(idx, offs, length):
        sig, st = np.full(64 * n, 0xA5, np.uint8), np.full(n, 0xA5, np.uint8)
        he.he_ks_sign_screened(keys.ctypes.data, pub.ctypes.data, m, n, blob.ctypes.data, length,
                               np.array(offs, np.uint64).ctypes.data, np.array(idx, np.uint32).ctypes.data,
                               sig.ctypes.data, st.ctypes.data)
        return sig.reshape(n, 64), st

    ref = np.zeros(64 * n, np.uint8)
    he.he_ed_signset_sign(keys.ctypes.data, pub.ctypes.data, n, blob.ctypes.data, np.array(off, np.uint64).ctypes.data,
                          np.array(key_idx, np.uint32).ctypes.data, ref.ctypes.data)
    ref = ref.reshape(n, 64)
    sig, st = run(key_idx, off, msgs_len)
    assert (sig == ref).all() and (st == ST_TRUE).all()
    sig, st = run(idx_bad, off_bad, msgs_len)
    screened = {}
    for i in range(n):
        a, b = off_bad[i], off_bad[i + 1]
        screened[i] = ST_BAD_KEY_INDEX if idx_bad[i] >= m else ST_BAD_ITEM if (b < a or b > msgs_len) else 0
    assert screened[1] == screened[17] == ST_BAD_KEY_INDEX
    assert screened[2] == screened[33] == screened[34] == ST_BAD_ITEM and screened[3] == 0

    def one(k, a, b):
        """The item signed alone: key k over blob[a:b]."""
        out = np.zeros(64, np.uint8)
        he.he_ed_signset_sign(keys.ctypes.data, pub.ctypes.data, 1, blob.ctypes.data, np.array([a, b], np.uint64).ctypes.data,
                              np.array([k], np.uint32).ctypes.data, out.ctypes.data)
        return out

    for i in range(n):
        if screened[i]:
            assert st[i] == screened[i] and not sig[i].any(), i
        else:
            assert st[i] == ST_TRUE and (sig[i] == one(idx_bad[i], off_bad[i], off_bad[i + 1])).all(), i
            if off_bad[i] == off[i] and off_bad[i + 1] == off[i + 1]:
                assert (sig[i] == ref[i]).all(), i


EXPORTS_DEV = {
    "eb200_scalar_mul_batch_keyed_dev": 6, "eb200_mul_add_batch_keyed_dev": 7, "eb200_ecdh_derive_batch_keyed_dev": 6,
    "eb200_ecdsa_recovery_param_batch_keyed_dev": 8, "eb200_eddsa_verify_batch_keyed_dev": 7,
    "eb200_x25519_derive_batch_keyed_dev": 6,
}


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
            for name, nptr in EXPORTS_DEV.items():
                assert getattr(lib, name)(None, n, *[ptr] * nptr) == _native.ERR_ARG, name
            assert lib.eb200_eddsa_verify_batch_keyed_msgs_dev(None, n, ptr, ptr, ptr, 0, ptr, ptr, ptr, ptr, None) == \
                _native.ERR_ARG
            assert lib.eb200_eddsa_sign_batch_keyed_dev(None, n, ptr, 0, ptr, ptr, ptr, ptr, ptr, None) == _native.ERR_ARG
        assert lib.eb200_keyset_dev_workspace_bytes(None, n) == 0
    assert (_native.ST_BAD_KEY_INDEX, _native.ST_BAD_ITEM) == (12, 13)
