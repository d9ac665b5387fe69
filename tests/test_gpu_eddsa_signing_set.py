"""EdDSA signing sets on the GPU: eb200_eddsa_sign_batch_keyed must write exactly the signatures eb200_eddsa_sign_batch
writes for the same messages with each item's key secret, for the reference's sign.input vectors and at the benchmark
shape over several chunks; plus the handle's contract and the Python EdSigningSet."""
import ctypes
import gzip
import json
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

p = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


def create(lib, secrets):
    from elliptic_b200 import _native as nat
    secrets = np.ascontiguousarray(secrets, np.uint8)
    pub, h = np.zeros((len(secrets), 32), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_signing_set_create(len(secrets), secrets.ctypes.data, pub.ctypes.data, ctypes.byref(h)))
    return h, pub


def keyed(lib, h, msgs, off, idx):
    from elliptic_b200 import _native as nat
    n = len(idx)
    sig, st = np.full((n, 64), 0xEE, np.uint8), np.zeros(n, np.uint8)
    nat.call(lib.eb200_eddsa_sign_batch_keyed, h, n, msgs if msgs.size else None, off, np.ascontiguousarray(idx, np.uint32),
             sig, st)
    assert (st == nat.ST_TRUE).all()
    return sig


def unkeyed(lib, secrets, msgs, off):
    from elliptic_b200 import _native as nat
    n = len(secrets)
    sig, pub, st = np.zeros((n, 64), np.uint8), np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    nat.call(lib.eb200_eddsa_sign_batch, n, np.ascontiguousarray(secrets), msgs if msgs.size else None, off, sig, pub, st)
    return sig, pub


def items(n, m, seed, max_len=200):
    """m random secrets, n messages of random lengths 0..max_len, random key indices."""
    rng = np.random.default_rng(seed)
    sec = rng.integers(0, 256, (m, 32), dtype=np.uint8)
    lens = rng.integers(0, max_len + 1, n)
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    msgs = rng.integers(0, 256, int(off[n]), dtype=np.uint8)
    idx = rng.integers(0, m, n).astype(np.uint32)
    return sec, msgs, off, idx


def test_sign_input_vectors(lib):
    from elliptic_b200 import _native as nat
    vecs = json.load(gzip.open(os.path.join(os.path.dirname(__file__), "golden", "ed25519_sign_input.json.gz"), "rt"))["vectors"]
    assert len(vecs) == 1024
    sec = np.frombuffer(b"".join(bytes.fromhex(v["secret"]) for v in vecs), np.uint8).reshape(-1, 32)
    ms = [bytes.fromhex(v["msg"]) for v in vecs]
    off = np.zeros(1025, np.uint64)
    off[1:] = np.cumsum([len(x) for x in ms])
    msgs = np.frombuffer(b"".join(ms), np.uint8)
    h, pub = create(lib, sec[::-1])                                     # key k holds vector 1023 - k
    try:
        assert [pub[1023 - i].tobytes().hex() for i in range(1024)] == [v["pk"] for v in vecs]
        sig = keyed(lib, h, msgs, off, 1023 - np.arange(1024))
        assert [sig[i].tobytes().hex() for i in range(1024)] == [v["sig"] for v in vecs]
        assert (sig == unkeyed(lib, sec, msgs, off)[0]).all()
    finally:
        nat.check(lib.eb200_keyset_destroy(h))


def test_benchmark_shape_mixed_lengths(lib):
    """2^20 items over 4096 keys, messages of 0..200 bytes, over several chunks: the unkeyed call's bytes, every
    signature verifies on the GPU, and libsodium agrees on a sample."""
    import nacl.signing
    from elliptic_b200 import _native as nat
    n, m = 1 << 20, 4096
    sec, msgs, off, idx = items(n, m, 1)
    h, pub = create(lib, sec)
    try:
        sig = keyed(lib, h, msgs, off, idx)
        t = nat.last_timing()
        assert t["launches"] % 3 == 0 and t["launches"] >= 12 and t["main_kernel_ms"] > 0
        want, upub = unkeyed(lib, sec[idx], msgs, off)
        bad = np.nonzero((sig != want).any(axis=1))[0]
        assert not len(bad), bad[:8]
        assert (upub == pub[idx]).all()
        st = np.zeros(n, np.uint8)
        nat.call(lib.eb200_eddsa_verify_batch_msgs, n, np.ascontiguousarray(sig[:, :32]), np.ascontiguousarray(sig[:, 32:]),
                 np.ascontiguousarray(pub[idx]), msgs, off, st)
        assert (st == nat.ST_TRUE).all()
        for i in range(0, n, n // 64):
            k = nacl.signing.SigningKey(sec[idx[i]].tobytes())
            assert k.verify_key.encode() == pub[idx[i]].tobytes()
            assert k.sign(msgs[int(off[i]):int(off[i + 1])].tobytes()).signature == sig[i].tobytes()
    finally:
        nat.check(lib.eb200_keyset_destroy(h))


@pytest.mark.parametrize("n", [1, 127, 129, (1 << 18) + 777])
def test_sizes(lib, n):
    from elliptic_b200 import _native as nat
    sec, msgs, off, idx = items(n, 37, n, max_len=90)
    h, _ = create(lib, sec)
    try:
        assert (keyed(lib, h, msgs, off, idx) == unkeyed(lib, sec[idx], msgs, off)[0]).all()
    finally:
        nat.check(lib.eb200_keyset_destroy(h))


def test_handle_contract(lib):
    from elliptic_b200 import _native as nat
    n, m = 256, 16
    sec, msgs, off, idx = items(n, m, 3)
    want = unkeyed(lib, sec[idx], msgs, off)[0]
    assert lib.eb200_keyset_destroy(None) == nat.OK
    h, pub = create(lib, sec)
    cv, mm, w, db = ctypes.c_int(7), ctypes.c_size_t(), ctypes.c_uint32(7), ctypes.c_size_t()
    nat.check(lib.eb200_keyset_info(h, ctypes.byref(cv), ctypes.byref(mm), ctypes.byref(w), ctypes.byref(db)))
    assert (cv.value, mm.value, w.value, db.value) == (nat.CURVE_ED25519, m, 0, 96 * m)
    # without out_pub; the same keys give the same set
    h2 = ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_signing_set_create(m, p(sec), None, ctypes.byref(h2)))
    assert (keyed(lib, h2, msgs, off, idx) == want).all()
    nat.check(lib.eb200_keyset_destroy(h2))
    # three launches per chunk; main_kernel_ms is the nonce kernel
    assert (keyed(lib, h, msgs, off, idx) == want).all()
    t = nat.last_timing()
    assert t["launches"] == 3 and 0 < t["main_kernel_ms"] <= t["kernel_ms"]
    # empty messages with msgs = NULL; n = 0
    z_off = np.zeros(5, np.uint64)
    assert (keyed(lib, h, np.zeros(0, np.uint8), z_off, [0, 1, 2, 3]) ==
            unkeyed(lib, sec[:4], np.zeros(0, np.uint8), z_off)[0]).all()
    assert lib.eb200_eddsa_sign_batch_keyed(h, 0, None, None, None, None, None) == nat.OK
    # key_idx >= m, decreasing offsets, NULL pointers: ERR_ARG with the outputs untouched
    sig, st = np.full((n, 64), 0xEE, np.uint8), np.full(n, 0xEE, np.uint8)
    bad = idx.copy(); bad[n - 1] = m
    assert lib.eb200_eddsa_sign_batch_keyed(h, n, p(msgs), p(off), p(bad), p(sig), p(st)) == nat.ERR_ARG
    boff = off.copy(); boff[5] = boff[6] + 1
    assert lib.eb200_eddsa_sign_batch_keyed(h, n, p(msgs), p(boff), p(idx), p(sig), p(st)) == nat.ERR_ARG
    assert lib.eb200_eddsa_sign_batch_keyed(h, n, None, p(off), p(idx), p(sig), p(st)) == nat.ERR_ARG
    assert lib.eb200_eddsa_sign_batch_keyed(h, n, p(msgs), p(off), p(idx), None, p(st)) == nat.ERR_ARG
    assert lib.eb200_eddsa_sign_batch_keyed(h, n, p(msgs), p(off), p(idx), p(sig), None) == nat.ERR_ARG
    assert (sig == 0xEE).all() and (st == 0xEE).all()
    # kind mismatches in both directions
    xy = np.frombuffer(b"".join(v.to_bytes(32, "big") for v in (0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798,
                                                                   0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8)), np.uint8).reshape(1, 64)
    ek, ekst = ctypes.c_void_p(), np.zeros(1, np.uint8)
    nat.check(lib.eb200_keyset_create(nat.CURVE_SECP256K1, 1, p(xy), 0, 4, p(ekst), ctypes.byref(ek)))
    vk, vkst = ctypes.c_void_p(), np.zeros(m, np.uint8)
    nat.check(lib.eb200_eddsa_keyset_create(m, p(pub), 4, p(vkst), ctypes.byref(vk)))
    z, zi, zs = np.zeros((4, 32), np.uint8), np.zeros(4, np.uint32), np.full(4, 0xEE, np.uint8)
    z64 = np.zeros((4, 64), np.uint8)
    for other in (ek, vk):
        assert lib.eb200_eddsa_sign_batch_keyed(other, 4, p(msgs), p(off), p(zi), p(z64), p(zs)) == nat.ERR_ARG
    assert lib.eb200_eddsa_verify_batch_keyed(h, 4, p(z), p(z), p(z), p(zi), p(zs)) == nat.ERR_ARG
    assert lib.eb200_eddsa_verify_batch_keyed_msgs(h, 4, p(z), p(z), p(msgs), p(off), p(zi), p(zs)) == nat.ERR_ARG
    assert lib.eb200_ecdsa_verify_batch_keyed(h, 4, p(z), p(z), p(z), p(zi), p(zs)) == nat.ERR_ARG
    assert lib.eb200_scalar_mul_batch_keyed(h, 4, p(z), p(zi), p(z64), p(zs)) == nat.ERR_ARG
    assert lib.eb200_mul_add_batch_keyed(h, 4, p(z), p(z), p(zi), p(z64), p(zs)) == nat.ERR_ARG
    assert lib.eb200_ecdh_derive_batch_keyed(h, 4, p(z), p(zi), p(z), p(zs)) == nat.ERR_ARG
    assert (zs == 0xEE).all()
    # the EdDSA verify set built from the signing set's public keys verifies its signatures
    sig = keyed(lib, h, msgs, off, idx)
    vst = np.zeros(n, np.uint8)
    nat.call(lib.eb200_eddsa_verify_batch_keyed_msgs, vk, n, np.ascontiguousarray(sig[:, :32]),
             np.ascontiguousarray(sig[:, 32:]), msgs, off, idx, vst)
    assert (vst == nat.ST_TRUE).all()
    nat.check(lib.eb200_keyset_destroy(ek))
    nat.check(lib.eb200_keyset_destroy(vk))
    # four threads on one set
    outs, errs = [None] * 4, []

    def run(t):
        try:
            outs[t] = keyed(lib, h, msgs, off, idx)
        except Exception as ex:                     # noqa: BLE001 -- reported below
            errs.append(ex)
    th = [threading.Thread(target=run, args=(t,)) for t in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs and all((o == want).all() for o in outs)
    nat.check(lib.eb200_keyset_destroy(h))


def test_ed_signing_set_equals_sign_batch(lib):
    from elliptic_b200.eddsa import EDDSA
    ed = EDDSA()
    sec, msgs, off, idx = items(300, 5, 9, max_len=120)
    secrets = [sec[0].tobytes().hex(), list(sec[1]), sec[2].tobytes(), bytearray(sec[3].tobytes()), sec[4].tobytes().hex()]
    messages = [msgs[int(off[i]):int(off[i + 1])].tobytes() for i in range(300)]
    messages = [x.hex() if i % 3 == 0 else (list(x) if i % 3 == 1 else x) for i, x in enumerate(messages)]
    want = ed.sign_batch(messages, [secrets[k] for k in idx])
    with ed.signing_set(secrets) as ss:
        assert ss.device_bytes == 96 * 5 and ss.public.shape == (5, 32)
        assert (ss.public == ed.public_from_secret_batch(sec)).all()
        assert not any(isinstance(v, np.ndarray) and v.shape == (5, 32) and (v == sec).all() for v in vars(ss).values())
        assert ss.sign_batch(messages, idx) == want
        assert (ss.sign_batch_packed(msgs, off, idx) == np.frombuffer(b"".join(want), np.uint8).reshape(300, 64)).all()


def test_two_devices(lib):
    from elliptic_b200 import _native as nat
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    nat.init_devices([0, 1])
    n, m = 1 << 16, 64
    sec, msgs, off, idx = items(n, m, 4)
    h, _ = create(lib, sec)
    assert (keyed(lib, h, msgs, off, idx) == unkeyed(lib, sec[idx], msgs, off)[0]).all()
    nat.check(lib.eb200_keyset_destroy(h))


def test_shutdown_leaves_not_init(lib):
    from elliptic_b200 import _native as nat
    sec, msgs, off, idx = items(128, 4, 5)
    h, _ = create(lib, sec)
    nat.shutdown()
    sig, st = np.zeros((128, 64), np.uint8), np.zeros(128, np.uint8)
    assert lib.eb200_eddsa_sign_batch_keyed(h, 128, p(msgs), p(off), p(idx), p(sig), p(st)) == nat.ERR_NOT_INIT
    assert lib.eb200_keyset_destroy(h) == nat.OK
    lib = nat.init(0)
    h, _ = create(lib, sec)
    assert (keyed(lib, h, msgs, off, idx) == unkeyed(lib, sec[idx], msgs, off)[0]).all()
    nat.check(lib.eb200_keyset_destroy(h))
