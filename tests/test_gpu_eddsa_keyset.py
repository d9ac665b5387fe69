"""EdDSA key sets on the GPU: eb200_eddsa_verify_batch_keyed[_msgs] must write exactly the status bytes
eb200_eddsa_verify_batch[_msgs] writes for the same items with the keys gathered, at every width, for honest,
throwing, small-order, mixed-order and non-canonical keys; plus the handle's contract and the Python EdKeySet."""
import ctypes
import threading

import numpy as np
import pytest

import benchdata
import ed_ks_items as K

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


def create(lib, A, bits=0):
    from elliptic_b200 import _native as nat
    A = np.ascontiguousarray(A, np.uint8)
    kst, h = np.zeros(len(A), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_keyset_create(len(A), A.ctypes.data, bits, kst.ctypes.data, ctypes.byref(h)))
    return h, kst


def keyed(lib, h, R, S, hh, idx):
    from elliptic_b200 import _native as nat
    st = np.full(len(idx), 0xEE, np.uint8)
    nat.call(lib.eb200_eddsa_verify_batch_keyed, h, len(idx), R, S, hh, np.ascontiguousarray(idx, np.uint32), st)
    return st


def keyed_msgs(lib, h, R, S, msgs, off, idx):
    from elliptic_b200 import _native as nat
    st = np.full(len(idx), 0xEE, np.uint8)
    nat.call(lib.eb200_eddsa_verify_batch_keyed_msgs, h, len(idx), R, S, msgs, off, np.ascontiguousarray(idx, np.uint32), st)
    return st


def unkeyed(lib, R, S, A, hh):
    from elliptic_b200 import _native as nat
    st = np.zeros(len(R), np.uint8)
    nat.call(lib.eb200_eddsa_verify_batch, len(R), R, S, np.ascontiguousarray(A), hh, st)
    return st


def dataset(n, m):
    ds = benchdata.gen_ed25519_verify(n, n_keys=m, cache_dir=benchdata.cache_dir(), with_msgs=True)
    keys, idx = np.ascontiguousarray(ds["A"][:m]), np.arange(n, dtype=np.uint32) % m
    assert (ds["A"] == keys[idx]).all()
    off = np.arange(n + 1, dtype=np.uint64) * 32
    return ds, keys, idx, np.ascontiguousarray(ds["msgs"].reshape(-1)), off


def test_keyed_equals_unkeyed(lib):
    from elliptic_b200 import _native as nat
    n, m = 1 << 16, 64
    ds, keys, idx, msgs, off = dataset(n, m)
    want = unkeyed(lib, ds["R"], ds["S"], ds["A"], ds["h"])
    assert (want == ds["expected"]).all()
    for bits in (4, 7, 8, 0):
        h, kst = create(lib, keys, bits)
        w = ctypes.c_uint32()
        nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), None))
        assert (kst == 1).all() and w.value == (bits or 8)
        got = keyed(lib, h, ds["R"], ds["S"], ds["h"], idx)
        got_m = keyed_msgs(lib, h, ds["R"], ds["S"], msgs, off, idx)
        nat.check(lib.eb200_keyset_destroy(h))
        assert (got == want).all(), (bits, np.nonzero(got != want)[0][:8])
        assert (got_m == want).all(), (bits, np.nonzero(got_m != want)[0][:8])


@pytest.mark.parametrize("bits", [4, 6, 8])
def test_adversarial_keys_against_oracle(lib, bits):
    from oracle.ref_py.eddsa import EDDSA
    ed = EDDSA()
    keys, items = K.cases(ed, vectors=64)
    want = np.array(K.answers(ed, keys, items), np.uint8)
    A, R, S, hh, idx = K.pack(keys, items)
    h, kst = create(lib, A, bits)
    try:
        assert list(kst) == [K.expected(ed, ed.encode_point(ed.g), K.le(1), a, 0) or 1 for a in keys]
        got = keyed(lib, h, R, S, hh, idx)
        assert (got == want).all(), np.nonzero(got != want)[0][:8]
        assert (unkeyed(lib, R, S, A[idx], hh) == want).all()
        sel, blob, off = K.msg_items(items)
        got_m = keyed_msgs(lib, h, np.ascontiguousarray(R[sel]), np.ascontiguousarray(S[sel]), blob, off, idx[sel])
        assert (got_m == want[sel]).all(), np.nonzero(got_m != want[sel])[0][:8]
    finally:
        from elliptic_b200 import _native as nat
        nat.check(lib.eb200_keyset_destroy(h))


def test_benchmark_shape(lib):
    """2^20 items over 4096 keys, the width chosen automatically (W = 7 under 1 GiB), through both calls."""
    from elliptic_b200 import _native as nat
    n, m = 1 << 20, 4096
    ds, keys, idx, msgs, off = dataset(n, m)
    h, kst = create(lib, keys)
    w, db = ctypes.c_uint32(), ctypes.c_size_t()
    nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), ctypes.byref(db)))
    assert w.value == 7 and db.value == m * (32 + 1 + 227328)
    assert (keyed(lib, h, ds["R"], ds["S"], ds["h"], idx) == ds["expected"]).all()
    assert (keyed_msgs(lib, h, ds["R"], ds["S"], msgs, off, idx) == ds["expected"]).all()
    nat.check(lib.eb200_keyset_destroy(h))


def test_handle_contract(lib):
    from elliptic_b200 import _native as nat
    n, m = 256, 16
    ds, keys, idx, msgs, off = dataset(n, m)
    h, _ = create(lib, keys, 5)
    cv, mm, w, db = ctypes.c_int(), ctypes.c_size_t(), ctypes.c_uint32(), ctypes.c_size_t()
    nat.check(lib.eb200_keyset_info(h, ctypes.byref(cv), ctypes.byref(mm), ctypes.byref(w), ctypes.byref(db)))
    assert (cv.value, mm.value, w.value, db.value) == (nat.CURVE_ED25519, m, 5, m * (33 + 78336))
    # launch counts per chunk: 1 from h, 3 from raw messages (gather, hash, main)
    keyed(lib, h, ds["R"], ds["S"], ds["h"], idx)
    assert nat.last_timing()["launches"] == 1 and nat.last_timing()["main_kernel_ms"] > 0
    keyed_msgs(lib, h, ds["R"], ds["S"], msgs, off, idx)
    assert nat.last_timing()["launches"] == 3
    # out-of-range indices and h >= n: ERR_ARG, status untouched
    st = np.full(n, 0xEE, np.uint8)
    bad = idx.copy(); bad[n - 1] = m
    p = lambda a: np.ascontiguousarray(a).ctypes.data
    assert lib.eb200_eddsa_verify_batch_keyed(h, n, p(ds["R"]), p(ds["S"]), p(ds["h"]), p(bad), p(st)) == nat.ERR_ARG
    assert lib.eb200_eddsa_verify_batch_keyed_msgs(h, n, p(ds["R"]), p(ds["S"]), p(msgs), p(off), p(bad), p(st)) == nat.ERR_ARG
    hn = ds["h"].copy(); hn[7] = np.frombuffer(K.le(K.N), np.uint8)
    assert lib.eb200_eddsa_verify_batch_keyed(h, n, p(ds["R"]), p(ds["S"]), p(hn), p(idx), p(st)) == nat.ERR_ARG
    assert (st == 0xEE).all()
    # ECDSA and EdDSA handles swapped; both kinds alive at once
    xy = np.frombuffer(b"".join(v.to_bytes(32, "big") for v in (0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798,
                                                                   0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8)), np.uint8).reshape(1, 64)
    ek, ekst = ctypes.c_void_p(), np.zeros(1, np.uint8)
    nat.check(lib.eb200_keyset_create(nat.CURVE_SECP256K1, 1, p(xy), 0, 4, p(ekst), ctypes.byref(ek)))
    z = np.zeros((4, 32), np.uint8)
    assert lib.eb200_eddsa_verify_batch_keyed(ek, 4, p(z), p(z), p(z), p(np.zeros(4, np.uint32)), p(st)) == nat.ERR_ARG
    assert lib.eb200_ecdsa_verify_batch_keyed(h, 4, p(z), p(z), p(z), p(np.zeros(4, np.uint32)), p(st)) == nat.ERR_ARG
    assert (keyed(lib, h, ds["R"], ds["S"], ds["h"], idx) == ds["expected"]).all()
    nat.check(lib.eb200_keyset_destroy(ek))
    # four threads on one set
    outs, errs = [None] * 4, []

    def run(t):
        try:
            outs[t] = keyed(lib, h, ds["R"], ds["S"], ds["h"], idx)
        except Exception as ex:                     # noqa: BLE001 -- reported below
            errs.append(ex)
    th = [threading.Thread(target=run, args=(t,)) for t in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs and all((o == ds["expected"]).all() for o in outs)
    nat.check(lib.eb200_keyset_destroy(h))


def test_ed_key_set_equals_verify_batch(lib):
    from elliptic_b200.eddsa import EDDSA
    n, m = 512, 8
    ds, keys, idx, msgs, off = dataset(n, m)
    ed = EDDSA()
    messages = [bytes(x) for x in ds["msgs"]]
    sigs = [bytes(ds["R"][i]) + bytes(ds["S"][i]) for i in range(n)]
    want = ed.verify_batch(messages, sigs, [bytes(a) for a in ds["A"]])
    with ed.key_set([bytes(k).hex() for k in keys], table_bits=6) as ks:
        assert ks.table_bits == 6 and (ks.status == 1).all() and ks.device_bytes == m * (33 + 132096)
        assert (ks.verify_batch(messages, sigs, idx) == want).all()
        assert (ks.verify_batch(messages, sigs, idx, gpu_hash=False) == want).all()
        assert (ks.verify_batch_packed(ds["R"], ds["S"], ds["h"], idx) == want).all()
    assert (want == ds["expected"]).all()


def test_two_devices(lib):
    from elliptic_b200 import _native as nat
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    nat.init_devices([0, 1])
    n, m = 1 << 16, 64
    ds, keys, idx, msgs, off = dataset(n, m)
    h, _ = create(lib, keys)
    assert (keyed(lib, h, ds["R"], ds["S"], ds["h"], idx) == ds["expected"]).all()
    assert (keyed_msgs(lib, h, ds["R"], ds["S"], msgs, off, idx) == ds["expected"]).all()
    nat.check(lib.eb200_keyset_destroy(h))


def test_shutdown_leaves_not_init(lib):
    from elliptic_b200 import _native as nat
    ds, keys, idx, msgs, off = dataset(128, 4)
    h, _ = create(lib, keys)
    nat.shutdown()
    st = np.zeros(128, np.uint8)
    p = lambda a: np.ascontiguousarray(a).ctypes.data
    assert lib.eb200_eddsa_verify_batch_keyed(h, 128, p(ds["R"]), p(ds["S"]), p(ds["h"]), p(idx), p(st)) == nat.ERR_NOT_INIT
    assert lib.eb200_keyset_destroy(h) == nat.OK
    nat.init(0)
