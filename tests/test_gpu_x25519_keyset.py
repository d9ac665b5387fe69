"""curve25519 key sets on the GPU: eb200_x25519_derive_batch_keyed must write exactly the bytes and statuses
eb200_x25519_derive_batch writes for the same private keys with the peer keys gathered, at every width, on the benchmark's
items and on small-order, mixed-order, non-canonical, twist and random keys against the oracle; plus the handle's
contract and the Python X25519KeySet."""
import ctypes
import threading

import numpy as np
import pytest

import benchdata
import torsion_cases as tc
from test_x25519_keyset import cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


def p(a):
    return np.ascontiguousarray(a).ctypes.data


def create(lib, pubx, bits=0):
    from elliptic_b200 import _native as nat
    pubx = np.ascontiguousarray(pubx, np.uint8)
    kst, h = np.zeros(len(pubx), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_x25519_keyset_create(len(pubx), pubx.ctypes.data, bits, kst.ctypes.data, ctypes.byref(h)))
    return h, kst


def keyed(lib, h, priv, idx):
    from elliptic_b200 import _native as nat
    n = len(idx)
    out, st = np.full((n, 32), 0xEE, np.uint8), np.full(n, 0xEE, np.uint8)
    nat.call(lib.eb200_x25519_derive_batch_keyed, h, n, np.ascontiguousarray(priv), np.ascontiguousarray(idx, np.uint32), out, st)
    return out, st


def unkeyed(lib, priv, pubx):
    from elliptic_b200 import _native as nat
    n = len(priv)
    out, st = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
    nat.call(lib.eb200_x25519_derive_batch, n, np.ascontiguousarray(priv), np.ascontiguousarray(pubx), out, st)
    return out, st


def dataset(n, m):
    """benchdata's items over m peer keys (one in 256 on the twist), the set's keys (the distinct pubx rows) and indices."""
    ds = benchdata.gen_x25519_derive(n, n_pubs=m, cache_dir=benchdata.cache_dir())
    keys, idx = np.unique(ds["pubx"].view("V32").reshape(-1), return_inverse=True)
    keys = np.ascontiguousarray(keys.view(np.uint8).reshape(-1, 32))
    idx = idx.reshape(-1).astype(np.uint32)
    assert (keys[idx] == ds["pubx"]).all()
    return ds, keys, idx


def test_keyed_equals_unkeyed_on_benchmark_items(lib):
    from elliptic_b200 import _native as nat
    n, m = 1 << 20, 4096
    ds, keys, idx = dataset(n, m)
    want_out, want_st = unkeyed(lib, ds["priv"], ds["pubx"])
    assert (want_st == ds["expected"]).all()
    for bits in (4, 5, 6, 7, 8, 0):
        h, kst = create(lib, keys, bits)
        w = ctypes.c_uint32()
        nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), None))
        out, st = keyed(lib, h, ds["priv"], idx)
        nat.check(lib.eb200_keyset_destroy(h))
        # the items use 4080 of the generator's peer keys (the other 16 slots hold twist points) and the 16 twist x
        assert w.value == (bits or 7) and len(keys) == m and (kst == 5).sum() == 16 and (kst == 1).sum() == m - 16
        assert (st == want_st).all(), (bits, np.nonzero(st != want_st)[0][:8])
        assert (out == want_out).all(), (bits, np.nonzero((out != want_out).any(1))[0][:8])


@pytest.mark.parametrize("bits", [4, 6, 8])
def test_adversarial_keys_against_oracle(lib, bits):
    from elliptic_b200 import _native as nat
    c = cases()
    us, items, want = c["us"], c["items"], c["want"]
    pubx = np.frombuffer(tc.be(us), np.uint8).reshape(-1, 32)
    priv = np.frombuffer(tc.be([k for _, k in items]), np.uint8).reshape(-1, 32)
    idx = np.array([j for j, _ in items], np.uint32)
    h, kst = create(lib, pubx, bits)
    try:
        out, st = keyed(lib, h, priv, idx)
    finally:
        nat.check(lib.eb200_keyset_destroy(h))
    got = [(int(st[i]), int.from_bytes(bytes(out[i]), "big")) for i in range(len(items))]
    assert got == want, [i for i in range(len(items)) if got[i] != want[i]][:8]
    uo, us_ = unkeyed(lib, priv, pubx[idx])
    assert (uo == out).all() and (us_ == st).all()


def test_handle_contract(lib):
    from elliptic_b200 import _native as nat
    n, m = 4096, 16
    ds, keys, idx = dataset(n, m)
    mk = len(keys)
    h, _ = create(lib, keys, 5)
    cv, mm, w, db = ctypes.c_int(), ctypes.c_size_t(), ctypes.c_uint32(), ctypes.c_size_t()
    nat.check(lib.eb200_keyset_info(h, ctypes.byref(cv), ctypes.byref(mm), ctypes.byref(w), ctypes.byref(db)))
    assert (cv.value, mm.value, w.value, db.value) == (nat.CURVE_CURVE25519, mk, 5, mk * (33 + 78336))
    out, st = keyed(lib, h, ds["priv"], idx)
    assert nat.last_timing()["launches"] == 2 and nat.last_timing()["main_kernel_ms"] > 0
    assert (st == ds["expected"]).all()
    assert lib.eb200_x25519_derive_batch_keyed(h, 0, None, None, None, None) == nat.OK
    # key_idx >= m, priv >= n and NULL pointers: ERR_ARG, outputs untouched
    o, s = np.full((n, 32), 0xEE, np.uint8), np.full(n, 0xEE, np.uint8)
    bad = idx.copy(); bad[n - 1] = mk
    assert lib.eb200_x25519_derive_batch_keyed(h, n, p(ds["priv"]), p(bad), p(o), p(s)) == nat.ERR_ARG
    for v in (tc.N, 2**256 - 1):
        pn = ds["priv"].copy(); pn[n // 2] = np.frombuffer(v.to_bytes(32, "big"), np.uint8)
        assert lib.eb200_x25519_derive_batch_keyed(h, n, p(pn), p(idx), p(o), p(s)) == nat.ERR_ARG
    assert lib.eb200_x25519_derive_batch_keyed(h, n, p(ds["priv"]), p(idx), None, p(s)) == nat.ERR_ARG
    assert (o == 0xEE).all() and (s == 0xEE).all()
    # other kinds of set on the new call, and the new set on every other keyed call
    xy = np.frombuffer(b"".join(v.to_bytes(32, "big") for v in (0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798,
                                                                   0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8)), np.uint8).reshape(1, 64)
    ek, ed, es, one = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p(), np.zeros(1, np.uint8)
    nat.check(lib.eb200_keyset_create(nat.CURVE_SECP256K1, 1, p(xy), 0, 4, p(one), ctypes.byref(ek)))
    A = np.frombuffer(bytes.fromhex("d75a980182b10ab7d54bfed3c964073a0ee172f3daa62325af021a68f707511a"), np.uint8).copy()
    nat.check(lib.eb200_eddsa_keyset_create(1, p(A), 4, p(one), ctypes.byref(ed)))
    nat.check(lib.eb200_eddsa_signing_set_create(1, p(np.zeros(32, np.uint8)), None, ctypes.byref(es)))
    z, zi, off = np.zeros((4, 32), np.uint8), np.zeros(4, np.uint32), np.zeros(5, np.uint64)
    zo, zs = np.zeros((4, 64), np.uint8), np.zeros(4, np.uint8)
    for other in (ek, ed, es):
        assert lib.eb200_x25519_derive_batch_keyed(other, 4, p(z), p(zi), p(zo), p(zs)) == nat.ERR_ARG
    assert lib.eb200_ecdsa_verify_batch_keyed(h, 4, p(z), p(z), p(z), p(zi), p(zs)) == nat.ERR_ARG
    assert lib.eb200_scalar_mul_batch_keyed(h, 4, p(z), p(zi), p(zo), p(zs)) == nat.ERR_ARG
    assert lib.eb200_mul_add_batch_keyed(h, 4, p(z), p(z), p(zi), p(zo), p(zs)) == nat.ERR_ARG
    assert lib.eb200_ecdh_derive_batch_keyed(h, 4, p(z), p(zi), p(zo), p(zs)) == nat.ERR_ARG
    assert lib.eb200_ecdsa_recovery_param_batch_keyed(h, 4, p(z), p(z), p(z), p(zi), p(zs), p(zs)) == nat.ERR_ARG
    assert lib.eb200_eddsa_verify_batch_keyed(h, 4, p(z), p(z), p(z), p(zi), p(zs)) == nat.ERR_ARG
    assert lib.eb200_eddsa_verify_batch_keyed_msgs(h, 4, p(z), p(z), None, p(off), p(zi), p(zs)) == nat.ERR_ARG
    assert lib.eb200_eddsa_sign_batch_keyed(h, 4, None, p(off), p(zi), p(zo), p(zs)) == nat.ERR_ARG
    for other in (ek, ed, es):
        nat.check(lib.eb200_keyset_destroy(other))
    # four threads on one set
    outs, errs = [None] * 4, []

    def run(t):
        try:
            outs[t] = keyed(lib, h, ds["priv"], idx)
        except Exception as ex:                     # noqa: BLE001 -- reported below
            errs.append(ex)
    th = [threading.Thread(target=run, args=(t,)) for t in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs and all((o_ == out).all() and (s_ == st).all() for o_, s_ in outs)
    nat.check(lib.eb200_keyset_destroy(h))


def test_x25519_key_set_equals_derive_batch(lib):
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC, EllipticError, X25519KeySet
    n, m = 1024, 8
    ds, keys, idx = dataset(n, m)
    ec = EC("curve25519")
    privs = [int.from_bytes(bytes(k), "big") for k in ds["priv"]]
    privs[3] += 5 * ec.n                                         # reduced mod n at import, as EC.derive_batch does
    pubs = [bytes(k) for k in keys]
    pubs[0] = int.from_bytes(pubs[0], "big") + 2**256 * 3          # wider than 256 bits: reduced mod p
    pubs[1] = pubs[1].hex()
    want, wst = ec.derive_batch(privs, [pubs[j] for j in idx])
    with ec.key_set(pubs, table_bits=6) as ks:
        assert isinstance(ks, X25519KeySet) and ks.table_bits == 6 and ks.device_bytes == len(keys) * (33 + 132096)
        assert (ks.status == 1).sum() == m and (ks.status == 5).sum() == len(keys) - m
        got, st = ks.derive_batch(privs, idx)
        assert got == want and (st == wst).all() and (st == ds["expected"]).all()
        o, s = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
        ro, rs = ks.derive_batch_packed(ds["priv"], idx, out=o, status=s)
        assert ro is o and rs is s
        wo, ws_ = ec.derive_batch_packed(ds["priv"], ds["pubx"])
        assert (o == wo).all() and (s == ws_).all()
        with pytest.raises(nat.NativeError):
            ks.derive_batch_packed(np.full((n, 32), 0xFF, np.uint8), idx)    # priv >= n: the library's ERR_ARG
    with pytest.raises(EllipticError):
        ks.derive_batch_packed(ds["priv"], idx)                      # closed


def test_two_devices(lib):
    from elliptic_b200 import _native as nat
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    nat.init_devices([0, 1])
    n, m = 1 << 16, 64
    ds, keys, idx = dataset(n, m)
    h, _ = create(lib, keys)
    out, st = keyed(lib, h, ds["priv"], idx)
    nat.check(lib.eb200_keyset_destroy(h))
    wo, ws_ = unkeyed(lib, ds["priv"], ds["pubx"])
    assert (out == wo).all() and (st == ws_).all() and (st == ds["expected"]).all()


def test_shutdown_leaves_not_init(lib):
    from elliptic_b200 import _native as nat
    ds, keys, idx = dataset(256, 4)
    h, _ = create(lib, keys)
    nat.shutdown()
    o, s = np.zeros((256, 32), np.uint8), np.zeros(256, np.uint8)
    assert lib.eb200_x25519_derive_batch_keyed(h, 256, p(ds["priv"]), p(idx), p(o), p(s)) == nat.ERR_NOT_INIT
    assert lib.eb200_keyset_destroy(h) == nat.OK
    nat.init(0)
