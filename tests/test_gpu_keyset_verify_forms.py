"""The DER and device-pointer forms of the keyed ECDSA verify on the GPU: eb200_ecdsa_verify_batch_keyed_der must write
exactly what eb200_ecdsa_verify_batch_der writes with the keys gathered, and eb200_ecdsa_verify_batch_keyed_dev exactly
what eb200_ecdsa_verify_batch_keyed writes, with BAD_KEY_INDEX for an index >= m; on the config-1 fixture in every key
format and on all six presets; plus their argument, lifetime, stream, thread and timing contract and
KeySet.verify_batch_der_packed."""
import ctypes
import gzip
import json
import os
import random
import threading

import numpy as np
import pytest

import ks_der_items as kd
from gpu_keyset_items import gpu_items
from ks_items import CURVES, adversarial_items, adversarial_keys

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
BY_NAME = {nm: (cid, ln) for nm, cid, ln in CURVES}


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


def create(lib, cid, pub, fmt=0, bits=0):
    from elliptic_b200 import _native as nat
    pub = np.ascontiguousarray(pub, np.uint8)
    kst, h = np.zeros(len(pub), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_keyset_create(cid, len(pub), pub.ctypes.data, fmt, bits, kst.ctypes.data, ctypes.byref(h)))
    return h, kst


def keyed_der(lib, h, e, ders, idx):
    from elliptic_b200 import _native as nat
    data, off = kd.blob(ders)
    st = np.full(len(ders), 0xEE, np.uint8)
    nat.call(lib.eb200_ecdsa_verify_batch_keyed_der, h, len(ders), np.ascontiguousarray(e), data, off,
             np.ascontiguousarray(idx, np.uint32), st)
    return st


def unkeyed_der(lib, cid, e, ders, pub, fmt=0):
    from elliptic_b200 import _native as nat
    data, off = kd.blob(ders)
    st = np.full(len(ders), 0xEE, np.uint8)
    nat.call(lib.eb200_ecdsa_verify_batch_der, cid, len(ders), np.ascontiguousarray(e), data, off, np.ascontiguousarray(pub),
             fmt, st)
    return st


def expected_launches(lib, n, per_chunk):
    """launches of a keyed host call of n items on a set held by every initialised device (run_sharded_on, make_plan)."""
    r128 = lambda x: (x + 127) & ~127

    def chunks(m):
        ch = 16 if m >= 1 << 22 else 4 if m >= 1 << 18 else 1
        per, pos, k = r128(-(-m // ch)), 0, 0
        if 1 < ch < 16 and r128(per // 4) < m:
            pos, k = r128(per // 4), 1
            per = r128(-(-(m - pos) // ch))
        while pos < m:
            pos, k = min(pos + per, m), k + 1
        return k
    use = max(1, min(lib.eb200_device_count(), n >> 14))
    per = r128(-(-n // use))
    return sum(per_chunk * chunks(min(per, n - lo)) for lo in range(0, n, per))


def wire_ders(ln, r, s, rnd):
    """The canonical DER of every item, with one item in 7 bit-flipped, one in 11 truncated, one in 13 with a
    long-form length and one in 17 with a padded r."""
    ders = []
    for i in range(len(r)):
        ri, si = int.from_bytes(r[i].tobytes(), "big"), int.from_bytes(s[i].tobytes(), "big")
        if i % 7 == 3 or i % 11 == 5 or i % 13 == 6 or i % 17 == 8:
            v = kd.variants(ri, si, rnd)
            ders.append(v[5] if i % 7 == 3 else v[3] if i % 11 == 5 else v[1] if i % 13 == 6 else v[2])
        else:
            ders.append(kd.canonical(ri, si))
    return ders


# ---- config 1 ---------------------------------------------------------------------------------------------------------

THROW = {"throw:invalid point": 2, "throw:Assertion failed": 5, "throw:Unknown point format": 6,
         "throw:Signature without r or s": 9}


def test_config1_fixture_in_every_key_format(lib):
    """All 1024 fixture items with DER signatures ({r, s} ones encoded with the oracle's to_der) through a KeySet over
    key sets over the fixture's keys as given, one per wire format ({x, y}; uncompressed and hybrid; compressed): equal to
    the oracle on the DER form, to the fixture's expectation wherever the encoding is the fixture's own, and to the
    unkeyed DER call; throwing (hybrid parity), off-curve and no-sqrt keys included."""
    from elliptic_b200 import _native as nat
    from oracle.ref_py.bn import RefError
    from oracle.ref_py.ec import EC as RefEC
    from oracle.ref_py.signature import Signature
    items = json.load(gzip.open(os.path.join(HERE, "golden", "secp256k1_verify_1024.json.gz"), "rt"))["items"]
    ref = RefEC("secp256k1")
    ders = [bytes.fromhex(it["sig"]) if isinstance(it["sig"], str) else bytes(Signature(it["sig"], "hex").to_der())
            for it in items]
    e = np.frombuffer(b"".join(bytes.fromhex(it["msg"]) for it in items), np.uint8).reshape(-1, 32)
    keys, key_idx = [], []
    for it in items:
        k = json.dumps(it["pub"], sort_keys=True)
        if k not in keys:
            keys.append(k)
        key_idx.append(keys.index(k))
    pubs = [json.loads(k) for k in keys]
    want = []
    for it, der in zip(items, ders):
        try:
            want.append(int(bool(ref.verify(it["msg"], der.hex(), it["pub"], "hex"))))
        except RefError as ex:
            want.append(THROW["throw:" + ex.args[0]])
        if isinstance(it["sig"], str):
            x = it["expected"]
            assert want[-1] == (THROW[x] if isinstance(x, str) else int(x)), it["i"]
    # one native set per wire format, with the keys' bytes as given: a key that throws is imported and throws there
    wire = []
    for p in pubs:
        if isinstance(p, dict):
            wire.append((nat.PUB_XY, bytes.fromhex(p["x"].rjust(64, "0")) + bytes.fromhex(p["y"].rjust(64, "0"))))
        else:
            b = bytes.fromhex(p)
            wire.append((nat.PUB_SEC1_65 if len(b) == 65 else nat.PUB_SEC1_33, b))
    got = np.full(len(items), 0xEE, np.uint8)
    for fmt in (nat.PUB_XY, nat.PUB_SEC1_65, nat.PUB_SEC1_33):
        kk = [j for j in range(len(pubs)) if wire[j][0] == fmt]
        sel = np.array([i for i in range(len(items)) if wire[key_idx[i]][0] == fmt])
        pos = {j: t for t, j in enumerate(kk)}
        h, kst = create(lib, 1, np.frombuffer(b"".join(wire[j][1] for j in kk), np.uint8).reshape(len(kk), -1), fmt)
        got[sel] = keyed_der(lib, h, e[sel], [ders[i] for i in sel], [pos[key_idx[i]] for i in sel])
        assert nat.last_timing()["launches"] == 5
        nat.check(lib.eb200_keyset_destroy(h))
        pub = np.frombuffer(b"".join(wire[key_idx[i]][1] for i in sel), np.uint8).reshape(len(sel), -1)
        assert np.array_equal(unkeyed_der(lib, 1, e[sel], [ders[i] for i in sel], pub, fmt), got[sel]), fmt
    assert [int(v) for v in got] == want, [i for i in range(len(want)) if got[i] != want[i]]
    assert {0, 1, 2, 5, 9} <= set(want)


# ---- all six presets --------------------------------------------------------------------------------------------------

_ITEMS = {}


def preset_items(lib, name):
    """Honest GPU-signed traffic large enough for several chunks (and for sharding on two GPUs), the adversarial keys'
    items, and their wire DER."""
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    if name not in _ITEMS:
        cid, ln = BY_NAME[name]
        n = (1 << 19) + 333 if ln <= 32 else (1 << 18) + 333
        xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, 256, n, seed=cid)
        ec = EC(name)
        adv = adversarial_keys(ec, cid, (4, 8))[:6]
        ai = adversarial_items(ec, cid, adv, 8 if cid == 1 else 6)
        col = lambda vals: np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in vals), np.uint8).reshape(-1, ln)
        axy = np.concatenate([col([Q.x for _, Q in adv]), col([Q.y for _, Q in adv])], axis=1)
        off_curve = axy[:1].copy()
        off_curve[0, -1] ^= 1                                            # imported, not validated, off the curve
        xy = np.concatenate([xy, axy, off_curve])
        ae, ar, as_ = col([it[0] for it in ai]), col([it[1] for it in ai]), col([it[2] for it in ai])
        aidx = np.array([256 + it[3] for it in ai] + [len(xy) - 1] * 4, np.uint32)
        e = np.concatenate([e, ae, ae[:4]]); r = np.concatenate([r, ar, ar[:4]]); s = np.concatenate([s, as_, as_[:4]])
        idx = np.concatenate([idx, aidx])
        ders = wire_ders(ln, r, s, random.Random(cid))
        _ITEMS[name] = (cid, ln, xy, e, r, s, idx, ders)
    return _ITEMS[name]


@pytest.mark.parametrize("name", [c[0] for c in CURVES])
def test_keyed_der_equals_unkeyed_der_on_every_preset(lib, name):
    from elliptic_b200 import _native as nat
    cid, ln, xy, e, r, s, idx, ders = preset_items(lib, name)
    want = unkeyed_der(lib, cid, e, ders, xy[idx])
    assert {0, 1, 9} <= set(int(v) for v in np.unique(want))
    for bits in (4, 8, 0):
        h, kst = create(lib, cid, xy, 0, bits)
        assert list(kst[-1:]) == [0] and (kst[:-1] == 1).all()
        got = keyed_der(lib, h, e, ders, idx)
        assert nat.last_timing()["launches"] == expected_launches(lib, len(idx), 5)
        nat.check(lib.eb200_keyset_destroy(h))
        assert (got == want).all(), (name, bits, np.nonzero(got != want)[0][:8])


def test_keyed_der_key_throws_and_sec1_sets(lib):
    """A compressed-key set whose keys include ones that throw (no square root, bad prefix): every item on such a key
    gets the key's throw, whatever its DER, as the unkeyed DER call gives it."""
    from elliptic_b200 import _native as nat
    cid, ln, xy, e, r, s, idx, ders = preset_items(lib, "secp256k1")
    m = 64
    comp = np.zeros((m, 33), np.uint8)
    comp[:, 0] = 2 + (xy[:m, 63] & 1)
    comp[:, 1:] = xy[:m, :32]
    comp[5, 0] = 5                                   # Unknown point format
    p = 2**256 - 2**32 - 977
    x = next(x for x in range(2, 1000) if pow(x**3 + 7, (p - 1) // 2, p) == p - 1)
    comp[9, 1:] = np.frombuffer(x.to_bytes(32, "big"), np.uint8)      # x^3 + 7 has no square root
    n = 1 << 15
    sel = np.nonzero(idx < m)[0][:n]
    h, kst = create(lib, cid, comp, nat.PUB_SEC1_33)
    assert kst[5] == nat.ST_THROW_POINT_FORMAT and kst[9] == nat.ST_THROW_INVALID_POINT
    got = keyed_der(lib, h, e[sel], [ders[i] for i in sel], idx[sel])
    want = unkeyed_der(lib, cid, e[sel], [ders[i] for i in sel], comp[idx[sel]], nat.PUB_SEC1_33)
    nat.check(lib.eb200_keyset_destroy(h))
    assert (got == want).all()
    assert (got[np.isin(idx[sel], [5, 9])] > nat.ST_TRUE).all() and (got == nat.ST_THROW_SIG_FORMAT).any()


def test_keyed_der_argument_errors(lib):
    from elliptic_b200 import _native as nat
    cid, ln, xy, e, r, s, idx, ders = preset_items(lib, "p256")
    h, _ = create(lib, cid, xy)
    data, off = kd.blob(ders[:8])
    st = np.full(8, 0xEE, np.uint8)
    good = (e[:8].copy(), data, off, np.zeros(8, np.uint32), st)
    f = lib.eb200_ecdsa_verify_batch_keyed_der
    args = lambda a: [x.ctypes.data if isinstance(x, np.ndarray) else x for x in a]
    for k in range(5):
        bad = list(good)
        bad[k] = None
        assert f(h, 8, *args(bad)) == nat.ERR_ARG
    dec = off.copy(); dec[3], dec[4] = dec[4], dec[3]
    assert f(h, 8, *args((good[0], data, dec, good[3], st))) == nat.ERR_ARG
    big = np.zeros(8, np.uint32); big[7] = len(xy)
    assert f(h, 8, *args((good[0], data, off, big, st))) == nat.ERR_ARG
    assert (st == 0xEE).all()
    assert f(h, 0, None, None, None, None, None) == nat.OK
    assert f(None, 8, *args(good)) == nat.ERR_ARG
    # EdDSA, signing and curve25519 sets are refused
    A = np.zeros((1, 32), np.uint8); A[0, 0] = 1                     # the identity's encoding: a valid key
    for mk in ("ed", "sign", "x"):
        oh, kst = ctypes.c_void_p(), np.zeros(1, np.uint8)
        if mk == "ed": nat.check(lib.eb200_eddsa_keyset_create(1, A.ctypes.data, 4, kst.ctypes.data, ctypes.byref(oh)))
        elif mk == "sign": nat.check(lib.eb200_eddsa_signing_set_create(1, A.ctypes.data, np.zeros(32, np.uint8).ctypes.data, ctypes.byref(oh)))
        else: nat.check(lib.eb200_x25519_keyset_create(1, (A + 8).ctypes.data, 4, kst.ctypes.data, ctypes.byref(oh)))
        assert f(oh, 8, *args(good)) == nat.ERR_ARG
        assert lib.eb200_ecdsa_verify_batch_keyed_dev(oh, 8, *[1] * 7) == nat.ERR_ARG
        assert lib.eb200_ecdsa_verify_keyed_workspace_bytes(oh, 8) == 0
        nat.check(lib.eb200_keyset_destroy(oh))
    nat.check(lib.eb200_keyset_destroy(h))


# ---- device pointers --------------------------------------------------------------------------------------------------

def dev_call(lib, h, e, r, s, idx, stream=None):
    import torch
    from elliptic_b200 import _native as nat
    n = len(idx)
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (e, r, s)]
    ti = torch.from_numpy(np.ascontiguousarray(idx, np.uint32).view(np.int32)).cuda()
    st = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    ws = torch.empty(lib.eb200_ecdsa_verify_keyed_workspace_bytes(h, n), dtype=torch.uint8, device="cuda")
    stream = stream or torch.cuda.current_stream()
    rc = lib.eb200_ecdsa_verify_batch_keyed_dev(h, n, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), ti.data_ptr(),
                                                st.data_ptr(), ws.data_ptr(), ctypes.c_void_p(stream.cuda_stream))
    nat.check(rc)
    stream.synchronize()
    return st.cpu().numpy()


@pytest.mark.parametrize("name", [c[0] for c in CURVES])
def test_dev_equals_host_keyed_with_bad_indices(lib, name):
    import torch
    from elliptic_b200 import _native as nat
    cid, ln, xy, e, r, s, idx, _ = preset_items(lib, name)
    n = min(len(idx), 1 << 17)
    e, r, s, idx = e[-n:], r[-n:], s[-n:], idx[-n:]
    h, _ = create(lib, cid, xy, 0, 0)
    want = np.zeros(n, np.uint8)
    nat.call(lib.eb200_ecdsa_verify_batch_keyed, h, n, np.ascontiguousarray(e), np.ascontiguousarray(r),
             np.ascontiguousarray(s), np.ascontiguousarray(idx), want)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = dev_call(lib, h, e, r, s, idx, side)
    assert nat.last_timing()["launches"] == 5
    assert (got == want).all(), np.nonzero(got != want)[0][:8]
    bad = idx.copy()
    pos = np.arange(0, n, 97)
    bad[pos] = np.resize(np.array([len(xy), 1 << 31, (1 << 32) - 1], np.uint32), len(pos))
    got = dev_call(lib, h, e, r, s, bad)
    assert (got[pos] == nat.ST_BAD_KEY_INDEX).all()
    keep = np.ones(n, bool); keep[pos] = False
    assert (got[keep] == want[keep]).all()
    nat.check(lib.eb200_keyset_destroy(h))


def test_dev_workspace_and_argument_errors(lib):
    import torch
    from elliptic_b200 import _native as nat
    cid, ln, xy, e, r, s, idx, _ = preset_items(lib, "secp256k1")
    h, _ = create(lib, cid, xy)
    a = lambda x: (x + 255) & ~255
    for n in (1, 1000, 1 << 20):
        # screened key_idx | verdicts | prep words (19 per item) | inversion scratch (8 per item), 256-byte aligned
        assert lib.eb200_ecdsa_verify_keyed_workspace_bytes(h, n) == a(n * 4) + a(n) + a(a(19 * n * 4) + 8 * n * 4)
    assert lib.eb200_ecdsa_verify_keyed_workspace_bytes(None, 8) == 0
    d = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda").data_ptr()
    f = lib.eb200_ecdsa_verify_batch_keyed_dev
    for k in range(7):
        args = [d] * 7
        args[k] = None
        if k == 6:
            continue                                   # the stream: NULL is the default stream
        assert f(h, 8, *args) == nat.ERR_ARG
    host = np.zeros(1 << 16, np.uint8)
    assert f(h, 8, d, d, d, d, host.ctypes.data, d, None) == nat.ERR_NOT_INIT      # d_status not device memory
    assert f(h, 0, None, None, None, None, None, None, None) == nat.OK
    if torch.cuda.device_count() > 1 and lib.eb200_device_count() == 1:
        with torch.cuda.device(1):
            d1 = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda:1").data_ptr()
        assert f(h, 8, d, d, d, d, d1, d, None) == nat.ERR_NOT_INIT            # device 1 not initialised
        nat.init_devices([0, 1])
        assert f(h, 8, d1, d1, d1, d1, d1, d1, None) == nat.ERR_ARG            # initialised, but not holding this set
    nat.check(lib.eb200_keyset_destroy(h))


def test_dev_threads_against_one_set(lib):
    import torch
    from elliptic_b200 import _native as nat
    cid, ln, xy, e, r, s, idx, _ = preset_items(lib, "secp256k1")
    n = 1 << 15
    h, _ = create(lib, cid, xy)
    want = np.zeros(n, np.uint8)
    nat.call(lib.eb200_ecdsa_verify_batch_keyed, h, n, np.ascontiguousarray(e[:n]), np.ascontiguousarray(r[:n]),
             np.ascontiguousarray(s[:n]), np.ascontiguousarray(idx[:n]), want)
    errs = []

    def work(k):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(3):
                    got = dev_call(lib, h, e[:n], r[:n], s[:n], idx[:n], st)
                    assert (got == want).all()
        except Exception as ex:                        # reported on the main thread
            errs.append(repr(ex))
    th = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in th: t.start()
    for t in th: t.join()
    nat.check(lib.eb200_keyset_destroy(h))
    assert not errs, errs


def test_python_keyset_der_equals_ec_der(lib):
    """KeySet.verify_batch_der_packed equals EC.verify_batch_der_packed with the keys gathered, on a set that mixes
    {x, y}, uncompressed and compressed keys (one native set per wire format the host mirror keeps)."""
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    cid, ln, xy, e, r, s, idx, ders = preset_items(lib, "secp256k1")
    m, n = 48, 20000
    sel = np.nonzero(idx < m)[0][:n]
    pubs = []
    for k in range(m):
        x, y = xy[k, :32].tobytes(), xy[k, 32:].tobytes()
        pubs.append({"x": x.hex(), "y": y.hex()} if k % 3 == 0 else ("04" + (x + y).hex()) if k % 3 == 1 else
                    ("%02x" % (2 + (y[-1] & 1)) + x.hex()))
    ec = EC("secp256k1")
    ks = ec.key_set(pubs, "hex")
    assert len(ks._sets) >= 2
    got = ks.verify_batch_der_packed(e[sel], [ders[i] for i in sel], idx[sel])
    want = ec.verify_batch_der_packed(e[sel], [ders[i] for i in sel], xy[idx[sel]], nat.PUB_XY)
    assert np.array_equal(got, want) and {0, 1, 9} <= set(int(v) for v in np.unique(want))
    with pytest.raises(ValueError):
        ks.verify_batch_der_packed(e[:2], ders[:2], [0, m])
    ks.close()


def test_released_set_answers_not_init():
    """Last in this file: eb200_shutdown releases the set's devices; both new calls then return ERR_NOT_INIT."""
    import torch
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    rnd = np.random.default_rng(5)
    d = rnd.integers(1, 255, size=(4, 32), dtype=np.uint8)
    xy, st = np.zeros((4, 64), np.uint8), np.zeros(4, np.uint8)
    nat.call(lib.eb200_scalar_mul_batch, 1, 4, d, None, xy, st)
    h, _ = create(lib, 1, xy)
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    nat.shutdown()
    try:
        data, off = kd.blob([b"\x30\x00"] * 4)
        assert lib.eb200_ecdsa_verify_batch_keyed_der(h, 4, np.zeros(128, np.uint8).ctypes.data, data.ctypes.data,
                                                      off.ctypes.data, np.zeros(4, np.uint32).ctypes.data,
                                                      np.zeros(4, np.uint8).ctypes.data) == nat.ERR_NOT_INIT
        assert lib.eb200_ecdsa_verify_batch_keyed_dev(h, 4, p, p, p, p, p, p, None) == nat.ERR_NOT_INIT
        nat.check(lib.eb200_keyset_destroy(h))
    finally:
        nat.init(0)
