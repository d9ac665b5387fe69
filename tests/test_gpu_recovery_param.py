"""eb200_ecdsa_recovery_param_batch (EC.getKeyRecoveryParam) on the GPU: parity with the oracle through the C ABI and the
host mirror, sign -> recover-parameter round trips, agreement with the answer composed from eb200_ecdsa_recover_batch,
return codes and launch counts with a device, and sharding over two devices."""
import numpy as np
import pytest

from krp_items import CURVES, NO_RECOVERY, krp_items
from test_recovery_param import RECOVER_NO_DEVICE, abi_cases, cases

pytestmark = pytest.mark.gpu

NMOD = {}


def order(name):
    if name not in NMOD:
        from elliptic_b200.ec import _CURVES
        NMOD[name] = (_CURVES[name]["n"], _CURVES[name]["p"])
    return NMOD[name]


def call(lib, cid, e, r, s, q):
    from elliptic_b200 import _native as nat
    n = e.shape[0]
    rid, st = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    arrs = [np.ascontiguousarray(a) for a in (e, r, s, q)]
    nat.check(lib.eb200_ecdsa_recovery_param_batch(cid, n, *[a.ctypes.data for a in arrs], rid.ctypes.data, st.ctypes.data))
    return rid, st


def pack(vals, ln):
    return np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in vals), np.uint8).reshape(len(vals), ln).copy()


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_abi_and_mirror_match_the_oracle(native, name, cid, ln):
    from elliptic_b200.ec import EC
    ec, items, truth, want = cases(name, ln)
    n = ec.n
    e = pack([it[0] % n for it in items], ln)
    r, s = pack([it[1] for it in items], ln), pack([it[2] for it in items], ln)
    q = np.concatenate([pack([it[3] for it in items], ln), pack([it[4] for it in items], ln)], axis=1)
    rid, st = call(native, cid, e, r, s, q)
    assert set(st.tolist()) <= {1, NO_RECOVERY} and not rid[st != 1].any()
    assert [int(j) if t == 1 else int(t) for j, t in zip(rid, st)] == want
    js, st2 = EC(name).get_key_recovery_param_batch([it[0] for it in items], [_sig(it) for it in items],
                                                    [(it[3], it[4]) for it in items])
    assert [j if t == 1 else int(t) for j, t in zip(js, st2)] == want


class _sig:                    # a Signature-like object: r = 0 / s = 0 do not pass the {r, s} dict form
    def __init__(self, it):
        self.r, self.s, self.recoveryParam = it[1], it[2], None


def _keys_and_sigs(name, ln, n, seed, canonical):
    """n signatures made on the GPU with their keys (mirror batch calls)."""
    from elliptic_b200.ec import EC
    rng = np.random.default_rng(seed)
    nn, _ = order(name)
    ec = EC(name)
    privs = [int.from_bytes(rng.bytes(ln + 8), "big") % (nn - 1) + 1 for _ in range(n)]
    msgs = [int.from_bytes(rng.bytes(ln), "big") >> max(0, 8 * ln - nn.bit_length() + 1) for _ in range(n)]
    rs, ss, rec = ec.sign_batch(msgs, privs, canonical=canonical)
    pubs = ec.g_mul_batch(privs)
    e = pack([m % nn for m in msgs], ln)
    q = np.concatenate([pack([x for x, _ in pubs], ln), pack([y for _, y in pubs], ln)], axis=1)
    return e, pack(rs, ln), pack(ss, ln), q, np.asarray(rec, np.uint8)


@pytest.mark.parametrize("name,cid,ln,n", [("secp256k1", 1, 32, 1 << 16), ("p256", 2, 32, 1 << 16), ("p384", 3, 48, 1 << 12),
                                           ("p521", 6, 66, 1 << 10), ("p192", 7, 24, 1 << 12), ("p224", 8, 28, 1 << 12)])
def test_round_trip_from_gpu_signatures(native, name, cid, ln, n):
    for canonical in (False, True):
        e, r, s, q, rec = _keys_and_sigs(name, ln, n, seed=cid * 10 + canonical, canonical=canonical)
        rid, st = call(native, cid, e, r, s, q)
        assert (st == 1).all() and np.array_equal(rid, rec), (name, canonical)
        bad = e.copy()
        bad[:, ln - 1] ^= 0x5A                                   # one byte of e
        rid, st = call(native, cid, bad, r, s, q)
        assert (st == NO_RECOVERY).all() and not rid.any(), (name, canonical)


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_agrees_with_composed_recover_calls(native, name, cid, ln):
    """First j whose eb200_ecdsa_recover_batch point equals Q, on valid, wrong-key and random items."""
    from elliptic_b200 import _native as nat
    n = 1 << 14 if ln < 66 else 1 << 12
    e, r, s, q, rec = _keys_and_sigs(name, ln, n, seed=100 + cid, canonical=False)
    rng = np.random.default_rng(200 + cid)
    third = n // 3
    q[third:2 * third] = np.roll(q[third:2 * third], 1, axis=0)                    # wrong keys
    nn, _ = order(name)
    r[2 * third:] = pack([int.from_bytes(rng.bytes(ln), "big") >> (8 * ln - nn.bit_length()) for _ in range(n - 2 * third)], ln)
    s[2 * third:] = pack([int.from_bytes(rng.bytes(ln), "big") % nn for _ in range(n - 2 * third)], ln)
    rid, st = call(native, cid, e, r, s, q)
    want = np.full(n, NO_RECOVERY, np.uint8)
    done = np.zeros(n, bool)
    for j in range(4):
        out, sj, js = np.zeros((n, 2 * ln), np.uint8), np.zeros(n, np.uint8), np.full(n, j, np.uint8)
        nat.check(native.eb200_ecdsa_recover_batch(cid, n, e.ctypes.data, r.ctypes.data, s.ctypes.data, js.ctypes.data,
                                                   out.ctypes.data, sj.ctypes.data))
        hit = ~done & (sj == 1) & (out == q).all(axis=1)
        want[hit] = j
        done |= hit
    got = np.where(st == 1, rid, st)
    assert np.array_equal(got, want)
    assert (got[:third] == rec[:third]).all() and (got[third:] == NO_RECOVERY).mean() > 0.9


def test_return_codes_and_launches_with_device(native):
    from elliptic_b200 import _native as nat
    cs, _keep = abi_cases()
    with_dev = {"curve77": -5, "ed25519": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3}
    assert {t: native.eb200_ecdsa_recover_batch(*a) for t, a in cs} == with_dev
    assert {t: native.eb200_ecdsa_recovery_param_batch(*a) for t, a in cs} == with_dev
    assert RECOVER_NO_DEVICE.keys() == with_dev.keys()
    for name, cid, ln in CURVES:
        e, r, s, q, rec = _keys_and_sigs(name, ln, 256, seed=cid, canonical=False)
        s[:3] = 0                                                   # the cold kernel has work too
        rid, st = call(native, cid, e, r, s, q)
        t = nat.last_timing()
        assert t["launches"] == 3 and t["main_kernel_ms"] > 0, name
        assert (st[3:] == 1).all() and np.array_equal(rid[3:], rec[3:])


def test_sharded_over_two_devices():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from elliptic_b200 import _native as nat
    lib = nat.init_devices([0, 1])
    n = (1 << 15) + 4099
    e, r, s, q, rec = _keys_and_sigs("secp256k1", 32, n, seed=77, canonical=True)
    rid, st = call(lib, 1, e, r, s, q)
    assert (st == 1).all() and np.array_equal(rid, rec)
