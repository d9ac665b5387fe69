"""Key sets on the GPU: eb200_ecdsa_verify_batch_keyed must write exactly the status bytes eb200_ecdsa_verify_batch
writes for the same items with the keys gathered, on every short preset and width, for honest, adversarial, throwing
and off-curve keys; plus the handle's lifetime, argument and timing contract and the Python KeySet."""
import ctypes
import threading

import numpy as np
import pytest

from gpu_keyset_items import gpu_items
from ks_items import CURVES, adversarial_items, adversarial_keys, expected, pack, seeded_set

pytestmark = pytest.mark.gpu


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


def keyed(lib, h, e, r, s, idx):
    from elliptic_b200 import _native as nat
    st = np.full(len(idx), 0xEE, np.uint8)
    nat.call(lib.eb200_ecdsa_verify_batch_keyed, h, len(idx), e, r, s, np.ascontiguousarray(idx, np.uint32), st)
    return st


def unkeyed(lib, cid, e, r, s, pub, fmt=0):
    from elliptic_b200 import _native as nat
    st = np.zeros(len(e), np.uint8)
    nat.call(lib.eb200_ecdsa_verify_batch, cid, len(e), e, r, s, np.ascontiguousarray(pub), fmt, st)
    return st


@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_keyed_equals_unkeyed_on_every_preset(lib, name, cid, ln):
    from elliptic_b200 import _native as nat
    xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, 64, 1 << 16, seed=cid)
    want = unkeyed(lib, cid, e, r, s, xy[idx])
    assert want.sum() == len(idx) - len(idx) // 64
    for bits in (4, 8, 0):
        h, kst = create(lib, cid, xy, 0, bits)
        w = ctypes.c_uint32()
        nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), None))
        assert (kst == 1).all() and w.value == (bits or 8)
        got = keyed(lib, h, e, r, s, idx)
        assert nat.last_timing()["launches"] == 3
        nat.check(lib.eb200_keyset_destroy(h))
        assert (got == want).all(), (name, bits, np.nonzero(got != want)[0][:8])


@pytest.mark.parametrize("name,cid,ln", [c for c in CURVES if c[0] in ("secp256k1", "p256", "p224")])
def test_adversarial_throwing_and_off_curve_keys(lib, name, cid, ln):
    """Keys sharing table entries with G (exceptional additions), against the oracle and the unkeyed call; then the
    same set in compressed form with a bad prefix and an x without a square root, and an off-curve {x, y} key."""
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    ec = EC(name)
    dims = [ctypes.c_int() for _ in range(3)]
    nat.check(lib.eb200_selftest_gtab_dims(cid, *(ctypes.byref(d) for d in dims)))
    keys, items = seeded_set(ec, ln, 3, 24)
    adv = adversarial_keys(ec, cid, (4, 8))
    base = len(keys)
    keys += [(Q.x, Q.y) for _, Q in adv]
    items += [it[:3] + (it[3] + base,) for it in adversarial_items(ec, cid, adv, dims[2].value)]
    keys.append((keys[0][0], (keys[0][1] + 1) % ec.curve.p))
    items += [(e, r, s, len(keys) - 1) for e, r, s, _ in items[:3]]
    xy, e, r, s, idx = pack(ln, keys, items)
    want = unkeyed(lib, cid, e, r, s, xy[idx])
    assert list(want) == expected(ec, keys, items)
    for bits in (4, 8):
        h, kst = create(lib, cid, xy, 0, bits)
        assert list(kst) == [1] * (len(keys) - 1) + [0]
        assert (keyed(lib, h, e, r, s, idx) == want).all()
        nat.check(lib.eb200_keyset_destroy(h))
    comp = np.concatenate([(2 + (xy[:, -1:] & 1)).astype(np.uint8), xy[:, :ln]], axis=1)
    comp[1, 0] = 5                                        # 'Unknown point format'
    x = 1
    while True:                                           # an x with no point: 'invalid point' (p224: the Tonelli-Shanks assertion)
        try:
            ec.curve.point_from_x(x, 0)
            x += 1
        except Exception:
            break
    comp[2, 1:] = np.frombuffer(x.to_bytes(ln, "big"), np.uint8)
    want = unkeyed(lib, cid, e, r, s, comp[idx], 2)
    h, kst = create(lib, cid, comp, 2, 0)
    assert kst[1] == nat.ST_THROW_POINT_FORMAT and kst[2] in (nat.ST_THROW_INVALID_POINT, nat.ST_THROW_ASSERT)
    got = keyed(lib, h, e, r, s, idx)
    assert (got == want).all() and {int(kst[1]), int(kst[2])} <= set(got.tolist())
    nat.check(lib.eb200_keyset_destroy(h))


def test_full_size_benchmark_shape(lib):
    """secp256k1, 2^20 items over 4096 keys (the benchmark's shape): the generator's expectation and the unkeyed call."""
    import benchdata
    from elliptic_b200 import _native as nat
    d = benchdata.gen_secp256k1_verify(1 << 20)
    keys, idx = np.unique(d["pub"], axis=0, return_inverse=True)
    assert len(keys) == 4096
    h, kst = create(lib, 1, keys)
    assert (kst == 1).all()
    got = keyed(lib, h, d["e"], d["r"], d["s"], idx.reshape(-1))
    nat.check(lib.eb200_keyset_destroy(h))
    assert (got == d["expected"]).all() and (got == unkeyed(lib, 1, d["e"], d["r"], d["s"], d["pub"])).all()


def test_handle_contract(lib):
    from elliptic_b200 import _native as nat
    xy, e, r, s, idx = gpu_items(lib, nat, 1, 32, 16, 4096, seed=77)
    want = unkeyed(lib, 1, e, r, s, xy[idx])
    h1, _ = create(lib, 1, xy, 0, 5)
    h2, _ = create(lib, 1, xy[::-1].copy(), 0, 6)
    m, db = ctypes.c_size_t(), ctypes.c_size_t()
    nat.check(lib.eb200_keyset_info(h1, None, ctypes.byref(m), None, ctypes.byref(db)))
    assert m.value == 16 and db.value == 16 * (64 + 1 + 27 * 16 * 64)
    bad = idx.copy(); bad[100] = 16
    st = np.full(len(idx), 0xEE, np.uint8)
    assert lib.eb200_ecdsa_verify_batch_keyed(h1, len(idx), e.ctypes.data, r.ctypes.data, s.ctypes.data, bad.ctypes.data,
                                              st.ctypes.data) == nat.ERR_ARG
    assert (st == 0xEE).all()
    nat.check(lib.eb200_keyset_destroy(h1))               # the other set still answers
    assert (keyed(lib, h2, e, r, s, 15 - idx) == want).all()
    out = [None] * 4

    def work(t):
        out[t] = keyed(lib, h2, e, r, s, 15 - idx)
    th = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert all((o == want).all() for o in out)
    nat.check(lib.eb200_keyset_destroy(h2))


def test_two_devices_give_the_same_statuses(lib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    from elliptic_b200 import _native as nat
    nat.init_devices([0, 1])
    xy, e, r, s, idx = gpu_items(lib, nat, 1, 32, 64, 1 << 16, seed=5)
    h, _ = create(lib, 1, xy)
    assert (keyed(lib, h, e, r, s, idx) == unkeyed(lib, 1, e, r, s, xy[idx])).all()
    nat.check(lib.eb200_keyset_destroy(h))


def test_python_key_set_matches_verify_batch():
    from elliptic_b200.ec import EC, EllipticError
    from oracle.ref_py.ec import EC as RefEC
    ref, ec = RefEC("secp256k1"), EC("secp256k1")
    ds = [11, 22, 33]
    pts = [ref.g.mul(d) for d in ds]
    keys = [{"x": pts[0].x, "y": pts[0].y}, "04%064x%064x" % (pts[1].x, pts[1].y), "%02x%064x" % (2 + (pts[2].y & 1), pts[2].x),
            {"x": pts[0].x, "y": pts[0].y + 1}]
    msgs, sigs, kidx = [], [], []
    for t in range(24):
        k = t % 3
        sg = ref.sign(1000 + t, ds[k])
        msgs.append(1000 + t + (t == 5)); sigs.append({"r": sg.r, "s": sg.s if t != 7 else ref.n}); kidx.append(k if t < 20 else 3)
    with ec.key_set(keys, "hex") as ks:
        assert list(ks.status) == [1, 1, 1, 0] and ks.table_bits == 8 and ks.device_bytes > 0
        got = ks.verify_batch(msgs, sigs, kidx)
    assert (got == ec.verify_batch(msgs, sigs, [keys[k] for k in kidx], "hex")).all() and got[:20].sum() == 18
    with pytest.raises(EllipticError, match="Unknown point format"):
        ec.key_set(["05" + "00" * 32], "hex")
