"""The device-pointer forms of the keyed calls on the GPU: each must write exactly what its host form writes, outputs and
statuses, with BAD_KEY_INDEX / BAD_ITEM and zeroed outputs for the arguments the host form refuses; on a non-default
stream whose own copies wrote the inputs, with a workspace of stale bytes and guard regions; plus the argument,
lifetime and secret-clearing contract."""
import ctypes

import numpy as np
import pytest

import benchdata
import ed_ks_items as eki
from gpu_keyset_items import gpu_items
from ks_items import CURVES

pytestmark = pytest.mark.gpu
N25519 = 2**252 + 27742317777372353535851937790883648493
GUARD = 512
NITEMS = 1 << 17


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


class Out:
    """An output buffer of `nbytes` for dev()."""
    def __init__(self, nbytes):
        self.nbytes = nbytes


def dev(lib, fn, h, n, args, launches=None):
    """fn(h, n, *args, workspace, stream) on a fresh non-default stream: numpy arrays are copied to the device by copies
    enqueued on that stream just before, Out(b) becomes a b-byte device buffer, ints pass through.  The workspace is
    sized by eb200_keyset_dev_workspace_bytes and filled with 0xA5; every buffer is followed by a guard that must stay
    unchanged.  Returns the outputs (numpy) and the workspace."""
    import torch
    from elliptic_b200 import _native as nat
    st = torch.cuda.Stream()
    wsb = lib.eb200_keyset_dev_workspace_bytes(h, n)
    bufs, outs, cargs = [], [], []
    with torch.cuda.stream(st):
        ws = torch.full((wsb + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        for a in args:
            if isinstance(a, np.ndarray):
                src = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy())
                t = torch.full((src.numel() + GUARD,), 0x5A, dtype=torch.uint8, device="cuda")
                t[:src.numel()].copy_(src, non_blocking=True)
                bufs.append((t, src.numel()))
                cargs.append(ctypes.c_void_p(t.data_ptr()))
            elif isinstance(a, Out):
                t = torch.full((a.nbytes + GUARD,), 0x5A, dtype=torch.uint8, device="cuda")
                outs.append((t, a.nbytes))
                cargs.append(ctypes.c_void_p(t.data_ptr()))
            elif a is None:
                cargs.append(None)
            else:
                cargs.append(ctypes.c_uint64(a))
        nat.check(fn(h, n, *cargs, ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(st.cuda_stream)))
    st.synchronize()
    tm = nat.last_timing()
    if launches is not None:
        assert tm["launches"] == launches
    for t, nb in bufs + outs + [(ws, wsb)]:
        g = t[nb:].cpu().numpy()
        assert (g == (0xA5 if t is ws else 0x5A)).all(), "guard overwritten"
    return [t[:nb].cpu().numpy() for t, nb in outs], ws[:wsb].cpu().numpy()


def host(fn, *args):
    from elliptic_b200 import _native as nat
    nat.call(fn, *args)


def body_at(n):
    """Offset of a workspace's body, behind the screened indices and the verdicts."""
    return ((n * 4 + 255) & ~255) + ((n + 255) & ~255)


def scatter_bad_idx(idx, m, step=97, start=5):
    bad = idx.copy()
    pos = np.arange(start, len(idx), step)
    bad[pos] = np.resize(np.array([m, 1 << 31, (1 << 32) - 1, m + 1], np.uint32), len(pos))
    return bad, pos


def check_rows(got_out, got_st, want_out, want_st, bad_pos, code, ol):
    keep = np.ones(len(want_st), bool)
    keep[bad_pos] = False
    assert (got_st[keep] == want_st[keep]).all(), np.nonzero(got_st[keep] != want_st[keep])[0][:8]
    assert (got_st[bad_pos] == code).all()
    if ol:
        go, wo = got_out.reshape(len(want_st), ol), want_out.reshape(len(want_st), ol)
        assert (go[keep] == wo[keep]).all()
        assert not go[bad_pos].any()


# ---- ECDSA sets ----------------------------------------------------------------------------------------------------------

def ecdsa_set(lib, cid, ln, n, seed):
    """A SEC1-uncompressed set of 64 keys from GPU signers, key 5 with a prefix that throws and key 9 off the curve
    (imported, replayed), with n items signed under those keys."""
    from elliptic_b200 import _native as nat
    m = 64
    xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, m, n, seed)
    pub = np.concatenate([np.full((m, 1), 4, np.uint8), xy], axis=1)
    pub[5, 0] = 5
    pub[9, -1] ^= 1
    kst, h = np.zeros(m, np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_keyset_create(cid, m, pub.ctypes.data, nat.PUB_SEC1_65, 0, kst.ctypes.data, ctypes.byref(h)))
    assert kst[9] == nat.ST_FALSE and kst[5] > nat.ST_TRUE
    return h, m, e, r, s, idx


@pytest.mark.parametrize("name", [c[0] for c in CURVES])
def test_ecdsa_calls_equal_host_forms(lib, name):
    from elliptic_b200 import _native as nat
    cid, ln = {c[0]: (c[1], c[2]) for c in CURVES}[name]
    n = NITEMS
    h, m, e, r, s, idx = ecdsa_set(lib, cid, ln, n, seed=cid)
    rng = np.random.default_rng(cid)
    k1, k2 = (rng.integers(0, 256, (n, ln), dtype=np.uint8) for _ in range(2))
    k1[::31] = 0
    bad, pos = scatter_bad_idx(idx, m)
    calls = [("mul", lib.eb200_scalar_mul_batch_keyed, lib.eb200_scalar_mul_batch_keyed_dev, [k2], 2 * ln),
             ("mul_add", lib.eb200_mul_add_batch_keyed, lib.eb200_mul_add_batch_keyed_dev, [k1, k2], 2 * ln),
             ("derive", lib.eb200_ecdh_derive_batch_keyed, lib.eb200_ecdh_derive_batch_keyed_dev, [k2], ln),
             ("recid", lib.eb200_ecdsa_recovery_param_batch_keyed, lib.eb200_ecdsa_recovery_param_batch_keyed_dev,
              [e, r, s], 1)]
    for what, hf, df, ins, ol in calls:
        want_o, want_s = np.zeros(n * ol, np.uint8), np.zeros(n, np.uint8)
        host(hf, h, n, *ins, idx, want_o, want_s)
        (got_o, got_s), ws = dev(lib, df, h, n, ins + [idx, Out(n * ol), Out(n)], launches=6)
        assert (got_o == want_o).all() and (got_s == want_s).all(), what
        assert (want_s[idx == 5] > nat.ST_TRUE).all(), what              # the key whose import threw
        if what == "derive":
            assert not ws[body_at(n):].any(), "derive left scalar-derived words in the workspace"
        (got_o, got_s), _ = dev(lib, df, h, n, ins + [bad, Out(n * ol), Out(n)])
        check_rows(got_o, got_s, want_o, want_s, pos, nat.ST_BAD_KEY_INDEX, ol)
    nat.check(lib.eb200_keyset_destroy(h))


# ---- EdDSA sets ----------------------------------------------------------------------------------------------------------

def ed_data(n):
    """The key-set cases (non-canonical, small-order, mixed-order and throwing keys) tiled to n items, and a message
    subset with mixed lengths (empty included)."""
    from oracle.ref_py.eddsa import EDDSA
    ed = EDDSA("ed25519")
    keys, items = eki.cases(ed, vectors=64)
    A, R, S, hh, idx = eki.pack(keys, items)
    reps = -(-n // len(idx))
    R, S, hh, idx = (np.ascontiguousarray(np.tile(x, (reps, 1))[:n] if x.ndim == 2 else np.tile(x, reps)[:n])
                     for x in (R, S, hh, idx))
    return A, R, S, hh, idx


def test_eddsa_verify_equals_host_forms(lib):
    from elliptic_b200 import _native as nat
    n = NITEMS
    A, R, S, hh, idx = ed_data(n)
    m = len(A)
    kst, h = np.zeros(m, np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_keyset_create(m, A.ctypes.data, 0, kst.ctypes.data, ctypes.byref(h)))
    want = np.zeros(n, np.uint8)
    host(lib.eb200_eddsa_verify_batch_keyed, h, n, R, S, hh, idx, want)
    (got,), _ = dev(lib, lib.eb200_eddsa_verify_batch_keyed_dev, h, n, [R, S, hh, idx, Out(n)], launches=3)
    assert (got == want).all() and {0, 1} <= set(np.unique(want).tolist())
    # bad h (n - 1 stays good) on keys away from the end of the table, bad indices elsewhere
    bad_h = hh.copy()
    hpos = np.arange(3, n, 101)
    hpos = hpos[idx[hpos] < m - 4]
    vals = [N25519, N25519 + 1, 2**252 + 2**253, 2**256 - 1]
    for j, p in enumerate(hpos):
        bad_h[p] = np.frombuffer(vals[j % 4].to_bytes(32, "little"), np.uint8)
    bidx, ipos = scatter_bad_idx(idx, m, 89, 7)
    both = np.intersect1d(hpos, ipos)
    (got,), _ = dev(lib, lib.eb200_eddsa_verify_batch_keyed_dev, h, n, [R, S, bad_h, bidx, Out(n)])
    exp = want.copy()
    exp[hpos] = nat.ST_BAD_ITEM
    exp[ipos] = nat.ST_BAD_KEY_INDEX                         # precedence over a bad h
    assert (got == exp).all() and len(both) > 0
    # raw messages: mixed lengths with empty ones, and a NULL buffer of length 0
    rng = np.random.default_rng(4)
    lens = rng.integers(0, 300, n)
    lens[::5] = 0
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    msgs = rng.integers(0, 256, int(off[n]) + 64, dtype=np.uint8)     # 64 spare bytes past msgs_len
    L = int(off[n])
    want = np.zeros(n, np.uint8)
    host(lib.eb200_eddsa_verify_batch_keyed_msgs, h, n, R, S, msgs, off, idx, want)
    (got,), _ = dev(lib, lib.eb200_eddsa_verify_batch_keyed_msgs_dev, h, n, [R, S, msgs, L, off, idx, Out(n)], launches=5)
    assert (got == want).all()
    z = np.zeros(n + 1, np.uint64)
    host(lib.eb200_eddsa_verify_batch_keyed_msgs, h, n, R, S, None, z, idx, want)
    (got,), _ = dev(lib, lib.eb200_eddsa_verify_batch_keyed_msgs_dev, h, n, [R, S, None, 0, z, idx, Out(n)])
    assert (got == want).all()
    # bad ranges that stay inside the buffer: the last item ends one past msgs_len, and a decreasing pair
    boff = off.copy()
    boff[n] = L + 1
    dpos = n // 2 + int(np.argmax(lens[n // 2:] > 0))
    boff[dpos + 1] = boff[dpos] - 1
    host(lib.eb200_eddsa_verify_batch_keyed_msgs, h, n, R, S, msgs, off, idx, want)
    (got,), _ = dev(lib, lib.eb200_eddsa_verify_batch_keyed_msgs_dev, h, n, [R, S, msgs, L, boff, bidx, Out(n)])
    changed = {n - 1, dpos, dpos + 1}
    for i in range(n):
        a, b = int(boff[i]), int(boff[i + 1])
        e = nat.ST_BAD_KEY_INDEX if bidx[i] >= m else nat.ST_BAD_ITEM if (b < a or b > L) else None
        if e is not None:
            assert got[i] == e, i
        elif i not in changed:
            assert got[i] == want[i], i
    assert got[n - 1] in (nat.ST_BAD_ITEM, nat.ST_BAD_KEY_INDEX)
    nat.check(lib.eb200_keyset_destroy(h))


def test_eddsa_sign_equals_host_form(lib):
    from elliptic_b200 import _native as nat
    n, m = NITEMS, 512
    rng = np.random.default_rng(8)
    sec = rng.integers(0, 256, (m, 32), dtype=np.uint8)
    lens = rng.integers(0, 200, n)
    lens[::7] = 0
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    L = int(off[n])
    msgs = rng.integers(0, 256, L + 64, dtype=np.uint8)
    idx = rng.integers(0, m, n).astype(np.uint32)
    pub, h = np.zeros((m, 32), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_signing_set_create(m, sec.ctypes.data, pub.ctypes.data, ctypes.byref(h)))
    want, wst = np.zeros(64 * n, np.uint8), np.zeros(n, np.uint8)
    host(lib.eb200_eddsa_sign_batch_keyed, h, n, msgs, off, idx, want, wst)
    (sig, st), ws = dev(lib, lib.eb200_eddsa_sign_batch_keyed_dev, h, n, [msgs, L, off, idx, Out(64 * n), Out(n)],
                        launches=5)
    assert (sig == want).all() and (st == wst).all() and (st == nat.ST_TRUE).all()
    body = ws[body_at(n):].view(np.uint32)
    assert not body[32 * n: 40 * n].any(), "nonces left in the workspace"
    # screened items, one of them in every normalisation batch position range: bad indices and bad ranges
    bidx, ipos = scatter_bad_idx(idx, m, 61, 0)
    boff = off.copy()
    boff[n] = L + 1
    (sig, st), _ = dev(lib, lib.eb200_eddsa_sign_batch_keyed_dev, h, n, [msgs, L, boff, bidx, Out(64 * n), Out(n)])
    bad = np.zeros(n, bool)
    bad[ipos] = True
    bad[n - 1] = True
    sig = sig.reshape(n, 64)
    want = want.reshape(n, 64)
    assert (st[ipos] == nat.ST_BAD_KEY_INDEX).all()
    assert st[n - 1] == (nat.ST_BAD_KEY_INDEX if bidx[n - 1] >= m else nat.ST_BAD_ITEM)
    assert not sig[bad].any()
    assert (sig[~bad] == want[~bad]).all() and (st[~bad] == nat.ST_TRUE).all()
    nat.check(lib.eb200_keyset_destroy(h))


def test_x25519_derive_equals_host_form(lib):
    from elliptic_b200 import _native as nat
    n = NITEMS
    ds = benchdata.gen_x25519_derive(n, n_pubs=4096, cache_dir=benchdata.cache_dir())
    keys, idx = np.unique(ds["pubx"].view("V32").reshape(-1), return_inverse=True)
    keys = np.ascontiguousarray(keys.view(np.uint8).reshape(-1, 32))
    idx = idx.reshape(-1).astype(np.uint32)
    m = len(keys)
    rng = np.random.default_rng(9)
    priv = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    priv[:, 0] &= 0x0F                                        # below 2^252 < n
    kst, h = np.zeros(m, np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_x25519_keyset_create(m, keys.ctypes.data, 0, kst.ctypes.data, ctypes.byref(h)))
    assert (kst == nat.ST_THROW_ASSERT).any()                 # twist keys
    want, wst = np.zeros(32 * n, np.uint8), np.zeros(n, np.uint8)
    host(lib.eb200_x25519_derive_batch_keyed, h, n, priv, idx, want, wst)
    (out, st), ws = dev(lib, lib.eb200_x25519_derive_batch_keyed_dev, h, n, [priv, idx, Out(32 * n), Out(n)], launches=4)
    assert (out == want).all() and (st == wst).all()
    assert nat.ST_THROW_ASSERT in wst
    assert not ws[body_at(n):].any(), "derive left scalar-derived words in the workspace"
    bp = priv.copy()
    ppos = np.arange(2, n, 103)
    ppos = ppos[idx[ppos] < m - 4]
    vals = [N25519 - 1, N25519, N25519 + 1, 2**256 - 1]
    for j, p in enumerate(ppos):
        bp[p] = np.frombuffer(vals[j % 4].to_bytes(32, "big"), np.uint8)
    bidx, ipos = scatter_bad_idx(idx, m, 89, 11)
    (out, st), _ = dev(lib, lib.eb200_x25519_derive_batch_keyed_dev, h, n, [bp, bidx, Out(32 * n), Out(n)])
    # n - 1 is a good scalar: recompute those items with the host form
    good_nm1 = ppos[np.arange(len(ppos)) % 4 == 0]
    w2, ws2 = np.zeros(32 * n, np.uint8), np.zeros(n, np.uint8)
    fix = priv.copy()
    fix[good_nm1] = bp[good_nm1]
    host(lib.eb200_x25519_derive_batch_keyed, h, n, fix, idx, w2, ws2)
    exp = ws2.copy()
    exp[np.setdiff1d(ppos, good_nm1)] = nat.ST_BAD_ITEM
    exp[ipos] = nat.ST_BAD_KEY_INDEX
    assert (st == exp).all()
    out, w2 = out.reshape(n, 32), w2.reshape(n, 32)
    bad = np.isin(np.arange(n), np.union1d(ipos, np.setdiff1d(ppos, good_nm1)))
    assert not out[bad].any() and (out[~bad] == w2[~bad]).all()
    nat.check(lib.eb200_keyset_destroy(h))


# ---- contract --------------------------------------------------------------------------------------------------------------

def small_sets(lib):
    """One set of each kind, four keys each: ECDSA (secp256k1), EdDSA, signing, curve25519."""
    from elliptic_b200 import _native as nat
    rnd = np.random.default_rng(5)
    d = rnd.integers(1, 255, size=(4, 32), dtype=np.uint8)
    xy, st = np.zeros((4, 64), np.uint8), np.zeros(4, np.uint8)
    nat.call(lib.eb200_scalar_mul_batch, 1, 4, d, None, xy, st)
    out = {}
    for kind, make in (("ecdsa", lambda h: lib.eb200_keyset_create(1, 4, xy.ctypes.data, 0, 4, st.ctypes.data, h)),
                       ("ed", lambda h: lib.eb200_eddsa_keyset_create(4, d.ctypes.data, 4, st.ctypes.data, h)),
                       ("sign", lambda h: lib.eb200_eddsa_signing_set_create(4, d.ctypes.data, None, h)),
                       ("x25519", lambda h: lib.eb200_x25519_keyset_create(4, d.ctypes.data, 4, st.ctypes.data, h))):
        h = ctypes.c_void_p()
        nat.check(make(ctypes.byref(h)))
        out[kind] = h
    return out


def calls(lib):
    """(function, set kind, argument count before the workspace, index of d_status, indices of ints)"""
    return [(lib.eb200_scalar_mul_batch_keyed_dev, "ecdsa", 4, 3, ()),
            (lib.eb200_mul_add_batch_keyed_dev, "ecdsa", 5, 4, ()),
            (lib.eb200_ecdh_derive_batch_keyed_dev, "ecdsa", 4, 3, ()),
            (lib.eb200_ecdsa_recovery_param_batch_keyed_dev, "ecdsa", 6, 5, ()),
            (lib.eb200_eddsa_verify_batch_keyed_dev, "ed", 5, 4, ()),
            (lib.eb200_eddsa_verify_batch_keyed_msgs_dev, "ed", 7, 6, (3,)),
            (lib.eb200_eddsa_sign_batch_keyed_dev, "sign", 6, 5, (1,)),
            (lib.eb200_x25519_derive_batch_keyed_dev, "x25519", 4, 3, ())]


def test_contract(lib):
    import torch
    from elliptic_b200 import _native as nat
    sets = small_sets(lib)
    bufs = [torch.zeros(1 << 16, dtype=torch.uint8, device="cuda") for _ in range(8)]
    dp = bufs[7].data_ptr()                                  # the workspace
    host_mem = np.zeros(1 << 16, np.uint8)
    for kind, h in sets.items():
        w = lib.eb200_keyset_dev_workspace_bytes(h, 1000)
        assert w > 0
        if kind == "ecdsa":
            for n in (1, 1000, 1 << 20):
                assert lib.eb200_keyset_dev_workspace_bytes(h, n) >= lib.eb200_ecdsa_verify_keyed_workspace_bytes(h, n)
    assert lib.eb200_keyset_dev_workspace_bytes(None, 8) == 0
    for fn, kind, na, si, ints in calls(lib):
        base = [0 if j in ints else bufs[j].data_ptr() for j in range(na)]
        for other, h in sets.items():
            if other != kind:
                assert fn(h, 8, *base, dp, None) == nat.ERR_ARG, (fn, other)
        h = sets[kind]
        assert fn(None, 8, *base, dp, None) == nat.ERR_ARG
        assert fn(h, 0, *[0 if j in ints else None for j in range(na)], None, None) == nat.OK
        for j in range(na):
            if j in ints:
                continue
            args = list(base)
            args[j] = None
            if kind in ("ed", "sign") and (j == ints[0] - 1 if ints else False):
                assert fn(h, 8, *args, dp, None) == nat.OK   # d_msgs NULL with msgs_len 0
                continue
            assert fn(h, 8, *args, dp, None) == nat.ERR_ARG, (fn, j)
        assert fn(h, 8, *base, None, None) == nat.ERR_ARG  # no workspace
        args = list(base)
        args[si] = host_mem.ctypes.data
        assert fn(h, 8, *args, dp, None) == nat.ERR_NOT_INIT   # d_status not device memory
        if ints:
            args = list(base)
            args[ints[0] - 1] = None
            args[ints[0]] = 5
            assert fn(h, 8, *args, dp, None) == nat.ERR_ARG     # NULL d_msgs with msgs_len > 0
    torch.cuda.synchronize()
    if torch.cuda.device_count() > 1:
        with torch.cuda.device(1):
            d1 = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda:1").data_ptr()
        if lib.eb200_device_count() == 1:
            for fn, kind, na, si, ints in calls(lib):
                args = [0 if j in ints else dp for j in range(na)]
                args[si] = d1
                assert fn(sets[kind], 8, *args, dp, None) == nat.ERR_NOT_INIT     # device 1 not initialised
        nat.init_devices([0, 1])
        for fn, kind, na, si, ints in calls(lib):
            args = [0 if j in ints else d1 for j in range(na)]
            assert fn(sets[kind], 8, *args, d1, None) == nat.ERR_ARG              # initialised, not holding the set
    for h in sets.values():
        nat.check(lib.eb200_keyset_destroy(h))


def test_released_sets_answer_not_init():
    """Last in this file: after eb200_shutdown every new call returns ERR_NOT_INIT for a set it released."""
    import torch
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    sets = small_sets(lib)
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    dp = buf.data_ptr()
    nat.shutdown()
    try:
        for fn, kind, na, si, ints in calls(lib):
            assert fn(sets[kind], 8, *[0 if j in ints else dp for j in range(na)], dp, None) == nat.ERR_NOT_INIT
        for h in sets.values():
            nat.check(lib.eb200_keyset_destroy(h))
    finally:
        nat.init(0)
