"""The tensor forms on the GPU: every `*_tensors` method writes exactly what its host form writes, outputs and statuses,
on every curve it takes; the keyed DER device-pointer call equals its host form on the six short presets; a key set of
mixed wire formats gives through every keyed tensor method what its packed method gives, and BAD_KEY_INDEX for indices
that are negative, >= m or beyond 32 bits; the calls run on the caller's stream without synchronising it."""
import ctypes

import numpy as np
import pytest

from gpu_keyset_items import gpu_items
from ks_items import CURVES
from test_gpu_keyset_dev import Out, dev
from test_gpu_unkeyed_dev import ALL, der, msg_block, rnd_rows, signed

pytestmark = pytest.mark.gpu
N = 300


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


def T(a, device="cuda"):
    """A numpy array as a CUDA tensor: uint64 offsets become int64."""
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.astype(np.int64)
    return torch.from_numpy(a.copy()).to(device)


def H(t):
    return t.cpu().numpy()


def host(fn, *args):
    from elliptic_b200 import _native as nat
    nat.call(fn, *args)


def assert_same(got, want, what):
    got = H(got).reshape(want.shape)
    assert (got == want).all(), (what, np.nonzero(got != want)[0][:8])


def throwing_key(make_set, cands):
    """The first candidate key whose import throws, found by importing them all into a probe set."""
    from elliptic_b200 import _native as nat
    with make_set(cands) as probe:
        return cands[int(np.flatnonzero(probe.status > nat.ST_TRUE)[0])]


def throwing_compressed(ec, ln):
    return throwing_key(ec.key_set, [bytes([2]) + v.to_bytes(ln, "big") for v in range(1, 17)])


# ---- EC: each tensor method against its host form --------------------------------------------------------------------

@pytest.mark.parametrize("name,cid,ln", ALL)
def test_ec_tensor_methods_equal_host_forms(lib, name, cid, ln):
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    ec = EC(name)
    e, d, r, s, rec, q = signed(lib, cid, ln, N, cid * 11)
    e[1::9, -1] ^= 1                                                # FALSE
    q2 = q.copy()
    q2[4::31, -1] ^= 1                                              # off-curve keys: replayed / NEEDS_HOST on ed25519
    sec1 = np.concatenate([np.full((N, 1), 4, np.uint8), q2], axis=1)
    sec1[8::37, 0] = 5                                              # a key that throws
    for pub, fmt in ((q2, nat.PUB_XY), (sec1, nat.PUB_SEC1_65)):
        assert_same(ec.verify_batch_tensors(T(e), T(r), T(s), T(pub), fmt), ec.verify_batch_packed(e, r, s, pub, fmt),
                    "verify")
        sigs, off = der(r, s)
        ders = [sigs[int(off[i]):int(off[i + 1])].tobytes() for i in range(N)]
        ders[6::15] = [b"\x31" + x[1:] for x in ders[6::15]]                 # rejected encodings
        blob = np.frombuffer(b"".join(ders), np.uint8)
        got = ec.verify_batch_der_tensors(T(e), T(blob), T(off), T(pub), fmt)
        want = ec.verify_batch_der_packed(e, ders, pub, fmt)
        assert_same(got, want, "der")
        assert {nat.ST_TRUE, nat.ST_FALSE, nat.ST_THROW_SIG_FORMAT} <= set(want.tolist())
    wsb = lib.eb200_dev_workspace_bytes(cid, N)
    assert wsb > 0
    # sign (plain, pers, k with RETRY rows) and keygen against the host calls the Python methods make
    rng = np.random.default_rng(cid)
    pers = rng.integers(0, 256, 40, dtype=np.uint8)
    k = rnd_rows(rng, N, ln, 0x7F)
    k[::5] = 0                                                      # RETRY
    for kw, hf, extra in (({}, lib.eb200_ecdsa_sign_batch, []), ({"pers": T(pers)}, lib.eb200_ecdsa_sign_batch_pers, [pers, 40]),
                          ({"k": T(k)}, lib.eb200_ecdsa_sign_batch_k, [k])):
        want = [np.zeros((N, ln), np.uint8), np.zeros((N, ln), np.uint8), np.zeros(N, np.uint8), np.zeros(N, np.uint8)]
        host(hf, cid, N, e, d, *extra, 1, *want)
        got = ec.sign_batch_tensors(T(e), T(d), canonical=True, **kw)
        assert_same(got[3], want[3], ("sign", sorted(kw), "status"))
        # a RETRY item gets no r, s or recid from the C call (the host form's bytes there are its staging buffer's):
        # those rows are compared where the status is TRUE, and read as zeros in the tensor form
        ok = want[3] == nat.ST_TRUE
        for g, w, what in zip(got[:3], want[:3], ("r", "s", "recid")):
            assert (H(g)[ok] == w[ok]).all(), ("sign", sorted(kw), what)
            assert not H(g)[~ok].any(), ("sign", sorted(kw), what, "RETRY rows")
        if "k" in kw:
            assert nat.ST_RETRY in want[3] and ok.any()
        else:
            assert ok.all()
    ent = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    want = [np.zeros((N, ln), np.uint8), np.zeros((N, 2 * ln), np.uint8), np.zeros(N, np.uint8)]
    host(lib.eb200_ec_keygen_batch, cid, N, ent, 32, pers, 10, *want)
    for g, w in zip(ec.gen_key_pair_batch_tensors(T(ent), T(pers[:10])), want):
        assert_same(g, w, "keygen")
    # mul (G and points), mulAdd, derive; INFINITY and off-curve points
    k1, k2 = rnd_rows(rng, N, ln), rnd_rows(rng, N, ln)
    k2[::29] = 0
    for got, fn, ins, ol in ((ec.mul_batch_tensors(T(k2)), lib.eb200_scalar_mul_batch, [k2, None], 2 * ln),
                             (ec.mul_batch_tensors(T(k2), T(q2)), lib.eb200_scalar_mul_batch, [k2, q2], 2 * ln),
                             (ec.mul_add_batch_tensors(T(k1), T(k2), T(q2)), lib.eb200_mul_add_batch, [k1, k2, q2], 2 * ln),
                             (ec.derive_batch_tensors(T(k2), T(q2)), lib.eb200_ecdh_derive_batch, [k2, q2], ln)):
        want = [np.zeros((N, ol), np.uint8), np.zeros(N, np.uint8)]
        host(fn, cid, N, *ins, *want)
        assert_same(got[0], want[0], fn.__name__)
        assert_same(got[1], want[1], fn.__name__)
    if name == "ed25519":
        return
    # recover and getKeyRecoveryParam: INFINITY, s = 0, second-key candidates, off-curve Q
    r2, s2, rec2 = r.copy(), s.copy(), rec.copy()
    r2[3::17] = 0
    s2[5::13] = 0
    rec2[::3] ^= 2
    want = [np.zeros((N, 2 * ln), np.uint8), np.zeros(N, np.uint8)]
    host(lib.eb200_ecdsa_recover_batch, cid, N, e, r2, s2, rec2, *want)
    for g, w in zip(ec.recover_pub_key_batch_tensors(T(e), T(r2), T(s2), T(rec2)), want):
        assert_same(g, w, "recover")
    assert len(set(want[1].tolist())) > 1
    want = [np.zeros(N, np.uint8), np.zeros(N, np.uint8)]
    host(lib.eb200_ecdsa_recovery_param_batch, cid, N, e, r2, s2, q2, *want)
    for g, w in zip(ec.get_key_recovery_param_batch_tensors(T(e), T(r2), T(s2), T(q2)), want):
        assert_same(g, w, "recovery param")
    assert {nat.ST_TRUE, nat.ST_THROW_NO_RECOVERY} <= set(want[1].tolist())


def test_curve25519_and_eddsa_tensor_methods_equal_host_forms(lib):
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    from elliptic_b200.eddsa import EDDSA
    rng = np.random.default_rng(25519)
    x = EC("curve25519")
    k, px = rng.integers(0, 256, (N, 32), dtype=np.uint8), rng.integers(0, 256, (N, 32), dtype=np.uint8)
    k[:, 0] &= 0x0F                                                 # below n, as derive takes them
    out, st = x.derive_batch_packed(k, px)
    got = x.derive_batch_tensors(T(k), T(px))
    assert_same(got[0], out, "x25519 derive")
    assert_same(got[1], st, "x25519 derive")
    assert {nat.ST_TRUE, nat.ST_THROW_ASSERT} <= set(st.tolist())
    want = [np.zeros((N, 32), np.uint8), np.zeros(N, np.uint8)]
    host(lib.eb200_x25519_mul_batch, N, k, px, *want)
    for g, w in zip(x.x_mul_batch_tensors(T(k), T(px)), want):
        assert_same(g, w, "x25519 mul")
    ed = EDDSA()
    sec = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    msgs, off, L = msg_block(rng, N)
    msgs = msgs[:L].copy()
    sig, pub = ed.sign_batch_packed(sec, msgs, off, want_pub=True)
    g_sig, g_pub, g_st = ed.sign_batch_tensors(T(sec), T(msgs), T(off), want_pub=True)
    assert_same(g_sig, sig, "eddsa sign")
    assert_same(g_pub, pub, "eddsa sign pub")
    assert (H(g_st) == nat.ST_TRUE).all()
    R, S, A = sig[:, :32].copy(), sig[:, 32:].copy(), pub.copy()
    R[3::17] = 0xFF                                                 # R that does not decode
    S[5::19, 31] ^= 0x10                                            # S >= n or a wrong S
    m2 = msgs.copy()
    m2[::53] ^= 1
    want = ed.verify_batch_msgs_packed(R, S, A, m2, off)
    assert_same(ed.verify_batch_msgs_tensors(T(R), T(S), T(A), T(m2), T(off)), want, "eddsa verify msgs")
    assert {nat.ST_TRUE, nat.ST_FALSE} <= set(want.tolist())
    h = np.frombuffer(b"".join(ed.hash_int(R[i], A[i], m2[off[i]:off[i + 1]]).to_bytes(32, "little") for i in range(N)),
                      np.uint8).reshape(N, 32)
    assert_same(ed.verify_batch_tensors(T(R), T(S), T(A), T(h)), ed.verify_batch_packed(R, S, A, h), "eddsa verify")


# ---- the keyed DER device-pointer call against its host form ----------------------------------------------------------

@pytest.mark.parametrize("name,cid,ln", CURVES)
def test_keyed_der_dev_equals_host_form(lib, name, cid, ln):
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    m, n = 64, 2000
    xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, m, n, seed=cid + 100)
    sigs, off = der(r, s)
    L = int(off[n])
    sigs[off[6::15].astype(np.int64)] = 0x31                        # rejected encodings
    s_hi = s.copy()
    s_hi[7::41] = 0xFF                                              # s out of range: FALSE
    sigs2, off2 = der(r, s_hi)
    comp = np.concatenate([(2 + (xy[:, -1] & 1)).astype(np.uint8)[:, None], xy[:, :ln]], axis=1)
    comp[3] = np.frombuffer(throwing_compressed(EC(name), ln), np.uint8)   # no square root: the key throws
    sec1 = np.concatenate([np.full((m, 1), 4, np.uint8), xy], axis=1)
    sec1[5, 0] = 5                                                  # a prefix that throws
    sec1[9, -1] ^= 1                                                # off the curve: replayed
    for pub, fmt in ((sec1, nat.PUB_SEC1_65), (comp, nat.PUB_SEC1_33), (xy, nat.PUB_XY)):
        kst, h = np.zeros(m, np.uint8), ctypes.c_void_p()
        nat.check(lib.eb200_keyset_create(cid, m, np.ascontiguousarray(pub).ctypes.data, fmt, 0, kst.ctypes.data,
                                          ctypes.byref(h)))
        try:
            seen = set()
            for blob, offs in ((sigs, off), (sigs2, off2)):
                Lb = int(offs[n])
                want = np.zeros(n, np.uint8)
                host(lib.eb200_ecdsa_verify_batch_keyed_der, h, n, e, blob, offs, idx, want)
                (got,), _ = dev(lib, lib.eb200_ecdsa_verify_batch_keyed_der_dev, h, n,
                                [e, blob, Lb, offs, idx, Out(n)], launches=6)
                assert (got == want).all(), (fmt, np.nonzero(got != want)[0][:8])
                seen |= set(want.tolist())
            assert {nat.ST_TRUE, nat.ST_FALSE, nat.ST_THROW_SIG_FORMAT} <= seen
            if fmt != nat.PUB_XY:
                assert (want[idx == (5 if fmt == nat.PUB_SEC1_65 else 3)] > nat.ST_TRUE).all()
            # BAD_KEY_INDEX, then BAD_ITEM for a decreasing range and the last past the end (over a key's throw)
            bad, boff = idx.copy(), off.copy()
            bad[5::97] = np.resize(np.array([m, 1 << 31, (1 << 32) - 1], np.uint32), len(bad[5::97]))
            boff[n] = L + 1
            boff[11] = boff[10] - 1
            thrower = 5 if fmt == nat.PUB_SEC1_65 else 3
            bad[10] = thrower
            want = np.zeros(n, np.uint8)
            host(lib.eb200_ecdsa_verify_batch_keyed_der, h, n, e, sigs, off, idx, want)
            (got,), _ = dev(lib, lib.eb200_ecdsa_verify_batch_keyed_der_dev, h, n,
                            [e, sigs, L, boff, bad, Out(n)])
            for i in range(n):
                a, b = int(boff[i]), int(boff[i + 1])
                if bad[i] >= m:
                    assert got[i] == nat.ST_BAD_KEY_INDEX, i
                elif b < a or b > L:
                    assert got[i] == nat.ST_BAD_ITEM, i
                elif a == off[i] and b == off[i + 1] and bad[i] == idx[i]:
                    assert got[i] == want[i], i
            assert got[10] == nat.ST_BAD_ITEM and got[n - 1] in (nat.ST_BAD_ITEM, nat.ST_BAD_KEY_INDEX)
        finally:
            nat.check(lib.eb200_keyset_destroy(h))


# ---- key sets: every keyed tensor method, mixed wire formats and bad indices -----------------------------------------

def bad_indices(idx, m):
    """int64 indices with -1, m, 2^32 + k and 2^33 scattered in; their positions."""
    import torch
    big = idx.astype(np.int64)
    pos = np.arange(3, len(idx), 23)
    big[pos] = np.resize(np.array([-1, m, (1 << 32) + 3, (1 << 32) + int(idx[0]), 1 << 33, -(1 << 32)], np.int64), len(pos))
    return torch.from_numpy(big).cuda(), pos


def check_keyed(got, want, pos, what):
    """Tensor outputs against the packed method's for the items with valid indices, BAD_KEY_INDEX and zero rows at pos."""
    from elliptic_b200 import _native as nat
    got = [H(g) for g in got]
    keep = np.ones(len(got[-1]), bool)
    keep[pos] = False
    for g, w in zip(got, want):
        g = g.reshape(len(keep), -1)
        w = w.reshape(int(keep.sum()), -1)
        assert (g[keep] == w).all(), (what, np.nonzero((g[keep] != w).any(axis=1))[0][:8])
    assert (got[-1][pos] == nat.ST_BAD_KEY_INDEX).all(), what
    for g in got[:-1]:
        assert not g.reshape(len(keep), -1)[pos].any(), what


@pytest.mark.parametrize("name,cid,ln", [CURVES[0], CURVES[2]])
def test_keyset_tensor_methods_mixed_formats(lib, name, cid, ln):
    import torch
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    ec = EC(name)
    m, n = 48, 1500
    xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, m, n, seed=cid + 7)
    keys = []
    for j in range(m):
        x, y = xy[j, :ln].tobytes(), xy[j, ln:].tobytes()
        keys.append({"x": x.hex(), "y": y.hex()} if j % 3 == 0 else b"\x04" + x + y if j % 3 == 1 else
                    bytes([2 + (y[-1] & 1)]) + x)
    keys[4] = throwing_compressed(ec, ln)                           # a compressed key that throws
    keys[7] = {"x": xy[7, :ln].tobytes().hex(), "y": (int.from_bytes(xy[7, ln:].tobytes(), "big") ^ 1)}  # off the curve
    ks = ec.key_set(keys)
    try:
        assert len(ks._sets) == 2 and ks.status[4] > nat.ST_TRUE and ks.status[7] == nat.ST_FALSE
        bidx, pos = bad_indices(idx, m)
        keep = np.ones(n, bool)
        keep[pos] = False
        ki = idx[keep]
        rng = np.random.default_rng(cid)
        k1, k2 = rnd_rows(rng, n, ln), rnd_rows(rng, n, ln)
        k2[::31] = 0
        sigs, off = der(r, s)
        ders = [sigs[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)]
        ders[6::15] = [b"\x31" + x[1:] for x in ders[6::15]]
        blob = np.frombuffer(b"".join(ders), np.uint8)
        for key_idx in (T(idx.astype(np.int64)), T(idx.astype(np.int32))):
            assert_same(ks.verify_batch_tensors(T(e), T(r), T(s), key_idx), ks.verify_batch_packed(e, r, s, idx), "verify")
        cases = [
            ("verify", lambda t: [ks.verify_batch_tensors(T(e), T(r), T(s), t)],
             lambda sel: [ks.verify_batch_packed(e[sel], r[sel], s[sel], ki)]),
            ("der", lambda t: [ks.verify_batch_der_tensors(T(e), T(blob), T(off), t)],
             lambda sel: [ks.verify_batch_der_packed(e[sel], [d for d, k in zip(ders, sel) if k], ki)]),
            ("mul", lambda t: ks.mul_batch_tensors(T(k2), t), lambda sel: ks.mul_batch_packed(k2[sel], ki)),
            ("mul_add", lambda t: ks.mul_add_batch_tensors(T(k1), T(k2), t),
             lambda sel: ks.mul_add_batch_packed(k1[sel], k2[sel], ki)),
            ("derive", lambda t: ks.derive_batch_tensors(T(k2), t), lambda sel: ks.derive_batch_packed(k2[sel], ki)),
            ("recid", lambda t: ks.recovery_param_batch_tensors(T(e), T(r), T(s), t),
             lambda sel: ks.recovery_param_batch_packed(e[sel], r[sel], s[sel], ki)),
        ]
        for what, tensor_form, packed_form in cases:
            want = packed_form(keep)
            got = tensor_form(bidx)
            if len(got) == 1:
                want = [want[0]]
            else:
                want = [want[0], want[1]]
            check_keyed(got, want, pos, what)
            st = want[-1]
            assert (st[ki == 4] > nat.ST_TRUE).all(), what
        # the same through a one-format set: one direct call
        one = ec.key_set([b"\x04" + xy[j].tobytes() for j in range(m)])
        try:
            assert len(one._sets) == 1
            check_keyed([one.verify_batch_tensors(T(e), T(r), T(s), bidx)], [one.verify_batch_packed(e[keep], r[keep], s[keep], ki)],
                        pos, "one-format verify")
            i32 = torch.from_numpy(np.where(keep, idx.astype(np.int64), -1).astype(np.int32)).cuda()
            check_keyed(one.mul_batch_tensors(T(k2), i32), list(one.mul_batch_packed(k2[keep], ki)), np.nonzero(~keep)[0],
                        "int32 -1")
        finally:
            one.close()
    finally:
        ks.close()
    with pytest.raises(Exception, match="closed"):
        ks.verify_batch_tensors(T(e), T(r), T(s), T(idx.astype(np.int64)))


def test_ed_and_x25519_sets_tensor_methods(lib):
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    from elliptic_b200.eddsa import EDDSA
    ed = EDDSA()
    rng = np.random.default_rng(5)
    m, n = 16, 700
    sec = rng.integers(0, 256, (m, 32), dtype=np.uint8)
    msgs, off, L = msg_block(rng, n)
    msgs = msgs[:L].copy()
    idx = rng.integers(0, m, n).astype(np.uint32)
    bidx, pos = bad_indices(idx, m)
    keep = np.ones(n, bool)
    keep[pos] = False
    with ed.signing_set([bytes(x) for x in sec]) as ss:
        sig = ss.sign_batch_packed(msgs, off, idx)
        g_sig, g_st = ss.sign_batch_tensors(T(msgs), T(off), T(idx.astype(np.int64)))
        assert_same(g_sig, sig, "signing set")
        assert (H(g_st) == nat.ST_TRUE).all()
        g = ss.sign_batch_tensors(T(msgs), T(off), bidx)
        assert (H(g[0])[keep] == sig[keep]).all() and not H(g[0])[pos].any()
        assert (H(g[1])[pos] == nat.ST_BAD_KEY_INDEX).all()
        pubs = ss.public.copy()
    pubs[2] = np.frombuffer(throwing_key(ed.key_set, [v.to_bytes(32, "little") for v in range(2, 18)]), np.uint8)
    R, S = sig[:, :32].copy(), sig[:, 32:].copy()
    S[5::19, 31] ^= 0x10
    with ed.key_set([bytes(p) for p in pubs]) as eks:
        want = eks.verify_batch_msgs_packed(R, S, msgs, off, idx)
        assert_same(eks.verify_batch_msgs_tensors(T(R), T(S), T(msgs), T(off), T(idx.astype(np.int32))), want, "ed msgs")
        h = np.frombuffer(b"".join(ed.hash_int(R[i], pubs[idx[i]], msgs[off[i]:off[i + 1]]).to_bytes(32, "little")
                                   for i in range(n)), np.uint8).reshape(n, 32)
        want = eks.verify_batch_packed(R, S, h, idx)
        assert_same(eks.verify_batch_tensors(T(R), T(S), T(h), T(idx.astype(np.int64))), want, "ed verify")
        # S >= n answers FALSE before the key's throw (eddsa/index.js order); every other item of key 2 throws
        assert {nat.ST_TRUE, nat.ST_FALSE} <= set(want.tolist())
        assert (want[idx == 2] > nat.ST_TRUE).any() and (want[idx == 2] != nat.ST_TRUE).all()
        check_keyed([eks.verify_batch_tensors(T(R), T(S), T(h), bidx)], [want[keep]], pos, "ed bad indices")
    x = EC("curve25519")
    pubx = rng.integers(0, 256, (m, 32), dtype=np.uint8)
    priv = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    priv[:, 0] &= 0x0F
    with x.key_set([p.tobytes() for p in pubx]) as xks:
        out, st = xks.derive_batch_packed(priv, idx)
        got = xks.derive_batch_tensors(T(priv), T(idx.astype(np.int64)))
        assert_same(got[0], out, "x25519 set")
        assert_same(got[1], st, "x25519 set")
        check_keyed(xks.derive_batch_tensors(T(priv), bidx), [out[keep], st[keep]], pos, "x25519 bad indices")


# ---- stream and synchronisation ----------------------------------------------------------------------------------------

def test_tensor_calls_run_on_the_callers_stream_without_synchronising(lib):
    import torch
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC
    cid, ln = 1, 32
    ec = EC("secp256k1")
    m, n = 24, 4096
    xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, m, n, seed=77)
    keys = [b"\x04" + xy[j].tobytes() if j % 2 else bytes([2 + (xy[j, -1] & 1)]) + xy[j, :ln].tobytes() for j in range(m)]
    ks = ec.key_set(keys)
    try:
        te, tr, ts, tq, ti = T(e), T(r), T(s), T(xy[idx]), T(idx.astype(np.int64))
        want_u = ec.verify_batch_packed(e, r, s, xy[idx])
        want_k = ks.verify_batch_packed(e, r, s, idx)
        ec.verify_batch_tensors(te, tr, ts, tq)                     # warm the tables and the mixed set's map
        ks.verify_batch_tensors(te, tr, ts, ti)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            torch.cuda._sleep(int(2e8))                             # about 100 ms at the H100's clocks
            got_u = ec.verify_batch_tensors(te, tr, ts, tq)
            got_k = ks.verify_batch_tensors(te, tr, ts, ti)
            assert not side.query(), "the call waited for the stream"
        side.synchronize()
        assert_same(got_u, want_u, "unkeyed on a side stream")
        assert_same(got_k, want_k, "mixed keyed on a side stream")
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = [ec.verify_batch_tensors(te, tr, ts, tq), ks.verify_batch_tensors(te, tr, ts, ti),
                   ks.mul_batch_tensors(tr, ti)[1], ks.verify_batch_tensors(te, tr, ts, ti.int())]
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        for g, w in zip(got, (want_u, want_k, None, want_k)):
            if w is not None:
                assert_same(g, w, "under sync debug mode")
    finally:
        ks.close()


def test_second_device(lib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the tensors-on-cuda:1 case needs two")
    from elliptic_b200.ec import EC
    from elliptic_b200 import _native as nat
    e, d, r, s, rec, q = signed(lib, 1, 32, N, 3)
    ec = EC("secp256k1")
    want = ec.verify_batch_packed(e, r, s, q)
    got = ec.verify_batch_tensors(T(e, "cuda:1"), T(r, "cuda:1"), T(s, "cuda:1"), T(q, "cuda:1"))
    assert got.device == torch.device("cuda:1")
    torch.cuda.synchronize(1)
    assert_same(got, want, "cuda:1")
    assert nat.ST_TRUE in want
