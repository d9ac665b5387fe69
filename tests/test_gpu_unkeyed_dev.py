"""The device-pointer forms of the unkeyed calls on the GPU: each must write exactly what its host form writes, outputs and
statuses, on every curve the host form takes, at sizes that end inside the normalisation and inversion batches; on a
non-default stream whose own copies wrote the inputs, with guard regions behind every buffer and a workspace whose stale
contents do not matter; plus BAD_ITEM for bad ranges, asynchrony, secret clearing and the return codes."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GUARD = 512
SIZES = [1, 127, (1 << 17) + 3]
SHORT = [("secp256k1", 1, 32), ("p256", 2, 32), ("p384", 3, 48), ("p521", 6, 66), ("p192", 7, 24), ("p224", 8, 28)]
ALL = SHORT + [("ed25519", 4, 32)]


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native as nat
    return nat.init(0)


class Out:
    """An output buffer of `nbytes` for dev()."""
    def __init__(self, nbytes):
        self.nbytes = nbytes


def dev(lib, fn, lead, args, wsb, fill=0xA5, stream=None):
    """fn(*lead, *args, [workspace,] stream) on a non-default stream: numpy arrays are copied to the device by copies
    enqueued on that stream just before, Out(b) becomes a b-byte device buffer, None stays NULL, ints pass as 64-bit
    values.  wsb: workspace bytes (None: the call takes no workspace), prefilled with `fill`.  Every buffer is followed
    by a guard that must stay unchanged.  Returns the outputs (numpy) and the workspace."""
    import torch
    from elliptic_b200 import _native as nat
    st = stream or torch.cuda.Stream()
    bufs, outs, cargs = [], [], []
    with torch.cuda.stream(st):
        ws = torch.full(((wsb or 0) + GUARD,), fill, dtype=torch.uint8, device="cuda")
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
                cargs.append(a)
        tail = [ctypes.c_void_p(ws.data_ptr())] if wsb is not None else []
        nat.check(fn(*lead, *cargs, *tail, ctypes.c_void_p(st.cuda_stream)))
    st.synchronize()
    for t, nb in bufs + outs + [(ws, wsb or 0)]:
        assert (t[nb:].cpu().numpy() == (fill if t is ws else 0x5A)).all(), "guard overwritten"
    return [t[:nb].cpu().numpy() for t, nb in outs], ws[:wsb or 0].cpu().numpy()


def host(fn, *args):
    from elliptic_b200 import _native as nat
    nat.call(fn, *args)


def same(lib, hf, df, lead, ins, outs, wsb, host_ins=None):
    """The host form into fresh outputs, the device form twice (workspace prefilled 0xA5, then 0x00): equal byte for byte.
    outs: output byte counts (None = a NULL output).  Returns the host outputs and the last workspace."""
    want = [np.zeros(b, np.uint8) if b is not None else None for b in outs]
    host(hf, *lead, *(host_ins if host_ins is not None else ins), *want)
    got = None
    for fill in (0xA5, 0x00):
        got, ws = dev(lib, df, lead, list(ins) + [Out(b) if b is not None else None for b in outs], wsb, fill)
        wn = [w for w in want if w is not None]
        for g, w in zip(got, wn):
            assert (g == w).all(), (df.__name__, fill, np.nonzero(g != w)[0][:8])
    return want, ws


def rnd_rows(rng, n, ln, top=None):
    a = rng.integers(0, 256, (n, ln), dtype=np.uint8)
    if ln == 66:
        a[:, 0] &= 1
    elif top is not None:
        a[:, 0] &= top
    return a


def signed(lib, cid, ln, n, seed):
    """n signatures by the library's host sign (e, priv, r, s, recid) and the signers' public points."""
    rng = np.random.default_rng(seed)
    e, d = rnd_rows(rng, n, ln, 0x7F), rnd_rows(rng, n, ln, 0x7F)
    d[:, -1] |= 1
    r, s, rec, st = np.zeros((n, ln), np.uint8), np.zeros((n, ln), np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    host(lib.eb200_ecdsa_sign_batch, cid, n, e, d, 0, r, s, rec, st)
    q = np.zeros((n, 2 * ln), np.uint8)
    host(lib.eb200_scalar_mul_batch, cid, n, d, None, q, st)
    return e, d, r, s, rec, q


def der(r, s):
    """DER of fixed-width big-endian rows r, s: concatenated bytes and n + 1 offsets."""
    def integer(b):
        b = b.lstrip(b"\0") or b"\0"
        if b[0] & 0x80:
            b = b"\0" + b
        return b"\x02" + bytes([len(b)]) + b

    parts = []
    for ri, si in zip(r, s):
        body = integer(ri.tobytes()) + integer(si.tobytes())
        ln = bytes([len(body)]) if len(body) < 128 else b"\x81" + bytes([len(body)])
        parts.append(b"\x30" + ln + body)
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in parts])
    return np.frombuffer(b"".join(parts) + b"\0" * 8, np.uint8).copy(), off


def msg_block(rng, n, maxlen=200):
    lens = rng.integers(0, maxlen, n)
    lens[::7] = 0
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    L = int(off[n])
    return rng.integers(0, 256, L + 64, dtype=np.uint8), off, L        # 64 spare bytes past msgs_len


# ---- each call against its host form -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("name,cid,ln", ALL)
def test_sign_and_keygen_equal_host_forms(lib, name, cid, ln, n):
    rng = np.random.default_rng(cid * 7 + n)
    wsb = lib.eb200_dev_workspace_bytes(cid, n)
    e, d = rnd_rows(rng, n, ln, 0x7F), rnd_rows(rng, n, ln, 0x7F)
    k = rnd_rows(rng, n, ln, 0x7F)
    k[::5] = 0                                                      # k outside [2, n - 2]: RETRY
    k[1::11] = 0xFF
    pers = rng.integers(0, 256, 40, dtype=np.uint8)
    outs = [n * ln, n * ln, n, n]
    want, _ = same(lib, lib.eb200_ecdsa_sign_batch, lib.eb200_ecdsa_sign_batch_dev, (cid, n), [e, d, 1], outs, wsb)
    assert (want[3] == 1).all()
    # sign with k: an item the reference retries (status 10) gets no r, s, recid (the host form's bytes there are its
    # staging buffer's), so those are compared where the status is TRUE
    want = [np.zeros(b, np.uint8) for b in outs]
    host(lib.eb200_ecdsa_sign_batch_k, cid, n, e, d, k, 0, *want)
    ok = want[3] == 1
    for fill in (0xA5, 0x00):
        (gr, gs, gid, gst), _ = dev(lib, lib.eb200_ecdsa_sign_batch_k_dev, (cid, n), [e, d, k, 0] + [Out(b) for b in outs], wsb,
                                    fill)
        assert (gst == want[3]).all()
        assert (gr.reshape(n, ln)[ok] == want[0].reshape(n, ln)[ok]).all() and (gid[ok] == want[2][ok]).all()
        assert (gs.reshape(n, ln)[ok] == want[1].reshape(n, ln)[ok]).all()
    if n > 1:
        assert 10 in want[3] and 1 in want[3]
    same(lib, lib.eb200_ecdsa_sign_batch_pers, lib.eb200_ecdsa_sign_batch_pers_dev, (cid, n), [e, d, pers, 40, 0], outs, wsb)
    same(lib, lib.eb200_ecdsa_sign_batch_pers, lib.eb200_ecdsa_sign_batch_pers_dev, (cid, n), [e, d, None, 0, 0], outs, wsb)
    ent = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    same(lib, lib.eb200_ec_keygen_batch, lib.eb200_ec_keygen_batch_dev, (cid, n), [ent, 32, pers, 10], [n * ln, 2 * n * ln, n],
         wsb)
    same(lib, lib.eb200_ec_keygen_batch, lib.eb200_ec_keygen_batch_dev, (cid, n), [ent, 32, None, 0], [n * ln, None, n], wsb)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("name,cid,ln", SHORT)
def test_recover_and_recovery_param_equal_host_forms(lib, name, cid, ln, n):
    from elliptic_b200 import _native as nat
    e, d, r, s, rec, q = signed(lib, cid, ln, n, cid + n)
    wsb = lib.eb200_dev_workspace_bytes(cid, n)
    r2, s2, rec2, q2 = r.copy(), s.copy(), rec.copy(), q.copy()
    r2[3::17] = 0                                                   # r = 0: infinity
    s2[5::13] = 0                                                   # s = 0 (mod n): the cold kernel
    rec2[::3] ^= 2                                                  # r + n candidates: often THROW_SECOND_KEY / invalid point
    q2[7::19, -1] ^= 1                                              # off-curve Q: THROW_NO_RECOVERY
    want, _ = same(lib, lib.eb200_ecdsa_recover_batch, lib.eb200_ecdsa_recover_batch_dev, (cid, n), [e, r2, s2, rec2],
                   [2 * n * ln, n], wsb)
    if n == SIZES[-1]:
        assert nat.ST_TRUE in want[1] and len(set(want[1].tolist())) > 1
    want, _ = same(lib, lib.eb200_ecdsa_recovery_param_batch, lib.eb200_ecdsa_recovery_param_batch_dev, (cid, n),
                   [e, r2, s2, q2], [n, n], wsb)
    if n == SIZES[-1]:
        assert {nat.ST_TRUE, nat.ST_THROW_NO_RECOVERY} <= set(want[1].tolist())


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("name,cid,ln", ALL)
def test_mul_mul_add_derive_equal_host_forms(lib, name, cid, ln, n):
    rng = np.random.default_rng(cid * 3 + n)
    wsb = lib.eb200_dev_workspace_bytes(cid, n)
    k1, k2 = rnd_rows(rng, n, ln), rnd_rows(rng, n, ln)
    k2[::29] = 0                                                    # k = 0: INFINITY
    st = np.zeros(n, np.uint8)
    pts = np.zeros((n, 2 * ln), np.uint8)
    host(lib.eb200_scalar_mul_batch, cid, n, rnd_rows(rng, n, ln, 0x7F), None, pts, st)
    pts[2::9, -1] ^= 1                                              # off-curve points: replayed (NEEDS_HOST on ed25519)
    same(lib, lib.eb200_scalar_mul_batch, lib.eb200_scalar_mul_batch_dev, (cid, n), [k2, None], [2 * n * ln, n], wsb)
    same(lib, lib.eb200_scalar_mul_batch, lib.eb200_scalar_mul_batch_dev, (cid, n), [k2, pts], [2 * n * ln, n], wsb)
    same(lib, lib.eb200_mul_add_batch, lib.eb200_mul_add_batch_dev, (cid, n), [k1, k2, pts], [2 * n * ln, n], wsb)
    _, ws = same(lib, lib.eb200_ecdh_derive_batch, lib.eb200_ecdh_derive_batch_dev, (cid, n), [k2, pts], [n * ln, n], wsb)
    assert not ws.any(), "derive left scalar-derived words in the workspace"


@pytest.mark.parametrize("n", SIZES[1:])
def test_torsion_and_twist_cases_equal_host_forms(lib, n):
    """ed25519 points with every torsion component and scalars at the edges of n and 8n (mul, mulAdd, derive), and
    curve25519 u of small and mixed order, non-canonical and on the twist (Point.mul), tiled to n items."""
    import torsion_cases as tc
    cases = tc.mul_cases()
    reps = -(-n // len(cases))
    cs = (cases * reps)[:n]
    pts = np.frombuffer(b"".join(tc.be([pt[0], pt[1]]) for _, pt, _ in cs), np.uint8).reshape(n, 64).copy()
    k = np.frombuffer(tc.be([kk for _, _, kk in cs]), np.uint8).reshape(n, 32).copy()
    k1 = np.ascontiguousarray(k[::-1])
    cid = 4
    wsb = lib.eb200_dev_workspace_bytes(cid, n)
    same(lib, lib.eb200_scalar_mul_batch, lib.eb200_scalar_mul_batch_dev, (cid, n), [k, pts], [64 * n, n], wsb)
    same(lib, lib.eb200_mul_add_batch, lib.eb200_mul_add_batch_dev, (cid, n), [k1, k, pts], [64 * n, n], wsb)
    same(lib, lib.eb200_ecdh_derive_batch, lib.eb200_ecdh_derive_batch_dev, (cid, n), [k, pts], [32 * n, n], wsb)
    us = [u for _, u in tc.x25519_us()]
    ks = tc.scalars()
    xc = [(u, kk) for u in us for kk in ks]
    xc = (xc * -(-n // len(xc)))[:n]
    px = np.frombuffer(tc.be([u for u, _ in xc]), np.uint8).reshape(n, 32).copy()
    kx = np.frombuffer(tc.be([kk for _, kk in xc]), np.uint8).reshape(n, 32).copy()
    same(lib, lib.eb200_x25519_mul_batch, lib.eb200_x25519_mul_batch_dev, (n,), [kx, px], [32 * n, n], None)


@pytest.mark.parametrize("n", SIZES)
def test_x25519_mul_equals_host_form(lib, n):
    rng = np.random.default_rng(n)
    k, px = rng.integers(0, 256, (n, 32), dtype=np.uint8), rng.integers(0, 256, (n, 32), dtype=np.uint8)
    k[::13] = 0
    same(lib, lib.eb200_x25519_mul_batch, lib.eb200_x25519_mul_batch_dev, (n,), [k, px], [n * 32, n], None)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("name,cid,ln", ALL)
def test_der_verify_equals_host_form(lib, name, cid, ln, n):
    from elliptic_b200 import _native as nat
    e, d, r, s, rec, q = signed(lib, cid, ln, n, cid * 5 + n)
    e[1::9, -1] ^= 1                                                # FALSE
    q[4::31, -1] ^= 1                                               # off-curve keys: replayed / NEEDS_HOST
    sigs, off = der(r, s)
    L = int(off[n])
    sigs[off[6::15].astype(np.int64)] = 0x31                        # rejected encodings
    wsb = lib.eb200_dev_workspace_bytes(cid, n)
    assert wsb >= lib.eb200_ecdsa_verify_workspace_bytes(cid, n)
    sec1 = np.concatenate([np.full((n, 1), 4, np.uint8), q], axis=1)
    sec1[8::37, 0] = 5                                              # a key that throws
    for pub, fmt in ((q, nat.PUB_XY), (sec1, nat.PUB_SEC1_65)):
        want = np.zeros(n, np.uint8)
        host(lib.eb200_ecdsa_verify_batch_der, cid, n, e, sigs, off, pub, fmt, want)
        for fill in (0xA5, 0):
            (got,), _ = dev(lib, lib.eb200_ecdsa_verify_batch_der_dev, (cid, n),
                            [e, sigs, ctypes.c_uint64(L), off, pub, ctypes.c_uint32(fmt), Out(n)], wsb, fill)
            assert (got == want).all(), (fmt, np.nonzero(got != want)[0][:8])
        if n == SIZES[-1]:
            assert {nat.ST_TRUE, nat.ST_FALSE, nat.ST_THROW_SIG_FORMAT} <= set(want.tolist())
    if n < 16:
        return
    # bad ranges: a decreasing pair and the last offset past the end; BAD_ITEM over a key's throw
    boff = off.copy()
    boff[n] = L + 1
    boff[11] = boff[10] - 1 if boff[10] > 0 else boff[11]
    (got,), _ = dev(lib, lib.eb200_ecdsa_verify_batch_der_dev, (cid, n),
                    [e, sigs, ctypes.c_uint64(L), boff, sec1, ctypes.c_uint32(nat.PUB_SEC1_65), Out(n)], wsb)
    for i in range(n):
        a, b = int(boff[i]), int(boff[i + 1])
        if b < a or b > L:
            assert got[i] == nat.ST_BAD_ITEM, i
        elif a == off[i] and b == off[i + 1]:
            assert got[i] == want[i], i


@pytest.mark.parametrize("n", SIZES)
def test_eddsa_sign_and_verify_equal_host_forms(lib, n):
    from elliptic_b200 import _native as nat
    rng = np.random.default_rng(40 + n)
    wsb = lib.eb200_dev_workspace_bytes(nat.CURVE_ED25519, n)
    assert wsb >= lib.eb200_eddsa_verify_workspace_bytes(n)
    sec = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    msgs, off, L = msg_block(rng, n)
    want, _ = same(lib, lib.eb200_eddsa_sign_batch, lib.eb200_eddsa_sign_batch_dev, (n,),
                   [sec, msgs, ctypes.c_uint64(L), off], [64 * n, 32 * n, n], wsb, host_ins=[sec, msgs, off])
    sig, pub = want[0].reshape(n, 64), want[1].reshape(n, 32)
    same(lib, lib.eb200_eddsa_sign_batch, lib.eb200_eddsa_sign_batch_dev, (n,), [sec, msgs, ctypes.c_uint64(L), off],
         [64 * n, None, n], wsb, host_ins=[sec, msgs, off])
    R, S, A = sig[:, :32].copy(), sig[:, 32:].copy(), pub.copy()
    R[3::17] = 0xFF                                                 # R that does not decode
    S[5::19, 31] ^= 0x10                                            # S >= n or a wrong S
    m2 = msgs.copy()
    m2[: L: 53] ^= 1                                                # FALSE for the items that held those bytes
    want, _ = same(lib, lib.eb200_eddsa_verify_batch_msgs, lib.eb200_eddsa_verify_batch_msgs_dev, (n,),
                   [R, S, A, m2, ctypes.c_uint64(L), off], [n], wsb, host_ins=[R, S, A, m2, off])
    if n == SIZES[-1]:
        assert {nat.ST_TRUE, nat.ST_FALSE} <= set(want[0].tolist())
    z = np.zeros(n + 1, np.uint64)                                  # every message empty, NULL buffer
    same(lib, lib.eb200_eddsa_verify_batch_msgs, lib.eb200_eddsa_verify_batch_msgs_dev, (n,), [R, S, A, None, 0, z], [n],
         wsb, host_ins=[R, S, A, None, z])


def test_bad_ranges_eddsa(lib):
    """Every kind of bad range gets BAD_ITEM and zeroed outputs; the other items are the host form's."""
    from elliptic_b200 import _native as nat
    n = 4096
    rng = np.random.default_rng(77)
    wsb = lib.eb200_dev_workspace_bytes(nat.CURVE_ED25519, n)
    sec = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    msgs, off, L = msg_block(rng, n, 120)
    sig, pub, st = np.zeros(64 * n, np.uint8), np.zeros(32 * n, np.uint8), np.zeros(n, np.uint8)
    host(lib.eb200_eddsa_sign_batch, n, sec, msgs, off, sig, pub, st)
    boff = off.copy()
    boff[n] = L + 1                                                 # the last item ends one past msgs_len
    dec = int(np.argmax((np.diff(off)[100:] > 0))) + 100
    boff[dec + 1] = boff[dec] - 1                                   # decreasing
    boff[2001] = L + 1000                                           # items 2000 and 2001: past the end, then decreasing
    (gs, gp, gst), _ = dev(lib, lib.eb200_eddsa_sign_batch_dev, (n,),
                           [sec, msgs, ctypes.c_uint64(L), boff, Out(64 * n), Out(32 * n), Out(n)], wsb)
    gs, gp, sig, pub = gs.reshape(n, 64), gp.reshape(n, 32), sig.reshape(n, 64), pub.reshape(n, 32)
    bad = np.array([int(boff[i + 1]) < int(boff[i]) or int(boff[i + 1]) > L for i in range(n)])
    assert bad[[n - 1, dec, 2000, 2001]].all() and bad.sum() == 4
    assert (gst[bad] == nat.ST_BAD_ITEM).all() and not gs[bad].any() and not gp[bad].any()
    intact = ~bad & (boff[:-1] == off[:-1]) & (boff[1:] == off[1:])
    assert (gst[intact] == nat.ST_TRUE).all() and (gs[intact] == sig[intact]).all() and (gp[intact] == pub[intact]).all()
    R, S = np.ascontiguousarray(sig[:, :32]), np.ascontiguousarray(sig[:, 32:])
    want = np.zeros(n, np.uint8)
    host(lib.eb200_eddsa_verify_batch_msgs, n, R, S, pub, msgs, off, want)
    (got,), _ = dev(lib, lib.eb200_eddsa_verify_batch_msgs_dev, (n,), [R, S, pub, msgs, ctypes.c_uint64(L), boff, Out(n)], wsb)
    assert (got[bad] == nat.ST_BAD_ITEM).all() and (got[intact] == want[intact]).all() and (want == nat.ST_TRUE).all()


# ---- asynchrony, secrets, return codes ---------------------------------------------------------------------------------------

def test_calls_are_asynchronous(lib):
    """After a warm-up, a call queued behind a sleep on the caller's stream returns before its work has run."""
    import torch
    from elliptic_b200 import _native as nat
    n, cid, ln = 1 << 12, 2, 32
    rng = np.random.default_rng(1)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        e, d = (torch.from_numpy(rnd_rows(rng, n, ln, 0x7F)).cuda() for _ in range(2))
        r, s, rec, sts = (torch.zeros(x, dtype=torch.uint8, device="cuda") for x in (n * ln, n * ln, n, n))
        ws = torch.zeros(lib.eb200_dev_workspace_bytes(cid, n), dtype=torch.uint8, device="cuda")
    args = [cid, n, e.data_ptr(), d.data_ptr(), 0, r.data_ptr(), s.data_ptr(), rec.data_ptr(), sts.data_ptr(), ws.data_ptr(),
            st.cuda_stream]
    nat.check(lib.eb200_ecdsa_sign_batch_dev(*args))                # warm-up (table build)
    st.synchronize()
    want = r.cpu().numpy().copy()
    r.zero_()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        torch.cuda._sleep(200_000_000)
        nat.check(lib.eb200_ecdsa_sign_batch_dev(*args))
        ev = torch.cuda.Event()
        ev.record(st)
    assert not ev.query(), "the call waited for its work"
    st.synchronize()
    assert (r.cpu().numpy() == want).all()
    tm = nat.last_timing()
    assert tm["launches"] == 3 and tm["kernel_ms"] >= tm["main_kernel_ms"] > 0


def windows(rows):
    """Every 16-byte window of every row, big- and little-endian, and of its 32-bit limbs in little-endian word order."""
    out = set()
    for row in rows:
        b = row.tobytes()
        pad = b"\0" * ((-len(b)) % 4) + b
        limbs = b"".join(pad[i:i + 4][::-1] for i in range(len(pad) - 4, -1, -4))
        for v in (b, b[::-1], limbs):
            for j in range(len(v) - 15):
                w = v[j:j + 16]
                if w.count(0) < 12:
                    out.add(w)
    return out


def leaks(ws, secrets):
    wb = ws.tobytes()
    return [w for w in windows(secrets) if w in wb]


@pytest.mark.parametrize("n", [1, 300])
@pytest.mark.parametrize("name,cid,ln", [("secp256k1", 1, 32), ("p384", 3, 48), ("ed25519", 4, 32)])
def test_secret_bearing_calls_clear_the_workspace(lib, name, cid, ln, n):
    """No 16-byte window of a private key, secret or caller nonce stays in the workspace.  The kernels keep per-item
    words item-interleaved, so at n = 1 an item's words are contiguous and a leak shows as a window."""
    rng = np.random.default_rng(cid + 100 + n)
    wsb = lib.eb200_dev_workspace_bytes(cid, n)
    e, d, k = (rnd_rows(rng, n, ln, 0x7F) for _ in range(3))
    outs = [Out(n * ln), Out(n * ln), Out(n), Out(n)]
    _, ws = dev(lib, lib.eb200_ecdsa_sign_batch_dev, (cid, n), [e, d, 0] + outs, wsb)
    assert not leaks(ws, d)
    _, ws = dev(lib, lib.eb200_ecdsa_sign_batch_k_dev, (cid, n), [e, d, k, 0] + outs, wsb)
    assert not leaks(ws, np.concatenate([d, k]))
    ent = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    (priv, _), ws = dev(lib, lib.eb200_ec_keygen_batch_dev, (cid, n), [ent, 32, None, 0, Out(n * ln), None, Out(n)], wsb)
    assert not leaks(ws, priv.reshape(n, ln))
    pts = np.zeros((n, 2 * ln), np.uint8)
    host(lib.eb200_scalar_mul_batch, cid, n, rnd_rows(rng, n, ln, 0x7F), None, pts, np.zeros(n, np.uint8))
    _, ws = dev(lib, lib.eb200_ecdh_derive_batch_dev, (cid, n), [d, pts, Out(n * ln), Out(n)], wsb)
    assert not leaks(ws, d)
    if cid == 4:
        msgs, off, L = msg_block(rng, n)
        sec = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        _, ws = dev(lib, lib.eb200_eddsa_sign_batch_dev, (n,),
                    [sec, msgs, ctypes.c_uint64(L), off, Out(64 * n), Out(32 * n), Out(n)], wsb)
        assert not leaks(ws, sec)


def calls(lib):
    """(function, leading ints, pointer-argument count before the workspace, index of d_status among them, takes a
    workspace, positions of size arguments among them)"""
    return [(lib.eb200_ecdsa_sign_batch_dev, 1, 7, 6, True, (2,)),
            (lib.eb200_ecdsa_sign_batch_k_dev, 1, 8, 7, True, (3,)),
            (lib.eb200_ecdsa_sign_batch_pers_dev, 1, 9, 8, True, (3, 4)),
            (lib.eb200_ec_keygen_batch_dev, 1, 7, 6, True, (1, 3)),
            (lib.eb200_ecdsa_recover_batch_dev, 1, 6, 5, True, ()),
            (lib.eb200_ecdsa_recovery_param_batch_dev, 1, 6, 5, True, ()),
            (lib.eb200_scalar_mul_batch_dev, 1, 4, 3, True, ()),
            (lib.eb200_mul_add_batch_dev, 1, 5, 4, True, ()),
            (lib.eb200_ecdh_derive_batch_dev, 1, 4, 3, True, ()),
            (lib.eb200_x25519_mul_batch_dev, 0, 4, 3, False, ()),
            (lib.eb200_ecdsa_verify_batch_der_dev, 1, 7, 6, True, (2, 5)),
            (lib.eb200_eddsa_verify_batch_msgs_dev, 0, 7, 6, True, (4,)),
            (lib.eb200_eddsa_sign_batch_dev, 0, 7, 6, True, (2,))]


def test_return_codes_on_the_device(lib):
    """d_status in host memory or on a device eb200_init did not set up: ERR_NOT_INIT; with a second device initialised,
    each device serves its own pointers."""
    import torch
    from elliptic_b200 import _native as nat
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    dp = buf.data_ptr()
    host_mem = np.zeros(1 << 12, np.uint8)
    def args_for(ptr, status_ptr, na, si, szs, fn):
        a = [(32 if fn is lib.eb200_ec_keygen_batch_dev and j == 1 else 0) if j in szs else ptr for j in range(na)]
        if fn is lib.eb200_ecdsa_verify_batch_der_dev:
            a[5] = nat.PUB_XY
        a[si] = status_ptr
        return a

    for fn, lead, na, si, has_ws, szs in calls(lib):
        pre = [1] if lead else []
        a = args_for(dp, host_mem.ctypes.data, na, si, szs, fn)
        assert fn(*pre, 8, *a, *([dp] if has_ws else []), None) == nat.ERR_NOT_INIT, fn.__name__
    torch.cuda.synchronize()
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the second-device case needs two")
    with torch.cuda.device(1):
        b1 = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda:1")
    d1 = b1.data_ptr()
    if lib.eb200_device_count() == 1:
        for fn, lead, na, si, has_ws, szs in calls(lib):
            pre = [1] if lead else []
            a = args_for(d1, d1, na, si, szs, fn)
            assert fn(*pre, 8, *a, *([d1] if has_ws else []), None) == nat.ERR_NOT_INIT, fn.__name__
    nat.init_devices([0, 1])
    n, ln = 64, 32
    rng = np.random.default_rng(9)
    with torch.cuda.device(1):
        k = torch.from_numpy(rnd_rows(rng, n, ln, 0x7F)).to("cuda:1")
        out, st = torch.zeros(2 * n * ln, dtype=torch.uint8, device="cuda:1"), torch.zeros(n, dtype=torch.uint8, device="cuda:1")
        ws = torch.zeros(lib.eb200_dev_workspace_bytes(1, n), dtype=torch.uint8, device="cuda:1")
        s1 = torch.cuda.Stream(device=1)
        nat.check(lib.eb200_scalar_mul_batch_dev(1, n, k.data_ptr(), None, out.data_ptr(), st.data_ptr(), ws.data_ptr(),
                                                 s1.cuda_stream))
        s1.synchronize()
    want, wst = np.zeros(2 * n * ln, np.uint8), np.zeros(n, np.uint8)
    host(lib.eb200_scalar_mul_batch, 1, n, k.cpu().numpy(), None, want, wst)
    assert (out.cpu().numpy() == want).all() and (st.cpu().numpy() == wst).all()
