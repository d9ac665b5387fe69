"""Signed items over a key set, made on the GPU by the library's own sign and mul calls (test and benchmark helper)."""
import numpy as np


def gpu_items(lib, nat, cid, ln, m, n, seed, corrupt_every=64):
    """m keys and n signatures (key of item i: key_idx[i]); one item in corrupt_every gets a damaged e.
    Returns (keys_xy (m, 2 ln), e, r, s (n, ln), key_idx (n,) uint32)."""
    rng = np.random.default_rng(seed)
    d = rng.integers(0, 256, size=(m, ln), dtype=np.uint8)
    e = rng.integers(0, 256, size=(n, ln), dtype=np.uint8)
    d[:, 0] &= 0x7F if ln != 66 else 0
    e[:, 0] &= 0x7F if ln != 66 else 0
    d[:, -1] |= 1
    idx = rng.integers(0, m, size=n).astype(np.uint32)
    di = np.ascontiguousarray(d[idx])
    r, s = np.zeros((n, ln), np.uint8), np.zeros((n, ln), np.uint8)
    rec, st = np.zeros(n, np.uint8), np.zeros(max(n, m), np.uint8)
    nat.call(lib.eb200_ecdsa_sign_batch, cid, n, e, di, 0, r, s, rec, st)
    xy = np.zeros((m, 2 * ln), np.uint8)
    nat.call(lib.eb200_scalar_mul_batch, cid, m, d, None, xy, st)
    assert (st[:m] == nat.ST_TRUE).all()
    e[::corrupt_every, -1] ^= 1
    return xy, e, r, s, idx
