"""EdDSA signing sets without a GPU: the create, nonce, normalise and challenge bodies run through the host emulation
against the reference's sign.input vectors, the oracle's EDDSA.sign and the unkeyed body; the batched normalisation
against the per-item encoder; the C entry points' return codes without a device, and EdSigningSet's argument checks."""
import ctypes
import gzip
import json
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2**255 - 19


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostemu")), "libed_signset_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", lib,
                    os.path.join(ROOT, "tests", "hostemu", "ed_signset_emu.cpp")], check=True)
    he = ctypes.CDLL(lib)
    he.he_ed_signset_create.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 3
    he.he_ed_signset_sign.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 4
    he.he_ed_sign_unkeyed.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 5
    he.he_ed_signset_normalise.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 5
    return he


def blob(msgs):
    off = np.zeros(len(msgs) + 1, np.uint64)
    off[1:] = np.cumsum([len(m) for m in msgs])
    return np.frombuffer(b"".join(msgs) + b"\x00", np.uint8).copy(), off


def keyed(he, secrets, msgs, idx):
    """(signatures, public keys) of the keyed pipeline: create over `secrets`, item i signed by key idx[i]."""
    m = len(secrets)
    sec = np.frombuffer(b"".join(secrets), np.uint8).copy()
    keys, pub = np.zeros(16 * m, np.uint32), np.zeros((m, 32), np.uint8)
    he.he_ed_signset_create(m, sec.ctypes.data, keys.ctypes.data, pub.ctypes.data)
    b, off = blob(msgs)
    idx = np.ascontiguousarray(idx, np.uint32)
    sig = np.zeros((len(msgs), 64), np.uint8)
    he.he_ed_signset_sign(keys.ctypes.data, pub.ctypes.data, len(msgs), b.ctypes.data, off.ctypes.data, idx.ctypes.data,
                          sig.ctypes.data)
    return sig, pub


def unkeyed(he, secrets, msgs):
    n = len(msgs)
    sec = np.frombuffer(b"".join(secrets), np.uint8).copy()
    b, off = blob(msgs)
    sig, pub = np.zeros((n, 64), np.uint8), np.zeros((n, 32), np.uint8)
    he.he_ed_sign_unkeyed(n, sec.ctypes.data, b.ctypes.data, off.ctypes.data, sig.ctypes.data, pub.ctypes.data)
    return sig, pub


def test_sign_input_vectors(he):
    """All 1024 sign.input lines, the set built over their secrets in a shuffled order: signatures and public keys equal
    the vectors, the unkeyed body and the oracle's EDDSA.sign."""
    from oracle.ref_py.eddsa import EDDSA
    vecs = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "ed25519_sign_input.json.gz"), "rt"))["vectors"]
    assert len(vecs) == 1024
    perm = list(range(1024))
    random.Random(5).shuffle(perm)
    secrets = [bytes.fromhex(vecs[j]["secret"]) for j in perm]
    where = {j: k for k, j in enumerate(perm)}
    msgs = [bytes.fromhex(v["msg"]) for v in vecs]
    sig, pub = keyed(he, secrets, msgs, [where[i] for i in range(1024)])
    assert [sig[i].tobytes().hex() for i in range(1024)] == [v["sig"] for v in vecs]
    assert [pub[where[i]].tobytes().hex() for i in range(1024)] == [v["pk"] for v in vecs]
    usig, upub = unkeyed(he, [bytes.fromhex(v["secret"]) for v in vecs], msgs)
    assert (usig == sig).all() and all(upub[i].tobytes() == pub[where[i]].tobytes() for i in range(1024))
    ed = EDDSA()
    assert all(ed.sign(msgs[i], bytes.fromhex(vecs[i]["secret"])) == sig[i].tobytes() for i in range(1024))


def test_every_message_length_matches_the_unkeyed_body(he):
    """8 keys signing messages of every length 0..300 (SHA-512 padding edges at 47/48 and 79/80 bytes), keys in a
    scattered order: byte for byte what ed25519_sign_item gives for the key's secret."""
    rnd = random.Random(11)
    secrets = [bytes(rnd.randrange(256) for _ in range(32)) for _ in range(8)]
    msgs = [bytes(rnd.randrange(256) for _ in range(L)) for L in range(301)]
    idx = [rnd.randrange(8) for _ in msgs]
    sig, _ = keyed(he, secrets, msgs, idx)
    usig, _ = unkeyed(he, [secrets[k] for k in idx], msgs)
    bad = [i for i in range(len(msgs)) if sig[i].tobytes() != usig[i].tobytes()]
    assert not bad, bad[:8]


def test_normalise_body_equals_per_item_encoding(he):
    """Batches with n < B and n mod B != 0, holding the identity (0 : 1 : 1), a scaled identity and points with Z != 1:
    the batched body writes exactly the bytes the per-item ed_encode writes, and both are the oracle's encodePoint."""
    from oracle.ref_py.eddsa import EDDSA
    ed = EDDSA()
    B = he.he_ed_signset_batch()
    assert B == 16
    rnd = random.Random(7)
    words = lambda v: [(v >> (32 * q)) & 0xFFFFFFFF for q in range(8)]
    for n in (1, 3, B - 1, B, B + 1, 2 * B + 5, 5 * B - 3):
        pts, want = [], []
        for i in range(n):
            pt = ed.g.mul(rnd.randrange(1, 2**252)) if i % 5 else ed.g.mul(0)      # every 5th: the identity
            lam = rnd.randrange(2, P) if i % 3 else 1                              # every 3rd: Z = 1
            pts.append((pt.get_x() * lam % P, pt.get_y() * lam % P, lam))
            want.append(ed.encode_point(pt))
        X, Y, Z = (np.array([words(p[c]) for p in pts], np.uint32).reshape(-1) for c in range(3))
        batched, single = np.zeros((n, 64), np.uint8), np.zeros((n, 32), np.uint8)
        he.he_ed_signset_normalise(n, X.ctypes.data, Y.ctypes.data, Z.ctypes.data, batched.ctypes.data, single.ctypes.data)
        assert (batched[:, :32] == single).all(), n
        assert [single[i].tobytes() for i in range(n)] == want, n
    assert pts[0] == (0, 1, 1)


def test_return_codes_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    buf = np.zeros(1 << 12, np.uint8)
    p = buf.ctypes.data
    out = ctypes.c_void_p(1)
    create = lambda *a: lib.eb200_eddsa_signing_set_create(*a, ctypes.byref(out))
    assert create(4, p, p) == _native.ERR_NOT_INIT and out.value is None
    assert create(4, p, None) == _native.ERR_NOT_INIT                     # out_pub is optional
    assert create(4, None, p) == _native.ERR_ARG
    assert lib.eb200_eddsa_signing_set_create(4, p, p, None) == _native.ERR_ARG
    assert create(0, p, p) == _native.ERR_ARG and create(1 << 32, p, p) == _native.ERR_ARG
    assert lib.eb200_eddsa_sign_batch_keyed(None, 4, p, p, p, p, p) == _native.ERR_ARG
    assert lib.eb200_eddsa_sign_batch_keyed(None, 0, None, None, None, None, None) == _native.ERR_ARG


def test_signing_set_argument_errors():
    from elliptic_b200.ec import EllipticError
    from elliptic_b200.eddsa import EDDSA, EdSigningSet
    with pytest.raises(EllipticError):
        EDDSA().signing_set(["00" * 31])                                # secret length, before any device is needed
    with pytest.raises(EllipticError):
        EDDSA().signing_set([list(range(33))])
    ss = EdSigningSet.__new__(EdSigningSet)                              # a set as built, without its native handle
    ss._ed, ss._sets, ss.public = EDDSA(), [], np.zeros((3, 32), np.uint8)
    assert not hasattr(ss, "_secrets")
    msgs, off = np.zeros(4, np.uint8), np.array([0, 1, 4], np.uint64)
    with pytest.raises(ValueError):
        ss.sign_batch_packed(msgs, off, [0, 3])                         # key_idx >= m
    with pytest.raises(ValueError):
        ss.sign_batch_packed(msgs, off, [0, -1])
    with pytest.raises(ValueError):
        ss.sign_batch_packed(msgs, off, [0])                            # n + 1 offsets
    with pytest.raises(ValueError):
        ss.sign_batch_packed(msgs, np.array([0, 1, 3], np.uint64), [0, 1])   # the last offset is len(msgs)
    with pytest.raises(ValueError):
        ss.sign_batch_packed(msgs, off, [[0, 1]])
    with pytest.raises(ValueError):
        ss.sign_batch(["", "00"], [0])
    with pytest.raises(EllipticError):
        ss.sign_batch_packed(msgs, off, [0, 1])                         # closed
    assert ss.sign_batch_packed(np.zeros(0, np.uint8), np.zeros(1, np.uint64), []).shape == (0, 64)
