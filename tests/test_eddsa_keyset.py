"""EdDSA key sets without a GPU: the build and keyed-verify bodies run through the host emulation against the oracle's
EDDSA.verify and the unkeyed body, the table geometry against the oracle's point arithmetic, the automatic width choice,
the C entry points' return codes without a device, and EdKeySet's argument checks."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import ed_ks_items as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_hostemu(root, out_dir):
    lib = os.path.join(out_dir, "libed_keyset_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", lib,
                    os.path.join(root, "tests", "hostemu", "ed_keyset_emu.cpp")], check=True)
    he = ctypes.CDLL(lib)
    he.he_ed_keyset_key_bytes.restype = ctypes.c_size_t
    he.he_ed_keyset_choose_bits.argtypes = [ctypes.c_size_t, ctypes.c_size_t]
    he.he_ed_keyset_verify.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 8
    he.he_ed_unkeyed_verify.argtypes = [ctypes.c_size_t] + [ctypes.c_void_p] * 5
    he.he_ed_keyset_table.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return he


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    return build_hostemu(ROOT, str(tmp_path_factory.mktemp("hostemu")))


_CASES = {}


def cases():
    """Keys, items and the oracle's answers: all 1024 sign.input vectors (valid and forged) and the adversarial keys."""
    if not _CASES:
        from oracle.ref_py.eddsa import EDDSA
        ed = EDDSA()
        keys, items = K.cases(ed)
        _CASES.update(ed=ed, keys=keys, items=items, want=K.answers(ed, keys, items))
    return _CASES


def run_keyed(he, W, keys, items, msgs=False):
    """Statuses of the keyed pipeline: from h, or (msgs) from the items' raw messages."""
    A, R, S, h, idx = K.pack(keys, items)
    kst = np.zeros(len(keys), np.uint8)
    if msgs:
        sel, blob, off = K.msg_items(items)
        R, S, idx = R[sel].copy(), S[sel].copy(), idx[sel].copy()
        st = np.zeros(len(sel), np.uint8)
        he.he_ed_keyset_verify(W, len(keys), A.ctypes.data, len(sel), R.ctypes.data, S.ctypes.data, None, blob.ctypes.data,
                               off.ctypes.data, idx.ctypes.data, kst.ctypes.data, st.ctypes.data)
    else:
        st = np.zeros(len(items), np.uint8)
        he.he_ed_keyset_verify(W, len(keys), A.ctypes.data, len(items), R.ctypes.data, S.ctypes.data, h.ctypes.data, None,
                               None, idx.ctypes.data, kst.ctypes.data, st.ctypes.data)
    return [int(v) for v in kst], [int(v) for v in st]


@pytest.mark.parametrize("W", [4, 5, 6, 7, 8])
def test_bodies_against_oracle(he, W):
    """Mutation checks (test_oracle_comparison_catches_a_broken_body): dropping a digit's sign, hashing a re-encoded key,
    or reading the key's verdict before R's decode each make this comparison fail."""
    c = cases()
    keys, items, want = c["keys"], c["items"], c["want"]
    kst, got = run_keyed(he, W, keys, items)
    assert kst == [K.expected(c["ed"], c["ed"].encode_point(c["ed"].g), K.le(1), A, 0) or 1 for A in keys]
    assert got == want, [i for i in range(len(items)) if got[i] != want[i]]
    sel = K.msg_items(items)[0]
    assert run_keyed(he, W, keys, items, msgs=True)[1] == [want[i] for i in sel]
    assert {0, 1, 2, 5} <= set(want) and sum(want) > len(want) // 3


def test_unkeyed_body_gives_the_same_bytes(he):
    c = cases()
    keys, items = c["keys"], c["items"]
    A, R, S, h, idx = K.pack(keys, items)
    Ai = A[idx].copy()
    st = np.zeros(len(items), np.uint8)
    he.he_ed_unkeyed_verify(len(items), R.ctypes.data, S.ctypes.data, Ai.ctypes.data, h.ctypes.data, st.ctypes.data)
    assert [int(v) for v in st] == c["want"]


@pytest.mark.parametrize("W", [4, 5, 6, 7, 8])
def test_table_geometry(he, W):
    """Entry (j, i) of a key's table is (i + 1) 2^(W j) (-A) as (y + x, y - x, 2 d x y), for a key with torsion."""
    from oracle.ref_py.eddsa import EDDSA
    ed = EDDSA()
    p = K.P
    d = -121665 * pow(121666, -1, p) % p
    A = ed.encode_point(ed.g.mul(0xC0FFEE).add(ed.decode_point(bytes.fromhex(K.ORDER8))))
    nw, E = K.windows(W), 1 << (W - 1)
    assert he.he_ed_keyset_windows(W) == nw and he.he_ed_keyset_key_bytes(W) == nw * E * 96
    out = np.zeros(nw * E * 24, np.uint32)
    he.he_ed_keyset_table(W, np.frombuffer(A, np.uint8).copy().ctypes.data, out.ctypes.data)
    val = lambda w: sum(int(v) << (32 * k) for k, v in enumerate(w))
    negA = ed.decode_point(A).neg()
    for j, i in {(0, 0), (0, E - 1), (1, 1), (nw // 2, E // 2), (nw - 1, 0), (nw - 1, E - 1)}:
        Pt = negA.mul((i + 1) << (W * j))
        x, y = Pt.get_x(), Pt.get_y()
        ent = out[(j * E + i) * 24:(j * E + i + 1) * 24]
        assert (val(ent[:8]), val(ent[8:16]), val(ent[16:])) == ((y + x) % p, (y - x) % p, 2 * d * x * y % p), (j, i)


def test_top_digit_fits_the_table():
    """h = n - 1, recoded low to high with a carry: the unsigned top digit stays <= 2^(W-1) at every width."""
    for W in range(4, 9):
        Kw, half, h, carry = K.windows(W), 1 << (W - 1), K.N - 1, 0
        for j in range(Kw):
            c = ((h >> (W * j)) & ((1 << W) - 1)) + carry
            carry = int(j < Kw - 1 and c >= half)
        assert c <= half, W


MUTATIONS = {
    "digit sign": ("acc = ed_add_niels(acc, ed_niels_neg_if(q, neg));", "acc = ed_add_niels(acc, q);"),
    "re-encoded key": ("const uint8_t* a = A + 32 * (size_t)key_idx[i];",
                       "uint8_t re[32]; { f25 x, y; ed_decode(A + 32 * (size_t)key_idx[i], &x, &y); ed_ext e = ed_identity(); "
                       "e.x = x; e.y = y; ed_encode(e, re); } const uint8_t* a = re;"),
    "verdict first": ("  uint8_t st = ed_decode(Rb + 32 * i, &rx, &ry);                  // sig.R()\n  if (st) return st;\n"
                      "  const u32 k = key_idx[i];\n  st = kst[k];                                                    // key.pub()\n"
                      "  if (st != 1) return st;\n",
                      "  const u32 k = key_idx[i];\n  uint8_t st = kst[k];\n  if (st != 1) return st;\n"
                      "  st = ed_decode(Rb + 32 * i, &rx, &ry);\n  if (st) return st;\n"),
}


@pytest.mark.parametrize("kind", sorted(MUTATIONS))
def test_oracle_comparison_catches_a_broken_body(tmp_path, kind):
    root = str(tmp_path)
    shutil.copytree(os.path.join(ROOT, "elliptic_b200", "csrc"), os.path.join(root, "elliptic_b200", "csrc"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(root, "include"))
    shutil.copytree(os.path.join(ROOT, "tests", "hostemu"), os.path.join(root, "tests", "hostemu"))
    path = os.path.join(root, "elliptic_b200", "csrc", "ed25519_keyset_body.cuh")
    old, new = MUTATIONS[kind]
    src = open(path).read()
    assert src.count(old) == 1, old
    open(path, "w").write(src.replace(old, new))
    bad = build_hostemu(root, root)
    c = cases()
    keys, items, want = c["keys"], c["items"], c["want"]
    if kind == "re-encoded key":
        sel = K.msg_items(items)[0]
        assert run_keyed(bad, 7, keys, items, msgs=True)[1] != [want[i] for i in sel]
    else:
        assert run_keyed(bad, 7, keys, items)[1] != want


def test_width_chooser(he):
    """The widest W in 4..8 whose m tables fit 1 GiB; 0 (the entry point then answers ERR_ARG) when W = 4 does not."""
    G = 1 << 30
    for m, W in ((1, 8), (64, 8), (2730, 8), (2731, 7), (4096, 7), (4723, 7), (4724, 6), (1 << 14, 4), (1 << 16, 0)):
        assert he.he_ed_keyset_choose_bits(m, G) == W, m
    assert [he.he_ed_keyset_key_bytes(W) for W in range(4, 9)] == [49152, 78336, 132096, 227328, 393216]


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
    create = lambda *a: lib.eb200_eddsa_keyset_create(*a, ctypes.byref(out))
    assert create(4, p, 0, p) == _native.ERR_NOT_INIT and out.value is None
    assert create(4, None, 0, p) == _native.ERR_ARG and create(4, p, 0, None) == _native.ERR_ARG
    assert lib.eb200_eddsa_keyset_create(4, p, 0, p, None) == _native.ERR_ARG
    assert create(0, p, 0, p) == _native.ERR_ARG and create(1 << 32, p, 0, p) == _native.ERR_ARG
    assert create(4, p, 3, p) == _native.ERR_ARG and create(4, p, 9, p) == _native.ERR_ARG
    assert create(1 << 16, p, 0, p) == _native.ERR_ARG                  # no width fits the default budget
    assert create(1 << 16, p, 4, p) == _native.ERR_NOT_INIT             # an explicit width is not held to it
    assert lib.eb200_eddsa_verify_batch_keyed(None, 4, p, p, p, p, p) == _native.ERR_ARG
    assert lib.eb200_eddsa_verify_batch_keyed_msgs(None, 4, p, p, p, p, p, p) == _native.ERR_ARG
    # the ECDSA entry point still answers as before, and an EdDSA handle never reaches it without a device
    assert lib.eb200_keyset_create(4, 4, p, 0, 0, p, ctypes.byref(out)) == _native.ERR_UNSUPPORTED


def test_ed_key_set_argument_errors():
    from elliptic_b200.ec import EllipticError
    from elliptic_b200.eddsa import EDDSA, EdKeySet
    with pytest.raises(EllipticError):
        EDDSA().key_set(["00" * 31])                                    # key length, before any device is needed
    ks = EdKeySet.__new__(EdKeySet)                                      # a set as built, without its native handle
    ks._ed, ks.status, ks._sets, ks._A = EDDSA(), np.ones(3, np.uint8), [], np.zeros((3, 32), np.uint8)
    z = np.zeros((2, 32), np.uint8)
    with pytest.raises(ValueError):
        ks.verify_batch_packed(z, np.zeros((2, 31), np.uint8), z, [0, 1])
    with pytest.raises(ValueError):
        ks.verify_batch_packed(z, z, np.zeros((1, 32), np.uint8), [0, 1])
    with pytest.raises(ValueError):
        ks.verify_batch_packed(z, z, z, [0, 3])
    with pytest.raises(ValueError):
        ks.verify_batch_packed(z, z, z, [0])
    with pytest.raises(ValueError):
        ks.verify_batch_msgs_packed(z, z, np.zeros(4, np.uint8), np.array([0, 1, 2], np.uint64), [0, 1])
    with pytest.raises(ValueError):
        ks.verify_batch(["", ""], ["00" * 64, "00" * 64], [0])
    with pytest.raises(EllipticError):
        ks.verify_batch([""], ["00" * 63], [0])                         # Signature has invalid size
    with pytest.raises(EllipticError):
        ks.verify_batch_packed(z, z, z, [0, 1])                          # closed
