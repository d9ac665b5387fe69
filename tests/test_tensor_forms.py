"""The tensor forms and the keyed DER device-pointer call without a GPU: the screened keyed DER decode through the host
emulation against a Python model of its precedence (whose mutants the cases must tell apart), the C entry point's
return codes without a device, and the tensor methods' argument checks, which refuse before any launch."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ST_FALSE, ST_TRUE, ST_THROW_INVALID_POINT, ST_THROW_POINT_FORMAT = 0, 1, 2, 6
ST_THROW_SIG_FORMAT, ST_BAD_KEY_INDEX, ST_BAD_ITEM = 9, 12, 13
P = ctypes.c_void_p
LEN = 32
KST = [ST_TRUE, ST_THROW_INVALID_POINT, ST_FALSE, ST_THROW_POINT_FORMAT]     # the set's key verdicts, m = 4
M = len(KST)
INDICES = [0, 1, 2, 3, M, (1 << 32) - 1]


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostemu")), "libkeyset_der_dev_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", lib,
                    os.path.join(ROOT, "tests", "hostemu", "keyset_der_dev_emu.cpp")], check=True)
    h = ctypes.CDLL(lib)
    h.he_ks_der_screened.argtypes = [ctypes.c_size_t, ctypes.c_uint32, P, ctypes.c_size_t, P, ctypes.c_uint64] + [P] * 6
    h.he_ks_der_plain.argtypes = [ctypes.c_size_t, ctypes.c_uint32] + [P] * 7
    return h


def der(r, s):
    return bytes([0x30, 4 + len(r) + len(s), 2, len(r)]) + r + bytes([2, len(s)]) + s


GOOD = der(bytes([0x11] * LEN), bytes([0x22] * LEN))
ENCODINGS = [GOOD, der(b"\x00\x7f", b"\x05"), b"\x31\x00", b"", der(bytes([0x80] * LEN), b"\x01")]


def cases():
    """Items of every index beside every kind of range: each encoding in place, a decreasing range, one ending at
    der_len, one ending one past it, and one wholly past it.  The bytes past der_len hold GOOD, so a body that read a
    range there would decode r, s != 0; spacer items make each range exactly the one intended."""
    blob, idx, off = bytearray(), [], [0]
    spans = []
    for i in INDICES:
        for enc in ENCODINGS:
            spans.append((i, len(blob), len(blob) + len(enc)))
            blob += enc
        spans.append((i, len(blob) + 5, len(blob) + 1))                # decreasing
    der_len = len(blob)
    spans.append((0, der_len - 1, der_len))                              # ends exactly at der_len
    for i in INDICES:
        spans.append((i, der_len - 3, der_len + 1))                      # one past the end
        spans.append((i, der_len, der_len + len(GOOD)))                  # wholly past it, over GOOD
    for i, a, b in spans:
        if off[-1] != a:
            idx.append(0)                                                # spacer item
            off.append(a)
        idx.append(i)
        off.append(b)
    buf = bytes(blob) + GOOD + bytes(64)
    return np.array(idx, np.uint32), np.array(off, np.uint64), np.frombuffer(buf, np.uint8).copy(), der_len


def run(he, fn_screened, idx, off, buf, der_len):
    n = len(idx)
    kst = np.array(KST, np.uint8)
    r, s = np.full(n * LEN, 0xA5, np.uint8), np.full(n * LEN, 0xA5, np.uint8)
    vd, idx_out = np.full(n, 0xA5, np.uint8), np.full(n, 0xA5A5A5A5, np.uint32)
    if fn_screened:
        he.he_ks_der_screened(n, LEN, idx.ctypes.data, M, buf.ctypes.data, der_len, off.ctypes.data, kst.ctypes.data,
                              idx_out.ctypes.data, r.ctypes.data, s.ctypes.data, vd.ctypes.data)
    else:
        he.he_ks_der_plain(n, LEN, buf.ctypes.data, off.ctypes.data, idx.ctypes.data, kst.ctypes.data, r.ctypes.data,
                           s.ctypes.data, vd.ctypes.data)
    return list(vd), r.reshape(n, LEN), s.reshape(n, LEN), list(idx_out)


def model(idx, a, b, der_len, der_ok, mut=None):
    """The verdict of one item: BAD_KEY_INDEX, BAD_ITEM, the key's import throw, THROW_SIG_FORMAT, else 0 (the keyed verify
    decides).  Mutants: item_first (BAD_ITEM before BAD_KEY_INDEX), throw_first (the key's throw before BAD_ITEM),
    sig_first (THROW_SIG_FORMAT before the key's throw), end_ge (a range ending at der_len is refused)."""
    bad_idx = idx >= M
    bad_range = b < a or (b >= der_len if mut == "end_ge" else b > der_len)
    throw = 0 if bad_idx or KST[idx] <= ST_TRUE else KST[idx]
    sig = 0 if der_ok else ST_THROW_SIG_FORMAT
    order = {None: [ST_BAD_KEY_INDEX, ST_BAD_ITEM, "throw", "sig"], "end_ge": [ST_BAD_KEY_INDEX, ST_BAD_ITEM, "throw", "sig"],
             "item_first": [ST_BAD_ITEM, ST_BAD_KEY_INDEX, "throw", "sig"],
             "throw_first": [ST_BAD_KEY_INDEX, "throw", ST_BAD_ITEM, "sig"],
             "sig_first": [ST_BAD_KEY_INDEX, ST_BAD_ITEM, "sig", "throw"]}[mut]
    for step in order:
        v = {ST_BAD_KEY_INDEX: ST_BAD_KEY_INDEX if bad_idx else 0, ST_BAD_ITEM: ST_BAD_ITEM if bad_range else 0,
             "throw": throw, "sig": sig}[step]
        if v:
            return v
    return 0


def test_screened_keyed_der_decode_precedence(he):
    """Against the model, with the decode itself taken from the unscreened body on a one-item view: every unscreened item
    gets exactly the host form's r, s and verdict; every screened item its screen verdict, r = s = 0 and index 0, and
    none of its range read (the screened ranges over GOOD would decode to r, s != 0).  Each mutant disagrees."""
    idx, off, buf, der_len = cases()
    n = len(idx)
    vd, r, s, idx_out = run(he, True, idx, off, buf, der_len)
    ok_idx = np.zeros(1, np.uint32)

    def alone(i, key):
        """The unscreened keyed DER decode of item i alone, with key `key`."""
        return run(he, False, np.array([key], np.uint32), off[i:i + 2].copy(), buf, der_len)

    der_ok, decoded = [], []
    for i in range(n):
        a, b = int(off[i]), int(off[i + 1])
        if b < a:
            der_ok.append(False)
            decoded.append(None)
            continue
        v1, r1, s1, _ = alone(i, int(ok_idx[0]))                        # key 0 is TRUE: the verdict is the encoding's
        der_ok.append(v1[0] == 0)
        decoded.append((r1[0], s1[0]))
    want = [model(int(idx[i]), int(off[i]), int(off[i + 1]), der_len, der_ok[i]) for i in range(n)]
    assert vd == want
    for i in range(n):
        a, b = int(off[i]), int(off[i + 1])
        screened = int(idx[i]) >= M or b < a or b > der_len
        if screened:
            assert not r[i].any() and not s[i].any() and idx_out[i] == 0, i
        else:
            v1, r1, s1, _ = alone(i, int(idx[i]))
            assert vd[i] == v1[0] and (r[i] == r1[0]).all() and (s[i] == s1[0]).all() and idx_out[i] == idx[i], i
    for v in (ST_BAD_KEY_INDEX, ST_BAD_ITEM, ST_THROW_INVALID_POINT, ST_THROW_POINT_FORMAT, ST_THROW_SIG_FORMAT, 0):
        assert v in want, v
    for mut in ("item_first", "throw_first", "sig_first", "end_ge"):
        assert vd != [model(int(idx[i]), int(off[i]), int(off[i + 1]), der_len, der_ok[i], mut) for i in range(n)], mut
    # a body that decoded screened ranges: some screened item over GOOD would have r, s != 0
    read = [i for i in range(n) if want[i] in (ST_BAD_KEY_INDEX, ST_BAD_ITEM) and decoded[i] is not None
            and decoded[i][0].any()]
    assert read and all(not r[i].any() for i in read)


def test_keyed_der_dev_return_codes_without_device():
    """No device: a NULL set is ERR_ARG for n = 0 and n = 4, with NULL in each pointer argument in turn."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    p = np.zeros(1 << 12, np.uint8).ctypes.data
    fn = lib.eb200_ecdsa_verify_batch_keyed_der_dev
    # (ks, n, d_e, d_sigs, sigs_len, d_sig_off, d_key_idx, d_status, d_workspace, stream)
    for n in (0, 4):
        for null in (None, 2, 3, 5, 6, 7, 8, 9):
            args = [None, n, p, p, 64, p, p, p, p, None]
            if null is not None:
                args[null] = None
            assert fn(*args) == _native.ERR_ARG, (n, null)
        assert fn(None, n, p, None, 0, p, p, p, p, None) == _native.ERR_ARG


def test_import_does_not_import_torch():
    code = "import sys, elliptic_b200, elliptic_b200.ec, elliptic_b200.eddsa; assert 'torch' not in sys.modules"
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)


def _closed(cls, **attrs):
    obj = cls.__new__(cls)
    obj._sets = []
    for k, v in attrs.items():
        setattr(obj, k, v)
    return obj


def test_tensor_argument_checks_without_device():
    """A CPU tensor, a wrong dtype, a wrong shape, a non-contiguous view, mismatched n and a closed set each raise before
    anything reaches the library (a launch without a device would raise NativeError instead)."""
    import torch
    from elliptic_b200.ec import EC, EllipticError, KeySet, X25519KeySet
    from elliptic_b200.eddsa import EDDSA, EdKeySet, EdSigningSet
    ec = EC("secp256k1")
    u8 = lambda *shape: torch.zeros(shape, dtype=torch.uint8)                               # noqa: E731
    e = u8(4, 32)
    cases = [
        (lambda: ec.verify_batch_tensors(e, e, e, u8(4, 64)), "CUDA"),                       # CPU tensors
        (lambda: ec.verify_batch_tensors(e.int(), e, e, u8(4, 64)), "uint8"),                # dtype
        (lambda: ec.verify_batch_tensors(u8(4, 31), e, e, u8(4, 64)), "(n, 32)"),            # shape
        (lambda: ec.verify_batch_tensors(e, u8(32, 4).t(), e, u8(4, 64)), "contiguous"),     # non-contiguous view
        (lambda: ec.verify_batch_tensors(e, u8(5, 32), e, u8(4, 64)), "n = 4"),              # mismatched n
        (lambda: ec.verify_batch_tensors(e, e, e, u8(4, 65), 2), "(n, 33)"),                 # shape of the format
        (lambda: ec.verify_batch_der_tensors(e, u8(10), torch.zeros(4, dtype=torch.int64), u8(4, 64)), "(n + 1,)"),
        (lambda: ec.verify_batch_der_tensors(e, u8(10), torch.zeros(5, dtype=torch.int32), u8(4, 64)), "int64"),
        (lambda: ec.sign_batch_tensors(e, e, k=u8(3, 32)), "n = 4"),
        (lambda: ec.mul_batch_tensors(e, u8(4, 32)), "(n, 64)"),
        (lambda: EC("curve25519").x_mul_batch_tensors(e, u8(4, 32).t().contiguous().t()), "contiguous"),
        (lambda: EDDSA().sign_batch_tensors(e, u8(2, 5), torch.zeros(5, dtype=torch.int64)), "1-D"),
        (lambda: EDDSA().verify_batch_tensors(e, e, e, [0] * 4), "torch.Tensor"),
    ]
    ks = KeySet.__new__(KeySet)
    ks._sets, ks.status, ks._ec = [object()], np.zeros(3, np.uint8), ec
    idx = torch.zeros(4, dtype=torch.int64)
    cases += [
        (lambda: ks.verify_batch_tensors(e, e, e, idx.to(torch.int16)), "int32"),
        (lambda: ks.verify_batch_tensors(e, e, e, torch.zeros(3, dtype=torch.int64)), "n = 4"),
        (lambda: ks.mul_batch_tensors(e, idx), "CUDA"),
    ]
    for i, (call, msg) in enumerate(cases):
        with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)").replace("+", r"\+")):
            call()
    closed = [
        lambda: _closed(KeySet, status=np.zeros(3, np.uint8), _ec=ec).verify_batch_der_tensors(e, u8(1), idx, idx),
        lambda: _closed(KeySet, status=np.zeros(3, np.uint8), _ec=ec).recovery_param_batch_tensors(e, e, e, idx),
        lambda: _closed(EdKeySet, status=np.zeros(3, np.uint8)).verify_batch_msgs_tensors(e, e, u8(1), idx, idx),
        lambda: _closed(EdSigningSet, public=np.zeros((3, 32), np.uint8)).sign_batch_tensors(u8(1), idx, idx),
        lambda: _closed(X25519KeySet, status=np.zeros(3, np.uint8)).derive_batch_tensors(e, idx),
    ]
    for call in closed:
        with pytest.raises(EllipticError, match="closed"):
            call()
