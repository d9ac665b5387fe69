"""The device-pointer forms of the unkeyed calls without a GPU: the range screen, the screened DER decode and a screened
EdDSA sign batch run through the host emulation on boundary cases, each compared with a small Python model (and the
model's mutants, which the cases must tell apart); the new entry points' return codes without a device, case by case;
and the one workspace size that serves every unkeyed device-pointer call on a curve."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ST_TRUE, ST_SIG_FORMAT, ST_BAD_ITEM = 1, 9, 13
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def he(tmp_path_factory):
    lib = os.path.join(str(tmp_path_factory.mktemp("hostemu")), "libunkeyed_dev_emu.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", lib,
                    os.path.join(ROOT, "tests", "hostemu", "unkeyed_dev_emu.cpp")], check=True)
    h = ctypes.CDLL(lib)
    h.he_ud_range_screen.argtypes = [ctypes.c_size_t, P, ctypes.c_uint64, P]
    h.he_ud_der_decode_screened.argtypes = [ctypes.c_size_t, ctypes.c_uint32, P, P, P, P, P, P, ctypes.c_int]
    h.he_ud_sign_screened.argtypes = [ctypes.c_size_t, P, P, ctypes.c_uint64, P, P, P, P]
    h.he_ed_sign_unkeyed.argtypes = [ctypes.c_size_t] + [P] * 5
    return h


def range_model(off, L, mut=None):
    out = []
    for i in range(len(off) - 1):
        a, b = off[i], off[i + 1]
        if mut == "end_ge":
            bad = b < a or b >= L
        elif mut == "no_decrease":
            bad = b > L
        elif mut == "start_past":
            bad = b < a or a > L
        else:
            bad = b < a or b > L
        out.append(ST_BAD_ITEM if bad else 0)
    return out


def test_range_screen_boundaries(he):
    """Empty ranges, a range equal to the whole buffer, one that ends at msgs_len and one past it, decreasing ranges, the
    last offset past the end, and offsets near 2^64."""
    L = 40
    off = [0, 0, 3, 3, L, L, 10, 9, L + 1, L + 1, 5, 20, 2**64 - 1, 7, L - 1, L]
    offs = np.array(off, np.uint64)
    vd = np.full(len(off) - 1, 0xA5, np.uint8)
    he.he_ud_range_screen(len(off) - 1, offs.ctypes.data, L, vd.ctypes.data)
    want = range_model(off, L)
    assert list(vd) == want
    B = ST_BAD_ITEM           # (40, 40) empty at the end is good; (41, 41) empty past the end is not
    assert want == [0, 0, 0, 0, 0, B, B, B, B, B, 0, B, B, 0, 0]
    for mut in ("end_ge", "no_decrease", "start_past"):
        assert list(vd) != range_model(off, L, mut), mut
    whole = np.array([0, L], np.uint64)                      # one item, the whole buffer; and one past it
    for end, v in ((L, 0), (L + 1, ST_BAD_ITEM)):
        whole[1] = end
        he.he_ud_range_screen(1, whole.ctypes.data, L, vd.ctypes.data)
        assert vd[0] == v


def der_int(v):
    b = v.to_bytes((v.bit_length() + 7) // 8 or 1, "big")
    return b"\x02" + bytes([len(b) + (b[0] >> 7)]) + (b"\0" if b[0] & 0x80 else b"") + b


def test_der_decode_screened(he):
    """A screened item reads no byte of its range (here: offsets far past the buffer), gets r = s = 0 and the status of
    a rejected encoding unless the key's status comes first; the others decode as der_decode_kernel does, with r = s = 0
    for a rejected encoding.  Mutants: screened items decoded, stale r / s kept, the key's status ignored."""
    rnd = random.Random(5)
    ln, n = 32, 24
    vals = [(rnd.getrandbits(256), rnd.getrandbits(256 - 8 * (i % 3))) for i in range(n)]
    parts = []
    for i, (r, s) in enumerate(vals):
        body = der_int(r) + der_int(s)
        p = b"\x30" + bytes([len(body)]) + body
        if i % 5 == 4:
            p = b"\x31" + p[1:]                              # rejected
        parts.append(p)
    blob = b"".join(parts)
    off = [0]
    for p in parts:
        off.append(off[-1] + len(p))
    screened = {2, 9, 15}
    soff = list(off)
    for i in sorted(screened):                               # the screen's verdict stands; the range is never read
        soff[i + 1] = 10**12 if i != 9 else soff[i + 1]
    # item 3 now starts at 10^12 too and is screened as well (its range decreases)
    screened = {i for i in range(n) if soff[i + 1] < soff[i] or soff[i + 1] > len(blob)}
    assert {2, 3, 15, 16} <= screened
    vd = np.zeros(n, np.uint8)
    he.he_ud_range_screen(n, np.array(soff, np.uint64).ctypes.data, len(blob), vd.ctypes.data)
    assert {i for i in range(n) if vd[i]} == screened
    keyst = [0] * n
    keyst[2], keyst[7] = 6, 2                                # a key that threw on a screened item and on a good one
    for pre_valid in (0, 1):
        r = np.full(n * ln, 0xA5, np.uint8)
        s = np.full(n * ln, 0xA5, np.uint8)
        pre = np.array(keyst if pre_valid else [0xEE] * n, np.uint8)
        der = np.frombuffer(blob, np.uint8).copy()
        he.he_ud_der_decode_screened(n, ln, vd.ctypes.data, der.ctypes.data, np.array(soff, np.uint64).ctypes.data,
                                     r.ctypes.data, s.ctypes.data, pre.ctypes.data, pre_valid)
        r, s = r.reshape(n, ln), s.reshape(n, ln)

        def model(mut=None):
            rows = []
            for i in range(n):
                ok = (i not in screened or mut == "read_screened") and i % 5 != 4
                k = keyst[i] if pre_valid and mut != "key_ignored" else 0
                st = k or (0 if ok else ST_SIG_FORMAT)
                rv = vals[i] if ok else (None if mut == "stale" else (0, 0))
                rows.append((st, rv))
            return rows

        got = [(int(pre[i]), None if (r[i] == 0xA5).all() else (int.from_bytes(r[i].tobytes(), "big"),
                                                                 int.from_bytes(s[i].tobytes(), "big"))) for i in range(n)]
        assert got == model()
        for mut in ("stale", "read_screened") + (("key_ignored",) if pre_valid else ()):
            assert got != model(mut), mut


def test_sign_screened_batch(he):
    """Bad ranges of every kind scattered through a batch: each gets BAD_ITEM and zeroed signature and public key; every
    other item equals a one-item signature of its own range (the items next to a bad offset included), and the batch
    with good offsets equals the unscreened body."""
    rnd = random.Random(3)
    n = 40
    sec = np.frombuffer(rnd.randbytes(32 * n), np.uint8).copy()
    msgs = [rnd.randbytes(rnd.choice([0, 5, 64, 130])) for _ in range(n)]
    msgs[0] = rnd.randbytes(7)
    off = [0]
    for mm in msgs:
        off.append(off[-1] + len(mm))
    L = off[-1]
    blob = np.frombuffer(b"".join(msgs) + b"\0" * 8, np.uint8).copy()

    def run(offs, pub=True):
        sig, pk, st = np.full(64 * n, 0xA5, np.uint8), np.full(32 * n, 0xA5, np.uint8), np.full(n, 0xA5, np.uint8)
        he.he_ud_sign_screened(n, sec.ctypes.data, blob.ctypes.data, L, np.array(offs, np.uint64).ctypes.data,
                               sig.ctypes.data, pk.ctypes.data if pub else None, st.ctypes.data)
        return sig.reshape(n, 64), pk.reshape(n, 32), st

    def one(i, a, b):
        sg, pk = np.zeros(64, np.uint8), np.zeros(32, np.uint8)
        he.he_ed_sign_unkeyed(1, sec[32 * i:].ctypes.data, blob.ctypes.data, np.array([a, b], np.uint64).ctypes.data,
                              sg.ctypes.data, pk.ctypes.data)
        return sg, pk

    ref_sig, ref_pub = np.zeros(64 * n, np.uint8), np.zeros(32 * n, np.uint8)
    he.he_ed_sign_unkeyed(n, sec.ctypes.data, blob.ctypes.data, np.array(off, np.uint64).ctypes.data, ref_sig.ctypes.data,
                          ref_pub.ctypes.data)
    sig, pk, st = run(off)
    assert (sig == ref_sig.reshape(n, 64)).all() and (pk == ref_pub.reshape(n, 32)).all() and (st == ST_TRUE).all()
    boff = list(off)
    boff[2 + 1] = boff[2] - 1                                # item 2 decreases; item 3 starts one byte earlier
    boff[20 + 1] = L + 1                                     # item 20 ends past the buffer, item 21 decreases
    boff[n] = L + 1                                          # the last offset past the end
    bad = {i for i in range(n) if boff[i + 1] < boff[i] or boff[i + 1] > L}
    assert bad == {2, 20, 21, n - 1}
    sig, pk, st = run(boff)
    for i in range(n):
        if i in bad:
            assert st[i] == ST_BAD_ITEM and not sig[i].any() and not pk[i].any(), i
        else:
            w_sig, w_pub = one(i, boff[i], boff[i + 1])
            assert st[i] == ST_TRUE and (sig[i] == w_sig).all() and (pk[i] == w_pub).all(), i
    sig2, _, st2 = run(boff, pub=False)                      # no public keys asked for
    assert (sig2 == sig).all() and (st2 == st).all()
    # mutant: a model that screens only decreasing ranges misses the items past the end
    assert bad != {i for i in range(n) if boff[i + 1] < boff[i]}


# ---- the C entry points without a device -------------------------------------------------------------------------------------

NS = [0, 1, 127, 128, (1 << 18) + 777, 1 << 20]
# eb200_dev_workspace_bytes(curve, n) for curve ids 0..9 and n in NS
DEV_WORKSPACE = {
    0: [0, 0, 0, 0, 0, 0],
    1: [0, 2304, 128256, 129024, 264499712, 1054867456],
    2: [0, 2304, 127232, 128000, 262396416, 1046478848],
    3: [0, 2816, 190464, 191488, 392805120, 1566572544],
    4: [0, 2304, 163328, 164352, 337065728, 1344274432],
    5: [0, 0, 0, 0, 0, 0],
    6: [0, 3328, 282112, 283648, 582108160, 2321547264],
    7: [0, 2304, 95744, 96256, 197191680, 786432000],
    8: [0, 2304, 125184, 125952, 258189312, 1029701632],
    9: [0, 0, 0, 0, 0, 0],
}

# (name, leading curve argument?, argument kinds after n: p = pointer, z = a size, u = a 32-bit value, o = an optional
# pointer, m = the buffer of the following length (NULL allowed when it is 0), w = workspace)
SIGS = {
    "eb200_ecdsa_sign_batch_dev": (True, "ppupppppw"),
    "eb200_ecdsa_sign_batch_k_dev": (True, "pppupppppw"),
    "eb200_ecdsa_sign_batch_pers_dev": (True, "ppmzupppppw"),
    "eb200_ec_keygen_batch_dev": (True, "pzmzpoppw"),
    "eb200_ecdsa_recover_batch_dev": (True, "ppppppw"),
    "eb200_ecdsa_recovery_param_batch_dev": (True, "ppppppw"),
    "eb200_scalar_mul_batch_dev": (True, "poppw"),
    "eb200_mul_add_batch_dev": (True, "pppppw"),
    "eb200_ecdh_derive_batch_dev": (True, "ppppw"),
    "eb200_x25519_mul_batch_dev": (False, "pppp"),
    "eb200_ecdsa_verify_batch_der_dev": (True, "pmzppupw"),
    "eb200_eddsa_verify_batch_msgs_dev": (False, "pppmzppw"),
    "eb200_eddsa_sign_batch_dev": (False, "pmzppopw"),
}
# return codes without a device (-3 ERR_ARG, -4 ERR_NOT_INIT, -5 ERR_UNSUPPORTED); nullK: NULL in argument K (counting
# from 0 with the curve and n); curve77 / ed25519: that curve id; fmt9: pub_fmt 9; big/zeroK: a size K of 2^20 + 1 / 0;
# all: every argument valid (the device check answers)
NO_DEVICE = {
    "eb200_ecdsa_sign_batch_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "null3": -3,
                                   "null5": -3, "null6": -3, "null7": -3, "null8": -3, "null9": -3, "null10": -4},
    "eb200_ecdsa_sign_batch_k_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "null3": -3,
                                     "null4": -3, "null6": -3, "null7": -3, "null8": -3, "null9": -3, "null10": -3,
                                     "null11": -4},
    "eb200_ecdsa_sign_batch_pers_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "null3": -3,
                                        "null4": -3, "null4_len0": -4, "big5": -3, "zero5": -4, "huge5": -3,
                                        "null7": -3, "null8": -3, "null9": -3, "null10": -3, "null11": -3,
                                        "null12": -4},
    "eb200_ec_keygen_batch_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "big3": -3,
                                  "zero3": -3, "huge3": -3, "null4": -3, "null4_len0": -4, "big5": -3, "zero5": -4,
                                  "huge5": -3, "null6": -3, "null7": -4, "null8": -3, "null9": -3, "null10": -4},
    "eb200_ecdsa_recover_batch_dev": {"all": -4, "curve77": -5, "ed25519": -5, "n0": -4, "null2": -3, "null3": -3,
                                      "null4": -3, "null5": -3, "null6": -3, "null7": -3, "null8": -3},
    "eb200_ecdsa_recovery_param_batch_dev": {"all": -4, "curve77": -5, "ed25519": -5, "n0": -4, "null2": -3,
                                             "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3,
                                             "null8": -3},
    "eb200_scalar_mul_batch_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "null3": -4,
                                   "null4": -3, "null5": -3, "null6": -3},
    "eb200_mul_add_batch_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "null3": -3,
                                "null4": -3, "null5": -3, "null6": -3, "null7": -3},
    "eb200_ecdh_derive_batch_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "null3": -3,
                                    "null4": -3, "null5": -3, "null6": -3},
    "eb200_x25519_mul_batch_dev": {"all": -4, "n0": -4, "null1": -3, "null2": -3, "null3": -3, "null4": -3},
    "eb200_ecdsa_verify_batch_der_dev": {"all": -4, "curve77": -5, "ed25519": -4, "n0": -4, "null2": -3, "null3": -3,
                                         "null3_len0": -4, "big4": -4, "zero4": -4, "huge4": -4, "null5": -3,
                                         "null6": -3, "fmt9": -5, "null8": -3, "null9": -3},
    "eb200_eddsa_verify_batch_msgs_dev": {"all": -4, "n0": -4, "null1": -3, "null2": -3, "null3": -3, "null4": -3,
                                          "null4_len0": -4, "big5": -4, "zero5": -4, "huge5": -4, "null6": -3,
                                          "null7": -3, "null8": -3},
    "eb200_eddsa_sign_batch_dev": {"all": -4, "n0": -4, "null1": -3, "null2": -3, "null2_len0": -4, "big3": -4,
                                   "zero3": -4, "huge3": -4, "null4": -3, "null5": -3, "null6": -4, "null7": -3,
                                   "null8": -3},
}


def cases(name):
    """(case, arguments) of `name` with host pointers standing for device buffers."""
    lead, kinds = SIGS[name]
    buf = np.zeros(1 << 12, np.uint8)
    p = buf.ctypes.data
    base = ([1] if lead else []) + [4]
    for k in kinds:
        base.append({"p": p, "o": p, "m": p, "w": p, "z": 16, "u": 0}[k])
    if name == "eb200_ec_keygen_batch_dev":
        base[2 + 1] = 32                                      # entropy_len
    out = [("all", list(base))]
    if lead:
        out.append(("curve77", [77] + base[1:]))
        out.append(("ed25519", [4] + base[1:]))
    a = list(base)
    a[1 if lead else 0] = 0
    out.append(("n0", a))
    for j, k in enumerate(kinds):
        pos = j + (2 if lead else 1)
        if k in "pomw":
            a = list(base)
            a[pos] = None
            out.append(("null%d" % pos, a))
        if k == "m":
            a = list(base)
            a[pos] = None
            a[pos + 1] = 0
            out.append(("null%d_len0" % pos, a))
        if k == "z":
            for tag, v in (("big", (1 << 20) + 1), ("zero", 0), ("huge", 1 << 40)):
                a = list(base)
                a[pos] = v
                out.append(("%s%d" % (tag, pos), a))
        if k == "u" and name == "eb200_ecdsa_verify_batch_der_dev":
            a = list(base)
            a[pos] = 9
            out.append(("fmt9", a))
    return buf, out


@pytest.fixture(scope="module")
def nodev():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from elliptic_b200 import _native, build
    build.build()
    lib = _native.load()
    assert lib.eb200_device_count() == 0
    return lib


def test_return_codes_without_device(nodev):
    got = {}
    for name in SIGS:
        buf, cs = cases(name)
        fn = getattr(nodev, name)
        got[name] = {case: fn(*args, None) for case, args in cs}
    assert got == NO_DEVICE


def test_dev_workspace_bytes(nodev):
    """One size per curve and n, pinned; never below the verify workspace nor, on ed25519, the EdDSA verify workspace."""
    lib = nodev
    got = {c: [lib.eb200_dev_workspace_bytes(c, n) for n in NS] for c in range(10)}
    assert got == DEV_WORKSPACE
    for c in range(10):
        for n in NS:
            w = lib.eb200_dev_workspace_bytes(c, n)
            assert w >= lib.eb200_ecdsa_verify_workspace_bytes(c, n)
            if c == 4:
                assert w >= lib.eb200_eddsa_verify_workspace_bytes(n)
    assert all(v == 0 for c in (0, 5, 9) for v in got[c])
