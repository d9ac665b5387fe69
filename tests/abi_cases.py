"""Argument and launch-count cases of the C ABI, shared by test_capi_contract.py (no device) and
test_gpu_properties.py (device initialised).  Each case is a name and a call; the tests compare what the calls
return (and, on the GPU, eb200_timing.launches) with literal tables."""
import ctypes

import numpy as np

# Argument kinds of every entry point, in header order.  c: curve id, n: item count, p: pointer, f: public-key
# format, u: flags, o: selftest op, z: a byte length or word count, d: eb200_short_curve descriptor, k: key set.
SIGNATURES = {
    "eb200_ecdsa_verify_batch": "cnppppfp",
    "eb200_ecdsa_verify_batch_der": "cnppppfp",
    "eb200_ecdsa_verify_batch_dev": "cnppppfppp",
    "eb200_ecdsa_sign_batch": "cnppupppp",
    "eb200_ecdsa_sign_batch_k": "cnpppupppp",
    "eb200_ecdsa_sign_batch_pers": "cnpppzupppp",
    "eb200_ec_keygen_batch": "cnpzpzppp",
    "eb200_ecdsa_recover_batch": "cnpppppp",
    "eb200_ecdsa_recovery_param_batch": "cnpppppp",
    "eb200_scalar_mul_batch": "cnpppp",
    "eb200_ecdh_derive_batch": "cnpppp",
    "eb200_mul_add_batch": "cnppppp",
    "eb200_eddsa_verify_batch": "nppppp",
    "eb200_eddsa_verify_batch_msgs": "npppppp",
    "eb200_eddsa_verify_batch_dev": "nppppppp",
    "eb200_eddsa_sign_batch": "npppppp",
    "eb200_x25519_derive_batch": "npppp",
    "eb200_x25519_derive_batch_dev": "nppppp",
    "eb200_x25519_mul_batch": "npppp",
    "eb200_curve_mul_batch": "dnpzppp",
    "eb200_curve_mul_add_batch": "dnppppzpp",
    "eb200_curve_add_batch": "dnpppp",
    "eb200_curve_dbl_batch": "dnppp",
    "eb200_curve_validate_batch": "dnpp",
    "eb200_ecdsa_verify_batch_keyed": "knppppp",
    "eb200_ecdsa_verify_batch_keyed_der": "knppppp",
    "eb200_ecdsa_verify_batch_keyed_dev": "knppppppp",
    "eb200_scalar_mul_batch_keyed": "knpppp",
    "eb200_mul_add_batch_keyed": "knppppp",
    "eb200_ecdh_derive_batch_keyed": "knpppp",
    "eb200_ecdsa_recovery_param_batch_keyed": "knpppppp",
    "eb200_eddsa_verify_batch_keyed": "knppppp",
    "eb200_eddsa_verify_batch_keyed_msgs": "knpppppp",
    "eb200_eddsa_sign_batch_keyed": "knppppp",
    "eb200_x25519_derive_batch_keyed": "knpppp",
    "eb200_ecdsa_verify_batch_keyed_der_dev": "knppzppppp",
    "eb200_scalar_mul_batch_keyed_dev": "knpppppp",
    "eb200_mul_add_batch_keyed_dev": "knppppppp",
    "eb200_ecdh_derive_batch_keyed_dev": "knpppppp",
    "eb200_ecdsa_recovery_param_batch_keyed_dev": "knpppppppp",
    "eb200_eddsa_verify_batch_keyed_dev": "knppppppp",
    "eb200_eddsa_verify_batch_keyed_msgs_dev": "knpppzppppp",
    "eb200_eddsa_sign_batch_keyed_dev": "knpzpppppp",
    "eb200_x25519_derive_batch_keyed_dev": "knpppppp",
    "eb200_selftest_fe": "conppp",
    "eb200_selftest_gtab": "cpz",
    "eb200_selftest_gtab_dims": "cppp",
    "eb200_last_timing": "p",
}
# the self-test hooks copy from their host pointers without checking them: no NULL cases with a device
HOOKS = ("eb200_selftest_fe", "eb200_selftest_gtab")


def set_kind(name):
    """The kind of key set a keyed entry point takes: ecdsa, ed (EdDSA public keys), sign (EdDSA secrets) or x25519."""
    return "sign" if "eddsa_sign" in name else "ed" if "eddsa" in name else "x25519" if "x25519" in name else "ecdsa"


WRONG_KIND = {"ecdsa": "ed", "ed": "sign", "sign": "ed", "x25519": "ecdsa"}


def small_sets(lib, curve=1, m=4):
    """One set of each kind, m keys each: ECDSA (on `curve`, secp256k1 or p256), EdDSA, signing, curve25519.  The
    EdDSA and curve25519 keys are random bytes (their import verdicts do not matter here)."""
    from elliptic_b200 import _native as nat
    rnd = np.random.default_rng(5)
    d = rnd.integers(1, 255, size=(m, 32), dtype=np.uint8)
    xy, st = np.zeros((m, 64), np.uint8), np.zeros(m, np.uint8)
    nat.call(lib.eb200_scalar_mul_batch, curve, m, d, None, xy, st)
    out = {}
    for kind, make in (("ecdsa", lambda h: lib.eb200_keyset_create(curve, m, xy.ctypes.data, 0, 4, st.ctypes.data, h)),
                       ("ed", lambda h: lib.eb200_eddsa_keyset_create(m, d.ctypes.data, 4, st.ctypes.data, h)),
                       ("sign", lambda h: lib.eb200_eddsa_signing_set_create(m, d.ctypes.data, None, h)),
                       ("x25519", lambda h: lib.eb200_x25519_keyset_create(m, d.ctypes.data, 4, st.ctypes.data, h))):
        h = ctypes.c_void_p()
        nat.check(make(ctypes.byref(h)))
        out[kind] = h
    return out


def argument_cases(with_device):
    """(case id, call) for every entry point: n == 0, a NULL in each pointer argument, an unknown curve, an unknown
    public-key format, a NULL descriptor and, with a device, a NULL key set and one of the wrong kind.  Every other
    argument is valid: 4 items, secp256k1, {x, y} keys, a set of the entry point's kind (a NULL set without a device)
    and pointers into one zeroed host buffer (so device-pointer calls find no owning device; zeros are valid key
    indices, h, scalars and offsets)."""
    from elliptic_b200 import _native as nat
    buf = np.zeros(1 << 16, np.uint8)
    ptr = buf.ctypes.data
    desc = nat.ShortCurveDesc(32, ptr, ptr, ptr)
    base = {"c": 1, "n": 4, "p": ptr, "f": 0, "u": 0, "o": 0, "z": 32, "d": ctypes.byref(desc)}
    sets = small_sets(nat.load()) if with_device else {}
    cases = []
    for name, kinds in SIGNATURES.items():
        variants = []
        for i, k in enumerate(kinds):
            if k == "n":
                variants.append(("n0", i, 0))
            elif k == "p" and not (with_device and name in HOOKS):
                variants.append(("null%d" % i, i, None))
            elif k == "c":
                variants.append(("curve77", i, 77))
            elif k == "f":
                variants.append(("fmt9", i, 9))
            elif k == "d":
                variants.append(("desc_null", i, None))
            elif k == "k" and with_device:
                variants += [("null%d" % i, i, None), ("wrong_set", i, sets[WRONG_KIND[set_kind(name)]])]
        for tag, pos, val in variants:
            args = [sets.get(set_kind(name)) if k == "k" else base[k] for k in kinds]
            args[pos] = val

            def call(lib, name=name, args=args):
                return getattr(lib, name)(*args)
            cases.append(("%s/%s" % (name, tag), call))
    return cases, (buf, desc, sets)


CURVES = {1: 32, 2: 32, 3: 48, 4: 32, 6: 66, 7: 24, 8: 28}     # EC-API curve id -> field bytes
SMALL = 256
CHUNKED = (1 << 18) + 777                                          # cut into chunks by the pipelined host calls


def launch_cases():
    """(case id, call) for every entry point x curve x mode; each call returns the entry point's return code and
    leaves its launch count in eb200_last_timing()."""
    import torch
    from elliptic_b200 import _native as nat
    rng = np.random.default_rng(7)
    keep = []

    def rnd(*shape):
        a = rng.integers(0, 256, size=shape, dtype=np.uint8)
        keep.append(a)
        return a.ctypes.data

    def out(*shape):
        a = np.zeros(shape, np.uint8)
        keep.append(a)
        return a.ctypes.data

    def dev(nbytes):
        t = torch.randint(0, 256, (max(nbytes, 1),), dtype=torch.uint8, device="cuda")
        keep.append(t)
        return t.data_ptr()

    def offsets(n, step):
        a = np.arange(n + 1, dtype=np.uint64) * step
        keep.append(a)
        return a.ctypes.data

    def synced(fn):
        def call(lib):
            rc = fn(lib)
            torch.cuda.synchronize()
            return rc
        return call

    cases = []
    n = SMALL
    for cv, ln in CURVES.items():
        for fmt, pb in ((nat.PUB_XY, 2 * ln), (nat.PUB_SEC1_65, 1 + 2 * ln), (nat.PUB_SEC1_33, 1 + ln)):
            args = (cv, n, rnd(n, ln), rnd(n, ln), rnd(n, ln), rnd(n, pb), fmt, out(n))
            cases.append(("verify/%d/fmt%d" % (cv, fmt), lambda lib, a=args: lib.eb200_ecdsa_verify_batch(*a)))
            args = (cv, n, rnd(n, ln), rnd(n * 8), offsets(n, 8), rnd(n, pb), fmt, out(n))
            cases.append(("verify_der/%d/fmt%d" % (cv, fmt), lambda lib, a=args: lib.eb200_ecdsa_verify_batch_der(*a)))
            args = (cv, n, dev(n * ln), dev(n * ln), dev(n * ln), dev(n * pb), fmt, dev(n),
                    dev(nat.load().eb200_ecdsa_verify_workspace_bytes(cv, n)), None)
            cases.append(("verify_dev/%d/fmt%d" % (cv, fmt), synced(lambda lib, a=args: lib.eb200_ecdsa_verify_batch_dev(*a))))
        for flags in (0, 1):
            args = (cv, n, rnd(n, ln), rnd(n, ln), flags, out(n, ln), out(n, ln), out(n), out(n))
            cases.append(("sign/%d/flags%d" % (cv, flags), lambda lib, a=args: lib.eb200_ecdsa_sign_batch(*a)))
        args = (cv, n, rnd(n, ln), rnd(n, ln), rnd(n, ln), 0, out(n, ln), out(n, ln), out(n), out(n))
        cases.append(("sign_k/%d" % cv, lambda lib, a=args: lib.eb200_ecdsa_sign_batch_k(*a)))
        for plen in (0, 5):
            args = (cv, n, rnd(n, ln), rnd(n, ln), rnd(8), plen, 0, out(n, ln), out(n, ln), out(n), out(n))
            cases.append(("sign_pers/%d/len%d" % (cv, plen), lambda lib, a=args: lib.eb200_ecdsa_sign_batch_pers(*a)))
        for pers in (False, True):
            args = (cv, n, rnd(n, 32), 32, rnd(8) if pers else None, 8 if pers else 0, out(n, ln), out(n, 2 * ln), out(n))
            cases.append(("keygen/%d/pers%d" % (cv, pers), lambda lib, a=args: lib.eb200_ec_keygen_batch(*a)))
        if cv != nat.CURVE_ED25519:
            args = (cv, n, rnd(n, ln), rnd(n, ln), rnd(n, ln), rnd(n), out(n, 2 * ln), out(n))
            cases.append(("recover/%d" % cv, lambda lib, a=args: lib.eb200_ecdsa_recover_batch(*a)))
        for pts in (False, True):
            args = (cv, n, rnd(n, ln), rnd(n, 2 * ln) if pts else None, out(n, 2 * ln), out(n))
            cases.append(("mul/%d/points%d" % (cv, pts), lambda lib, a=args: lib.eb200_scalar_mul_batch(*a)))
        args = (cv, n, rnd(n, ln), rnd(n, ln), rnd(n, 2 * ln), out(n, 2 * ln), out(n))
        cases.append(("mul_add/%d" % cv, lambda lib, a=args: lib.eb200_mul_add_batch(*a)))
        args = (cv, n, rnd(n, ln), rnd(n, 2 * ln), out(n, ln), out(n))
        cases.append(("derive/%d" % cv, lambda lib, a=args: lib.eb200_ecdh_derive_batch(*a)))

    for m in (n, CHUNKED):
        args = (m, rnd(m, 32), rnd(m, 32), rnd(m, 32), rnd(m, 32), out(m))
        cases.append(("eddsa_verify/%d" % m, lambda lib, a=args: lib.eb200_eddsa_verify_batch(*a)))
        args = (m, rnd(m, 32), rnd(m, 32), rnd(m, 32), rnd(m * 4), offsets(m, 4), out(m))
        cases.append(("eddsa_verify_msgs/%d" % m, lambda lib, a=args: lib.eb200_eddsa_verify_batch_msgs(*a)))
        args = (m, rnd(m, 32), rnd(m, 32), out(m, 32), out(m))
        cases.append(("x25519_derive/%d" % m, lambda lib, a=args: lib.eb200_x25519_derive_batch(*a)))
        args = (m, rnd(m, 32), rnd(m, 32), out(m, 32), out(m))
        cases.append(("x25519_mul/%d" % m, lambda lib, a=args: lib.eb200_x25519_mul_batch(*a)))
    for cv in (1, 2):
        args = (cv, CHUNKED, rnd(CHUNKED, 32), rnd(CHUNKED, 32), rnd(CHUNKED, 32), rnd(CHUNKED, 64), 0, out(CHUNKED))
        cases.append(("verify/%d/chunked" % cv, lambda lib, a=args: lib.eb200_ecdsa_verify_batch(*a)))
    args = (n, dev(32 * n), dev(32 * n), dev(32 * n), dev(32 * n), dev(n), dev(nat.load().eb200_eddsa_verify_workspace_bytes(n)), None)
    cases.append(("eddsa_verify_dev", synced(lambda lib, a=args: lib.eb200_eddsa_verify_batch_dev(*a))))
    args = (n, dev(32 * n), dev(32 * n), dev(32 * n), dev(n), None)
    cases.append(("x25519_derive_dev", synced(lambda lib, a=args: lib.eb200_x25519_derive_batch_dev(*a))))
    for pub in (False, True):
        args = (n, rnd(n, 32), rnd(n * 4), offsets(n, 4), out(n, 64), out(n, 32) if pub else None, out(n))
        cases.append(("eddsa_sign/pub%d" % pub, lambda lib, a=args: lib.eb200_eddsa_sign_batch(*a)))

    # keyed calls: host forms at SMALL and CHUNKED, device-pointer forms at SMALL, against sets of 16 keys
    lib = nat.load()
    nkeys = 16
    sets = {cv: small_sets(lib, cv, nkeys) for cv in (1, 2)}
    keep.append(sets)

    def idx(m):
        a = rng.integers(0, nkeys, size=m, dtype=np.uint32)
        keep.append(a)
        return a

    def below_n(m, top):                                   # 25519 scalars below the group order; top: the high byte
        a = rng.integers(0, 256, size=(m, 32), dtype=np.uint8)
        a[:, top] &= 0x0F
        keep.append(a)
        return a.ctypes.data

    def dev_of(a):
        t = torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).cuda()
        keep.append(t)
        return t.data_ptr()

    def dev_off(m, step):
        return dev_of(np.arange(m + 1, dtype=np.int64) * step)

    for cv in (1, 2):
        ks = sets[cv]["ecdsa"]
        for m in (n, CHUNKED):
            cases += [
                ("verify_keyed/%d/%d" % (cv, m), lambda lib, a=(ks, m, rnd(m, 32), rnd(m, 32), rnd(m, 32), idx(m).ctypes.data, out(m)):
                    lib.eb200_ecdsa_verify_batch_keyed(*a)),
                ("verify_keyed_der/%d/%d" % (cv, m), lambda lib, a=(ks, m, rnd(m, 32), rnd(m * 8), offsets(m, 8), idx(m).ctypes.data, out(m)):
                    lib.eb200_ecdsa_verify_batch_keyed_der(*a)),
                ("mul_keyed/%d/%d" % (cv, m), lambda lib, a=(ks, m, rnd(m, 32), idx(m).ctypes.data, out(m, 64), out(m)):
                    lib.eb200_scalar_mul_batch_keyed(*a)),
                ("mul_add_keyed/%d/%d" % (cv, m), lambda lib, a=(ks, m, rnd(m, 32), rnd(m, 32), idx(m).ctypes.data, out(m, 64), out(m)):
                    lib.eb200_mul_add_batch_keyed(*a)),
                ("derive_keyed/%d/%d" % (cv, m), lambda lib, a=(ks, m, rnd(m, 32), idx(m).ctypes.data, out(m, 32), out(m)):
                    lib.eb200_ecdh_derive_batch_keyed(*a)),
                ("recovery_param_keyed/%d/%d" % (cv, m),
                    lambda lib, a=(ks, m, rnd(m, 32), rnd(m, 32), rnd(m, 32), idx(m).ctypes.data, out(m), out(m)):
                    lib.eb200_ecdsa_recovery_param_batch_keyed(*a)),
            ]
        ws = dev(lib.eb200_keyset_dev_workspace_bytes(ks, n))
        cases += [
            ("verify_keyed_dev/%d" % cv, synced(lambda lib, a=(ks, n, dev(32 * n), dev(32 * n), dev(32 * n), dev_of(idx(n)), dev(n),
                                                               dev(lib.eb200_ecdsa_verify_keyed_workspace_bytes(ks, n)), None):
                                                lib.eb200_ecdsa_verify_batch_keyed_dev(*a))),
            ("verify_keyed_der_dev/%d" % cv, synced(lambda lib, a=(ks, n, dev(32 * n), dev(8 * n), 8 * n, dev_off(n, 8), dev_of(idx(n)),
                                                                   dev(n), ws, None):
                                                    lib.eb200_ecdsa_verify_batch_keyed_der_dev(*a))),
            ("mul_keyed_dev/%d" % cv, synced(lambda lib, a=(ks, n, dev(32 * n), dev_of(idx(n)), dev(64 * n), dev(n), ws, None):
                                             lib.eb200_scalar_mul_batch_keyed_dev(*a))),
            ("mul_add_keyed_dev/%d" % cv, synced(lambda lib, a=(ks, n, dev(32 * n), dev(32 * n), dev_of(idx(n)), dev(64 * n), dev(n), ws,
                                                                None):
                                                 lib.eb200_mul_add_batch_keyed_dev(*a))),
            ("derive_keyed_dev/%d" % cv, synced(lambda lib, a=(ks, n, dev(32 * n), dev_of(idx(n)), dev(32 * n), dev(n), ws, None):
                                                lib.eb200_ecdh_derive_batch_keyed_dev(*a))),
            ("recovery_param_keyed_dev/%d" % cv, synced(lambda lib, a=(ks, n, dev(32 * n), dev(32 * n), dev(32 * n), dev_of(idx(n)), dev(n),
                                                                       dev(n), ws, None):
                                                        lib.eb200_ecdsa_recovery_param_batch_keyed_dev(*a))),
        ]
    ed, sg, xs = sets[1]["ed"], sets[1]["sign"], sets[1]["x25519"]
    for m in (n, CHUNKED):
        cases += [
            ("eddsa_verify_keyed/%d" % m, lambda lib, a=(ed, m, rnd(m, 32), rnd(m, 32), below_n(m, 31), idx(m).ctypes.data, out(m)):
                lib.eb200_eddsa_verify_batch_keyed(*a)),
            ("eddsa_verify_keyed_msgs/%d" % m, lambda lib, a=(ed, m, rnd(m, 32), rnd(m, 32), rnd(m * 4), offsets(m, 4), idx(m).ctypes.data,
                                                              out(m)):
                lib.eb200_eddsa_verify_batch_keyed_msgs(*a)),
            ("eddsa_sign_keyed/%d" % m, lambda lib, a=(sg, m, rnd(m * 4), offsets(m, 4), idx(m).ctypes.data, out(m, 64), out(m)):
                lib.eb200_eddsa_sign_batch_keyed(*a)),
            ("x25519_derive_keyed/%d" % m, lambda lib, a=(xs, m, below_n(m, 0), idx(m).ctypes.data, out(m, 32), out(m)):
                lib.eb200_x25519_derive_batch_keyed(*a)),
        ]
    ws = {k: dev(lib.eb200_keyset_dev_workspace_bytes(s, n)) for k, s in (("ed", ed), ("sign", sg), ("x25519", xs))}
    cases += [
        ("eddsa_verify_keyed_dev", synced(lambda lib, a=(ed, n, dev(32 * n), dev(32 * n), dev(32 * n), dev_of(idx(n)), dev(n), ws["ed"], None):
                                          lib.eb200_eddsa_verify_batch_keyed_dev(*a))),
        ("eddsa_verify_keyed_msgs_dev", synced(lambda lib, a=(ed, n, dev(32 * n), dev(32 * n), dev(4 * n), 4 * n, dev_off(n, 4), dev_of(idx(n)),
                                                              dev(n), ws["ed"], None):
                                               lib.eb200_eddsa_verify_batch_keyed_msgs_dev(*a))),
        ("eddsa_sign_keyed_dev", synced(lambda lib, a=(sg, n, dev(4 * n), 4 * n, dev_off(n, 4), dev_of(idx(n)), dev(64 * n), dev(n), ws["sign"],
                                                       None):
                                        lib.eb200_eddsa_sign_batch_keyed_dev(*a))),
        ("x25519_derive_keyed_dev", synced(lambda lib, a=(xs, n, dev(32 * n), dev_of(idx(n)), dev(32 * n), dev(n), ws["x25519"], None):
                                           lib.eb200_x25519_derive_batch_keyed_dev(*a))),
    ]

    primes = {"p256": 2**256 - 2**224 + 2**192 + 2**96 - 1, "p384": 2**384 - 2**128 - 2**96 + 2**32 - 1, "p521": 2**521 - 1}
    for name, pv in primes.items():                        # the 8-, 12- and 18-limb run-time curve kernels
        ln = (pv.bit_length() + 7) // 8
        p, a, b = (np.frombuffer(v.to_bytes(ln, "big"), np.uint8).copy() for v in (pv, pv - 3, 7))
        keep.extend((p, a, b))
        desc = nat.ShortCurveDesc(ln, p.ctypes.data, a.ctypes.data, b.ctypes.data)
        keep.append(desc)
        d = ctypes.byref(desc)
        cases += [
            ("curve_mul/%s" % name, lambda lib, a=(d, n, rnd(n, 32), 32, rnd(n, 2 * ln), out(n, 2 * ln), out(n)): lib.eb200_curve_mul_batch(*a)),
            ("curve_mul_add/%s" % name, lambda lib, a=(d, n, rnd(n, 32), rnd(n, 2 * ln), rnd(n, 32), rnd(n, 2 * ln), 32, out(n, 2 * ln), out(n)):
                lib.eb200_curve_mul_add_batch(*a)),
            ("curve_add/%s" % name, lambda lib, a=(d, n, rnd(n, 2 * ln), rnd(n, 2 * ln), out(n, 2 * ln), out(n)): lib.eb200_curve_add_batch(*a)),
            ("curve_dbl/%s" % name, lambda lib, a=(d, n, rnd(n, 2 * ln), out(n, 2 * ln), out(n)): lib.eb200_curve_dbl_batch(*a)),
            ("curve_validate/%s" % name, lambda lib, a=(d, n, rnd(n, 2 * ln), out(n)): lib.eb200_curve_validate_batch(*a)),
        ]
    return cases, keep
