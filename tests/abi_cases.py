"""Argument and launch-count cases of the C ABI, shared by test_capi_contract.py (no device) and
test_gpu_properties.py (device initialised).  Each case is a name and a call; the tests compare what the calls
return (and, on the GPU, eb200_timing.launches) with literal tables."""
import ctypes

import numpy as np

# Argument kinds of every entry point, in header order.  c: curve id, n: item count, p: pointer, f: public-key
# format, u: flags, o: selftest op, z: a byte length or word count, d: eb200_short_curve descriptor.
SIGNATURES = {
    "eb200_ecdsa_verify_batch": "cnppppfp",
    "eb200_ecdsa_verify_batch_der": "cnppppfp",
    "eb200_ecdsa_verify_batch_dev": "cnppppfppp",
    "eb200_ecdsa_sign_batch": "cnppupppp",
    "eb200_ecdsa_sign_batch_k": "cnpppupppp",
    "eb200_ecdsa_sign_batch_pers": "cnpppzupppp",
    "eb200_ec_keygen_batch": "cnpzpzppp",
    "eb200_ecdsa_recover_batch": "cnpppppp",
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
    "eb200_selftest_fe": "conppp",
    "eb200_selftest_gtab": "cpz",
    "eb200_selftest_gtab_dims": "cppp",
    "eb200_last_timing": "p",
}
# the self-test hooks copy from their host pointers without checking them: no NULL cases with a device
HOOKS = ("eb200_selftest_fe", "eb200_selftest_gtab")


def argument_cases(with_device):
    """(case id, call) for every entry point: n == 0, a NULL in each pointer argument, an unknown curve, an unknown
    public-key format and a NULL descriptor.  Every other argument is valid: 4 items, secp256k1, {x, y} keys and
    pointers into one zeroed host buffer (so device-pointer calls find no owning device)."""
    from elliptic_b200 import _native as nat
    buf = np.zeros(1 << 16, np.uint8)
    ptr = buf.ctypes.data
    desc = nat.ShortCurveDesc(32, ptr, ptr, ptr)
    base = {"c": 1, "n": 4, "p": ptr, "f": 0, "u": 0, "o": 0, "z": 32, "d": ctypes.byref(desc)}
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
        for tag, pos, val in variants:
            args = [base[k] for k in kinds]
            args[pos] = val

            def call(lib, name=name, args=args):
                return getattr(lib, name)(*args)
            cases.append(("%s/%s" % (name, tag), call))
    return cases, (buf, desc)


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
