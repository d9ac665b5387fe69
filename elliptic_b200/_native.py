"""ctypes binding of libelliptic_b200.so (the C ABI in include/elliptic_b200.h).

There is deliberately no CPU fallback: if the shared library is missing or no
CUDA device is usable, every compute call raises.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# EB200_LIB lets the tuning scripts load an alternative build of the same library
LIB_PATH = os.environ.get("EB200_LIB") or os.path.join(_HERE, "libelliptic_b200.so")

OK, ERR_NO_DEVICE, ERR_CUDA, ERR_ARG, ERR_NOT_INIT, ERR_UNSUPPORTED = 0, -1, -2, -3, -4, -5
ST_FALSE, ST_TRUE, ST_THROW_INVALID_POINT, ST_THROW_NOT_VALIDATED, ST_NEEDS_HOST, ST_THROW_ASSERT, \
    ST_THROW_POINT_FORMAT = range(7)
ST_INFINITY, ST_THROW_SECOND_KEY, ST_THROW_SIG_FORMAT, ST_RETRY, ST_THROW_NO_RECOVERY = 7, 8, 9, 10, 11
ST_BAD_KEY_INDEX, ST_BAD_ITEM = 12, 13
CURVE_SECP256K1, CURVE_P256, CURVE_P384, CURVE_ED25519, CURVE_CURVE25519, CURVE_P521, CURVE_P192, CURVE_P224 = 1, 2, 3, 4, 5, 6, 7, 8
PUB_XY, PUB_SEC1_65, PUB_SEC1_33 = 0, 1, 2
KEYSET_MIN_BITS, KEYSET_MAX_BITS, KEYSET_DEFAULT_BUDGET = 4, 8, 1 << 30

EXPORTS = [
    "eb200_init", "eb200_shutdown", "eb200_device_count", "eb200_strerror", "eb200_last_error", "eb200_last_timing",
    "eb200_ecdsa_verify_batch", "eb200_ecdsa_verify_workspace_bytes", "eb200_ecdsa_verify_batch_dev",
    "eb200_selftest_fe", "eb200_selftest_gtab", "eb200_selftest_gtab_dims",
    "eb200_eddsa_verify_batch", "eb200_eddsa_verify_workspace_bytes", "eb200_eddsa_verify_batch_dev",
    "eb200_x25519_derive_batch", "eb200_x25519_derive_batch_dev", "eb200_ecdsa_recover_batch", "eb200_ecdsa_sign_batch",
    "eb200_eddsa_verify_batch_msgs", "eb200_scalar_mul_batch", "eb200_mul_add_batch",
    "eb200_ecdsa_verify_batch_der", "eb200_ecdh_derive_batch", "eb200_eddsa_sign_batch",
    "eb200_ecdsa_sign_batch_k", "eb200_ecdsa_sign_batch_pers", "eb200_ec_keygen_batch", "eb200_x25519_mul_batch",
    "eb200_curve_mul_batch", "eb200_curve_mul_add_batch", "eb200_curve_add_batch", "eb200_curve_dbl_batch", "eb200_curve_validate_batch",
    "eb200_ecdsa_recovery_param_batch",
    "eb200_keyset_create", "eb200_keyset_info", "eb200_keyset_destroy", "eb200_ecdsa_verify_batch_keyed",
    "eb200_eddsa_keyset_create", "eb200_eddsa_verify_batch_keyed", "eb200_eddsa_verify_batch_keyed_msgs",
    "eb200_scalar_mul_batch_keyed", "eb200_mul_add_batch_keyed", "eb200_ecdh_derive_batch_keyed",
    "eb200_eddsa_signing_set_create", "eb200_eddsa_sign_batch_keyed", "eb200_ecdsa_recovery_param_batch_keyed",
    "eb200_x25519_keyset_create", "eb200_x25519_derive_batch_keyed",
    "eb200_ecdsa_verify_batch_keyed_der", "eb200_ecdsa_verify_keyed_workspace_bytes", "eb200_ecdsa_verify_batch_keyed_dev",
    "eb200_keyset_dev_workspace_bytes", "eb200_scalar_mul_batch_keyed_dev", "eb200_mul_add_batch_keyed_dev",
    "eb200_ecdh_derive_batch_keyed_dev", "eb200_ecdsa_recovery_param_batch_keyed_dev", "eb200_eddsa_verify_batch_keyed_dev",
    "eb200_eddsa_verify_batch_keyed_msgs_dev", "eb200_eddsa_sign_batch_keyed_dev", "eb200_x25519_derive_batch_keyed_dev",
    "eb200_dev_workspace_bytes", "eb200_ecdsa_sign_batch_dev", "eb200_ecdsa_sign_batch_k_dev", "eb200_ecdsa_sign_batch_pers_dev",
    "eb200_ec_keygen_batch_dev", "eb200_ecdsa_recover_batch_dev", "eb200_ecdsa_recovery_param_batch_dev",
    "eb200_scalar_mul_batch_dev", "eb200_mul_add_batch_dev", "eb200_ecdh_derive_batch_dev", "eb200_x25519_mul_batch_dev",
    "eb200_ecdsa_verify_batch_der_dev", "eb200_eddsa_verify_batch_msgs_dev", "eb200_eddsa_sign_batch_dev",
    "eb200_ecdsa_verify_batch_keyed_der_dev",
]


class Timing(ctypes.Structure):
    _fields_ = [("h2d_ms", ctypes.c_float), ("kernel_ms", ctypes.c_float), ("d2h_ms", ctypes.c_float),
                ("main_kernel_ms", ctypes.c_float), ("launches", ctypes.c_uint32)]


class ShortCurveDesc(ctypes.Structure):
    _fields_ = [("len", ctypes.c_uint32), ("p", ctypes.c_void_p), ("a", ctypes.c_void_p), ("b", ctypes.c_void_p)]


def short_curve(pab):
    """The eb200_short_curve over the rows p, a, b of a (3, len) uint8 array, which the caller keeps alive."""
    return ShortCurveDesc(pab.shape[1], *(row.ctypes.data for row in pab))


class NativeError(RuntimeError):
    pass


_lib = None


def load():
    """dlopen the library (no CUDA call yet)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            "libelliptic_b200.so is not built (run `python -m elliptic_b200.build`); "
            "elliptic_b200 has no CPU fallback")
    lib = ctypes.CDLL(LIB_PATH)
    c = ctypes
    lib.eb200_init.argtypes = [c.POINTER(c.c_int), c.c_int, c.c_uint32]
    lib.eb200_strerror.restype = c.c_char_p
    lib.eb200_strerror.argtypes = [c.c_int]
    lib.eb200_last_error.restype = c.c_char_p
    lib.eb200_last_timing.argtypes = [c.POINTER(Timing)]
    lib.eb200_ecdsa_verify_batch.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 4 + [c.c_uint32, c.c_void_p]
    lib.eb200_ecdsa_verify_workspace_bytes.restype = c.c_size_t
    lib.eb200_ecdsa_verify_workspace_bytes.argtypes = [c.c_int, c.c_size_t]
    lib.eb200_ecdsa_verify_batch_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 4 + [c.c_uint32] + [c.c_void_p] * 3
    lib.eb200_eddsa_verify_batch.argtypes = [c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_eddsa_verify_workspace_bytes.restype = c.c_size_t
    lib.eb200_eddsa_verify_workspace_bytes.argtypes = [c.c_size_t]
    lib.eb200_eddsa_verify_batch_dev.argtypes = [c.c_size_t] + [c.c_void_p] * 7
    lib.eb200_x25519_derive_batch.argtypes = [c.c_size_t] + [c.c_void_p] * 4
    D = c.POINTER(ShortCurveDesc)
    lib.eb200_curve_mul_batch.argtypes = [D, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p]
    lib.eb200_curve_mul_add_batch.argtypes = [D, c.c_size_t] + [c.c_void_p] * 4 + [c.c_size_t, c.c_void_p, c.c_void_p]
    lib.eb200_curve_add_batch.argtypes = [D, c.c_size_t] + [c.c_void_p] * 4
    lib.eb200_curve_dbl_batch.argtypes = [D, c.c_size_t] + [c.c_void_p] * 3
    lib.eb200_curve_validate_batch.argtypes = [D, c.c_size_t] + [c.c_void_p] * 2
    lib.eb200_x25519_mul_batch.argtypes = [c.c_size_t] + [c.c_void_p] * 4
    lib.eb200_x25519_derive_batch_dev.argtypes = [c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_eddsa_verify_batch_msgs.argtypes = [c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_eddsa_sign_batch.argtypes = [c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_ecdsa_sign_batch_k.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_uint32] + [c.c_void_p] * 4
    lib.eb200_ecdsa_sign_batch_pers.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p, c.c_size_t, c.c_uint32] + [c.c_void_p] * 4
    lib.eb200_ec_keygen_batch.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t] + [c.c_void_p] * 3
    lib.eb200_ecdsa_sign_batch.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_void_p, c.c_uint32] + [c.c_void_p] * 4
    lib.eb200_ecdsa_recover_batch.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_ecdsa_recovery_param_batch.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_keyset_create.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_uint32, c.c_uint32, c.c_void_p, c.POINTER(c.c_void_p)]
    lib.eb200_keyset_info.argtypes = [c.c_void_p, c.POINTER(c.c_int), c.POINTER(c.c_size_t), c.POINTER(c.c_uint32), c.POINTER(c.c_size_t)]
    lib.eb200_keyset_destroy.argtypes = [c.c_void_p]
    lib.eb200_ecdsa_verify_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_ecdsa_verify_batch_keyed_der.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_ecdsa_verify_keyed_workspace_bytes.restype = c.c_size_t
    lib.eb200_ecdsa_verify_keyed_workspace_bytes.argtypes = [c.c_void_p, c.c_size_t]
    lib.eb200_ecdsa_verify_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 7
    lib.eb200_ecdsa_verify_batch_keyed_der_dev.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_uint64] + \
        [c.c_void_p] * 5
    lib.eb200_keyset_dev_workspace_bytes.restype = c.c_size_t
    lib.eb200_keyset_dev_workspace_bytes.argtypes = [c.c_void_p, c.c_size_t]
    lib.eb200_scalar_mul_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_mul_add_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 7
    lib.eb200_ecdh_derive_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_ecdsa_recovery_param_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 8
    lib.eb200_eddsa_verify_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 7
    lib.eb200_eddsa_verify_batch_keyed_msgs_dev.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p,
                                                            c.c_uint64] + [c.c_void_p] * 5
    lib.eb200_eddsa_sign_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t, c.c_void_p, c.c_uint64] + [c.c_void_p] * 6
    lib.eb200_x25519_derive_batch_keyed_dev.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_dev_workspace_bytes.restype = c.c_size_t
    lib.eb200_dev_workspace_bytes.argtypes = [c.c_int, c.c_size_t]
    lib.eb200_ecdsa_sign_batch_dev.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_void_p, c.c_uint32] + [c.c_void_p] * 6
    lib.eb200_ecdsa_sign_batch_k_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 3 + [c.c_uint32] + [c.c_void_p] * 6
    lib.eb200_ecdsa_sign_batch_pers_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 3 + [c.c_size_t, c.c_uint32] + \
        [c.c_void_p] * 6
    lib.eb200_ec_keygen_batch_dev.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_size_t, c.c_void_p, c.c_size_t] + \
        [c.c_void_p] * 5
    lib.eb200_ecdsa_recover_batch_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 8
    lib.eb200_ecdsa_recovery_param_batch_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 8
    lib.eb200_scalar_mul_batch_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_mul_add_batch_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 7
    lib.eb200_ecdh_derive_batch_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_x25519_mul_batch_dev.argtypes = [c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_ecdsa_verify_batch_der_dev.argtypes = [c.c_int, c.c_size_t, c.c_void_p, c.c_void_p, c.c_uint64, c.c_void_p,
                                                     c.c_void_p, c.c_uint32] + [c.c_void_p] * 3
    lib.eb200_eddsa_verify_batch_msgs_dev.argtypes = [c.c_size_t] + [c.c_void_p] * 4 + [c.c_uint64] + [c.c_void_p] * 4
    lib.eb200_eddsa_sign_batch_dev.argtypes = [c.c_size_t, c.c_void_p, c.c_void_p, c.c_uint64] + [c.c_void_p] * 6
    lib.eb200_scalar_mul_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 4
    lib.eb200_mul_add_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_ecdh_derive_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 4
    lib.eb200_ecdsa_recovery_param_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_eddsa_keyset_create.argtypes = [c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.POINTER(c.c_void_p)]
    lib.eb200_eddsa_verify_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_eddsa_verify_batch_keyed_msgs.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 6
    lib.eb200_eddsa_signing_set_create.argtypes = [c.c_size_t, c.c_void_p, c.c_void_p, c.POINTER(c.c_void_p)]
    lib.eb200_eddsa_sign_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_x25519_keyset_create.argtypes = [c.c_size_t, c.c_void_p, c.c_uint32, c.c_void_p, c.POINTER(c.c_void_p)]
    lib.eb200_x25519_derive_batch_keyed.argtypes = [c.c_void_p, c.c_size_t] + [c.c_void_p] * 4
    lib.eb200_ecdsa_verify_batch_der.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 4 + [c.c_uint32, c.c_void_p]
    lib.eb200_ecdh_derive_batch.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 4
    lib.eb200_scalar_mul_batch.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 4
    lib.eb200_mul_add_batch.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 5
    lib.eb200_selftest_gtab_dims.argtypes = [c.c_int] + [c.c_void_p] * 3
    lib.eb200_selftest_fe.argtypes = [c.c_int, c.c_int, c.c_size_t, c.c_void_p, c.c_void_p, c.c_void_p]
    lib.eb200_selftest_gtab.argtypes = [c.c_int, c.c_void_p, c.c_size_t]
    _lib = lib
    return lib


def check(rc):
    if rc != OK:
        lib = load()
        raise NativeError("%s [%s]" % (lib.eb200_strerror(rc).decode(), lib.eb200_last_error().decode()))


def call(fn, *args):
    """fn(*args) with every numpy array passed as the address of its data (the caller keeps it contiguous) and None
    as NULL; raises NativeError unless fn returns OK."""
    check(fn(*(a.ctypes.data if isinstance(a, np.ndarray) else a for a in args)))


_inited = set()
INIT_ALL_TABLES = 1


def init(device=0, flags=0):
    """Make sure a context exists on CUDA device `device` (idempotent; further devices are added, not replaced)."""
    return init_devices([device], flags)


def init_devices(devices=None, flags=0):
    """eb200_init(devices[], ndev, flags): one context per listed device (None: every visible device).  Host-pointer
    calls are then sharded over all initialised devices inside the library."""
    lib = load()
    if devices is None:
        check(lib.eb200_init(None, 0, flags))
        _inited.add("all")
        return lib
    new = [d for d in devices if d not in _inited]
    if new or flags:
        arr = (ctypes.c_int * len(devices))(*devices)
        check(lib.eb200_init(arr, len(devices), flags))
        _inited.update(devices)
    return lib


def shutdown():
    lib = load()
    check(lib.eb200_shutdown())
    _inited.clear()


def last_timing():
    t = Timing()
    check(load().eb200_last_timing(ctypes.byref(t)))
    return {"h2d_ms": t.h2d_ms, "kernel_ms": t.kernel_ms, "d2h_ms": t.d2h_ms,
            "main_kernel_ms": t.main_kernel_ms, "launches": t.launches}
