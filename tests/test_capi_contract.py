"""What the C ABI answers without computing anything: workspace sizes, fixed-base table geometry, and the return
code of every entry point for empty batches, NULL pointers and unknown curves / formats when no device is
initialised.  The order in which an entry point checks its arguments decides these codes, so they are pinned
case by case (tests/abi_cases.py builds the calls)."""
import ctypes

import pytest

from abi_cases import argument_cases

NS = [0, 1, 127, 128, (1 << 18) + 777, 1 << 20]
# eb200_ecdsa_verify_workspace_bytes(curve, n) for curve ids 0..9 and n in NS
ECDSA_WORKSPACE = {
    0: [0, 0, 0, 0, 0, 0],
    1: [0, 1792, 119808, 120576, 247409408, 986710016],
    2: [0, 1792, 118784, 119552, 245306112, 978321408],
    3: [0, 2304, 177920, 178944, 367301376, 1464860672],
    4: [0, 1792, 154880, 155904, 319975424, 1276116992],
    5: [0, 0, 0, 0, 0, 0],
    6: [0, 2816, 264960, 266496, 547139328, 2182086656],
    7: [0, 1792, 89344, 89856, 184308224, 735051776],
    8: [0, 1792, 117760, 118528, 243202560, 969932800],
    9: [0, 0, 0, 0, 0, 0],
}
EDDSA_WORKSPACE = [0, 1280, 146432, 147456, 302885120, 1207959552]
# eb200_selftest_gtab_dims(curve) -> (return code, windows, entries, wbits); -1: left untouched.  ed25519
# reports the p224 geometry.
GTAB_DIMS = {
    0: (-5, -1, -1, -1), 1: (0, 13, 524288, 20), 2: (0, 20, 4096, 13), 3: (0, 30, 4096, 13), 4: (0, 18, 4096, 13),
    5: (-5, -1, -1, -1), 6: (0, 41, 4096, 13), 7: (0, 15, 4096, 13), 8: (0, 18, 4096, 13), 9: (-5, -1, -1, -1),
}
# return codes without a device (-3 ERR_ARG, -4 ERR_NOT_INIT, -5 ERR_UNSUPPORTED); nullK: NULL in argument K.  The
# keyed calls get a NULL set here, which they refuse before they look for a device.
NO_DEVICE = {
    "eb200_ecdsa_verify_batch": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4, "fmt9": -4, "null7": -4},
    "eb200_ecdsa_verify_batch_der": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4, "fmt9": -4, "null7": -4},
    "eb200_ecdsa_verify_batch_dev": {"curve77": -5, "n0": -4, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "fmt9": -5, "null7": -3,
                                     "null8": -3, "null9": -4},
    "eb200_ecdsa_sign_batch": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null5": -4, "null6": -4, "null7": -4, "null8": -4},
    "eb200_ecdsa_sign_batch_k": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null6": -4, "null7": -4, "null8": -4,
                                 "null9": -4},
    "eb200_ecdsa_sign_batch_pers": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null7": -4, "null8": -4, "null9": -4,
                                    "null10": -4},
    "eb200_ec_keygen_batch": {"curve77": -4, "n0": -4, "null2": -4, "null4": -4, "null6": -4, "null7": -4, "null8": -4},
    "eb200_ecdsa_recover_batch": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4, "null6": -4, "null7": -4},
    "eb200_ecdsa_recovery_param_batch": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4,
                                         "null6": -4, "null7": -4},
    "eb200_scalar_mul_batch": {"curve77": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4},
    "eb200_ecdh_derive_batch": {"curve77": -4, "n0": -4, "null2": -4, "null3": -3, "null4": -4, "null5": -4},
    "eb200_mul_add_batch": {"curve77": -4, "n0": -4, "null2": -3, "null3": -4, "null4": -3, "null5": -4, "null6": -4},
    "eb200_eddsa_verify_batch": {"n0": -4, "null1": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4},
    "eb200_eddsa_verify_batch_msgs": {"n0": -4, "null1": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4, "null6": -4},
    "eb200_eddsa_verify_batch_dev": {"n0": -4, "null1": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -4},
    "eb200_eddsa_sign_batch": {"n0": -4, "null1": -4, "null2": -4, "null3": -4, "null4": -4, "null5": -4, "null6": -4},
    "eb200_x25519_derive_batch": {"n0": -4, "null1": -4, "null2": -4, "null3": -4, "null4": -4},
    "eb200_x25519_derive_batch_dev": {"n0": -4, "null1": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -4},
    "eb200_x25519_mul_batch": {"n0": -4, "null1": -4, "null2": -4, "null3": -4, "null4": -4},
    "eb200_curve_mul_batch": {"desc_null": -4, "n0": -4, "null2": -3, "null4": -4, "null5": -4, "null6": -4},
    "eb200_curve_mul_add_batch": {"desc_null": -4, "n0": -4, "null2": -3, "null3": -4, "null4": -3, "null5": -3, "null7": -4, "null8": -4},
    "eb200_curve_add_batch": {"desc_null": -4, "n0": -4, "null2": -4, "null3": -3, "null4": -4, "null5": -4},
    "eb200_curve_dbl_batch": {"desc_null": -4, "n0": -4, "null2": -4, "null3": -4, "null4": -4},
    "eb200_curve_validate_batch": {"desc_null": -4, "n0": -4, "null2": -4, "null3": -4},
    "eb200_ecdsa_verify_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_ecdsa_verify_batch_keyed_der": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_ecdsa_verify_batch_keyed_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                           "null7": -3, "null8": -3},
    "eb200_scalar_mul_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3},
    "eb200_mul_add_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_ecdh_derive_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3},
    "eb200_ecdsa_recovery_param_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                               "null7": -3},
    "eb200_eddsa_verify_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_eddsa_verify_batch_keyed_msgs": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                            "null7": -3},
    "eb200_eddsa_sign_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_x25519_derive_batch_keyed": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3},
    "eb200_ecdsa_verify_batch_keyed_der_dev": {"n0": -3, "null2": -3, "null3": -3, "null5": -3, "null6": -3, "null7": -3,
                                               "null8": -3, "null9": -3},
    "eb200_scalar_mul_batch_keyed_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3},
    "eb200_mul_add_batch_keyed_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3,
                                      "null8": -3},
    "eb200_ecdh_derive_batch_keyed_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3},
    "eb200_ecdsa_recovery_param_batch_keyed_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                                   "null7": -3, "null8": -3, "null9": -3},
    "eb200_eddsa_verify_batch_keyed_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                           "null7": -3, "null8": -3},
    "eb200_eddsa_verify_batch_keyed_msgs_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null6": -3, "null7": -3,
                                                "null8": -3, "null9": -3, "null10": -3},
    "eb200_eddsa_sign_batch_keyed_dev": {"n0": -3, "null2": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3, "null8": -3,
                                         "null9": -3},
    "eb200_x25519_derive_batch_keyed_dev": {"n0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                            "null7": -3},
    "eb200_selftest_fe": {"curve77": -4, "n0": -4, "null3": -4, "null4": -4, "null5": -4},
    "eb200_selftest_gtab": {"curve77": -4, "null1": -4},
    "eb200_selftest_gtab_dims": {"curve77": -5, "null1": -3, "null2": -3, "null3": -3},
    "eb200_last_timing": {"null0": -3},
}


@pytest.fixture(scope="module")
def lib():
    from elliptic_b200 import _native, build
    build.build()
    return _native.load()


def test_workspace_bytes(lib):
    for curve, want in ECDSA_WORKSPACE.items():
        assert [lib.eb200_ecdsa_verify_workspace_bytes(curve, n) for n in NS] == want, curve
    assert [lib.eb200_eddsa_verify_workspace_bytes(n) for n in NS] == EDDSA_WORKSPACE


def test_gtab_dims(lib):
    for curve, want in GTAB_DIMS.items():
        w, e, b = ctypes.c_int(-1), ctypes.c_int(-1), ctypes.c_int(-1)
        rc = lib.eb200_selftest_gtab_dims(curve, ctypes.byref(w), ctypes.byref(e), ctypes.byref(b))
        assert (rc, w.value, e.value, b.value) == want, curve


def test_return_codes_without_device(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    assert lib.eb200_device_count() == 0
    cases, _keep = argument_cases(with_device=False)
    got = {}
    for cid, call in cases:
        name, tag = cid.split("/")
        got.setdefault(name, {})[tag] = call(lib)
    assert got == NO_DEVICE
