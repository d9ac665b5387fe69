"""Size-independent properties at 2^16 items per call, all through the C ABI with packed arrays:
sign -> verify -> recover round trips, linearity of mulAdd, ECDH agreement, EdDSA expectation of the
bench generator, and spot checks against independent implementations (OpenSSL via `cryptography`,
libsodium via PyNaCl) where those agree with the reference by construction (well-formed inputs)."""
import ctypes
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 1 << 16
K256_N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141


def _ints(a):
    return [int.from_bytes(row.tobytes(), "big") for row in a]


def _be(vals, ln=32):
    return np.frombuffer(b"".join(v.to_bytes(ln, "big") for v in vals), np.uint8).reshape(-1, ln).copy()


def test_k256_sign_verify_recover_round_trip(native):
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC as GpuEC
    lib = nat.init(0)
    rng = np.random.default_rng(2024)
    e = rng.integers(0, 256, size=(N, 32), dtype=np.uint8)
    e[:, 0] &= 0x7F                                             # below n, so recover's `new BN(msg)` sees the same e
    priv = rng.integers(0, 256, size=(N, 32), dtype=np.uint8)
    priv[:, 0] &= 0x7F
    priv[:, 31] |= 1
    r = np.zeros((N, 32), np.uint8); s = np.zeros((N, 32), np.uint8); rec = np.zeros(N, np.uint8); st = np.zeros(N, np.uint8)
    pub = np.zeros((N, 64), np.uint8)
    nat.check(lib.eb200_scalar_mul_batch(1, N, priv.ctypes.data, None, pub.ctypes.data, st.ctypes.data))      # keygen
    assert (st == 1).all()
    for flags in (0, 1):
        nat.check(lib.eb200_ecdsa_sign_batch(1, N, e.ctypes.data, priv.ctypes.data, flags, r.ctypes.data, s.ctypes.data,
                                             rec.ctypes.data, st.ctypes.data))
        assert (st == 1).all()
        if flags:                                              # canonical: s <= n/2
            half = _be([K256_N >> 1])[0]
            assert all(row.tobytes() <= half.tobytes() for row in s[::97])
        ver = GpuEC("secp256k1").verify_batch_packed(e, r, s, pub)
        assert (ver == 1).all()
        out = np.zeros((N, 64), np.uint8)
        nat.check(lib.eb200_ecdsa_recover_batch(1, N, e.ctypes.data, r.ctypes.data, s.ctypes.data, rec.ctypes.data,
                                                out.ctypes.data, st.ctypes.data))
        assert (st == 1).all() and np.array_equal(out, pub)
        # a forged message must not verify, and must recover a different key
        e2 = e.copy(); e2[:, 31] ^= 1
        assert (GpuEC("secp256k1").verify_batch_packed(e2, r, s, pub) == 0).all()
    # independent implementation on a sample: OpenSSL accepts what we signed
    from cryptography.hazmat.primitives.asymmetric import ec as cec, utils as cutils
    from cryptography.hazmat.primitives import hashes
    for i in range(0, N, N // 64):
        x, y = int.from_bytes(pub[i, :32].tobytes(), "big"), int.from_bytes(pub[i, 32:].tobytes(), "big")
        key = cec.EllipticCurvePublicNumbers(x, y, cec.SECP256K1()).public_key()
        sig = cutils.encode_dss_signature(int.from_bytes(r[i].tobytes(), "big"), int.from_bytes(s[i].tobytes(), "big"))
        key.verify(sig, e[i].tobytes(), cec.ECDSA(cutils.Prehashed(hashes.SHA256())))


def test_k256_mul_add_is_linear(native):
    """k1*G + k2*(d*G) == ((k1 + k2*d) mod n)*G, and k*(d*G) == (k*d mod n)*G, for 2^16 random items."""
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    rnd = random.Random(5)
    ds = [rnd.randrange(1, K256_N) for _ in range(256)]
    dpub = np.zeros((256, 64), np.uint8); st8 = np.zeros(256, np.uint8)
    dk = _be(ds)
    nat.check(lib.eb200_scalar_mul_batch(1, 256, dk.ctypes.data, None, dpub.ctypes.data, st8.ctypes.data))
    rng = np.random.default_rng(11)
    k1 = rng.integers(0, 256, size=(N, 32), dtype=np.uint8)
    k2 = rng.integers(0, 256, size=(N, 32), dtype=np.uint8)
    idx = np.arange(N) % 256
    pts = dpub[idx].copy()
    k1i, k2i = _ints(k1), _ints(k2)
    lhs = np.zeros((N, 64), np.uint8); rhs = np.zeros((N, 64), np.uint8); st = np.zeros(N, np.uint8); st2 = np.zeros(N, np.uint8)
    comb = _be([(a + b * ds[i % 256]) % K256_N for i, (a, b) in enumerate(zip(k1i, k2i))])
    nat.check(lib.eb200_mul_add_batch(1, N, k1.ctypes.data, k2.ctypes.data, pts.ctypes.data, lhs.ctypes.data, st.ctypes.data))
    nat.check(lib.eb200_scalar_mul_batch(1, N, comb.ctypes.data, None, rhs.ctypes.data, st2.ctypes.data))
    assert np.array_equal(st, st2) and np.array_equal(lhs, rhs)
    comb = _be([b * ds[i % 256] % K256_N for i, b in enumerate(k2i)])
    nat.check(lib.eb200_scalar_mul_batch(1, N, k2.ctypes.data, pts.ctypes.data, lhs.ctypes.data, st.ctypes.data))
    nat.check(lib.eb200_scalar_mul_batch(1, N, comb.ctypes.data, None, rhs.ctypes.data, st2.ctypes.data))
    assert np.array_equal(st, st2) and np.array_equal(lhs, rhs)


def test_ed25519_generator_expectation_and_libsodium(native):
    import benchdata
    from elliptic_b200.eddsa import EDDSA as GpuEd
    ds = benchdata.gen_ed25519_verify(N, cache_dir=benchdata.cache_dir(), with_msgs=True)
    ged = GpuEd()
    st = ged.verify_batch_packed(ds["R"], ds["S"], ds["A"], ds["h"])
    assert np.array_equal(st, ds["expected"])
    off = np.arange(N + 1, dtype=np.uint64) * 32
    st2 = ged.verify_batch_msgs_packed(ds["R"], ds["S"], ds["A"], ds["msgs"].reshape(-1), off)      # SHA-512 on the GPU
    assert np.array_equal(st2, ds["expected"])
    assert 0 in set(ds["expected"].tolist()) and 1 in set(ds["expected"].tolist())
    import nacl.signing, nacl.exceptions
    for i in list(range(0, N, N // 96)) + list(range(63, N, 64))[:32]:
        vk = nacl.signing.VerifyKey(ds["A"][i].tobytes())
        try:
            vk.verify(ds["msgs"][i].tobytes(), ds["R"][i].tobytes() + ds["S"][i].tobytes())
            ok = 1
        except nacl.exceptions.BadSignatureError:
            ok = 0
        assert ok == int(st[i]), i


def test_curve25519_ecdh_agreement(native):
    """derive(a, b*9) == derive(b, a*9) for 2^15 pairs of unclamped scalars (test/ecdh-test.js:8-29),
    plus RFC 7748-style cross-check with OpenSSL X25519 for clamped scalars."""
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    n25519 = 2**252 + 27742317777372353535851937790883648493
    rnd = random.Random(8)
    half = N // 2
    a = [rnd.randrange(1, n25519) for _ in range(half)]
    b = [rnd.randrange(1, n25519) for _ in range(half)]
    nine = _be([9] * N)
    ks = _be(a + b)
    pubs = np.zeros((N, 32), np.uint8); st = np.zeros(N, np.uint8)
    nat.check(lib.eb200_x25519_derive_batch(N, ks.ctypes.data, nine.ctypes.data, pubs.ctypes.data, st.ctypes.data))
    assert (st == 1).all()
    swapped = np.concatenate([pubs[half:], pubs[:half]])
    shared = np.zeros((N, 32), np.uint8)
    nat.check(lib.eb200_x25519_derive_batch(N, ks.ctypes.data, swapped.ctypes.data, shared.ctypes.data, st.ctypes.data))
    assert (st == 1).all()
    assert np.array_equal(shared[:half], shared[half:])
    from cryptography.hazmat.primitives.asymmetric.x25519 import X25519PrivateKey, X25519PublicKey
    from cryptography.hazmat.primitives import serialization as ser
    for i in range(32):
        sk = bytearray(rnd.randbytes(32))
        sk[0] &= 248; sk[31] &= 127; sk[31] |= 64             # already clamped: OpenSSL's k equals ours
        k = int.from_bytes(bytes(sk), "little")
        if k >= n25519 * 8:
            continue
        peer = pubs[i].tobytes()                                # big-endian x
        want = X25519PrivateKey.from_private_bytes(bytes(sk)).exchange(X25519PublicKey.from_public_bytes(peer[::-1]))
        # the reference reduces the private key mod n (ec/key.js:76-82); peer points here have prime order,
        # so k and k mod n give the same multiple
        kb = _be([k % n25519]); px = np.frombuffer(peer, np.uint8).reshape(1, 32).copy()
        o = np.zeros((1, 32), np.uint8); s1 = np.zeros(1, np.uint8)
        nat.check(lib.eb200_x25519_derive_batch(1, kb.ctypes.data, px.ctypes.data, o.ctypes.data, s1.ctypes.data))
        assert s1[0] == 1 and o[0].tobytes()[::-1] == want


@pytest.mark.parametrize("name", ["secp256k1", "p256", "p384"])
def test_openssl_signatures_verify_and_forgeries_do_not(native, name):
    """Independent implementation as the producer: 2^12 ECDSA signatures made by OpenSSL (`cryptography`)
    must all verify through the C ABI -- with DER signatures and SEC1 keys straight off the wire, parsed on
    the GPU -- and none may verify once the digest is altered."""
    from cryptography.hazmat.primitives.asymmetric import ec as cec, utils as cutils
    from cryptography.hazmat.primitives import hashes, serialization as ser
    from elliptic_b200.ec import EC as GpuEC
    from elliptic_b200 import _native as nat
    curve, h, ln = {"secp256k1": (cec.SECP256K1(), hashes.SHA256(), 32), "p256": (cec.SECP256R1(), hashes.SHA256(), 32),
                    "p384": (cec.SECP384R1(), hashes.SHA384(), 48)}[name]
    rnd = random.Random(99)
    keys = [cec.generate_private_key(curve) for _ in range(16)]
    pubs65 = [k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.UncompressedPoint) for k in keys]
    pubs33 = [k.public_key().public_bytes(ser.Encoding.X962, ser.PublicFormat.CompressedPoint) for k in keys]
    n = 1 << 12
    digests = [rnd.randbytes(ln) for _ in range(n)]
    ders = [keys[i % 16].sign(digests[i], cec.ECDSA(cutils.Prehashed(h))) for i in range(n)]
    g = GpuEC(name)
    e = np.frombuffer(b"".join(digests), np.uint8).reshape(n, ln)          # digest length = n's byte length: no shift
    for fmt, pubs in ((nat.PUB_SEC1_65, pubs65), (nat.PUB_SEC1_33, pubs33)):
        pub = np.frombuffer(b"".join(pubs[i % 16] for i in range(n)), np.uint8).reshape(n, -1)
        st = g.verify_batch_der_packed(e, ders, pub, fmt)
        assert (st == 1).all(), np.nonzero(st != 1)[0][:5]
        e2 = e.copy(); e2[:, ln - 1] ^= 0x10
        assert (g.verify_batch_der_packed(e2, ders, pub, fmt) == 0).all()


# return codes with cuda:0 initialised (argument_cases(with_device=True)); nullK: NULL in argument K
WITH_DEVICE = {
    "eb200_curve_add_batch": {"desc_null": -3, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3},
    "eb200_curve_dbl_batch": {"desc_null": -3, "n0": 0, "null2": -3, "null3": -3, "null4": -3},
    "eb200_curve_mul_add_batch": {"desc_null": -3, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null7": -3, "null8": -3},
    "eb200_curve_mul_batch": {"desc_null": -3, "n0": 0, "null2": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_curve_validate_batch": {"desc_null": -3, "n0": 0, "null2": -3, "null3": -3},
    "eb200_ec_keygen_batch": {"curve77": -5, "n0": 0, "null2": -3, "null4": -3, "null6": -3, "null7": 0, "null8": -3},
    "eb200_ecdh_derive_batch": {"curve77": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3},
    "eb200_ecdsa_recover_batch": {"curve77": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3},
    "eb200_ecdsa_sign_batch": {"curve77": -5, "n0": 0, "null2": -3, "null3": -3, "null5": -3, "null6": -3, "null7": -3, "null8": -3},
    "eb200_ecdsa_sign_batch_k": {"curve77": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null6": -3, "null7": -3, "null8": -3, "null9": -3},
    "eb200_ecdsa_sign_batch_pers": {"curve77": -5, "n0": 0, "null10": -3, "null2": -3, "null3": -3, "null4": -3, "null7": -3, "null8": -3, "null9": -3},
    "eb200_ecdsa_verify_batch": {"curve77": -5, "fmt9": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null7": -3},
    "eb200_ecdsa_verify_batch_der": {"curve77": -5, "fmt9": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null7": -3},
    "eb200_ecdsa_verify_batch_dev": {"curve77": -5, "fmt9": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null7": -3, "null8": -3, "null9": -4},
    "eb200_eddsa_sign_batch": {"n0": 0, "null1": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_eddsa_verify_batch": {"n0": 0, "null1": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3},
    "eb200_eddsa_verify_batch_dev": {"n0": 0, "null1": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -4},
    "eb200_eddsa_verify_batch_msgs": {"n0": 0, "null1": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_last_timing": {"null0": -3},
    "eb200_mul_add_batch": {"curve77": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3},
    "eb200_scalar_mul_batch": {"curve77": -5, "n0": 0, "null2": -3, "null3": 0, "null4": -3, "null5": -3},
    "eb200_selftest_fe": {"curve77": -5, "n0": 0},
    "eb200_selftest_gtab": {"curve77": -5},
    "eb200_selftest_gtab_dims": {"curve77": -5, "null1": -3, "null2": -3, "null3": -3},
    "eb200_x25519_derive_batch": {"n0": 0, "null1": -3, "null2": -3, "null3": -3, "null4": -3},
    "eb200_x25519_derive_batch_dev": {"n0": 0, "null1": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -4},
    "eb200_x25519_mul_batch": {"n0": 0, "null1": -3, "null2": -3, "null3": -3, "null4": -3},
    "eb200_ecdh_derive_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "wrong_set": -3},
    "eb200_ecdh_derive_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                          "null7": -4, "wrong_set": -3},
    "eb200_ecdsa_recovery_param_batch": {"curve77": -5, "n0": 0, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                         "null7": -3},
    "eb200_ecdsa_recovery_param_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3,
                                               "null6": -3, "null7": -3, "wrong_set": -3},
    "eb200_ecdsa_recovery_param_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3,
                                                   "null6": -3, "null7": -3, "null8": -3, "null9": -4, "wrong_set": -3},
    "eb200_ecdsa_verify_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                       "wrong_set": -3},
    "eb200_ecdsa_verify_batch_keyed_der": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                           "wrong_set": -3},
    "eb200_ecdsa_verify_batch_keyed_der_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null5": -3, "null6": -3,
                                               "null7": -3, "null8": -3, "null9": -4, "wrong_set": -3},
    "eb200_ecdsa_verify_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                           "null7": -3, "null8": -4, "wrong_set": -3},
    "eb200_eddsa_sign_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                     "wrong_set": -3},
    "eb200_eddsa_sign_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null4": -3, "null5": -3, "null6": -3, "null7": -3,
                                         "null8": -3, "null9": -4, "wrong_set": -3},
    "eb200_eddsa_verify_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                       "wrong_set": -3},
    "eb200_eddsa_verify_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                           "null7": -3, "null8": -4, "wrong_set": -3},
    "eb200_eddsa_verify_batch_keyed_msgs": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3,
                                            "null6": -3, "null7": -3, "wrong_set": -3},
    "eb200_eddsa_verify_batch_keyed_msgs_dev": {"n0": 0, "null0": -3, "null10": -4, "null2": -3, "null3": -3, "null4": -3,
                                                "null6": -3, "null7": -3, "null8": -3, "null9": -3, "wrong_set": -3},
    "eb200_mul_add_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                  "wrong_set": -3},
    "eb200_mul_add_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                      "null7": -3, "null8": -4, "wrong_set": -3},
    "eb200_scalar_mul_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "wrong_set": -3},
    "eb200_scalar_mul_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3, "null6": -3,
                                         "null7": -4, "wrong_set": -3},
    "eb200_x25519_derive_batch_keyed": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3,
                                        "wrong_set": -3},
    "eb200_x25519_derive_batch_keyed_dev": {"n0": 0, "null0": -3, "null2": -3, "null3": -3, "null4": -3, "null5": -3,
                                            "null6": -3, "null7": -4, "wrong_set": -3},
}
# eb200_timing.launches after each call of launch_cases(): kernels launched per entry point x curve x mode
# (curve ids as in the header; fmtF: public-key format; 262921 items and `chunked`: cut into chunks; *_keyed: against
# sets of 16 keys, the ECDSA ones on the curve named)
LAUNCHES = {
    "curve_add/p256": 1, "curve_add/p384": 1, "curve_add/p521": 1,
    "curve_dbl/p256": 1, "curve_dbl/p384": 1, "curve_dbl/p521": 1,
    "curve_mul/p256": 1, "curve_mul/p384": 1, "curve_mul/p521": 1,
    "curve_mul_add/p256": 1, "curve_mul_add/p384": 1, "curve_mul_add/p521": 1,
    "curve_validate/p256": 1, "curve_validate/p384": 1, "curve_validate/p521": 1,
    "derive/1": 3, "derive/2": 3, "derive/3": 3, "derive/4": 1, "derive/6": 3, "derive/7": 3, "derive/8": 3,
    "eddsa_sign/pub0": 1, "eddsa_sign/pub1": 1,
    "eddsa_verify/256": 1, "eddsa_verify/262921": 5,
    "eddsa_verify_dev": 1,
    "eddsa_verify_msgs/256": 2, "eddsa_verify_msgs/262921": 10,
    "keygen/1/pers0": 2, "keygen/1/pers1": 2, "keygen/2/pers0": 2, "keygen/2/pers1": 2, "keygen/3/pers0": 2,
    "keygen/3/pers1": 2, "keygen/4/pers0": 2, "keygen/4/pers1": 2, "keygen/6/pers0": 2, "keygen/6/pers1": 2,
    "keygen/7/pers0": 2, "keygen/7/pers1": 2, "keygen/8/pers0": 2, "keygen/8/pers1": 2,
    "mul/1/points0": 1, "mul/1/points1": 3, "mul/2/points0": 1, "mul/2/points1": 3, "mul/3/points0": 1,
    "mul/3/points1": 3, "mul/4/points0": 1, "mul/4/points1": 1, "mul/6/points0": 1, "mul/6/points1": 3,
    "mul/7/points0": 1, "mul/7/points1": 3, "mul/8/points0": 1, "mul/8/points1": 3,
    "mul_add/1": 3, "mul_add/2": 3, "mul_add/3": 3, "mul_add/4": 1, "mul_add/6": 3, "mul_add/7": 3, "mul_add/8": 3,
    "recover/1": 2, "recover/2": 2, "recover/3": 2, "recover/6": 2, "recover/7": 2, "recover/8": 2,
    "sign/1/flags0": 3, "sign/1/flags1": 3, "sign/2/flags0": 3, "sign/2/flags1": 3, "sign/3/flags0": 3,
    "sign/3/flags1": 3, "sign/4/flags0": 1, "sign/4/flags1": 1, "sign/6/flags0": 3, "sign/6/flags1": 3,
    "sign/7/flags0": 3, "sign/7/flags1": 3, "sign/8/flags0": 3, "sign/8/flags1": 3,
    "sign_k/1": 3, "sign_k/2": 3, "sign_k/3": 3, "sign_k/4": 1, "sign_k/6": 3, "sign_k/7": 3, "sign_k/8": 3,
    "sign_pers/1/len0": 1, "sign_pers/1/len5": 1, "sign_pers/2/len0": 1, "sign_pers/2/len5": 1, "sign_pers/3/len0": 1,
    "sign_pers/3/len5": 1, "sign_pers/4/len0": 1, "sign_pers/4/len5": 1, "sign_pers/6/len0": 1, "sign_pers/6/len5": 1,
    "sign_pers/7/len0": 1, "sign_pers/7/len5": 1, "sign_pers/8/len0": 1, "sign_pers/8/len5": 1,
    "verify/1/chunked": 15, "verify/1/fmt0": 3, "verify/1/fmt1": 4, "verify/1/fmt2": 4, "verify/2/chunked": 15,
    "verify/2/fmt0": 3, "verify/2/fmt1": 4, "verify/2/fmt2": 4, "verify/3/fmt0": 3, "verify/3/fmt1": 4,
    "verify/3/fmt2": 4, "verify/4/fmt0": 1, "verify/4/fmt1": 2, "verify/4/fmt2": 2, "verify/6/fmt0": 3,
    "verify/6/fmt1": 4, "verify/6/fmt2": 4, "verify/7/fmt0": 3, "verify/7/fmt1": 4, "verify/7/fmt2": 4,
    "verify/8/fmt0": 3, "verify/8/fmt1": 4, "verify/8/fmt2": 4,
    "verify_der/1/fmt0": 4, "verify_der/1/fmt1": 5, "verify_der/1/fmt2": 5, "verify_der/2/fmt0": 4,
    "verify_der/2/fmt1": 5, "verify_der/2/fmt2": 5, "verify_der/3/fmt0": 4, "verify_der/3/fmt1": 5,
    "verify_der/3/fmt2": 5, "verify_der/4/fmt0": 2, "verify_der/4/fmt1": 3, "verify_der/4/fmt2": 3,
    "verify_der/6/fmt0": 4, "verify_der/6/fmt1": 5, "verify_der/6/fmt2": 5, "verify_der/7/fmt0": 4,
    "verify_der/7/fmt1": 5, "verify_der/7/fmt2": 5, "verify_der/8/fmt0": 4, "verify_der/8/fmt1": 5,
    "verify_der/8/fmt2": 5,
    "verify_dev/1/fmt0": 3, "verify_dev/1/fmt1": 4, "verify_dev/1/fmt2": 4, "verify_dev/2/fmt0": 3,
    "verify_dev/2/fmt1": 4, "verify_dev/2/fmt2": 4, "verify_dev/3/fmt0": 3, "verify_dev/3/fmt1": 4,
    "verify_dev/3/fmt2": 4, "verify_dev/4/fmt0": 1, "verify_dev/4/fmt1": 2, "verify_dev/4/fmt2": 2,
    "verify_dev/6/fmt0": 3, "verify_dev/6/fmt1": 4, "verify_dev/6/fmt2": 4, "verify_dev/7/fmt0": 3,
    "verify_dev/7/fmt1": 4, "verify_dev/7/fmt2": 4, "verify_dev/8/fmt0": 3, "verify_dev/8/fmt1": 4,
    "verify_dev/8/fmt2": 4,
    "x25519_derive/256": 1, "x25519_derive/262921": 5,
    "x25519_derive_dev": 1,
    "x25519_mul/256": 1, "x25519_mul/262921": 5,
    "derive_keyed/1/256": 4, "derive_keyed/1/262921": 20, "derive_keyed/2/256": 4, "derive_keyed/2/262921": 20,
    "derive_keyed_dev/1": 6, "derive_keyed_dev/2": 6, "eddsa_sign_keyed/256": 3, "eddsa_sign_keyed/262921": 15,
    "eddsa_sign_keyed_dev": 5, "eddsa_verify_keyed/256": 1, "eddsa_verify_keyed/262921": 5, "eddsa_verify_keyed_dev": 3,
    "eddsa_verify_keyed_msgs/256": 3, "eddsa_verify_keyed_msgs/262921": 15, "eddsa_verify_keyed_msgs_dev": 5,
    "mul_add_keyed/1/256": 4, "mul_add_keyed/1/262921": 20, "mul_add_keyed/2/256": 4, "mul_add_keyed/2/262921": 20,
    "mul_add_keyed_dev/1": 6, "mul_add_keyed_dev/2": 6, "mul_keyed/1/256": 4, "mul_keyed/1/262921": 20,
    "mul_keyed/2/256": 4, "mul_keyed/2/262921": 20, "mul_keyed_dev/1": 6, "mul_keyed_dev/2": 6,
    "recovery_param_keyed/1/256": 4, "recovery_param_keyed/1/262921": 20, "recovery_param_keyed/2/256": 4,
    "recovery_param_keyed/2/262921": 20, "recovery_param_keyed_dev/1": 6, "recovery_param_keyed_dev/2": 6,
    "verify_keyed/1/256": 3, "verify_keyed/1/262921": 15, "verify_keyed/2/256": 3, "verify_keyed/2/262921": 15,
    "verify_keyed_der/1/256": 5, "verify_keyed_der/1/262921": 25, "verify_keyed_der/2/256": 5,
    "verify_keyed_der/2/262921": 25, "verify_keyed_der_dev/1": 6, "verify_keyed_der_dev/2": 6, "verify_keyed_dev/1": 5,
    "verify_keyed_dev/2": 5, "x25519_derive_keyed/256": 2, "x25519_derive_keyed/262921": 10, "x25519_derive_keyed_dev": 4,
}


def test_c_abi_argument_and_error_behaviour(native):
    """The boundary's own contract (include/elliptic_b200.h): empty batches succeed without touching the output,
    NULL pointers and unknown curves / formats come back as error codes, never as a crash, and the library
    stays usable afterwards.  Every entry point's codes for those cases and its launch count per curve and mode
    are pinned in WITH_DEVICE and LAUNCHES."""
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    z = np.zeros((4, 64), np.uint8); st = np.full(4, 0xEE, np.uint8)
    assert lib.eb200_ecdsa_verify_batch(1, 0, None, None, None, None, 0, None) == nat.OK
    assert lib.eb200_ecdsa_verify_batch(1, 4, None, z.ctypes.data, z.ctypes.data, z.ctypes.data, 0, st.ctypes.data) == -3      # EB200_ERR_ARG
    assert lib.eb200_ecdsa_verify_batch(77, 4, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, 0, st.ctypes.data) == -5  # UNSUPPORTED
    assert lib.eb200_ecdsa_verify_batch(1, 4, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, 9, st.ctypes.data) == -5
    assert (st == 0xEE).all()
    assert lib.eb200_ecdsa_sign_batch(5, 4, z.ctypes.data, z.ctypes.data, 0, z.ctypes.data, z.ctypes.data, st.ctypes.data, st.ctypes.data) == -5
    assert lib.eb200_mul_add_batch(1, 4, None, z.ctypes.data, z.ctypes.data, z.ctypes.data, st.ctypes.data) == -3
    assert lib.eb200_strerror(-3).decode() == "invalid argument"
    # all-zero inputs are legal inputs: r = s = 0 -> FALSE for every item
    assert lib.eb200_ecdsa_verify_batch(1, 4, z.ctypes.data, z.ctypes.data, z.ctypes.data, z.ctypes.data, 0, st.ctypes.data) == nat.OK
    assert (st == 0).all()
    # every entry point: n == 0, NULL pointers, unknown curves / formats
    from abi_cases import argument_cases, launch_cases
    cases, _keep = argument_cases(with_device=True)
    got = {}
    for cid, call in cases:
        name, tag = cid.split("/")
        got.setdefault(name, {})[tag] = call(lib)
    assert got == WITH_DEVICE
    # the kernels each call launches, counted where they are launched
    cases, _keep = launch_cases()
    got = {}
    for cid, call in cases:
        assert call(lib) == nat.OK, cid
        got[cid] = nat.last_timing()["launches"]
    assert got == LAUNCHES, {k: (v, LAUNCHES.get(k)) for k, v in got.items() if LAUNCHES.get(k) != v}


def test_chunked_host_pipeline_equals_single_launch(native):
    """eb200_ecdsa_verify_batch splits batches of 2^18 and more into chunks on two alternating compute streams
    with per-chunk workspaces; an odd-sized batch must give the generator's statuses and exactly the statuses
    of the unchunked path (EB200_CHUNKS=1), for every chunk count the knob allows."""
    import os
    import benchdata
    from elliptic_b200.ec import EC as GpuEC
    n = (1 << 18) + 777
    ds = benchdata.gen_secp256k1_verify(n, cache_dir=benchdata.cache_dir())
    g = GpuEC("secp256k1")
    old = os.environ.get("EB200_CHUNKS")
    try:
        res = {}
        for chunks in ("1", "3", "4", "7", "16"):
            os.environ["EB200_CHUNKS"] = chunks
            res[chunks] = g.verify_batch_packed(ds["e"], ds["r"], ds["s"], ds["pub"]).copy()
        os.environ.pop("EB200_CHUNKS")
        res["default"] = g.verify_batch_packed(ds["e"], ds["r"], ds["s"], ds["pub"]).copy()
    finally:
        if old is None:
            os.environ.pop("EB200_CHUNKS", None)
        else:
            os.environ["EB200_CHUNKS"] = old
    for k, st in res.items():
        assert np.array_equal(st, ds["expected"]), k
