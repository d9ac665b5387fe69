/* elliptic_b200.h -- C ABI of libelliptic_b200.so, the drop-in boundary.
 *
 * The reference (indutny/elliptic, pure JavaScript) has no FFI of its own
 * (SURVEY.md 8b); these are the entry points an N-API addon for
 * `require('elliptic')` binds so that whole batches of the reference's
 * single-item calls run on H100 GPUs.  Each function names the reference
 * method whose per-item semantics it reproduces bit-exactly.
 *
 * Conventions: field elements / scalars are fixed-width big-endian byte
 * strings (32 bytes for secp256k1, the reference's toArray('be', len),
 * lib/elliptic/curve/base.js:298-306); arrays are item-major and contiguous
 * (item i of `r` is r[32*i .. 32*i+31]).  The caller owns every buffer.
 * Every function returns EB200_OK (0) or a negative error code; nothing
 * throws or aborts.  Per-item outcomes are written to `status`.
 * There is NO CPU fallback: without a usable CUDA device every compute entry
 * point returns EB200_ERR_NO_DEVICE.
 */
#ifndef ELLIPTIC_B200_H
#define ELLIPTIC_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define EB200_OK 0
#define EB200_ERR_NO_DEVICE (-1)   /* no CUDA device / driver */
#define EB200_ERR_CUDA (-2)        /* a CUDA call failed: eb200_last_error() */
#define EB200_ERR_ARG (-3)         /* bad argument (NULL buffer, unknown curve/format) */
#define EB200_ERR_NOT_INIT (-4)    /* eb200_init() has not succeeded */
#define EB200_ERR_UNSUPPORTED (-5) /* curve / format not built yet */

/* per-item status byte: what the reference's call would have done */
#define EB200_ST_FALSE 0                /* returned false */
#define EB200_ST_TRUE 1                 /* returned true */
#define EB200_ST_THROW_INVALID_POINT 2  /* threw Error('invalid point')  short.js:195, edwards.js:84 */
#define EB200_ST_THROW_NOT_VALIDATED 3  /* threw Error('public point not validated')  ec/key.js:104 */
#define EB200_ST_NEEDS_HOST 4           /* internal: the fast kernel's flag for an off-curve un-validated key
                                           (SURVEY 8a Q1).  Every verify entry point re-runs flagged items
                                           through an exact replay of the reference's own schedule on the GPU,
                                           so callers never see this value */
#define EB200_ST_THROW_ASSERT 5         /* threw Error('Assertion failed') (bn.js sqrt / hybrid parity) */
#define EB200_ST_THROW_POINT_FORMAT 6   /* threw Error('Unknown point format')  base.js:291 */
#define EB200_ST_INFINITY 7             /* (recover) returned the point at infinity */
#define EB200_ST_THROW_SECOND_KEY 8     /* (recover) threw Error('Unable to find sencond key candinate')  ec/index.js:244 */
#define EB200_ST_THROW_SIG_FORMAT 9     /* threw Error('Signature without r or s')  ec/signature.js:15 (DER rejected by _importDER) */
#define EB200_ST_RETRY 10               /* (sign with caller nonces) the reference's loop `continue`s: k outside [2, n-2], r = 0 or s = 0;
                                           the caller supplies its next k(iter), ec/index.js:153-185 */
#define EB200_ST_THROW_NO_RECOVERY 11   /* (getKeyRecoveryParam) threw Error('Unable to find valid recovery factor')  ec/index.js:277 */
#define EB200_ST_BAD_KEY_INDEX 12       /* (device-pointer keyed calls) key_idx[i] >= m: nothing was computed for the item */
#define EB200_ST_BAD_ITEM 13            /* (device-pointer keyed calls) an argument the host form refuses with EB200_ERR_ARG:
                                           nothing was computed for the item */

/* curve ids (names of lib/elliptic/curves.js presets) */
#define EB200_CURVE_SECP256K1 1
#define EB200_CURVE_P256 2
#define EB200_CURVE_P384 3
#define EB200_CURVE_ED25519 4
#define EB200_CURVE_CURVE25519 5
#define EB200_CURVE_P521 6       /* 66-byte fields; verify / recover / mul / mulAdd / derive */
#define EB200_CURVE_P192 7       /* 24-byte fields; same entry points as p521 */
#define EB200_CURVE_P224 8       /* 28-byte fields; p = 1 mod 4: compressed keys go through bn.js's Tonelli-Shanks */

/* public-key encodings accepted by eb200_ecdsa_verify_batch (KeyPair._importPublic,
 * lib/elliptic/ec/key.js:84-99 -> BaseCurve.decodePoint, curve/base.js:270-292) */
#define EB200_PUB_XY 0          /* {x, y}: 2*len bytes per item, NOT validated (as the reference) */
#define EB200_PUB_SEC1_65 1     /* 04|06|07 || x || y : 1+2*len bytes per item */
#define EB200_PUB_SEC1_33 2     /* 02|03 || x : 1+len bytes per item (pointFromX, short.js:187-204) */

typedef struct eb200_timing {
  float h2d_ms;     /* host->device copies of the last host-buffer call */
  float kernel_ms;  /* all kernels of the last call (CUDA events on the launch stream) */
  float d2h_ms;     /* device->host copy of the results */
  float main_kernel_ms; /* the dominant kernel only */
  uint32_t launches; /* kernels launched by the last call */
} eb200_timing;

/* Create (or keep) one context per listed CUDA ordinal and build the fixed-base tables there
 * (SURVEY 8b: eb200_init(devices[], ndev, flags)).  devices == NULL or ndev <= 0: every visible device.
 * Idempotent per device; later calls add devices.  Host-pointer entry points split a batch into contiguous
 * blocks over the initialised devices (no exchange between blocks, SURVEY 8e) when it has at least 2^14 items per
 * device, each block driven by its own host thread; smaller calls take one device, rotating, so that concurrent
 * callers spread out.  Device-pointer (`_dev`) entry points run on the device that owns `d_status`.
 * Every entry point is safe to call from several threads. */
#define EB200_INIT_ALL_TABLES 1u   /* build every curve's fixed-base table now instead of on first use */
int eb200_init(const int* devices, int ndev, uint32_t flags);
int eb200_shutdown(void);
int eb200_device_count(void);          /* devices initialised so far */
const char* eb200_strerror(int code);
const char* eb200_last_error(void);   /* text of the last CUDA error on this thread's context */
int eb200_last_timing(eb200_timing* out);

/* Batch of EC.prototype.verify (lib/elliptic/ec/index.js:188-229) for `curve`.
 *   e   : n x len  message hashes already truncated as _truncateToN does for a len-byte
 *                  input (ec/index.js:81-108); values >= n are accepted like the reference
 *   r,s : n x len  signature halves (Signature{r,s}, ec/signature.js:8-22)
 *   pub : n x (pub_fmt-dependent) public keys
 *   status : n bytes out
 * Host pointers (pinned or pageable: pageable buffers are staged through an internal pinned ring with a
 * parallel memcpy, so an unpinned caller such as a Node.js Buffer gets the pinned transfer rate); copies are done internally on the library's stream. */
int eb200_ecdsa_verify_batch(int curve, size_t n, const uint8_t* e, const uint8_t* r,
                             const uint8_t* s, const uint8_t* pub, uint32_t pub_fmt,
                             uint8_t* status);

/* Same call with the signatures as the reference takes them off the wire: DER (`new Signature(der)`,
 * lib/elliptic/ec/signature.js:73-134), parsed on the GPU.
 *   sigs    : the DER encodings back to back
 *   sig_off : n + 1 byte offsets into `sigs` (item i is sigs[sig_off[i] .. sig_off[i+1]))
 * status adds THROW_SIG_FORMAT for an encoding _importDER rejects; a key that throws takes precedence
 * (keyFromPublic runs before new Signature, ec/index.js:194-195). */
int eb200_ecdsa_verify_batch_der(int curve, size_t n, const uint8_t* e, const uint8_t* sigs, const uint64_t* sig_off,
                                 const uint8_t* pub, uint32_t pub_fmt, uint8_t* status);

/* Same, with DEVICE pointers and a caller-supplied CUDA stream (cudaStream_t cast to void*;
 * NULL = the CUDA default stream).  Asynchronous: the caller synchronises the stream.
 * `workspace` must hold eb200_ecdsa_verify_workspace_bytes(curve, n) bytes of device memory. */
size_t eb200_ecdsa_verify_workspace_bytes(int curve, size_t n);
int eb200_ecdsa_verify_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r,
                                 const uint8_t* d_s, const uint8_t* d_pub, uint32_t pub_fmt,
                                 uint8_t* d_status, void* d_workspace, void* stream);

/* Batch of EC.prototype.sign (lib/elliptic/ec/index.js:110-186) on every short preset (len = the curve's field
 * byte length), with the curve's default hash (sha256; sha384 on p384, sha512 on p521; curves.js:43-206) and no
 * `pers` / custom `k`:
 * the RFC 6979 nonces come from HMAC-DRBG over that hash, generated on the GPU.
 *   e    : n x len  _truncateToN(msg) (ec/index.js:127) including its final `- n`, i.e. e < n, big-endian
 *   priv : n x len  private scalars as the key pair holds them (reduced mod n at import, ec/key.js:76-82)
 *   flags: EB200_SIGN_CANONICAL = the `canonical` option (s <= n/2, recovery bit flipped)
 *   out_r, out_s : n x len big-endian; out_recid : n bytes (recoveryParam)
 * status: TRUE for every item (the reference's retry loop runs inside the kernel). */
#define EB200_SIGN_CANONICAL 1u
int eb200_ecdsa_sign_batch(int curve, size_t n, const uint8_t* e, const uint8_t* priv, uint32_t flags,
                           uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid, uint8_t* status);

/* Batch of EC.prototype.recoverPubKey (lib/elliptic/ec/index.js:231-259) on secp256k1 / p256 / p384 / p521
 * (len = 32 / 32 / 48 / 66 in place of the 32 and 64 below):
 *   e     : n x 32  `new BN(msg)` reduced mod n (NOT truncated -- the reference does not truncate here)
 *   r, s  : n x 32  signature halves (no range check in the reference: r = 0 yields the point at infinity)
 *   recid : n bytes, the recovery parameter j in 0..3 (bit 0 = y parity, bit 1 = use r + n)
 *   out_xy: n x 64  recovered public key x || y big-endian (zeroed unless status is TRUE)
 * status: TRUE (point written), INFINITY, THROW_INVALID_POINT (pointFromX, short.js:195), THROW_SECOND_KEY. */
int eb200_ecdsa_recover_batch(int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                              const uint8_t* recid, uint8_t* out_xy, uint8_t* status);

/* Batch of EC.prototype.getKeyRecoveryParam (lib/elliptic/ec/index.js:261-278) on the six short presets: the first j in
 * 0..3 whose recoverPubKey(e, sig, j) equals Q.  One double-scalar multiplication per item instead of up to four
 * recoveries: the groups have prime order, so r^-1 (s R - e G) = Q exactly when R = s^-1 (e G + r Q).
 *   e, r, s : n x len as eb200_ecdsa_recover_batch takes them (e reduced mod n; r, s any value below 2^(8 len))
 *   q_xy    : n x 2len public points x || y big-endian, reduced mod p like curve.point; not validated (an off-curve Q
 *             never equals a recovered point)
 *   out_recid : n bytes, the parameter 0..3 (0 unless status is TRUE)
 * status: TRUE or THROW_NO_RECOVERY.  The caller answers a signature that already carries its recoveryParam
 * (ec/index.js:263-264).  ed25519: EB200_ERR_UNSUPPORTED, as recover. */
int eb200_ecdsa_recovery_param_batch(int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                                     const uint8_t* q_xy, uint8_t* out_recid, uint8_t* status);

/* Batch of BasePoint.mul (lib/elliptic/curve/short.js:422-432) on secp256k1 / p256 / p384 (len = 32/32/48):
 *   k         : n x len big-endian scalars, any value below 2^(8 len) (the reference does not reduce them)
 *   points_xy : n x 2len x || y big-endian, or NULL for the base point (G.mul(k) -> _fixedNafMul, base.js:52-84)
 *   out_xy    : n x 2len affine result as Point.toP / getX / getY give it (zeroed unless status is TRUE)
 * status: TRUE (point written) or INFINITY.  Points are not validated, exactly as `curve.point(x, y)`
 * (short.js:251-271); an off-curve point gets the result of the reference's own add/double sequence. */
int eb200_scalar_mul_batch(int curve, size_t n, const uint8_t* k, const uint8_t* points_xy, uint8_t* out_xy,
                           uint8_t* status);

/* Batch of KeyPair.prototype.derive (lib/elliptic/ec/key.js:102-107) on the short curves: ECDH shared x.
 *   priv   : n x len private scalars, big-endian (reduced mod n as _importPrivate does, ec/key.js:76-82)
 *   pub_xy : n x 2len peer points x || y
 *   out_x  : n x len  pub.mul(priv).getX(), big-endian (zeroed unless status is TRUE)
 * status: TRUE, THROW_NOT_VALIDATED (the peer point is not on the curve), INFINITY (priv = 0 mod n: the
 * reference then dies with a TypeError inside getX()).  curve25519 has its own entry point below. */
int eb200_ecdh_derive_batch(int curve, size_t n, const uint8_t* priv, const uint8_t* pub_xy, uint8_t* out_x,
                            uint8_t* status);

/* Batch of G.mulAdd(k1, P2, k2) = k1*G + k2*P2 (lib/elliptic/curve/short.js:434-441; _endoWnafMulAdd
 * short.js:218-249 on secp256k1, _wnafMulAdd base.js:128-253 on p256 / p384).  Arguments and status as
 * eb200_scalar_mul_batch. */
int eb200_mul_add_batch(int curve, size_t n, const uint8_t* k1, const uint8_t* k2, const uint8_t* p2_xy,
                        uint8_t* out_xy, uint8_t* status);

/* Batch of EDDSA.prototype.verify (lib/elliptic/eddsa/index.js:52-63) on ed25519.
 *   R, S : the two 32-byte halves of each signature as on the wire (eddsa/signature.js:17-40)
 *   A    : 32-byte encoded public keys (eddsa/key.js:17-30)
 *   h    : SHA512(R || A || M) as a little-endian integer reduced mod n, 32 bytes LE (hashInt,
 *          eddsa/index.js:65-70) -- computed by the caller (the host wrapper hashes with hashlib /
 *          the N-API shim with hash.js); h MUST be < n.
 * status: TRUE / FALSE, or THROW_INVALID_POINT / THROW_ASSERT where the reference throws while
 * decoding R or A (edwards.js:84, bn.js Red.sqrt assertion). */
int eb200_eddsa_verify_batch(size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* A,
                             const uint8_t* h, uint8_t* status);
/* Same, hashing on the GPU: msgs = all messages concatenated, message i = msgs[msg_off[i] .. msg_off[i+1])
 * (msg_off has n+1 entries).  h = SHA512(R || A || M) mod n is computed in a first kernel. */
int eb200_eddsa_verify_batch_msgs(size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* A,
                                  const uint8_t* msgs, const uint64_t* msg_off, uint8_t* status);
size_t eb200_eddsa_verify_workspace_bytes(size_t n);
int eb200_eddsa_verify_batch_dev(size_t n, const uint8_t* d_R, const uint8_t* d_S, const uint8_t* d_A,
                                 const uint8_t* d_h, uint8_t* d_status, void* d_workspace, void* stream);

/* Batch of KeyPair.prototype.derive (lib/elliptic/ec/key.js:102-107) on curve25519:
 *   priv : n x 32 bytes big-endian, the key pair's private scalar as the reference holds it
 *          (reduced mod n at import, ec/key.js:76-82; no clamping)
 *   pubx : n x 32 bytes big-endian x coordinate of the peer point (mont.js:46-48 decodePoint)
 *   out  : n x 32 bytes big-endian shared x (BN -> toArray('be', 32)); zeroed when the call throws
 * status: TRUE = value returned; THROW_ASSERT = the reference throws inside validate()
 *         (twist point: Red.sqrt assertion, mont.js:21-28). */
int eb200_x25519_derive_batch(size_t n, const uint8_t* priv, const uint8_t* pubx, uint8_t* out, uint8_t* status);
int eb200_x25519_derive_batch_dev(size_t n, const uint8_t* d_priv, const uint8_t* d_pubx, uint8_t* d_out,
                                  uint8_t* d_status, void* stream);

/* EC.prototype.sign with the `k` option (options.k(iter), lib/elliptic/ec/index.js:154-157): one attempt of the
 * reference's loop with the caller's nonces.  k: n x len bytes big-endian, what k(iter) returned (it goes through
 * _truncateToN(k, true) here).  status: EB200_ST_TRUE, or EB200_ST_RETRY where the reference would call k(iter + 1). */
int eb200_ecdsa_sign_batch_k(int curve, size_t n, const uint8_t* e, const uint8_t* priv, const uint8_t* k, uint32_t flags,
                             uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid, uint8_t* status);
/* EC.prototype.sign with the `pers` option (ec/index.js:143-151): HMAC-DRBG seeded with key || msg || pers; pers is the
 * personalisation string after `persEnc` decoding, shared by the whole batch. */
int eb200_ecdsa_sign_batch_pers(int curve, size_t n, const uint8_t* e, const uint8_t* priv, const uint8_t* pers, size_t pers_len,
                                uint32_t flags, uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid, uint8_t* status);
/* EC.prototype.genKeyPair({entropy, pers}) (ec/index.js:55-79): per item HMAC-DRBG(hash, entropy_i, nonce = n.toArray(),
 * pers), the first candidate <= n - 2 plus one as the private key, and its public point.
 *   entropy : n x entropy_len bytes (the reference requires >= hmacStrength / 8 = 24);  out_priv : n x len;
 *   out_pub_xy : n x 2 len or NULL */
int eb200_ec_keygen_batch(int curve, size_t n, const uint8_t* entropy, size_t entropy_len, const uint8_t* pers, size_t pers_len,
                          uint8_t* out_priv, uint8_t* out_pub_xy, uint8_t* status);

/* The `ec` / `.curve` API over the other two curve types of lib/elliptic/curves.js:
 *  - EB200_CURVE_ED25519 is accepted by eb200_ecdsa_verify_batch (+ _der, SEC1 formats: BaseCurve.decodePoint and
 *    EdwardsCurve.pointFromX, edwards.js:46-69), eb200_ecdsa_sign_batch (+ _k, _pers), eb200_ec_keygen_batch,
 *    eb200_scalar_mul_batch / eb200_mul_add_batch (Point.mul / mulAdd, edwards.js:362-375; 32-byte big-endian x || y,
 *    the neutral element is the ordinary point (0, 1); the point's scalar is used as given, any value below 2^256, so
 *    that k P is exact for points with a torsion component too (the group has order 8n), and G's scalar is reduced
 *    mod n) and eb200_ecdh_derive_batch: new elliptic.ec('ed25519')
 *    (test/ecdsa-test.js:130, test/ecdh-test.js:26; eqXToP edwards.js:415-431).  An un-validated off-curve point is
 *    reported as EB200_ST_NEEDS_HOST (the reference's answer then depends on its own wNAF schedule, which is not
 *    replayed for this curve); eb200_ecdsa_recover_batch returns EB200_ERR_UNSUPPORTED.
 *  - curve25519 points are x-only: eb200_x25519_mul_batch is MontCurve Point.mul(k).getX() (mont.js:130-153) without
 *    the validation that eb200_x25519_derive_batch (KeyPair.derive) performs; mulAdd throws in the reference. */
int eb200_x25519_mul_batch(size_t n, const uint8_t* k, const uint8_t* px, uint8_t* out_x, uint8_t* status);

/* Short Weierstrass curves given at run time -- the batch form of `new elliptic.curve.short({p, a, b})`
 * (lib/elliptic/curve/short.js:10-24) and of Point.mul / mulAdd / add / dbl / validate on its points
 * (short.js:365-450, 206-216).  p: any odd prime > 3 of up to 576 bits; p, a, b: `len` bytes big-endian; points:
 * x || y, `len` bytes each (values >= p are reduced on entry like toRed); scalars: `klen` bytes big-endian, any value.
 * status: EB200_ST_TRUE = affine point written, EB200_ST_INFINITY = the point at infinity (output zeroed),
 * EB200_ST_NEEDS_HOST = an input does not satisfy the curve equation (the reference does not validate and its result
 * is then an artefact of its own schedule: not accelerated); validate: EB200_ST_TRUE / EB200_ST_FALSE.
 * The six presets keep their tuned entry points above; this generic path is not tuned (one thread per item,
 * double-and-add). */
typedef struct eb200_short_curve { uint32_t len; const uint8_t* p; const uint8_t* a; const uint8_t* b; } eb200_short_curve;
int eb200_curve_mul_batch(const eb200_short_curve* curve, size_t n, const uint8_t* k, size_t klen, const uint8_t* points_xy,
                          uint8_t* out_xy, uint8_t* status);
int eb200_curve_mul_add_batch(const eb200_short_curve* curve, size_t n, const uint8_t* k1, const uint8_t* p1_xy, const uint8_t* k2,
                              const uint8_t* p2_xy, size_t klen, uint8_t* out_xy, uint8_t* status);
int eb200_curve_add_batch(const eb200_short_curve* curve, size_t n, const uint8_t* p1_xy, const uint8_t* p2_xy, uint8_t* out_xy,
                          uint8_t* status);
int eb200_curve_dbl_batch(const eb200_short_curve* curve, size_t n, const uint8_t* p_xy, uint8_t* out_xy, uint8_t* status);
int eb200_curve_validate_batch(const eb200_short_curve* curve, size_t n, const uint8_t* p_xy, uint8_t* status);

/* Batch of EDDSA.prototype.sign (lib/elliptic/eddsa/index.js:34-44) with keys given as 32-byte secrets
 * (eddsa.keyFromSecret, eddsa/key.js:52-75: SHA-512 of the secret, clamped scalar, message prefix).
 *   secrets : n x 32 bytes;  msgs / msg_off : concatenated raw messages and n + 1 offsets
 *   out_sig : n x 64 bytes  Rencoded || S (little-endian), byte-identical to sig.toBytes()
 *   out_pub : n x 32 bytes  key.getPublic('bytes'), or NULL
 *   status  : n bytes, always EB200_ST_TRUE (the reference cannot fail on a 32-byte secret)
 * Everything (three SHA-512 per item, two fixed-base multiplications, the arithmetic mod n) runs on the GPU. */
int eb200_eddsa_sign_batch(size_t n, const uint8_t* secrets, const uint8_t* msgs, const uint64_t* msg_off,
                           uint8_t* out_sig, uint8_t* out_pub, uint8_t* status);

/* Key sets: the batch form of the reference's key objects -- `key = ec.keyFromPublic(pub, enc)` once,
 * `key.getPublic().precompute()` (lib/elliptic/curve/base.js:312-327), then `key.verify(msg, sig)` many times
 * (lib/elliptic/ec/key.js:20-28, 84-99, 114-116).  A set holds m public keys of one short preset (secp256k1, p256, p384,
 * p521, p192, p224; the 25519 curves return EB200_ERR_UNSUPPORTED here: ed25519 EdDSA keys have
 * eb200_eddsa_keyset_create and curve25519 ECDH keys eb200_x25519_keyset_create below) on the GPU: decoded once, checked
 * against the curve
 * once, and each on-curve key with a table of its multiples (2i+1) 2^(W j) Q over W-bit windows, so that a keyed verify
 * needs no doubling and no per-item table.
 *   pub, pub_fmt : m keys, exactly what eb200_ecdsa_verify_batch takes
 *   table_bits   : the window width W, EB200_KEYSET_MIN_BITS..EB200_KEYSET_MAX_BITS, or 0 for the widest of them whose
 *                  tables (m * (floor(mbits / W) + 1) * 2^(W-1) entries of x || y limbs; mbits = 131 on secp256k1, whose
 *                  windows cover a GLV half, else bits(n) - 1) fit EB200_KEYSET_DEFAULT_BUDGET bytes per device.  If
 *                  not even the narrowest fits, or for any other value: EB200_ERR_ARG (an explicit width is not held
 *                  to the budget; there is no silent fallback to the unkeyed path)
 *   key_status   : m bytes out -- EB200_ST_THROW_* = keyFromPublic throws that error; EB200_ST_TRUE = imported and
 *                  pub.validate() is true; EB200_ST_FALSE = imported but off the curve ({x, y} and uncompressed keys
 *                  are not validated by the reference)
 * The tables are built on every device initialised at the time of the call and the keyed calls stay on those devices;
 * a device added by a later eb200_init does not serve this set.  A failed allocation returns EB200_ERR_CUDA, leaves
 * *out NULL and frees what it had allocated.  m = 0, m >= 2^32 or a NULL pointer: EB200_ERR_ARG.
 * eb200_last_timing after create: kernel_ms = main_kernel_ms = the build kernels of the slowest device; launches = 3
 * per device (4 with a SEC1 format: the decoder).
 * A set is read-only once created: several threads may verify against it at once and several sets may be alive.
 * Destroying a set while a call uses it is the caller's error.  eb200_shutdown frees the device memory of surviving
 * sets; their handles then answer EB200_ERR_NOT_INIT and must still be passed to eb200_keyset_destroy. */
#define EB200_KEYSET_MIN_BITS 4
#define EB200_KEYSET_MAX_BITS 8
#define EB200_KEYSET_DEFAULT_BUDGET ((size_t)1 << 30)
typedef struct eb200_keyset eb200_keyset;
int eb200_keyset_create(int curve, size_t m, const uint8_t* pub, uint32_t pub_fmt, uint32_t table_bits,
                        uint8_t* key_status, eb200_keyset** out);
/* Any out pointer may be NULL.  device_bytes: what the set holds on EACH of its devices. */
int eb200_keyset_info(const eb200_keyset* ks, int* curve, size_t* m, uint32_t* table_bits, size_t* device_bytes);
int eb200_keyset_destroy(eb200_keyset* ks);          /* NULL is a no-op returning EB200_OK */

/* Batch of key.verify(msg, sig): item i is checked against key key_idx[i] of the set.  e, r, s as
 * eb200_ecdsa_verify_batch takes them (host pointers, sharded over the set's devices).  status[i] is exactly the byte
 * eb200_ecdsa_verify_batch writes for the same e, r, s with pub[i] = key key_idx[i] in the set's format: the key's throw
 * first, then TRUE / FALSE, and for an off-curve key the reference's schedule-dependent answer, replayed on the GPU from
 * the key's coordinates.  A key_idx[i] >= m returns EB200_ERR_ARG before anything is written.
 * eb200_last_timing: main_kernel_ms = the keyed main kernel; launches = 3 per chunk (prep, main, replay).
 * The same call takes DER signatures (eb200_ecdsa_verify_batch_keyed_der) and device pointers on the caller's stream
 * (eb200_ecdsa_verify_batch_keyed_dev), below. */
int eb200_ecdsa_verify_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* e, const uint8_t* r,
                                   const uint8_t* s, const uint32_t* key_idx, uint8_t* status);

/* Keyed verify of DER signatures off the wire, parsed on the GPU: e, sigs and sig_off as eb200_ecdsa_verify_batch_der
 * takes them (n + 1 absolute offsets).  status[i] is exactly the byte eb200_ecdsa_verify_batch_der writes for the same e
 * and DER with pub[i] = key key_idx[i] in the set's format; the first of these that applies: the key's import throw
 * (keyFromPublic runs before new Signature, ec/index.js:194-195), THROW_SIG_FORMAT for an encoding _importDER rejects,
 * FALSE for r or s out of range, then the keyed verify's TRUE / FALSE (for an off-curve key, the keyed replay's answer).
 * An EdDSA, signing or curve25519 set, a NULL pointer, decreasing offsets or a key_idx[i] >= m returns EB200_ERR_ARG;
 * a set released by eb200_shutdown EB200_ERR_NOT_INIT; both before anything is written.  n = 0 returns EB200_OK.
 * Host pointers, sharded over the set's devices and chunked with copy / compute overlap as eb200_ecdsa_verify_batch_keyed.
 * eb200_last_timing: main_kernel_ms = the keyed main kernel; launches = 5 per chunk (keyed DER decode, prep, keyed main,
 * keyed replay, verdict merge). */
int eb200_ecdsa_verify_batch_keyed_der(const eb200_keyset* ks, size_t n, const uint8_t* e, const uint8_t* sigs,
                                       const uint64_t* sig_off, const uint32_t* key_idx, uint8_t* status);

/* Keyed verify with DEVICE pointers (e, r, s: n x len; key_idx: n words; status: n bytes) on a caller-supplied CUDA
 * stream (cudaStream_t cast to void*; NULL = the CUDA default stream), on the device that owns d_status.  Asynchronous,
 * as eb200_ecdsa_verify_batch_dev: the caller synchronises the stream.  d_workspace must hold
 * eb200_ecdsa_verify_keyed_workspace_bytes(ks, n) bytes of device memory on that device (0 for NULL or a set that is not
 * an ECDSA set).  For d_key_idx[i] < m, d_status[i] is exactly what eb200_ecdsa_verify_batch_keyed writes; an index >= m
 * cannot be refused before launch without synchronising the caller's stream, so its item gets EB200_ST_BAD_KEY_INDEX
 * and the index never addresses the set.  Returned before any launch: EB200_ERR_ARG for an EdDSA, signing or
 * curve25519 set, a NULL pointer, or d_status on an initialised device that does not hold this set (one added after
 * the set was created); EB200_ERR_NOT_INIT for a set released by eb200_shutdown or d_status on a device eb200_init has
 * not set up.  n = 0 returns EB200_OK.
 * eb200_last_timing (after the caller has synchronised the stream): kernel_ms = the whole call, main_kernel_ms = the keyed
 * main kernel; launches = 5 (index screen, prep, keyed main, keyed replay, verdict merge). */
size_t eb200_ecdsa_verify_keyed_workspace_bytes(const eb200_keyset* ks, size_t n);
int eb200_ecdsa_verify_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_e, const uint8_t* d_r,
                                       const uint8_t* d_s, const uint32_t* d_key_idx, uint8_t* d_status,
                                       void* d_workspace, void* stream);

/* Point.mul / G.mulAdd / KeyPair.derive against the keys of a set (`pub = key.getPublic(); pub.precompute()` once, then
 * `pub.mul(k)`, `G.mulAdd(k1, pub, k2)`, `keyPair.derive(pub)` many times; curve/short.js:422-441, ec/key.js:102-107):
 * item i uses key key_idx[i].  For a key that imported (key_status TRUE or FALSE), out and status[i] are byte for byte
 * what eb200_scalar_mul_batch / eb200_mul_add_batch / eb200_ecdh_derive_batch write for the same scalars with the point
 * = that key's decoded x || y; for a key whose import threw, status[i] is that throw and the output is zeroed.  Scalars
 * are any value below 2^(8 len), as in the unkeyed calls (an on-curve key reduces them mod n; k = 0 mod n gives
 * INFINITY).  An off-curve key (an {x, y} or uncompressed key is not validated) follows the UNKEYED call: mul / mulAdd
 * replay the unkeyed call's schedule for an arbitrary point on the key's coordinates, derive is THROW_NOT_VALIDATED.
 * That is not the reference's _fixedNafMul schedule for a precomputed point, whose answer for an off-curve point
 * differs; eb200_ecdsa_verify_batch_keyed follows the same convention.
 * An EdDSA or curve25519 set, a key_idx[i] >= m or a NULL pointer: EB200_ERR_ARG; a set whose devices eb200_shutdown
 * released: EB200_ERR_NOT_INIT; both before anything is written.  n = 0: EB200_OK.  Host pointers, sharded over the set's
 * devices and chunked with copy / compute overlap as eb200_ecdsa_verify_batch_keyed.  derive clears the private scalars, their
 * digit words and the Jacobian results from the library's device buffers before it returns.
 * eb200_last_timing: main_kernel_ms = the keyed main kernel; launches = 4 per chunk (scalar prep, keyed main, batched
 * normalisation to affine, then the keyed replay of off-curve-key items, or for derive the status map). */
int eb200_scalar_mul_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* k, const uint32_t* key_idx, uint8_t* out_xy,
                                 uint8_t* status);
int eb200_mul_add_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* k1, const uint8_t* k2, const uint32_t* key_idx,
                              uint8_t* out_xy, uint8_t* status);
int eb200_ecdh_derive_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* priv, const uint32_t* key_idx, uint8_t* out_x,
                                  uint8_t* status);

/* getKeyRecoveryParam against the keys of a set (`ec.getKeyRecoveryParam(msg, sig, key.getPublic())`, ec/index.js:261-278,
 * for a signer that does not report the recovery bit): item i uses key key_idx[i].  e, r, s as
 * eb200_ecdsa_recovery_param_batch takes them (e reduced mod n; r, s any value below 2^(8 len)).  For a key
 * that imported (key_status TRUE or FALSE), out_recid[i] and status[i] are byte for byte what
 * eb200_ecdsa_recovery_param_batch writes with q = that key's decoded x || y: an off-curve key gets THROW_NO_RECOVERY (a
 * recovered point is always on the curve), so no item is replayed.  For a key whose import threw, status[i] is that
 * throw and out_recid[i] = 0.  u1 G + u2 Q comes from the key's table and the fixed table without doublings, and the
 * parity of y from one inversion per batch of items.
 * Argument and lifetime contract as eb200_scalar_mul_batch_keyed: an EdDSA or curve25519 set, a key_idx[i] >= m or a
 * NULL pointer:
 * EB200_ERR_ARG; a set whose devices eb200_shutdown released: EB200_ERR_NOT_INIT; both before anything is written.
 * n = 0: EB200_OK.  Host pointers, sharded over the set's devices and chunked with copy / compute overlap.
 * eb200_last_timing: main_kernel_ms = the keyed main kernel; launches = 4 per chunk (the unkeyed call's scalar prep,
 * keyed main, recid normalisation, then the cold kernel for s = 0 (mod n)). */
int eb200_ecdsa_recovery_param_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* e, const uint8_t* r,
                                           const uint8_t* s, const uint32_t* key_idx, uint8_t* out_recid, uint8_t* status);

/* EdDSA key sets: `key = eddsa.keyFromPublic(bytes)` once, then `eddsa.verify(msg, sig, key)` many times
 * (lib/elliptic/eddsa/index.js:52-63, eddsa/key.js:17-44), on ed25519.  The handle is the same eb200_keyset: _info
 * reports EB200_CURVE_ED25519, _destroy and eb200_shutdown treat it as any other set, and passing it to
 * eb200_ecdsa_verify_batch_keyed (or an ECDSA set to the calls below) returns EB200_ERR_ARG.
 *   A          : m x 32 encoded public keys, kept as given (hashInt reads key.pubBytes(), which for a key made from
 *                bytes is those bytes, a non-canonical y >= p included)
 *   table_bits : W = EB200_KEYSET_MIN_BITS..EB200_KEYSET_MAX_BITS, or 0 for the widest whose tables fit
 *                EB200_KEYSET_DEFAULT_BUDGET bytes per device; a key's table is ceil(253 / W) windows of 2^(W-1) affine
 *                niels entries i 2^(W j) (-A) of 96 bytes (W = 7: 227,328 bytes, 4,723 keys per GiB).  Otherwise as
 *                eb200_keyset_create: no width fits -> EB200_ERR_ARG, an explicit width is not held to the budget.
 *   key_status : m bytes out -- EB200_ST_TRUE = the key decodes, else the throw of decoding it (THROW_INVALID_POINT,
 *                THROW_ASSERT).  There is no FALSE verdict: a decoded key is on the curve.
 * m = 0, m >= 2^32 or a NULL pointer: EB200_ERR_ARG; no device: EB200_ERR_NOT_INIT; a failed allocation: EB200_ERR_CUDA
 * with *out NULL and everything freed.  device_bytes = 32 m + m + the tables.  eb200_last_timing after create: the
 * build kernels of the slowest device; launches = 3 per device (classify, window bases, table windows). */
int eb200_eddsa_keyset_create(size_t m, const uint8_t* A, uint32_t table_bits, uint8_t* key_status, eb200_keyset** out);
/* Batch of eddsa.verify against the set: item i uses key key_idx[i].  R, S, h as eb200_eddsa_verify_batch takes them;
 * status[i] is the byte eb200_eddsa_verify_batch writes for the same R, S, h and A = that key's bytes, in the reference's
 * order: S >= n -> FALSE, then R's throw, then the key's, then TRUE / FALSE.  A key_idx[i] >= m or an h[i] >= n returns
 * EB200_ERR_ARG before anything is written.  Host pointers, sharded over the set's devices and chunked as the unkeyed
 * call.  eb200_last_timing: main_kernel_ms = the keyed main kernel; launches = 1 per chunk. */
int eb200_eddsa_verify_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* h,
                                   const uint32_t* key_idx, uint8_t* status);
/* Same from raw messages, as eb200_eddsa_verify_batch_msgs takes them: h = SHA512(R || A_raw[key_idx[i]] || M) mod n on
 * the GPU.  launches = 3 per chunk (key-byte gather, hash, keyed main). */
int eb200_eddsa_verify_batch_keyed_msgs(const eb200_keyset* ks, size_t n, const uint8_t* R, const uint8_t* S,
                                        const uint8_t* msgs, const uint64_t* msg_off, const uint32_t* key_idx,
                                        uint8_t* status);

/* EdDSA signing sets: `key = eddsa.keyFromSecret(secret)` once, then `key.sign(msg)` many times (lib/elliptic/eddsa/
 * key.js:40-75, eddsa/index.js:34-44), on ed25519.  Create runs, per key, SHA-512 of the secret, the clamp, the message
 * prefix and A = a G, and encodes A, all on the GPU.  The set keeps a, the 32-byte prefix and the 32 bytes of A on each
 * device, not the secret: device_bytes = 96 m.  The handle is the same eb200_keyset: _info reports EB200_CURVE_ED25519
 * and table_bits = 0 (no table width applies), _destroy and eb200_shutdown treat it as any other set and clear its
 * secret words before they free them.  A signing set passed to any verify / mul / derive keyed call, or a public-key
 * set passed to eb200_eddsa_sign_batch_keyed, returns EB200_ERR_ARG.
 *   secrets : m x 32 bytes;  out_pub : m x 32 bytes key.getPublic('bytes'), or NULL
 * m = 0, m >= 2^32 or a NULL secrets / out: EB200_ERR_ARG; no device: EB200_ERR_NOT_INIT; a failed allocation:
 * EB200_ERR_CUDA with *out NULL and everything freed.  The staged secrets are cleared from the library's device
 * buffers before the call returns.  eb200_last_timing after create: launches = 1 per device. */
int eb200_eddsa_signing_set_create(size_t m, const uint8_t* secrets, uint8_t* out_pub, eb200_keyset** out);
/* Batch of key.sign(msg): item i is signed by key key_idx[i].  msgs / msg_off as eb200_eddsa_sign_batch takes them
 * (msgs may be NULL when every message is empty).  out_sig: n x 64 bytes Rencoded || S, byte-identical to what
 * eb200_eddsa_sign_batch writes with secrets[i] = that key's secret; status: n bytes, always EB200_ST_TRUE.
 * A NULL pointer, decreasing offsets or a key_idx[i] >= m: EB200_ERR_ARG; a set whose devices eb200_shutdown released:
 * EB200_ERR_NOT_INIT; both before anything is written.  n = 0: EB200_OK.  Host pointers, sharded over the set's
 * devices and chunked with copy / compute overlap.  Per chunk: the nonce kernel (r = SHA512(prefix || M) mod n,
 * R = r G), a batched normalisation of R (one inversion per 16 items) that writes Rencoded, and the challenge kernel
 * (S = r + SHA512(Rencoded || A || M) a mod n); the nonces r are cleared from the library's workspace before the call
 * returns.  eb200_last_timing: main_kernel_ms = the nonce kernel; launches = 3 per chunk. */
int eb200_eddsa_sign_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* msgs, const uint64_t* msg_off,
                                 const uint32_t* key_idx, uint8_t* out_sig, uint8_t* status);

/* curve25519 key sets: `pub = ec.keyFromPublic(x)` once, then `keyPair.derive(pub)` many times (lib/elliptic/ec/key.js:
 * 102-107), on curve25519.  The handle is the same eb200_keyset: _info reports EB200_CURVE_CURVE25519, _destroy and
 * eb200_shutdown treat it as any other set, and passing it to any short-curve or EdDSA keyed call (or any other set to
 * eb200_x25519_derive_batch_keyed) returns EB200_ERR_ARG.  Each key is kept as its image on edwards25519,
 * y = (u - 1) / (u + 1), a group isomorphism, with the table of an EdDSA key set: a derive is about 37 table additions
 * at W = 7 and no doubling, instead of the 256-step ladder.
 *   pubx       : m x 32 bytes big-endian, as eb200_x25519_derive_batch takes them (any value below 2^256, read mod p)
 *   table_bits : W as eb200_eddsa_keyset_create (same geometry: ceil(253 / W) windows of 2^(W-1) entries of 96 bytes;
 *                0 = the widest whose tables fit EB200_KEYSET_DEFAULT_BUDGET bytes per device)
 *   key_status : m bytes out -- EB200_ST_TRUE if u^3 + 486662 u^2 + u is 0 or a square mod p (MontCurve.validate,
 *                mont.js:21-28, the unkeyed call's check), else EB200_ST_THROW_ASSERT (a point on the twist)
 * m = 0, m >= 2^32 or a NULL pointer: EB200_ERR_ARG; no device: EB200_ERR_NOT_INIT; a failed allocation: EB200_ERR_CUDA
 * with *out NULL and everything freed.  device_bytes = 32 m + m + the tables.  eb200_last_timing after create: the
 * build kernels of the slowest device; launches = 3 per device (classify, window bases, table windows). */
int eb200_x25519_keyset_create(size_t m, const uint8_t* pubx, uint32_t table_bits, uint8_t* key_status, eb200_keyset** out);
/* Batch of keyPair(priv).derive(pub): item i uses key key_idx[i].  priv: n x 32 bytes big-endian, each below n (reduced
 * mod n at import, as eb200_x25519_derive_batch expects them; the tables cover 253 bits).  out_x and status[i] are byte
 * for byte what eb200_x25519_derive_batch writes for the same priv with pubx = that key's bytes: TRUE and x(priv P),
 * 0 for the point at infinity; THROW_ASSERT and 32 zero bytes for a key on the twist.
 * A NULL pointer, a key_idx[i] >= m or a priv[i] >= n: EB200_ERR_ARG; a set whose devices eb200_shutdown released:
 * EB200_ERR_NOT_INIT; both before anything is written.  n = 0: EB200_OK.  Host pointers, sharded over the set's
 * devices and chunked with copy / compute overlap.  Per chunk: the keyed main kernel (one table gather and one
 * addition per window of priv) and a normalisation (one inversion per 16 items).  The main kernel's table gathers are
 * indexed by the digits of the private scalar, as in the keyed short-curve derive and the fixed-base signing paths
 * (the unkeyed ladder's memory accesses do not depend on it).  The staged private scalars and the workspace that holds
 * the per-item results are cleared from the library's device buffers before the call returns.
 * eb200_last_timing: main_kernel_ms = the keyed main kernel; launches = 2 per chunk. */
int eb200_x25519_derive_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* priv, const uint32_t* key_idx,
                                    uint8_t* out_x, uint8_t* status);

/* Device-pointer forms of the keyed calls above, for CUDA callers whose data is already on the GPU.  Each takes its host
 * form's arguments as DEVICE pointers, then d_workspace and a CUDA stream (cudaStream_t cast to void*; NULL = the CUDA
 * default stream), as eb200_ecdsa_verify_batch_keyed_dev, and runs asynchronously on that stream on the device that owns
 * d_status; the caller synchronises the stream.  d_workspace must hold eb200_keyset_dev_workspace_bytes(ks, n) bytes of
 * device memory on that device; the call never reads it before writing it.
 * Outputs and statuses: for every item whose arguments the host form accepts, byte for byte what the host form writes.
 * An argument the host form refuses with EB200_ERR_ARG cannot be refused before launch without synchronising the stream,
 * so the item gets a status instead, its outputs are zeroed and nothing is computed from the bad value (a bad index
 * never addresses the set, a bad scalar never reaches its tables, a bad range is never read):
 *   EB200_ST_BAD_KEY_INDEX for d_key_idx[i] >= m; otherwise
 *   EB200_ST_BAD_ITEM for an EdDSA h >= n (little-endian), a curve25519 priv >= n (big-endian), or a message range with
 *     d_msg_off[i + 1] < d_msg_off[i] or d_msg_off[i + 1] > msgs_len (d_msg_off: n + 1 offsets into the msgs_len bytes
 *     at d_msgs, which may be NULL only when msgs_len = 0).
 * Returned before any launch: EB200_ERR_ARG for a set of another kind (as the host form), a NULL pointer, or d_status
 * on an initialised device that does not hold the set; EB200_ERR_NOT_INIT for a set released by eb200_shutdown or
 * d_status on a device eb200_init has not set up.  n = 0 returns EB200_OK.
 * ECDH derive, curve25519 derive and EdDSA sign clear, on the stream before their work ends, every workspace region that
 * held scalar-derived data (screened scalar copies, digit words, per-item results, nonces); the caller's own buffers
 * are the caller's.
 * eb200_last_timing (after the caller has synchronised the stream): kernel_ms = the whole call, main_kernel_ms = the keyed
 * main kernel (the nonce kernel for sign); launches as stated per call. */
size_t eb200_keyset_dev_workspace_bytes(const eb200_keyset* ks, size_t n);   /* 0 for NULL; for an ECDSA set at least
                                                                                eb200_ecdsa_verify_keyed_workspace_bytes */
/* Keyed verify of DER signatures (eb200_ecdsa_verify_batch_keyed_der) on device pointers: d_e (n x len), d_key_idx, and
 * the sigs_len bytes at d_sigs (NULL only when sigs_len = 0) with n + 1 offsets d_sig_off into them.  For every item the
 * host form accepts, d_status[i] is byte for byte what the host form writes, in its precedence: the key's import throw,
 * THROW_SIG_FORMAT, FALSE for r or s out of range, then the keyed verdict (for an off-curve key, the keyed replay's).
 * Otherwise BAD_KEY_INDEX for d_key_idx[i] >= m, else BAD_ITEM for a range that decreases or ends past sigs_len, which is
 * never read; BAD_ITEM takes precedence over a key's throw, as in eb200_ecdsa_verify_batch_der_dev.  main = the keyed
 * main kernel; launches = 6: index and range screen, screened keyed DER decode, prep, keyed main, keyed replay, merge. */
int eb200_ecdsa_verify_batch_keyed_der_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_e, const uint8_t* d_sigs,
                                           uint64_t sigs_len, const uint64_t* d_sig_off, const uint32_t* d_key_idx,
                                           uint8_t* d_status, void* d_workspace, void* stream);
/* ECDSA sets.  launches = 6: index screen, scalar prep, keyed main, normalisation, keyed replay (derive: the status
 * map), merge. */
int eb200_scalar_mul_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_k, const uint32_t* d_key_idx,
                                     uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace, void* stream);
int eb200_mul_add_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_k1, const uint8_t* d_k2,
                                  const uint32_t* d_key_idx, uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace,
                                  void* stream);
int eb200_ecdh_derive_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_priv, const uint32_t* d_key_idx,
                                      uint8_t* d_out_x, uint8_t* d_status, void* d_workspace, void* stream);
/* launches = 6: index screen, prep, keyed main, recid normalisation, cold kernel, merge. */
int eb200_ecdsa_recovery_param_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_e, const uint8_t* d_r,
                                               const uint8_t* d_s, const uint32_t* d_key_idx, uint8_t* d_out_recid,
                                               uint8_t* d_status, void* d_workspace, void* stream);
/* EdDSA sets.  launches = 3 (index and h screen, keyed main, merge), or 5 for raw messages (index and range screen,
 * key-byte gather, hash, keyed main, merge). */
int eb200_eddsa_verify_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_R, const uint8_t* d_S,
                                       const uint8_t* d_h, const uint32_t* d_key_idx, uint8_t* d_status, void* d_workspace,
                                       void* stream);
int eb200_eddsa_verify_batch_keyed_msgs_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_R, const uint8_t* d_S,
                                            const uint8_t* d_msgs, uint64_t msgs_len, const uint64_t* d_msg_off,
                                            const uint32_t* d_key_idx, uint8_t* d_status, void* d_workspace, void* stream);
/* EdDSA signing sets.  d_status[i] = EB200_ST_TRUE for an accepted item.  launches = 5: index and range screen, nonce,
 * normalisation, challenge, merge. */
int eb200_eddsa_sign_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_msgs, uint64_t msgs_len,
                                     const uint64_t* d_msg_off, const uint32_t* d_key_idx, uint8_t* d_out_sig,
                                     uint8_t* d_status, void* d_workspace, void* stream);
/* curve25519 sets.  launches = 4: index and priv screen, keyed main, normalisation, merge. */
int eb200_x25519_derive_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_priv, const uint32_t* d_key_idx,
                                        uint8_t* d_out_x, uint8_t* d_status, void* d_workspace, void* stream);

/* Device-pointer forms of the unkeyed calls (every compute entry point above except the eb200_curve_* calls), for CUDA
 * callers whose data is already on the GPU.  Each takes its host form's arguments as DEVICE pointers (d_*), then
 * d_workspace and a CUDA stream (cudaStream_t cast to void*; NULL = the CUDA default stream), and runs asynchronously on
 * that stream on the device that owns d_status; the caller synchronises the stream.  The call does not synchronise the
 * stream or the device, except for the first-use build of a curve's fixed-base table on that device, which
 * eb200_ecdsa_verify_batch_dev shares.  d_workspace (device memory on that device) must hold
 * eb200_dev_workspace_bytes(curve, n) bytes, one size for every unkeyed device-pointer call on the curve (those on ed25519
 * included, and the existing eb200_ecdsa_verify_batch_dev and eb200_eddsa_verify_batch_dev); the call never reads it
 * before writing it.  The curve25519 calls take no workspace.
 * Outputs and statuses: for every item whose arguments the host form accepts, byte for byte what the host form writes,
 * every status included (off-curve points replayed on the short curves, NEEDS_HOST for an off-curve ed25519 point, RETRY,
 * INFINITY, THROW_SECOND_KEY, THROW_NO_RECOVERY, the cold path for s = 0 mod n).
 * The calls with variable-length ranges take `len` bytes at d_sigs / d_msgs (NULL only when len = 0) and n + 1 offsets
 * into them.  A host form refuses a decreasing offset with EB200_ERR_ARG; a device call cannot without synchronising the
 * stream, so an item with off[i + 1] < off[i] or off[i + 1] > len gets EB200_ST_BAD_ITEM, its outputs are zeroed and its
 * range is never read.  For DER verify BAD_ITEM takes precedence over a key's throw (the host form refuses the whole
 * call).
 * Returned before any launch, in this order: EB200_ERR_UNSUPPORTED for an unknown curve or pub_fmt; for n = 0, EB200_OK
 * when a device is initialised, else EB200_ERR_NOT_INIT; EB200_ERR_ARG for a NULL pointer (other than those stated) or a
 * pers_len / entropy_len the host form refuses; EB200_ERR_NOT_INIT for d_status on a device eb200_init has not set up.
 * recover and getKeyRecoveryParam on ed25519 return EB200_ERR_UNSUPPORTED after the pointer checks, as their host forms.
 * Secrets: sign (all three forms), keygen, ECDH derive and EdDSA sign clear, on the stream before their work ends, every
 * workspace region that held scalar-derived data -- sign: the nonces, k G and the finish kernel's inversion scratch;
 * keygen: k G (when d_out_pub_xy is NULL) and the multiplication's statuses; derive: the scalars' digit words, the
 * per-item tables and the results x || y; EdDSA sign keeps nothing secret in the workspace (the range verdicts only).
 * The caller's own buffers are the caller's.
 * eb200_last_timing (after the caller has synchronised the stream): kernel_ms = the whole call, main_kernel_ms = the
 * dominant kernel (named per call below), launches as stated per call. */
size_t eb200_dev_workspace_bytes(int curve, size_t n);   /* 0 for an unknown curve and for curve25519; at least
                                                            eb200_ecdsa_verify_workspace_bytes(curve, n), and on ed25519
                                                            eb200_eddsa_verify_workspace_bytes(n) */
/* Sign: main = the nonce kernel (the whole loop with pers, and on ed25519).  launches = 3 (nonce, finish, then the slow
 * path, or for _k the RETRY map), 1 with pers or on ed25519.  With _k, an item whose status is RETRY gets no r, s or
 * recid: those output bytes are left as they were (the host form returns its staging buffer's bytes there). */
int eb200_ecdsa_sign_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_priv, uint32_t flags, uint8_t* d_out_r,
                               uint8_t* d_out_s, uint8_t* d_out_recid, uint8_t* d_status, void* d_workspace, void* stream);
int eb200_ecdsa_sign_batch_k_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_priv, const uint8_t* d_k,
                                 uint32_t flags, uint8_t* d_out_r, uint8_t* d_out_s, uint8_t* d_out_recid, uint8_t* d_status,
                                 void* d_workspace, void* stream);
int eb200_ecdsa_sign_batch_pers_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_priv, const uint8_t* d_pers,
                                    size_t pers_len, uint32_t flags, uint8_t* d_out_r, uint8_t* d_out_s, uint8_t* d_out_recid,
                                    uint8_t* d_status, void* d_workspace, void* stream);
/* Keygen: d_status gets the keygen verdicts; d_out_pub_xy may be NULL.  main = the keygen kernel; launches = 2 (keygen,
 * k G). */
int eb200_ec_keygen_batch_dev(int curve, size_t n, const uint8_t* d_entropy, size_t entropy_len, const uint8_t* d_pers,
                              size_t pers_len, uint8_t* d_out_priv, uint8_t* d_out_pub_xy, uint8_t* d_status, void* d_workspace,
                              void* stream);
/* recoverPubKey: main = the recovery kernel; launches = 2 (prep, recovery).  getKeyRecoveryParam: main = its main
 * kernel; launches = 3 (prep, main, cold kernel for s = 0 mod n). */
int eb200_ecdsa_recover_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r, const uint8_t* d_s,
                                  const uint8_t* d_recid, uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace, void* stream);
int eb200_ecdsa_recovery_param_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r, const uint8_t* d_s,
                                         const uint8_t* d_q_xy, uint8_t* d_out_recid, uint8_t* d_status, void* d_workspace,
                                         void* stream);
/* Point.mul (d_points_xy NULL = the base point), mulAdd, ECDH derive: main = the multiplication kernel; launches = 3
 * (scalar prep, main, replay; derive: the status map), 1 for G.mul and on ed25519.  derive writes x to d_out_x with a
 * strided device-to-device copy of the x || y it keeps in the workspace. */
int eb200_scalar_mul_batch_dev(int curve, size_t n, const uint8_t* d_k, const uint8_t* d_points_xy, uint8_t* d_out_xy,
                               uint8_t* d_status, void* d_workspace, void* stream);
int eb200_mul_add_batch_dev(int curve, size_t n, const uint8_t* d_k1, const uint8_t* d_k2, const uint8_t* d_p2_xy,
                            uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace, void* stream);
int eb200_ecdh_derive_batch_dev(int curve, size_t n, const uint8_t* d_priv, const uint8_t* d_pub_xy, uint8_t* d_out_x,
                                uint8_t* d_status, void* d_workspace, void* stream);
/* curve25519 Point.mul: no workspace, as eb200_x25519_derive_batch_dev.  main = the ladder; launches = 1. */
int eb200_x25519_mul_batch_dev(size_t n, const uint8_t* d_k, const uint8_t* d_px, uint8_t* d_out_x, uint8_t* d_status,
                               void* stream);
/* Verify from DER: d_sig_off holds n + 1 offsets into the sigs_len bytes at d_sigs.  main = the verify kernel; launches =
 * the host form's (SEC1 decode when pub_fmt is not XY, DER decode, prep, verify, replay; on ed25519 no prep and no
 * replay) + 2 (range screen, merge); the DER decode is a screened form of the host form's, which reads no byte of a
 * screened item. */
int eb200_ecdsa_verify_batch_der_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_sigs, uint64_t sigs_len,
                                     const uint64_t* d_sig_off, const uint8_t* d_pub, uint32_t pub_fmt, uint8_t* d_status,
                                     void* d_workspace, void* stream);
/* EdDSA verify from raw messages (workspace: eb200_dev_workspace_bytes(EB200_CURVE_ED25519, n)).  main = the verify
 * kernel; launches = 4 (range screen, screened hash, verify, merge). */
int eb200_eddsa_verify_batch_msgs_dev(size_t n, const uint8_t* d_R, const uint8_t* d_S, const uint8_t* d_A,
                                      const uint8_t* d_msgs, uint64_t msgs_len, const uint64_t* d_msg_off, uint8_t* d_status,
                                      void* d_workspace, void* stream);
/* EdDSA sign (workspace as above); d_out_pub may be NULL.  main = the sign kernel; launches = 3 (range screen, screened
 * sign, merge). */
int eb200_eddsa_sign_batch_dev(size_t n, const uint8_t* d_secrets, const uint8_t* d_msgs, uint64_t msgs_len,
                               const uint64_t* d_msg_off, uint8_t* d_out_sig, uint8_t* d_out_pub, uint8_t* d_status,
                               void* d_workspace, void* stream);

/* Self-test hooks used by the parity tests (device arithmetic vs the oracle).
 * a, b, out: n elements of L little-endian 32-bit limbs each (host pointers); L = 8, except p192 6, p384 12 and
 * p521 18.  An op the curve does not know returns a (short curves) or 0 (secp256k1, ed25519 / curve25519).
 * Coordinate field, on plain integers:
 *   0 mul, 1 sqr, 2 add, 3 sub, 4 neg, 7 inv (all curves);
 *   secp256k1 and the 25519 curves (weakly reduced results): 5 mul_small(b[0]), 6 normalize, 8 sqrt candidate
 *     (secp256k1) / a^((p-5)/8) (25519);
 *   p192 .. p521 (canonical results): 8 3ab, 9 4ab, 10 8a^2, 11 2a -- mul_k<3>, mul_k<4>, sqr_k<8> and dbl as the
 *     doubling calls them.
 * Scalar field mod n (mod l on the 25519 curves), on the words as given, Montgomery radix R = 2^(32 L):
 *   16 a b R^-1 (a < R, b < n), 17 to Montgomery form (a R mod n), 18 from Montgomery form (a R^-1 mod n),
 *   19 add, 20 sub (canonical operands), 21 inverse in Montgomery form (a^(n-2) R^(3-n) mod n; 0 -> 0).
 *   On secp256k1 ops 16, 17, 18 and 21 run sc_mont_mul / sc_mont_inv, the calls of the verify prep.
 * secp256k1 GLV split of a (< n) into odd halves k1 + k2 lambda = a (mod n), |ki| = 2 mi + 1:
 *   24 writes m1, 25 writes m2 (limbs 0..4), then the signs of k1 and k2 (limbs 5, 6: 1 = negative), limb 7 = 0. */
int eb200_selftest_fe(int curve, int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out);
/* Geometry of the fixed-base table: entry (j, i) = (2i+1) * 2^(wbits*j) * G, 16 words (x||y limbs). */
int eb200_selftest_gtab_dims(int curve, int* windows, int* entries, int* wbits);
/* Copy the fixed-base table of `curve` to the host (n_words 32-bit words available). */
int eb200_selftest_gtab(int curve, uint32_t* out, size_t n_words);

#ifdef __cplusplus
}
#endif
#endif
