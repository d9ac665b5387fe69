/* N-API addon: thin marshalling between JS typed arrays and the C ABI of libelliptic_b200.so
 * (include/elliptic_b200.h).  No arithmetic here.  Build (in a Node.js toolchain):
 *   cc -shared -fPIC -DEB200_HAVE_NODE_API_H -I../include elliptic_b200_napi.c -L../elliptic_b200 -lelliptic_b200 \
 *      -Wl,-rpath,'$ORIGIN/../elliptic_b200' -o elliptic_b200.node
 * This image has no node / node_api.h, so the file is compile-checked against binding/node_api_min.h only
 * (tests/test_capi_load.py) and cannot be loaded here.
 *
 * Every entry point validates EVERY buffer length against n * (the curve's field length) before it calls into the
 * library: the library reads and writes exactly n * len bytes per array and trusts its caller. */
#ifdef EB200_HAVE_NODE_API_H
#include <node_api.h>
#else
#include "node_api_min.h"
#endif
#include <stdlib.h>
#include <string.h>
#include "../include/elliptic_b200.h"

/* bytes of a field element / scalar on the wire; 0 = not an (x, y) curve of the ec API */
static size_t field_len(int curve) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: case EB200_CURVE_P256: case EB200_CURVE_ED25519: return 32;
    case EB200_CURVE_P384: return 48;
    case EB200_CURVE_P521: return 66;
    case EB200_CURVE_P192: return 24;
    case EB200_CURVE_P224: return 28;
    default: return 0;
  }
}
static size_t pub_bytes(size_t len, uint32_t fmt) {
  return fmt == EB200_PUB_XY ? 2 * len : fmt == EB200_PUB_SEC1_65 ? 1 + 2 * len : fmt == EB200_PUB_SEC1_33 ? 1 + len : 0;
}

static int u8(napi_env env, napi_value v, uint8_t** p, size_t* len) {
  napi_typedarray_type t; napi_value ab; size_t off; void* data;
  if (napi_get_typedarray_info(env, v, &t, len, &data, &ab, &off) != napi_ok || t != napi_uint8_array) return 0;
  *p = (uint8_t*)data;
  return 1;
}
/* null / undefined -> pointer 0, length 0 (optional arguments) */
static int u8_opt(napi_env env, napi_value v, uint8_t** p, size_t* len) {
  *p = 0; *len = 0;
  bool is_arr = false;
  if (napi_is_typedarray(env, v, &is_arr) != napi_ok || !is_arr) return 1;
  return u8(env, v, p, len);
}
static napi_value fail(napi_env env, int rc) {
  napi_throw_error(env, "EB200", rc == EB200_ERR_CUDA ? eb200_last_error() : eb200_strerror(rc));
  return 0;
}
static napi_value out_u8(napi_env env, size_t n, uint8_t** data) {
  napi_value ab, arr;
  napi_create_arraybuffer(env, n, (void**)data, &ab);
  napi_create_typedarray(env, napi_uint8_array, n, ab, 0, &arr);
  return arr;
}
static napi_value obj(napi_env env) { napi_value o; napi_create_object(env, &o); return o; }
#define ARGS(k) size_t argc = (k); napi_value argv[(k)]; napi_get_cb_info(env, info, &argc, argv, 0, 0); if (argc < (k)) return fail(env, EB200_ERR_ARG)
#define I32(i, var) int32_t var; if (napi_get_value_int32(env, argv[i], &var) != napi_ok) return fail(env, EB200_ERR_ARG)
#define U32(i, var) uint32_t var; if (napi_get_value_uint32(env, argv[i], &var) != napi_ok) return fail(env, EB200_ERR_ARG)
#define BUF(i, p, l) uint8_t* p; size_t l; if (!u8(env, argv[i], &p, &l)) return fail(env, EB200_ERR_ARG)
#define OPT(i, p, l) uint8_t* p; size_t l; if (!u8_opt(env, argv[i], &p, &l)) return fail(env, EB200_ERR_ARG)
#define SET(o, name, v) napi_set_named_property(env, o, name, v)

/* init(devices: Int32Array-like array of CUDA ordinals | undefined, flags) -- eb200_init(devices[], ndev, flags) */
static napi_value Init(napi_env env, napi_callback_info info) {
  size_t argc = 2; napi_value argv[2]; napi_value undef;
  napi_get_cb_info(env, info, &argc, argv, 0, 0);
  int devs[16]; int nd = 0; uint32_t flags = 0, alen = 0;
  bool is_array = false;
  if (argc >= 1 && napi_is_array(env, argv[0], &is_array) == napi_ok && is_array) {
    napi_get_array_length(env, argv[0], &alen);
    for (uint32_t i = 0; i < alen && nd < 16; i++) {
      napi_value v; int32_t d;
      if (napi_get_element(env, argv[0], i, &v) != napi_ok || napi_get_value_int32(env, v, &d) != napi_ok) return fail(env, EB200_ERR_ARG);
      devs[nd++] = d;
    }
  }
  if (argc >= 2) napi_get_value_uint32(env, argv[1], &flags);
  int rc = eb200_init(nd ? devs : 0, nd, flags);
  if (rc) return fail(env, rc);
  napi_get_undefined(env, &undef);
  return undef;
}

/* ecdsaVerifyBatch(curveId, e, r, s, pub, pubFmt) -> Uint8Array(n) of statuses
 * (EC.prototype.verify semantics per item, lib/elliptic/ec/index.js:188-229) */
static napi_value EcdsaVerifyBatch(napi_env env, napi_callback_info info) {
  ARGS(6); I32(0, curve); BUF(1, e, le); BUF(2, r, lr); BUF(3, s, ls); BUF(4, pub, lp); U32(5, fmt);
  size_t len = field_len(curve), pb = pub_bytes(len, fmt);
  if (!len || !pb) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = le / len;
  if (le != n * len || lr != le || ls != le || lp != n * pb) return fail(env, EB200_ERR_ARG);
  uint8_t* st; napi_value arr = out_u8(env, n, &st);
  int rc = eb200_ecdsa_verify_batch(curve, n, e, r, s, pub, fmt, st);
  return rc ? fail(env, rc) : arr;
}

/* ecdsaVerifyBatchAsync(curveId, e, r, s, pub, pubFmt) -> Promise<Uint8Array>: the same call on a libuv worker
 * thread (napi_create_async_work); the input arrays are kept alive by references until completion. */
typedef struct {
  napi_async_work work; napi_deferred deferred; napi_ref refs[5];
  int curve; size_t n; uint32_t fmt; uint8_t *e, *r, *s, *pub, *st; int rc; char err[256];
} verify_job;
static void verify_exec(napi_env env, void* data) {
  (void)env;
  verify_job* j = (verify_job*)data;
  j->rc = eb200_ecdsa_verify_batch(j->curve, j->n, j->e, j->r, j->s, j->pub, j->fmt, j->st);
  if (j->rc) { strncpy(j->err, j->rc == EB200_ERR_CUDA ? eb200_last_error() : eb200_strerror(j->rc), sizeof j->err - 1); j->err[sizeof j->err - 1] = 0; }
}
static void verify_done(napi_env env, napi_status status, void* data) {
  verify_job* j = (verify_job*)data;
  napi_value out;
  napi_get_reference_value(env, j->refs[4], &out);
  if (status == napi_ok && j->rc == 0) napi_resolve_deferred(env, j->deferred, out);
  else {
    napi_value msg, err;
    napi_create_string_utf8(env, j->rc ? j->err : "async work cancelled", NAPI_AUTO_LENGTH, &msg);
    napi_create_error(env, 0, msg, &err);
    napi_reject_deferred(env, j->deferred, err);
  }
  for (int i = 0; i < 5; i++) napi_delete_reference(env, j->refs[i]);
  napi_delete_async_work(env, j->work);
  free(j);
}
static napi_value EcdsaVerifyBatchAsync(napi_env env, napi_callback_info info) {
  ARGS(6); I32(0, curve); BUF(1, e, le); BUF(2, r, lr); BUF(3, s, ls); BUF(4, pub, lp); U32(5, fmt);
  size_t len = field_len(curve), pb = pub_bytes(len, fmt);
  if (!len || !pb) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = le / len;
  if (le != n * len || lr != le || ls != le || lp != n * pb) return fail(env, EB200_ERR_ARG);
  verify_job* j = (verify_job*)calloc(1, sizeof *j);
  if (!j) return fail(env, EB200_ERR_ARG);
  napi_value promise, name, arr = out_u8(env, n, &j->st);
  j->curve = curve; j->n = n; j->fmt = fmt; j->e = e; j->r = r; j->s = s; j->pub = pub;
  for (int i = 0; i < 4; i++) napi_create_reference(env, argv[1 + i], 1, &j->refs[i]);
  napi_create_reference(env, arr, 1, &j->refs[4]);
  napi_create_promise(env, &j->deferred, &promise);
  napi_create_string_utf8(env, "eb200.ecdsaVerifyBatch", NAPI_AUTO_LENGTH, &name);
  napi_create_async_work(env, 0, name, verify_exec, verify_done, j, &j->work);
  napi_queue_async_work(env, j->work);
  return promise;
}

/* ecdsaVerifyBatchDer(curveId, e, sigs, sigOff (n + 1 little-endian u64 offsets, as a Uint8Array view), pub, pubFmt) -> Uint8Array(n)
 * DER signatures as `new Signature(der)` takes them (ec/signature.js:73-134), parsed on the GPU */
static napi_value EcdsaVerifyBatchDer(napi_env env, napi_callback_info info) {
  ARGS(6); I32(0, curve); BUF(1, e, le); BUF(2, sig, lsg); BUF(3, off, lo); BUF(4, pub, lp); U32(5, fmt);
  size_t len = field_len(curve), pb = pub_bytes(len, fmt);
  if (!len || !pb) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = le / len;
  if (le != n * len || lo != 8 * (n + 1) || lp != n * pb || ((uintptr_t)off & 7)) return fail(env, EB200_ERR_ARG);
  const uint64_t* o = (const uint64_t*)off;
  for (size_t i = 0; i < n; i++) if (o[i + 1] < o[i]) return fail(env, EB200_ERR_ARG);
  if (o[n] > lsg) return fail(env, EB200_ERR_ARG);
  uint8_t* st; napi_value arr = out_u8(env, n, &st);
  int rc = eb200_ecdsa_verify_batch_der(curve, n, e, sig, o, pub, fmt, st);
  return rc ? fail(env, rc) : arr;
}

/* ecdsaSignBatch(curveId, e, priv, flags, k | null, pers | null) -> {r, s, recid, status}
 * (EC.prototype.sign, ec/index.js:110-186: RFC 6979 nonces on the GPU; k: options.k candidates for one attempt,
 * status 10 = ask k(iter + 1); pers: options.pers bytes) */
static napi_value EcdsaSignBatch(napi_env env, napi_callback_info info) {
  ARGS(6); I32(0, curve); BUF(1, e, le); BUF(2, d, ld); U32(3, flags); OPT(4, k, lk); OPT(5, pers, lpers);
  size_t len = field_len(curve);
  if (!len) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = le / len;
  if (le != n * len || ld != le || (k && lk != le) || (k && pers)) return fail(env, EB200_ERR_ARG);
  uint8_t *r, *s, *id, *st;
  napi_value ar = out_u8(env, le, &r), as = out_u8(env, le, &s), ai = out_u8(env, n, &id), ast = out_u8(env, n, &st);
  int rc = k ? eb200_ecdsa_sign_batch_k(curve, n, e, d, k, flags, r, s, id, st)
             : pers ? eb200_ecdsa_sign_batch_pers(curve, n, e, d, pers, lpers, flags, r, s, id, st)
                    : eb200_ecdsa_sign_batch(curve, n, e, d, flags, r, s, id, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "r", ar); SET(res, "s", as); SET(res, "recid", ai); SET(res, "status", ast);
  return res;
}

/* ecKeygenBatch(curveId, entropy (n x entropyLen), entropyLen, pers | null) -> {priv, pub, status}   (genKeyPair, ec/index.js:55-79) */
static napi_value EcKeygenBatch(napi_env env, napi_callback_info info) {
  ARGS(4); I32(0, curve); BUF(1, ent, lent); U32(2, elen); OPT(3, pers, lpers);
  size_t len = field_len(curve);
  if (!len) return fail(env, EB200_ERR_UNSUPPORTED);
  if (!elen || lent % elen) return fail(env, EB200_ERR_ARG);
  size_t n = lent / elen;
  uint8_t *priv, *pub, *st;
  napi_value ap = out_u8(env, n * len, &priv), aq = out_u8(env, 2 * n * len, &pub), ast = out_u8(env, n, &st);
  int rc = eb200_ec_keygen_batch(curve, n, ent, elen, pers, lpers, priv, pub, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "priv", ap); SET(res, "pub", aq); SET(res, "status", ast);
  return res;
}

/* ecdsaRecoverBatch(curveId, e, r, s, recid) -> {pub, status}   (recoverPubKey, ec/index.js:231-259) */
static napi_value EcdsaRecoverBatch(napi_env env, napi_callback_info info) {
  ARGS(5); I32(0, curve); BUF(1, e, le); BUF(2, r, lr); BUF(3, s, ls); BUF(4, id, li);
  size_t len = field_len(curve);
  if (!len) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = le / len;
  if (le != n * len || lr != le || ls != le || li != n) return fail(env, EB200_ERR_ARG);
  uint8_t *out, *st;
  napi_value ao = out_u8(env, 2 * len * n, &out), ast = out_u8(env, n, &st);
  int rc = eb200_ecdsa_recover_batch(curve, n, e, r, s, id, out, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "pub", ao); SET(res, "status", ast);
  return res;
}

/* ecdsaRecoveryParamBatch(curveId, e, r, s, pubXY) -> {recid, status}   (getKeyRecoveryParam, ec/index.js:261-278) */
static napi_value EcdsaRecoveryParamBatch(napi_env env, napi_callback_info info) {
  ARGS(5); I32(0, curve); BUF(1, e, le); BUF(2, r, lr); BUF(3, s, ls); BUF(4, q, lq);
  size_t len = field_len(curve);
  if (!len) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = le / len;
  if (le != n * len || lr != le || ls != le || lq != 2 * le) return fail(env, EB200_ERR_ARG);
  uint8_t *id, *st;
  napi_value ai = out_u8(env, n, &id), ast = out_u8(env, n, &st);
  int rc = eb200_ecdsa_recovery_param_batch(curve, n, e, r, s, q, id, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "recid", ai); SET(res, "status", ast);
  return res;
}

/* mulAddBatch(curveId, k1 | null, k2, points | null) -> {points, status}
 * k1 null: Point.mul (short.js:422-432, edwards.js:362-367); points null: G.mul; both: G.mulAdd(k1, P, k2) */
static napi_value MulAddBatch(napi_env env, napi_callback_info info) {
  ARGS(4); I32(0, curve); OPT(1, k1, l1); BUF(2, k2, l2); OPT(3, pts, lp);
  size_t len = field_len(curve);
  if (!len) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = l2 / len;
  if (l2 != n * len || (k1 && l1 != l2) || (pts && lp != 2 * l2) || (k1 && !pts)) return fail(env, EB200_ERR_ARG);
  uint8_t *out, *st;
  napi_value ao = out_u8(env, 2 * len * n, &out), ast = out_u8(env, n, &st);
  int rc = k1 ? eb200_mul_add_batch(curve, n, k1, k2, pts, out, st) : eb200_scalar_mul_batch(curve, n, k2, pts, out, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "points", ao); SET(res, "status", ast);
  return res;
}

/* ecdhDeriveBatch(curveId, priv, pubXY) -> {out, status}   (KeyPair.derive, ec/key.js:102-107) */
static napi_value EcdhDeriveBatch(napi_env env, napi_callback_info info) {
  ARGS(3); I32(0, curve); BUF(1, k, lk); BUF(2, pts, lp);
  size_t len = field_len(curve);
  if (!len) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t n = lk / len;
  if (lk != n * len || lp != 2 * lk) return fail(env, EB200_ERR_ARG);
  uint8_t *out, *st;
  napi_value ao = out_u8(env, lk, &out), ast = out_u8(env, n, &st);
  int rc = eb200_ecdh_derive_batch(curve, n, k, pts, out, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "out", ao); SET(res, "status", ast);
  return res;
}

/* curveOpBatch(op, len, p, a, b, k1 | null, p1, k2 | null, p2 | null, klen) -> {points, status}
 * run-time short curves (curve/short.js:10-24): op 0 mul / mulAdd, 1 add, 2 dbl, 3 validate */
static napi_value CurveOpBatch(napi_env env, napi_callback_info info) {
  ARGS(10); I32(0, op); U32(1, len); BUF(2, p, lp_); BUF(3, a, la); BUF(4, b, lb); OPT(5, k1, lk1); BUF(6, p1, l1); OPT(7, k2, lk2);
  OPT(8, p2, l2); U32(9, klen);
  if (!len || lp_ != len || la != len || lb != len || l1 % (2 * len)) return fail(env, EB200_ERR_ARG);
  size_t n = l1 / (2 * len);
  if ((p2 && l2 != l1) || (k1 && lk1 != n * klen) || (k2 && lk2 != n * klen)) return fail(env, EB200_ERR_ARG);
  eb200_short_curve cv = {len, p, a, b};
  uint8_t *out, *st;
  napi_value ao = out_u8(env, l1, &out), ast = out_u8(env, n, &st);
  int rc = op == 0 ? (k2 ? eb200_curve_mul_add_batch(&cv, n, k1, p1, k2, p2, klen, out, st) : eb200_curve_mul_batch(&cv, n, k1, klen, p1, out, st))
         : op == 1 ? eb200_curve_add_batch(&cv, n, p1, p2, out, st)
         : op == 2 ? eb200_curve_dbl_batch(&cv, n, p1, out, st) : eb200_curve_validate_batch(&cv, n, p1, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "points", ao); SET(res, "status", ast);
  return res;
}

/* eddsaVerifyBatch(R, S, A, h | null, msgs | null, msgOff | null) -> Uint8Array(n)   (EDDSA.prototype.verify, eddsa/index.js:52-63;
 * h = hashInt supplied by the caller, or the raw messages: SHA-512 on the GPU) */
static napi_value EddsaVerifyBatch(napi_env env, napi_callback_info info) {
  ARGS(6); BUF(0, R, a); BUF(1, S, b); BUF(2, A, c); OPT(3, h, d); OPT(4, msgs, lm); OPT(5, off, lo);
  size_t n = a / 32;
  if (a % 32 || b != a || c != a || (h && d != a) || (!h && (lo != 8 * (n + 1) || ((uintptr_t)off & 7)))) return fail(env, EB200_ERR_ARG);
  if (!h) {
    const uint64_t* o = (const uint64_t*)off;
    for (size_t i = 0; i < n; i++) if (o[i + 1] < o[i]) return fail(env, EB200_ERR_ARG);
    if (o[n] > lm) return fail(env, EB200_ERR_ARG);
  }
  uint8_t* st; napi_value arr = out_u8(env, n, &st);
  int rc = h ? eb200_eddsa_verify_batch(n, R, S, A, h, st) : eb200_eddsa_verify_batch_msgs(n, R, S, A, msgs, (const uint64_t*)off, st);
  return rc ? fail(env, rc) : arr;
}

/* eddsaSignBatch(secrets, msgs, msgOff) -> {sig, pub, status}   (EDDSA.prototype.sign, eddsa/index.js:34-44) */
static napi_value EddsaSignBatch(napi_env env, napi_callback_info info) {
  ARGS(3); BUF(0, sec, ls); OPT(1, msgs, lm); BUF(2, off, lo);
  size_t n = ls / 32;
  if (ls % 32 || lo != 8 * (n + 1) || ((uintptr_t)off & 7)) return fail(env, EB200_ERR_ARG);
  const uint64_t* o = (const uint64_t*)off;
  for (size_t i = 0; i < n; i++) if (o[i + 1] < o[i]) return fail(env, EB200_ERR_ARG);
  if (o[n] > lm) return fail(env, EB200_ERR_ARG);
  uint8_t *sig, *pub, *st;
  napi_value asig = out_u8(env, 64 * n, &sig), apub = out_u8(env, 32 * n, &pub), ast = out_u8(env, n, &st);
  int rc = eb200_eddsa_sign_batch(n, sec, msgs, o, sig, pub, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "sig", asig); SET(res, "pub", apub); SET(res, "status", ast);
  return res;
}

/* x25519Batch(k, x, validate) -> {out, status}: KeyPair.derive (validate = true, ec/key.js:102-107) or MontCurve Point.mul (mont.js:130-153) */
static napi_value X25519Batch(napi_env env, napi_callback_info info) {
  ARGS(3); BUF(0, k, a); BUF(1, x, b); U32(2, validate);
  if (a % 32 || a != b) return fail(env, EB200_ERR_ARG);
  uint8_t *out, *st;
  napi_value o = out_u8(env, a, &out), s = out_u8(env, a / 32, &st);
  int rc = validate ? eb200_x25519_derive_batch(a / 32, k, x, out, st) : eb200_x25519_mul_batch(a / 32, k, x, out, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "out", o); SET(res, "status", s);
  return res;
}

/* Key sets (eb200_keyset_*): the handle travels as an external whose box is shared with the finalizer, so that
 * keysetDestroy and garbage collection free the set exactly once.
 * keysetCreate(curveId, pub, pubFmt, tableBits) -> {handle, status: Uint8Array(m), tableBits, deviceBytes} */
typedef struct { eb200_keyset* ks; } keyset_box;
static void keyset_finalize(napi_env env, void* data, void* hint) {
  (void)env; (void)hint;
  keyset_box* b = (keyset_box*)data;
  eb200_keyset_destroy(b->ks);
  free(b);
}
/* the result object of a create call (rc: its return code; the box is freed on failure) */
static napi_value keyset_out(napi_env env, int rc, keyset_box* b, napi_value status) {
  if (rc) { free(b); return fail(env, rc); }
  uint32_t w = 0; size_t bytes = 0;
  eb200_keyset_info(b->ks, 0, 0, &w, &bytes);
  napi_value o = obj(env), h, vw, vb;
  napi_create_external(env, b, keyset_finalize, 0, &h);
  napi_create_uint32(env, w, &vw);
  napi_create_double(env, (double)bytes, &vb);
  SET(o, "handle", h); SET(o, "status", status); SET(o, "tableBits", vw); SET(o, "deviceBytes", vb);
  return o;
}
static napi_value KeysetCreate(napi_env env, napi_callback_info info) {
  ARGS(4); I32(0, curve); BUF(1, pub, lp); U32(2, fmt); U32(3, bits);
  size_t len = field_len(curve), pb = pub_bytes(len, fmt);
  if (!len || !pb) return fail(env, EB200_ERR_UNSUPPORTED);
  size_t m = lp / pb;
  if (lp != m * pb) return fail(env, EB200_ERR_ARG);
  keyset_box* b = (keyset_box*)calloc(1, sizeof *b);
  if (!b) return fail(env, EB200_ERR_ARG);
  uint8_t* st; napi_value arr = out_u8(env, m, &st);
  int rc = eb200_keyset_create(curve, m, pub, fmt, bits, st, &b->ks);
  return keyset_out(env, rc, b, arr);
}
/* eddsaKeysetCreate(A: m x 32 encoded keys, tableBits) -> {handle, status: Uint8Array(m), tableBits, deviceBytes} */
static napi_value EddsaKeysetCreate(napi_env env, napi_callback_info info) {
  ARGS(2); BUF(0, A, la); U32(1, bits);
  size_t m = la / 32;
  if (la % 32) return fail(env, EB200_ERR_ARG);
  keyset_box* b = (keyset_box*)calloc(1, sizeof *b);
  if (!b) return fail(env, EB200_ERR_ARG);
  uint8_t* st; napi_value arr = out_u8(env, m, &st);
  int rc = eb200_eddsa_keyset_create(m, A, bits, st, &b->ks);
  return keyset_out(env, rc, b, arr);
}
/* x25519KeysetCreate(pubx: m x 32 big-endian, tableBits) -> {handle, status: Uint8Array(m), tableBits, deviceBytes} */
static napi_value X25519KeysetCreate(napi_env env, napi_callback_info info) {
  ARGS(2); BUF(0, x, lx); U32(1, bits);
  size_t m = lx / 32;
  if (lx % 32) return fail(env, EB200_ERR_ARG);
  keyset_box* b = (keyset_box*)calloc(1, sizeof *b);
  if (!b) return fail(env, EB200_ERR_ARG);
  uint8_t* st; napi_value arr = out_u8(env, m, &st);
  int rc = eb200_x25519_keyset_create(m, x, bits, st, &b->ks);
  return keyset_out(env, rc, b, arr);
}
/* keysetDestroy(handle): frees the set now; the handle stays valid and answers EB200_ERR_ARG afterwards */
static napi_value KeysetDestroy(napi_env env, napi_callback_info info) {
  ARGS(1);
  void* p = 0; napi_value undef;
  if (napi_get_value_external(env, argv[0], &p) != napi_ok || !p) return fail(env, EB200_ERR_ARG);
  keyset_box* b = (keyset_box*)p;
  int rc = eb200_keyset_destroy(b->ks);
  b->ks = 0;
  if (rc) return fail(env, rc);
  napi_get_undefined(env, &undef);
  return undef;
}
/* ecdsaVerifyBatchKeyed(handle, e, r, s, keyIdx: Uint8Array over n little-endian uint32) -> Uint8Array(n) of statuses */
static napi_value EcdsaVerifyBatchKeyed(napi_env env, napi_callback_info info) {
  ARGS(5); BUF(1, e, le); BUF(2, r, lr); BUF(3, s, ls); BUF(4, idx, li);
  void* p = 0;
  if (napi_get_value_external(env, argv[0], &p) != napi_ok || !p || !((keyset_box*)p)->ks) return fail(env, EB200_ERR_ARG);
  eb200_keyset* ks = ((keyset_box*)p)->ks;
  int curve = 0;
  eb200_keyset_info(ks, &curve, 0, 0, 0);
  size_t len = field_len(curve), n = li / 4;
  if (!len || li != 4 * n || le != n * len || lr != le || ls != le || ((uintptr_t)idx & 3)) return fail(env, EB200_ERR_ARG);
  uint8_t* st; napi_value arr = out_u8(env, n, &st);
  int rc = eb200_ecdsa_verify_batch_keyed(ks, n, e, r, s, (const uint32_t*)(const void*)idx, st);
  return rc ? fail(env, rc) : arr;
}

/* ecdsaVerifyBatchKeyedDer(handle, e, sigs, sigOff (n + 1 little-endian u64 offsets, as a Uint8Array view),
 * keyIdx: Uint8Array over n little-endian uint32) -> Uint8Array(n) of statuses (DER parsed on the GPU) */
static napi_value EcdsaVerifyBatchKeyedDer(napi_env env, napi_callback_info info) {
  ARGS(5); BUF(1, e, le); BUF(2, sig, lsg); BUF(3, off, lo); BUF(4, idx, li);
  void* p = 0;
  if (napi_get_value_external(env, argv[0], &p) != napi_ok || !p || !((keyset_box*)p)->ks) return fail(env, EB200_ERR_ARG);
  eb200_keyset* ks = ((keyset_box*)p)->ks;
  int curve = 0;
  eb200_keyset_info(ks, &curve, 0, 0, 0);
  size_t len = field_len(curve), n = li / 4;
  if (!len || li != 4 * n || le != n * len || lo != 8 * (n + 1) || ((uintptr_t)off & 7) || ((uintptr_t)idx & 3))
    return fail(env, EB200_ERR_ARG);
  const uint64_t* o = (const uint64_t*)(const void*)off;
  for (size_t i = 0; i < n; i++) if (o[i + 1] < o[i]) return fail(env, EB200_ERR_ARG);
  if (o[n] > lsg) return fail(env, EB200_ERR_ARG);
  uint8_t* st; napi_value arr = out_u8(env, n, &st);
  int rc = eb200_ecdsa_verify_batch_keyed_der(ks, n, e, sig, o, (const uint32_t*)(const void*)idx, st);
  return rc ? fail(env, rc) : arr;
}

/* the ECDSA set behind a handle and its field length, or 0 */
static eb200_keyset* ecdsa_set(napi_env env, napi_value v, size_t* len) {
  void* p = 0;
  int curve = 0;
  if (napi_get_value_external(env, v, &p) != napi_ok || !p || !((keyset_box*)p)->ks) return 0;
  eb200_keyset_info(((keyset_box*)p)->ks, &curve, 0, 0, 0);
  *len = curve == EB200_CURVE_ED25519 || curve == EB200_CURVE_CURVE25519 ? 0 : field_len(curve);
  return *len ? ((keyset_box*)p)->ks : 0;
}
/* mulAddBatchKeyed(handle, k1 | null, k2, keyIdx: Uint8Array over n little-endian uint32) -> {points, status}
 * k1 null: pub.mul(k2) (short.js:422-432); else G.mulAdd(k1, pub, k2) (short.js:434-441), pub = key keyIdx[i] */
static napi_value MulAddBatchKeyed(napi_env env, napi_callback_info info) {
  ARGS(4); OPT(1, k1, l1); BUF(2, k2, l2); BUF(3, idx, li);
  size_t len = 0;
  eb200_keyset* ks = ecdsa_set(env, argv[0], &len);
  if (!ks) return fail(env, EB200_ERR_ARG);
  size_t n = li / 4;
  if (li != 4 * n || l2 != n * len || (k1 && l1 != l2) || ((uintptr_t)idx & 3)) return fail(env, EB200_ERR_ARG);
  const uint32_t* ki = (const uint32_t*)(const void*)idx;
  uint8_t *out, *st;
  napi_value ao = out_u8(env, 2 * len * n, &out), ast = out_u8(env, n, &st);
  int rc = k1 ? eb200_mul_add_batch_keyed(ks, n, k1, k2, ki, out, st) : eb200_scalar_mul_batch_keyed(ks, n, k2, ki, out, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "points", ao); SET(res, "status", ast);
  return res;
}
/* ecdhDeriveBatchKeyed(handle, priv, keyIdx: Uint8Array over n little-endian uint32) -> {out, status}
 * (KeyPair.derive, ec/key.js:102-107, against key keyIdx[i]) */
static napi_value EcdhDeriveBatchKeyed(napi_env env, napi_callback_info info) {
  ARGS(3); BUF(1, k, lk); BUF(2, idx, li);
  size_t len = 0;
  eb200_keyset* ks = ecdsa_set(env, argv[0], &len);
  if (!ks) return fail(env, EB200_ERR_ARG);
  size_t n = li / 4;
  if (li != 4 * n || lk != n * len || ((uintptr_t)idx & 3)) return fail(env, EB200_ERR_ARG);
  uint8_t *out, *st;
  napi_value ao = out_u8(env, lk, &out), ast = out_u8(env, n, &st);
  int rc = eb200_ecdh_derive_batch_keyed(ks, n, k, (const uint32_t*)(const void*)idx, out, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "out", ao); SET(res, "status", ast);
  return res;
}

/* ecdsaRecoveryParamBatchKeyed(handle, e, r, s, keyIdx: Uint8Array over n little-endian uint32) -> {recid, status}
 * (getKeyRecoveryParam, ec/index.js:261-278, against key keyIdx[i]) */
static napi_value EcdsaRecoveryParamBatchKeyed(napi_env env, napi_callback_info info) {
  ARGS(5); BUF(1, e, le); BUF(2, r, lr); BUF(3, s, ls); BUF(4, idx, li);
  size_t len = 0;
  eb200_keyset* ks = ecdsa_set(env, argv[0], &len);
  if (!ks) return fail(env, EB200_ERR_ARG);
  size_t n = li / 4;
  if (li != 4 * n || le != n * len || lr != le || ls != le || ((uintptr_t)idx & 3)) return fail(env, EB200_ERR_ARG);
  uint8_t *id, *st;
  napi_value ai = out_u8(env, n, &id), ast = out_u8(env, n, &st);
  int rc = eb200_ecdsa_recovery_param_batch_keyed(ks, n, e, r, s, (const uint32_t*)(const void*)idx, id, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "recid", ai); SET(res, "status", ast);
  return res;
}

/* eddsaVerifyBatchKeyed(handle, R, S, h | null, msgs | null, msgOff | null, keyIdx: Uint8Array over n little-endian
 * uint32) -> Uint8Array(n) of statuses   (eddsa.verify against keys of an EdDSA set; h as eddsaVerifyBatch) */
static napi_value EddsaVerifyBatchKeyed(napi_env env, napi_callback_info info) {
  ARGS(7); BUF(1, R, a); BUF(2, S, b); OPT(3, h, d); OPT(4, msgs, lm); OPT(5, off, lo); BUF(6, idx, li);
  void* p = 0;
  if (napi_get_value_external(env, argv[0], &p) != napi_ok || !p || !((keyset_box*)p)->ks) return fail(env, EB200_ERR_ARG);
  eb200_keyset* ks = ((keyset_box*)p)->ks;
  size_t n = a / 32;
  if (a % 32 || b != a || li != 4 * n || ((uintptr_t)idx & 3) || (h && d != a) ||
      (!h && (lo != 8 * (n + 1) || ((uintptr_t)off & 7)))) return fail(env, EB200_ERR_ARG);
  if (!h) {
    const uint64_t* o = (const uint64_t*)off;
    for (size_t i = 0; i < n; i++) if (o[i + 1] < o[i]) return fail(env, EB200_ERR_ARG);
    if (o[n] > lm) return fail(env, EB200_ERR_ARG);
  }
  const uint32_t* ki = (const uint32_t*)(const void*)idx;
  uint8_t* st; napi_value arr = out_u8(env, n, &st);
  int rc = h ? eb200_eddsa_verify_batch_keyed(ks, n, R, S, h, ki, st)
             : eb200_eddsa_verify_batch_keyed_msgs(ks, n, R, S, msgs, (const uint64_t*)off, ki, st);
  return rc ? fail(env, rc) : arr;
}

/* x25519DeriveBatchKeyed(handle, priv: n x 32 big-endian (< n), keyIdx: Uint8Array over n little-endian uint32)
 * -> {out, status}   (KeyPair.derive, ec/key.js:102-107, against key keyIdx[i] of a curve25519 set) */
static napi_value X25519DeriveBatchKeyed(napi_env env, napi_callback_info info) {
  ARGS(3); BUF(1, k, lk); BUF(2, idx, li);
  void* p = 0;
  if (napi_get_value_external(env, argv[0], &p) != napi_ok || !p || !((keyset_box*)p)->ks) return fail(env, EB200_ERR_ARG);
  eb200_keyset* ks = ((keyset_box*)p)->ks;
  size_t n = li / 4;
  if (li != 4 * n || lk != 32 * n || ((uintptr_t)idx & 3)) return fail(env, EB200_ERR_ARG);
  uint8_t *out, *st;
  napi_value ao = out_u8(env, lk, &out), ast = out_u8(env, n, &st);
  int rc = eb200_x25519_derive_batch_keyed(ks, n, k, (const uint32_t*)(const void*)idx, out, st);
  if (rc) return fail(env, rc);
  napi_value res = obj(env);
  SET(res, "out", ao); SET(res, "status", ast);
  return res;
}

/* eddsaSigningSetCreate(secrets: m x 32) -> {handle, pub: Uint8Array(32 m)}   (eddsa.keyFromSecret for m keys) */
static napi_value EddsaSigningSetCreate(napi_env env, napi_callback_info info) {
  ARGS(1); BUF(0, sec, ls);
  size_t m = ls / 32;
  if (ls % 32) return fail(env, EB200_ERR_ARG);
  keyset_box* b = (keyset_box*)calloc(1, sizeof *b);
  if (!b) return fail(env, EB200_ERR_ARG);
  uint8_t* pub; napi_value apub = out_u8(env, 32 * m, &pub);
  int rc = eb200_eddsa_signing_set_create(m, sec, pub, &b->ks);
  if (rc) { free(b); return fail(env, rc); }
  napi_value o = obj(env), h;
  napi_create_external(env, b, keyset_finalize, 0, &h);
  SET(o, "handle", h); SET(o, "pub", apub);
  return o;
}
/* eddsaSignBatchKeyed(handle, msgs | null, msgOff, keyIdx: Uint8Array over n little-endian uint32) -> Uint8Array(64 n)
 * of signatures Rencoded || S   (key.sign(msg) for keys of a signing set) */
static napi_value EddsaSignBatchKeyed(napi_env env, napi_callback_info info) {
  ARGS(4); OPT(1, msgs, lm); BUF(2, off, lo); BUF(3, idx, li);
  void* p = 0;
  if (napi_get_value_external(env, argv[0], &p) != napi_ok || !p || !((keyset_box*)p)->ks) return fail(env, EB200_ERR_ARG);
  eb200_keyset* ks = ((keyset_box*)p)->ks;
  size_t n = li / 4;
  if (li != 4 * n || ((uintptr_t)idx & 3) || lo != 8 * (n + 1) || ((uintptr_t)off & 7)) return fail(env, EB200_ERR_ARG);
  const uint64_t* o = (const uint64_t*)off;
  for (size_t i = 0; i < n; i++) if (o[i + 1] < o[i]) return fail(env, EB200_ERR_ARG);
  if (o[n] > lm) return fail(env, EB200_ERR_ARG);
  uint8_t *sig, *st;
  napi_value asig = out_u8(env, 64 * n, &sig);
  out_u8(env, n, &st);                                                 /* always EB200_ST_TRUE */
  int rc = eb200_eddsa_sign_batch_keyed(ks, n, msgs, o, (const uint32_t*)(const void*)idx, sig, st);
  return rc ? fail(env, rc) : asig;
}

static napi_value Register(napi_env env, napi_value exports) {
  static const struct { const char* name; napi_callback cb; } fns[] = {
      {"init", Init}, {"ecdsaVerifyBatch", EcdsaVerifyBatch}, {"ecdsaVerifyBatchAsync", EcdsaVerifyBatchAsync},
      {"ecdsaVerifyBatchDer", EcdsaVerifyBatchDer}, {"ecdsaSignBatch", EcdsaSignBatch}, {"ecKeygenBatch", EcKeygenBatch},
      {"ecdsaRecoverBatch", EcdsaRecoverBatch}, {"ecdsaRecoveryParamBatch", EcdsaRecoveryParamBatch},
      {"mulAddBatch", MulAddBatch}, {"ecdhDeriveBatch", EcdhDeriveBatch},
      {"curveOpBatch", CurveOpBatch}, {"eddsaVerifyBatch", EddsaVerifyBatch}, {"eddsaSignBatch", EddsaSignBatch},
      {"x25519Batch", X25519Batch},
      {"keysetCreate", KeysetCreate}, {"keysetDestroy", KeysetDestroy}, {"ecdsaVerifyBatchKeyed", EcdsaVerifyBatchKeyed},
      {"ecdsaVerifyBatchKeyedDer", EcdsaVerifyBatchKeyedDer},
      {"eddsaKeysetCreate", EddsaKeysetCreate}, {"eddsaVerifyBatchKeyed", EddsaVerifyBatchKeyed},
      {"mulAddBatchKeyed", MulAddBatchKeyed}, {"ecdhDeriveBatchKeyed", EcdhDeriveBatchKeyed},
      {"ecdsaRecoveryParamBatchKeyed", EcdsaRecoveryParamBatchKeyed},
      {"eddsaSigningSetCreate", EddsaSigningSetCreate}, {"eddsaSignBatchKeyed", EddsaSignBatchKeyed},
      {"x25519KeysetCreate", X25519KeysetCreate}, {"x25519DeriveBatchKeyed", X25519DeriveBatchKeyed}};
  for (unsigned i = 0; i < sizeof fns / sizeof fns[0]; i++) {
    napi_value f;
    napi_create_function(env, fns[i].name, NAPI_AUTO_LENGTH, fns[i].cb, 0, &f);
    napi_set_named_property(env, exports, fns[i].name, f);
  }
  return exports;
}
static napi_module eb200_module = {1, 0, __FILE__, Register, "elliptic_b200", 0, {0}};
__attribute__((constructor)) static void eb200_register(void) { napi_module_register(&eb200_module); }
