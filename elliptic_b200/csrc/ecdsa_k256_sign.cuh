// ecdsa_k256_sign.cuh -- batch ECDSA signing on secp256k1 (SURVEY 8f row 1 / 8a row a20).
//
// Reference: EC.prototype.sign, lib/elliptic/ec/index.js:110-186 -- RFC 6979 nonces from
// HMAC-DRBG(SHA-256) seeded with key || msg (hmac-drbg, dist/elliptic.js:8686-8800), the retry loop
// (:153-185), k*G by Point.mul -> _fixedNafMul (short.js:422-432, base.js:52-84), JPoint.toP
// (short.js:516-526), s = k^-1 (r d + e) mod n, recoveryParam, and the `canonical` option.
// Everything, including the DRBG, runs in one thread per signature; k*G reuses the verify
// kernel's fixed-base table (16-bit signed-odd windows: 16 mixed adds, no doublings).
#pragma once
#include "ecdsa_k256_body.cuh"
#include "sha2.cuh"

namespace eb {

// a^(p-2) by the standard secp256k1 addition chain (255 squarings + 15 multiplications)
EB_HD fe fe_sqr_n(fe a, int n) { for (int i = 0; i < n; i++) a = fe_sqr(a); return a; }
EB_HD fe fe_inv_chain(const fe& a) {
  fe x2 = fe_mul(fe_sqr(a), a);
  fe x3 = fe_mul(fe_sqr(x2), a);
  fe x6 = fe_mul(fe_sqr_n(x3, 3), x3);
  fe x9 = fe_mul(fe_sqr_n(x6, 3), x3);
  fe x11 = fe_mul(fe_sqr_n(x9, 2), x2);
  fe x22 = fe_mul(fe_sqr_n(x11, 11), x11);
  fe x44 = fe_mul(fe_sqr_n(x22, 22), x22);
  fe x88 = fe_mul(fe_sqr_n(x44, 44), x44);
  fe x176 = fe_mul(fe_sqr_n(x88, 88), x88);
  fe x220 = fe_mul(fe_sqr_n(x176, 44), x44);
  fe x223 = fe_mul(fe_sqr_n(x220, 3), x3);
  // p - 2 = 2^256 - 2^32 - 979: bits 255..33 all ones except bit 32; low 32 bits 0xFFFFFC2D
  fe t = fe_mul(fe_sqr_n(x223, 23), x22);
  t = fe_mul(fe_sqr_n(t, 5), a);
  t = fe_mul(fe_sqr_n(t, 3), x2);
  t = fe_mul(fe_sqr_n(t, 2), a);
  return t;
}

struct hmac_drbg { uint8_t K[32], V[32]; };

// HmacDRBG._update, dist:8735-8752
EB_HD void drbg_update(hmac_drbg* d, const uint8_t* seed, size_t n) {
  uint8_t b0 = 0x00, b1 = 0x01, t[32];
  hmac_sha256(d->K, d->V, 32, &b0, 1, seed, n, t);
  for (int i = 0; i < 32; i++) d->K[i] = t[i];
  hmac_sha256(d->K, d->V, 32, 0, 0, 0, 0, t);
  for (int i = 0; i < 32; i++) d->V[i] = t[i];
  if (!n) return;
  hmac_sha256(d->K, d->V, 32, &b1, 1, seed, n, t);
  for (int i = 0; i < 32; i++) d->K[i] = t[i];
  hmac_sha256(d->K, d->V, 32, 0, 0, 0, 0, t);
  for (int i = 0; i < 32; i++) d->V[i] = t[i];
}
// HmacDRBG ctor + _init, dist:8692-8733: seed = entropy || nonce || pers (pers empty here)
EB_HD void drbg_init(hmac_drbg* d, const uint8_t* entropy32, const uint8_t* nonce32) {
  for (int i = 0; i < 32; i++) { d->K[i] = 0x00; d->V[i] = 0x01; }
  uint8_t seed[64];
  for (int i = 0; i < 32; i++) { seed[i] = entropy32[i]; seed[32 + i] = nonce32[i]; }
  drbg_update(d, seed, 64);
}
// HmacDRBG.generate(32), dist:8771-8797
EB_HD void drbg_generate32(hmac_drbg* d, uint8_t* out) {
  uint8_t t[32];
  hmac_sha256(d->K, d->V, 32, 0, 0, 0, 0, t);
  for (int i = 0; i < 32; i++) { d->V[i] = t[i]; out[i] = t[i]; }
  drbg_update(d, 0, 0);
}

// k*G for 0 < k < n via the fixed table of ecdsa_k256_body.cuh; affine canonical result.
EB_HD ge_aff k256_mul_g(const u32* k, const u32* gtab) {
  u32 nn[8], kk[8];
  K256N::n(nn);
  copy_n<8>(kk, k);
  bool negg = (kk[0] & 1) == 0;
  if (negg) sub_n<8>(kk, nn, kk);                 // n - k is odd; (n-k) G = -(k G)
  u32 m[8];
  for (int w = 0; w < 8; w++) m[w] = (kk[w] >> 1) | ((w < 7 ? kk[w + 1] : 0u) << 31);
  ge_jac acc = jac_infinity();
  for (int j = 0; j < GTAB_WINDOWS; j++) {
    const int pos = GTAB_W * j;
    u32 lo = 0, hi = 0;
    for (int w = 0; w < 8; w++) { lo = (w == (pos >> 5)) ? m[w] : lo; hi = (w == (pos >> 5) + 1) ? m[w] : hi; }
    u64 both = ((u64)hi << 32) | lo;
    u32 chunk = (u32)(both >> (pos & 31)) & ((1u << GTAB_W) - 1);
    const u32 half = 1u << (GTAB_W - 1);
    bool dneg = (j != GTAB_WINDOWS - 1) && (chunk < half);
    u32 idx = (j == GTAB_WINDOWS - 1) ? (chunk & (half - 1)) : (dneg ? half - 1 - chunk : chunk - half);
    const u32* ent = gtab + ((size_t)j * GTAB_ENTRIES + idx) * 16;
    ge_aff P;
    P.x = load_fe(ent);
    P.y = load_fe(ent + 8);
    acc = jac_madd(acc, aff_neg_if(P, dneg != negg));
  }
  fe zi = fe_inv_chain(acc.z);                    // JPoint.toP, short.js:516-526
  fe zi2 = fe_sqr(zi);
  ge_aff r;
  r.x = fe_normalize(fe_mul(acc.x, zi2));
  r.y = fe_normalize(fe_mul(fe_mul(acc.y, zi2), zi));
  return r;
}

// G.mul(k) (short.js:422-427 -> _fixedNafMul, base.js:52-84) for any 256-bit k: affine x||y, or infinity.
EB_HD uint8_t k256_mul_g_item(size_t i, const uint8_t* k, const u32* gtab, uint8_t* out) {
  u32 nn[8], kv[8];
  K256N::n(nn);
  load_be<8>(kv, k + 32 * i);
  if (geq_n<8>(kv, nn)) sub_n<8>(kv, kv, nn);
  for (int b = 0; b < 64; b++) out[64 * i + b] = 0;
  if (is_zero_n<8>(kv)) return ST_INFINITY;
  ge_aff r = k256_mul_g(kv, gtab);
  store_be<8>(out + 64 * i, r.x.v);
  store_be<8>(out + 64 * i + 32, r.y.v);
  return ST_TRUE;
}

// getKeyRecoveryParam for the items recovery_param_item leaves as ST_NEEDS_HOST: s = 0, r != 0 (mod n).  There
// s2 = s rInv = 0, so recoverPubKey(e, sig, j) returns s1 G = ((n - e) / r) G for every j whose candidate exists, and the
// answer is the first such j when Q is that point.  Candidates exist as recover_item finds them: j = 0 (and 1) when
// r is an x coordinate, j = 2 (and 3) when r + n < p is one.
EB_HD uint8_t recovery_param_cold_item(size_t i, const uint8_t* e, const uint8_t* r, const uint8_t* q, const u32* gtab,
                                       uint8_t* recid) {
  u32 R2[8], nn[8], rv[8], ev[8], rm[8], rinv[8], k[8];
  K256N::r2(R2); K256N::n(nn);
  load_be<8>(rv, r + 32 * i);
  load_be<8>(ev, e + 32 * i);
  sc_mont_mul(rm, rv, R2);                        // r mod n, Montgomery form
  sc_mont_inv(rinv, rm);
  sc_mont_mul(k, ev, rinv);                       // e / r
  if (is_zero_n<8>(k)) return ST_THROW_NO_RECOVERY;   // s1 = 0: every Q' is the point at infinity
  sub_n<8>(k, nn, k);                             // (n - e) / r
  ge_aff T = k256_mul_g(k, gtab);
  if (!fe_eq(fe_from_be(q + 64 * i), T.x) || !fe_eq(fe_from_be(q + 64 * i + 32), T.y)) return ST_THROW_NO_RECOVERY;
  const u32 pmn[8] = {0x2fc9baeeu, 0x402da172u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0, 0, 0};  // p mod n = p - n
  for (u32 j = 0; j < 4; j += 2) {
    if (j == 2 && geq_n<8>(rv, pmn)) break;       // 'Unable to find sencond key candinate'
    fe x;
    copy_n<8>(x.v, rv);
    if (j == 2) add_n<8>(x.v, rv, nn);
    fe seven = fe_zero(); seven.v[0] = 7;
    fe y2 = fe_add(fe_mul(fe_sqr(x), x), seven);
    fe y = fe_sqrt_candidate(y2);
    if (fe_eq(fe_sqr(y), y2)) { recid[i] = (uint8_t)j; return ST_TRUE; }
  }
  return ST_THROW_NO_RECOVERY;
}

// One attempt of the loop body of ec/index.js:153-185 for a given nonce k (little-endian limbs, already
// _truncateToN(k, true)'d): false = the reference `continue`s (k out of range, r = 0 or s = 0).
EB_HD bool k256_sign_try(size_t i, const u32* k, const u32* ev, const u32* dv, u32 canonical, const u32* gtab,
                         uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid) {
  u32 nn[8], R2[8], ns1[8], one8[8] = {1, 0, 0, 0, 0, 0, 0, 0};
  K256N::n(nn); K256N::r2(R2);
  sub_n<8>(ns1, nn, one8);
  bool le1 = (k[0] <= 1) && ((k[1] | k[2] | k[3] | k[4] | k[5] | k[6] | k[7]) == 0);
  if (le1 || geq_n<8>(k, ns1)) return false;       // ec/index.js:158-159
  ge_aff kp = k256_mul_g(k, gtab);
  u32 r[8];
  copy_n<8>(r, kp.x.v);
  bool xr_differ = geq_n<8>(r, nn);
  if (xr_differ) sub_n<8>(r, r, nn);               // kpX.umod(n)
  if (is_zero_n<8>(r)) return false;
  u32 km[8], kinv[8], dm[8], rd[8], t[8], s[8];
  sc_mont_mul(km, k, R2);
  sc_mont_inv(kinv, km);                           // k^-1, Montgomery form
  sc_mont_mul(dm, dv, R2);
  sc_mont_mul(rd, r, dm);                          // r * d mod n
  u32 cy = add_n<8>(t, rd, ev);
  if (cy || geq_n<8>(t, nn)) sub_n<8>(t, t, nn);   // + e mod n
  sc_mont_mul(s, t, kinv);                         // k^-1 (r d + e) mod n
  if (is_zero_n<8>(s)) return false;
  u32 rec = (kp.y.v[0] & 1) | (xr_differ ? 2u : 0u);
  if (canonical) {
    u32 nh[8];
    for (int w = 0; w < 8; w++) nh[w] = (nn[w] >> 1) | ((w < 7 ? nn[w + 1] : 0u) << 31);
    u32 d2[8];
    bool gt = sub_n<8>(d2, nh, s) != 0;            // s > n/2
    if (gt) { sub_n<8>(s, nn, s); rec ^= 1; }
  }
  store_be<8>(out_r + 32 * i, r);
  store_be<8>(out_s + 32 * i, s);
  out_recid[i] = (uint8_t)rec;
  return true;
}

// One signature.  e: _truncateToN(msg) (32 bytes BE, < n); priv: the key pair's private scalar
// (32 bytes BE, already reduced mod n, ec/key.js:76-82).  Writes r, s (32 B BE) and the recovery param.
EB_HD uint8_t k256_sign_item(size_t i, const uint8_t* e, const uint8_t* priv, u32 canonical, const u32* gtab,
                             uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid) {
  u32 ev[8], dv[8];
  load_be<8>(ev, e + 32 * i);
  load_be<8>(dv, priv + 32 * i);
  hmac_drbg drbg;
  drbg_init(&drbg, priv + 32 * i, e + 32 * i);    // entropy = bkey, nonce = msg (ec/index.js:135-148)
  for (int iter = 0; iter < 128; iter++) {
    uint8_t kb[32];
    drbg_generate32(&drbg, kb);
    u32 k[8];
    load_be<8>(k, kb);                             // _truncateToN(k, true): 32 bytes, no shift
    if (k256_sign_try(i, k, ev, dv, canonical, gtab, out_r, out_s, out_recid)) return ST_TRUE;
  }
  return ST_FALSE;   // unreachable in practice (2^-128 per iteration)
}

}  // namespace eb
