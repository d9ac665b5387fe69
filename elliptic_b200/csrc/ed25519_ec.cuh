// ed25519_ec.cuh -- the `ec` API over the twisted Edwards preset: new elliptic.ec('ed25519')
// (the reference exercises it at test/ecdsa-test.js:130 and test/ecdh-test.js:26).
//
// Path replaced: EC.verify / sign / genKeyPair / KeyPair.derive (lib/elliptic/ec/index.js:55-229, ec/key.js:102-107)
// running on EdwardsCurve points: Point.mul / mulAdd / jmulAdd (curve/edwards.js:362-375 -> base.js:86-253),
// eqXToP (:415-431), isInfinity (:167-172), validate (:99-112), pointFromX (:46-69), BaseCurve.decodePoint
// (curve/base.js:270-292), and -- as batch entry points of the .curve API -- Point.mul / mulAdd themselves.
// Scalars run mod n on the CIOS Montgomery field of fp_mont.cuh; points use the extended-coordinate
// formulas and tables of ed25519_body.cuh (regular signed windows instead of the reference's wNAF: same
// group element for every on-curve input; un-validated off-curve points are flagged, status 4).
#pragma once
#include "ed25519_body.cuh"
#include "hmac_drbg_w.cuh"

namespace eb {

typedef Fp<ED25519_FN> EdS;

EB_HD f25 f25_from_be(const uint8_t* p) {           // toRed: any 256-bit value, reduced on use
  f25 r;
  load_be<8>(r.v, p);
  return r;
}
EB_HD void f25_to_be(uint8_t* p, const f25& a) {
  f25 n = f25_normalize(a);
  store_be<8>(p, n.v);
}
// a x^2 + y^2 == 1 + d x^2 y^2 with a = -1  (EdwardsCurve.validate, edwards.js:99-112)
EB_HD bool ed_on_curve(const f25& x, const f25& y) {
  f25 x2 = f25_sqr(x), y2 = f25_sqr(y);
  f25 lhs = f25_sub(y2, x2);
  f25 rhs = f25_add(f25_one(), f25_mul(f25_d(), f25_mul(x2, y2)));
  return f25_eq(lhs, rhs);
}
// sqrt(u / v): 0 and the root bn.js's Red.sqrt would be normalised from (the caller fixes the sign), or 5 when
// u / v is a non-residue (bn.js Tonelli-Shanks 'Assertion failed', dist:7220)
EB_HD uint8_t ed_sqrt_ratio(const f25& u, const f25& v, f25* root) {
  if (f25_is_zero(u)) { *root = f25_zero(); return 0; }
  f25 v3 = f25_mul(f25_sqr(v), v);
  f25 v7 = f25_mul(f25_sqr(v3), v);
  f25 xx = f25_mul(f25_mul(u, v3), f25_pow_p58(f25_mul(u, v7)));
  f25 vxx = f25_mul(v, f25_sqr(xx));
  if (!f25_eq(vxx, u)) {
    if (f25_eq(vxx, f25_neg(u))) xx = f25_mul(xx, f25_sqrt_m1());
    else return 5;
  }
  *root = xx;
  return 0;
}
// BaseCurve.decodePoint for the Edwards preset.  fmt 1: 04|06|07 || x || y (65 B); fmt 2: 02|03 || x (33 B,
// EdwardsCurve.pointFromX: y^2 = (1 + x^2) / (1 - d x^2)).  Writes x || y big-endian and a pre-status.
EB_HD uint8_t ed_ec_decode_pub(const uint8_t* in, u32 fmt, uint8_t* xy) {
  uint8_t tag = in[0];
  if (fmt == 1) {
    for (int k = 0; k < 64; k++) xy[k] = in[1 + k];
    if (tag != 4 && tag != 6 && tag != 7) return ST_THROW_POINT_FORMAT;
    if ((tag == 6 && (in[64] & 1)) || (tag == 7 && !(in[64] & 1))) return ST_THROW_ASSERT;      // base.js:278-281
    return 0;
  }
  for (int k = 0; k < 64; k++) xy[k] = 0;
  if (tag != 2 && tag != 3) return ST_THROW_POINT_FORMAT;
  f25 x = f25_from_be(in + 1);
  f25 x2 = f25_sqr(x);
  f25 u = f25_add(f25_one(), x2), v = f25_sub(f25_one(), f25_mul(f25_d(), x2));
  f25 y;
  uint8_t st = ed_sqrt_ratio(u, v, &y);
  if (st) return st;
  if (f25_is_odd(y) != (tag == 3)) y = f25_neg(y);
  f25_to_be(xy, x);
  f25_to_be(xy + 32, y);
  return 0;
}

// acc += s * G (fixed-base niels table), s < 2^255 little-endian limbs
EB_HD ed_ext ed_add_mul_base(ed_ext acc, const u32* s, const u32* gtab) {
  u32 S[8];
  {
    const u32 c19[8] = {0x02001000u, 0x00080040u, 0x04002001u, 0x00100080u, 0x08004002u, 0x00200100u, 0x10008004u, 0x00400200u};
    add_n<8>(S, s, c19);
  }
  for (int j = 0; j < ED_GWINDOWS; j++) {
    int pos = ED_GW * j, wi = pos >> 5;
    u32 lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) { lo = (k == wi) ? S[k] : lo; hi = (k == wi + 1) ? S[k] : hi; }
    u64 both = ((u64)hi << 32) | lo;
    int chunk = (int)((u32)(both >> (pos & 31)) & ((1u << ED_GW) - 1));
    int dg = (j == ED_GWINDOWS - 1) ? chunk : chunk - (1 << (ED_GW - 1));
    bool neg = dg < 0;
    u32 idx = (u32)(neg ? -dg : dg);
    const u32* ent = gtab + ((size_t)j * ED_GENTRIES + idx) * 24;
    ed_niels q;
    q.ypx = f25_load(ent); q.ymx = f25_load(ent + 8); q.t2d = f25_load(ent + 16);
    acc = ed_add_niels(acc, ed_niels_neg_if(q, neg));
  }
  return acc;
}
// k * P for an on-curve affine P (k: little-endian limbs): signed 4-bit windows over the per-item cached table
// {0..8} P in `tab` (ED_ATAB_WORDS words).  WINDOWS = 64 covers k < 2^253 (verify's u2 < n); WINDOWS = 65 covers any
// 256-bit k, the extra top window taking the carry out of the recoding (a digit of 0 or 1).
template <int WINDOWS>
EB_HD ed_ext ed_mul_var(const u32* k, const f25& px, const f25& py, u32* tab) {
  static_assert(WINDOWS == 64 || WINDOWS == 65, "ed_mul_var: 64 or 65 windows");
  {
    ed_ext p; p.x = px; p.y = py; p.z = f25_one(); p.t = f25_mul(px, py);
    ed_cached c1 = ed_to_cached(p);
    ed_ext acc = ed_identity();
    for (int m = 0; m <= 8; m++) {
      ed_cached c = ed_to_cached(acc);
      f25_store(tab + 32 * m, c.ypx); f25_store(tab + 32 * m + 8, c.ymx);
      f25_store(tab + 32 * m + 16, c.z); f25_store(tab + 32 * m + 24, c.t2d);
      if (m < 8) acc = ed_add_cached(acc, c1);
    }
  }
  u32 h[8], top;
  {
    const u32 off[8] = {0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u};
    top = add_n<8>(h, k, off);
  }
  ed_ext acc = ed_identity();
  if constexpr (WINDOWS == 65) {
    ed_cached c;
    c.ypx = f25_load(tab + 32 * top); c.ymx = f25_load(tab + 32 * top + 8);
    c.z = f25_load(tab + 32 * top + 16); c.t2d = f25_load(tab + 32 * top + 24);
    acc = ed_add_cached(acc, c);
  }
  for (int w = 63; w >= 0; w--) {
    if (WINDOWS == 65 || w != 63)
      for (int d = 0; d < 4; d++) acc = ed_dbl(acc);
    u32 word = 0;
#pragma unroll
    for (int m = 0; m < 8; m++) word = (m == (w >> 3)) ? h[m] : word;
    int dg = (int)((word >> (4 * (w & 7))) & 15) - 8;
    bool neg = dg < 0;
    u32 idx = (u32)(neg ? -dg : dg);
    ed_cached c;
    c.ypx = f25_load(tab + 32 * idx); c.ymx = f25_load(tab + 32 * idx + 8);
    c.z = f25_load(tab + 32 * idx + 16); c.t2d = f25_load(tab + 32 * idx + 24);
    acc = ed_add_cached(acc, ed_cached_neg_if(c, neg));
  }
  return acc;
}
// any 256-bit big-endian integer -> residue mod n as plain little-endian limbs
EB_HD void ed_scalar_mod_n(u32* out, const uint8_t* be32) {
  EdS::fe v;
  load_be<8>(v.v, be32);
  EdS::fe r = EdS::from_mont(EdS::to_mont(v));
  for (int w = 0; w < 8; w++) out[w] = r.v[w];
}

// EC.prototype.verify (ec/index.js:188-229) on ed25519.  e, r, s: 32 B big-endian; xy: x || y big-endian.
EB_HD uint8_t ed_ec_verify_item(size_t i, const uint8_t* e, const uint8_t* r, const uint8_t* s, const uint8_t* xy,
                                const uint8_t* pre, const u32* gtab, u32* atab) {
  if (pre && pre[i]) return pre[i];
  u32 nn[8], rv[8], sv[8];
  ed_n(nn);
  load_be<8>(rv, r + 32 * i);
  load_be<8>(sv, s + 32 * i);
  if (is_zero_n<8>(rv) || geq_n<8>(rv, nn) || is_zero_n<8>(sv) || geq_n<8>(sv, nn)) return ST_FALSE;   // :199-202
  f25 qx = f25_from_be(xy + 64 * i), qy = f25_from_be(xy + 64 * i + 32);
  if (!ed_on_curve(qx, qy)) return ST_NEEDS_HOST;                 // not validated by the reference (ec/key.js:95)
  EdS::fe sm, em, rm;
  copy_n<8>(sm.v, sv);
  load_be<8>(em.v, e + 32 * i);
  copy_n<8>(rm.v, rv);
  EdS::fe sinv = EdS::inv(EdS::to_mont(sm));
  EdS::fe u1 = EdS::from_mont(EdS::mul(EdS::to_mont(em), sinv));  // e s^-1 mod n
  EdS::fe u2 = EdS::from_mont(EdS::mul(EdS::to_mont(rm), sinv));  // r s^-1 mod n
  ed_ext acc = ed_mul_var<64>(u2.v, qx, qy, atab + (size_t)i * ED_ATAB_WORDS);
  acc = ed_add_mul_base(acc, u1.v, gtab);
  // p.isInfinity(): x == 0 && y == z  (edwards.js:167-172)
  if (f25_is_zero(acc.x) && f25_eq(acc.y, acc.z)) return ST_FALSE;
  // eqXToP (edwards.js:415-431): X == (r + j n) Z while r + j n < p
  f25 rz; copy_n<8>(rz.v, rv);
  f25 cur = f25_mul(rz, acc.z);
  if (f25_eq(acc.x, cur)) return ST_TRUE;
  f25 nf; copy_n<8>(nf.v, nn);
  f25 step = f25_mul(nf, acc.z);
  const u32 p25[8] = {0xffffffedu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x7fffffffu};
  u32 xc[8];
  copy_n<8>(xc, rv);
  for (int j = 0; j < 9; j++) {
    if (add_n<8>(xc, xc, nn)) return ST_FALSE;
    if (geq_n<8>(xc, p25)) return ST_FALSE;
    cur = f25_add(cur, step);
    if (f25_eq(acc.x, cur)) return ST_TRUE;
  }
  return ST_FALSE;
}

// One attempt of EC.sign's loop body for a nonce k (little-endian limbs, already truncated).
EB_HD bool ed_ec_sign_try(size_t i, const u32* k, const uint8_t* e, const uint8_t* priv, u32 canonical, const u32* gtab,
                          uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid) {
  u32 nn[8], ns1[8], one8[8] = {1, 0, 0, 0, 0, 0, 0, 0};
  ed_n(nn);
  sub_n<8>(ns1, nn, one8);
  bool le1 = (k[0] <= 1) && ((k[1] | k[2] | k[3] | k[4] | k[5] | k[6] | k[7]) == 0);
  if (le1 || geq_n<8>(k, ns1)) return false;                       // ec/index.js:158-159
  ed_ext kp = ed_add_mul_base(ed_identity(), k, gtab);
  f25 zi = f25_inv(kp.z);
  f25 x = f25_normalize(f25_mul(kp.x, zi)), y = f25_normalize(f25_mul(kp.y, zi));
  EdS::fe xm; copy_n<8>(xm.v, x.v);
  EdS::fe rmont = EdS::to_mont(xm);                                // kpX.umod(n)
  EdS::fe rp = EdS::from_mont(rmont);
  if (is_zero_n<8>(rp.v)) return false;
  EdS::fe km, dm, em;
  copy_n<8>(km.v, k);
  load_be<8>(dm.v, priv + 32 * i);
  load_be<8>(em.v, e + 32 * i);
  EdS::fe kinv = EdS::inv(EdS::to_mont(km));
  EdS::fe t = EdS::add(EdS::mul(rmont, EdS::to_mont(dm)), EdS::to_mont(em));
  EdS::fe sp = EdS::from_mont(EdS::mul(kinv, t));                  // k^-1 (r d + e) mod n
  if (is_zero_n<8>(sp.v)) return false;
  u32 rec = (y.v[0] & 1) | (eq_n<8>(x.v, rp.v) ? 0u : 2u);
  if (canonical) {
    u32 nh[8], d2[8];
    for (int w = 0; w < 8; w++) nh[w] = (nn[w] >> 1) | ((w < 7 ? nn[w + 1] : 0u) << 31);
    if (sub_n<8>(d2, nh, sp.v) != 0) { sub_n<8>(sp.v, nn, sp.v); rec ^= 1; }
  }
  store_be<8>(out_r + 32 * i, rp.v);
  store_be<8>(out_s + 32 * i, sp.v);
  out_recid[i] = (uint8_t)rec;
  return true;
}
// _truncateToN(k, true) for a 32-byte big-endian value against the 253-bit n
EB_HD void ed_ec_truncate_k(u32* k, const uint8_t* kb) {
  load_be<8>(k, kb);
  int top = 0;
  while (top < 32 && kb[top] == 0) top++;
  int delta = 8 * (32 - top) - 253;
  if (delta > 0)
    for (int w = 0; w < 8; w++) k[w] = (k[w] >> delta) | ((w + 1 < 8 ? k[w + 1] : 0u) << (32 - delta));
}
// EC.sign (ec/index.js:110-186) on ed25519: RFC 6979 nonces (HMAC-DRBG over SHA-256, curves.js:159), optionally
// with `pers`; or the caller's nonce for one attempt (kgiven, status EB200_ST_RETRY = 10 when the loop continues)
EB_HD uint8_t ed_ec_sign_item(size_t i, const uint8_t* e, const uint8_t* priv, const uint8_t* kgiven, const uint8_t* pers, int np,
                              u32 canonical, const u32* gtab, uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid) {
  u32 k[8];
  if (kgiven) {
    ed_ec_truncate_k(k, kgiven + 32 * i);
    return ed_ec_sign_try(i, k, e, priv, canonical, gtab, out_r, out_s, out_recid) ? ST_TRUE : (uint8_t)10;
  }
  HmacDrbgB<Sha256W> g;
  g.init(priv + 32 * i, 32, e + 32 * i, 32, pers, np);
  for (int iter = 0; iter < 256; iter++) {
    uint8_t kb[32];
    g.generate(kb, 32);
    ed_ec_truncate_k(k, kb);
    if (ed_ec_sign_try(i, k, e, priv, canonical, gtab, out_r, out_s, out_recid)) return ST_TRUE;
  }
  return ST_FALSE;
}
// EC.genKeyPair({entropy, pers}) (ec/index.js:55-79) on ed25519
EB_HD uint8_t ed_ec_keygen_item(size_t i, const uint8_t* entropy, int ne, const uint8_t* pers, int np, uint8_t* out_priv) {
  u32 nn[8], ns2[8], two[8] = {2, 0, 0, 0, 0, 0, 0, 0}, one[8] = {1, 0, 0, 0, 0, 0, 0, 0};
  ed_n(nn);
  sub_n<8>(ns2, nn, two);
  uint8_t nb[32];
  store_be<8>(nb, nn);
  HmacDrbgB<Sha256W> g;
  g.init(entropy + (size_t)ne * i, ne, nb, 32, pers, np);
  for (int iter = 0; iter < 65536; iter++) {
    uint8_t kb[32];
    g.generate(kb, 32);
    u32 k[8];
    load_be<8>(k, kb);
    if (geq_n<8>(k, ns2) && !eq_n<8>(k, ns2)) continue;            // priv.cmp(ns2) > 0
    add_n<8>(k, k, one);
    store_be<8>(out_priv + 32 * i, k);
    return ST_TRUE;
  }
  return ST_FALSE;
}

// Point.mul / Point.mulAdd (edwards.js:362-375) and KeyPair.derive (ec/key.js:102-107) on ed25519:
// k1 == NULL: k2 * P;  pts == NULL: k2 * G;  both: k1 * G + k2 * P.  Scalars: 32 B big-endian.  The reference uses k as
// given and the group has order 8n (cofactor 8), so P's scalar runs over all its 256 bits: reducing it mod n would
// change k2 * P whenever P has a torsion component.  G has order n and its scalars are reduced mod n; so is the
// private key of derive, as _importPrivate (ec/key.js:76-82) holds it.
// out: x || y big-endian (the neutral element is the ordinary point (0, 1)).  derive: x only semantics are
// applied by the host wrapper; an off-curve P is status 3 ('public point not validated') there, 4 otherwise.
EB_HD uint8_t ed_ec_mul_add_item(size_t i, const uint8_t* k1, const uint8_t* k2, const uint8_t* pts, bool derive,
                                 const u32* gtab, u32* atab, uint8_t* out) {
  for (int b = 0; b < 64; b++) out[64 * i + b] = 0;
  u32 s1[8], s2[8];
  ed_ext acc = ed_identity();
  if (pts) {
    f25 px = f25_from_be(pts + 64 * i), py = f25_from_be(pts + 64 * i + 32);
    if (!ed_on_curve(px, py)) return derive ? ST_THROW_NOT_VALIDATED : ST_NEEDS_HOST;
    if (derive) ed_scalar_mod_n(s2, k2 + 32 * i);
    else load_be<8>(s2, k2 + 32 * i);
    acc = ed_mul_var<65>(s2, px, py, atab + (size_t)i * ED_ATAB_WORDS);
    if (k1) { ed_scalar_mod_n(s1, k1 + 32 * i); acc = ed_add_mul_base(acc, s1, gtab); }
  } else {
    ed_scalar_mod_n(s2, k2 + 32 * i);
    acc = ed_add_mul_base(acc, s2, gtab);
  }
  f25 zi = f25_inv(acc.z);
  f25_to_be(out + 64 * i, f25_mul(acc.x, zi));
  f25_to_be(out + 64 * i + 32, f25_mul(acc.y, zi));
  return ST_TRUE;
}

}  // namespace eb
