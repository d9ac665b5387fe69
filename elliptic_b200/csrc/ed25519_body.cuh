// ed25519_body.cuh -- batch EdDSA (ed25519) verify and curve25519 ECDH bodies.
//
// Reference paths (lib/elliptic):
//   eddsa/index.js:52-63   EDDSA.verify: S < n; h = SHA512(R||A||M) mod n; accept iff
//                          R + h*A == S*G as affine points; throws on undecodable R / A
//   eddsa/index.js:100-109 decodePoint -> curve/edwards.js:71-97 pointFromY
//   curve/edwards.js:174-205, 279-309  _extDbl / _extAdd (a = -1 extended coordinates)
//   curve/base.js:52-126   _fixedNafMul (S*G) and _wnafMul (h*A)
//   ec/key.js:102-107      KeyPair.derive -> curve/mont.js:21-28 validate, :130-153 ladder, :173-178 getX
// Same outputs, GPU schedule: one thread per item, complete twisted-Edwards formulas (no
// exceptional cases for points on the curve, small-order ones included), h*A by fixed signed
// 4-bit windows over a per-item table of -A multiples, S*G by 13-bit windows over a fixed table;
// one exponentiation per decompression instead of inversion + Tonelli-Shanks.
#pragma once
#include "fe_25519.cuh"
#include "sw_params.cuh"
#include "sha2.cuh"

namespace eb {

struct ed_ext { f25 x, y, z, t; };
struct ed_cached { f25 ypx, ymx, z, t2d; };
struct ed_niels { f25 ypx, ymx, t2d; };

constexpr int ED_GW = 13;                         // fixed-base window width
constexpr int ED_GWINDOWS = 20;                   // 19 signed windows + an unsigned top one (bits 247..)
constexpr int ED_GENTRIES = (1 << (ED_GW - 1)) + 1;   // i * 2^(13 j) * G, i = 0..4096
constexpr int ED_ATAB_WORDS = 9 * 32;             // per item: 0..8 multiples of -A in cached form

EB_HD ed_ext ed_identity() { ed_ext r; r.x = f25_zero(); r.y = f25_one(); r.z = f25_one(); r.t = f25_zero(); return r; }

// dbl-2008-hwcd, a = -1  (edwards.js:174-205)
EB_HD ed_ext ed_dbl_inl(const ed_ext& p) {
  f25 a = f25_sqr_hot(p.x);
  f25 b = f25_sqr_hot(p.y);
  f25 c = f25_dbl(f25_sqr_hot(p.z));
  f25 d = f25_neg(a);
  f25 e = f25_sub(f25_sub(f25_sqr_hot(f25_add(p.x, p.y)), a), b);
  f25 g = f25_add(d, b);
  f25 f = f25_sub(g, c);
  f25 h = f25_sub(d, b);
  ed_ext r;
  r.x = f25_mul(e, f);
  r.y = f25_mul(g, h);
  r.t = f25_mul(e, h);
  r.z = f25_mul(f, g);
  return r;
}

// add-2008-hwcd-3 with the second operand pre-arranged (edwards.js:279-309)
EB_HD ed_ext ed_add_cached_inl(const ed_ext& p, const ed_cached& q) {
  f25 a = f25_mul(f25_sub(p.y, p.x), q.ymx);
  f25 b = f25_mul(f25_add(p.y, p.x), q.ypx);
  f25 c = f25_mul(p.t, q.t2d);
  f25 d = f25_dbl(f25_mul(p.z, q.z));
  f25 e = f25_sub(b, a);
  f25 f = f25_sub(d, c);
  f25 g = f25_add(d, c);
  f25 h = f25_add(b, a);
  ed_ext r;
  r.x = f25_mul(e, f);
  r.y = f25_mul(g, h);
  r.t = f25_mul(e, h);
  r.z = f25_mul(f, g);
  return r;
}
EB_HD ed_ext ed_add_niels_inl(const ed_ext& p, const ed_niels& q) {
  f25 a = f25_mul(f25_sub(p.y, p.x), q.ymx);
  f25 b = f25_mul(f25_add(p.y, p.x), q.ypx);
  f25 c = f25_mul(p.t, q.t2d);
  f25 d = f25_dbl(p.z);
  f25 e = f25_sub(b, a);
  f25 f = f25_sub(d, c);
  f25 g = f25_add(d, c);
  f25 h = f25_add(b, a);
  ed_ext r;
  r.x = f25_mul(e, f);
  r.y = f25_mul(g, h);
  r.t = f25_mul(e, h);
  r.z = f25_mul(f, g);
  return r;
}
#if defined(__CUDACC__)
#define EB_EDFN __host__ __device__ __noinline__
#else
#define EB_EDFN
#endif
EB_EDFN ed_ext ed_dbl(ed_ext p) { return ed_dbl_inl(p); }
EB_EDFN ed_ext ed_add_cached(ed_ext p, ed_cached q) { return ed_add_cached_inl(p, q); }
EB_EDFN ed_ext ed_add_niels(ed_ext p, ed_niels q) { return ed_add_niels_inl(p, q); }

EB_HD ed_cached ed_to_cached(const ed_ext& p) {
  ed_cached c;
  c.ypx = f25_add(p.y, p.x);
  c.ymx = f25_sub(p.y, p.x);
  c.z = p.z;
  c.t2d = f25_mul(p.t, f25_2d());
  return c;
}
EB_HD ed_cached ed_cached_neg_if(const ed_cached& c, bool neg) {
  ed_cached r;
  r.ypx = f25_cmov(c.ypx, c.ymx, neg);
  r.ymx = f25_cmov(c.ymx, c.ypx, neg);
  r.z = c.z;
  r.t2d = f25_cmov(c.t2d, f25_neg(c.t2d), neg);
  return r;
}
EB_HD ed_niels ed_niels_neg_if(const ed_niels& c, bool neg) {
  ed_niels r;
  r.ypx = f25_cmov(c.ypx, c.ymx, neg);
  r.ymx = f25_cmov(c.ymx, c.ypx, neg);
  r.t2d = f25_cmov(c.t2d, f25_neg(c.t2d), neg);
  return r;
}

EB_HD void ed_G(f25* x, f25* y) {
  const u32 gx[8] = {0x8f25d51au, 0xc9562d60u, 0x9525a7b2u, 0x692cc760u, 0xfdd6dc5cu, 0xc0a4e231u, 0xcd6e53feu, 0x216936d3u};
  const u32 gy[8] = {0x66666658u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u, 0x66666666u};
  for (int i = 0; i < 8; i++) { x->v[i] = gx[i]; y->v[i] = gy[i]; }
}
EB_HD void ed_n(u32* r) {
  const u32 v[8] = {0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0, 0, 0, 0x10000000u};
  for (int i = 0; i < 8; i++) r[i] = v[i];
}

// EdwardsCurve.pointFromY on the 32-byte wire form (eddsa/index.js:100-109 + edwards.js:71-97).
// Returns 0 when the reference decodes the point, else the status of the Error it throws:
// ST 2 'invalid point' (x = 0 with the sign bit set), ST 5 'Assertion failed' (bn.js Red.sqrt on a
// non-residue, dist:7220).  Non-canonical y (>= p) is accepted and reduced, as `toRed` does.
EB_HD uint8_t ed_decode(const uint8_t* enc, f25* x, f25* y) {
  f25 yy;
  load_le<8>(yy.v, enc);
  bool odd = (yy.v[7] >> 31) != 0;
  yy.v[7] &= 0x7FFFFFFFu;
  f25 y2 = f25_sqr(yy);
  f25 u = f25_sub(y2, f25_one());
  f25 v = f25_add(f25_mul(y2, f25_d()), f25_one());
  *y = yy;
  if (f25_is_zero(u)) {                       // x^2 = 0
    *x = f25_zero();
    return odd ? 2 : 0;
  }
  f25 v3 = f25_mul(f25_sqr(v), v);
  f25 v7 = f25_mul(f25_sqr(v3), v);
  f25 xx = f25_mul(f25_mul(u, v3), f25_pow_p58(f25_mul(u, v7)));
  f25 vxx = f25_mul(v, f25_sqr(xx));
  if (!f25_eq(vxx, u)) {
    if (f25_eq(vxx, f25_neg(u))) xx = f25_mul(xx, f25_sqrt_m1());
    else return 5;
  }
  if (f25_is_odd(xx) != odd) xx = f25_neg(xx);
  *x = xx;
  return 0;
}

// fixed-base entry (j, i) = i * 2^(13 j) * G in niels form, i = 0..4096
EB_HD void ed_gtab_entry(int j, int idx, u32* out24) {
  ed_ext g = ed_identity();
  ed_G(&g.x, &g.y);
  g.t = f25_mul(g.x, g.y);
  for (int k = 0; k < ED_GW * j; k++) g = ed_dbl(g);
  ed_cached base = ed_to_cached(g);
  ed_ext acc = ed_identity();
  for (int k = ED_GW - 1; k >= 0; k--) {
    acc = ed_dbl(acc);
    if ((idx >> k) & 1) acc = ed_add_cached(acc, base);
  }
  f25 zi = f25_inv(acc.z);
  f25 x = f25_mul(acc.x, zi), y = f25_mul(acc.y, zi);
  ed_niels n;
  n.ypx = f25_normalize(f25_add(y, x));
  n.ymx = f25_normalize(f25_sub(y, x));
  n.t2d = f25_normalize(f25_mul(f25_mul(x, y), f25_2d()));
  f25_store(out24, n.ypx); f25_store(out24 + 8, n.ymx); f25_store(out24 + 16, n.t2d);
}

// One signature.  R, S, A, h: N x 32 bytes little-endian (wire format; h = SHA512(R||A||M) mod n,
// eddsa/index.js:65-70, computed by the caller).  atab: N x ED_ATAB_WORDS words of scratch.
EB_HD uint8_t ed25519_verify_item(size_t i, const uint8_t* Rb, const uint8_t* Sb, const uint8_t* Ab,
                                  const uint8_t* hb, const u32* gtab, u32* atab) {
  u32 S[8], n[8];
  load_le<8>(S, Sb + 32 * i);
  ed_n(n);
  if (geq_n<8>(S, n)) return 0;                                   // eddsa/index.js:55-57
  f25 rx, ry, ax, ay;
  uint8_t st = ed_decode(Rb + 32 * i, &rx, &ry);                  // sig.R()
  if (st) return st;
  st = ed_decode(Ab + 32 * i, &ax, &ay);                          // key.pub()
  if (st) return st;

  // table of k * (-A), k = 0..8, cached form
  u32* tab = atab + (size_t)i * ED_ATAB_WORDS;
  {
    ed_ext na; na.x = f25_neg(ax); na.y = ay; na.z = f25_one(); na.t = f25_mul(na.x, ay);
    ed_cached c1 = ed_to_cached(na);
    ed_ext acc = ed_identity();
    for (int k = 0; k <= 8; k++) {
      ed_cached c = ed_to_cached(acc);
      f25_store(tab + 32 * k, c.ypx); f25_store(tab + 32 * k + 8, c.ymx);
      f25_store(tab + 32 * k + 16, c.z); f25_store(tab + 32 * k + 24, c.t2d);
      if (k < 8) acc = ed_add_cached(acc, c1);
    }
  }
  // h' = h + 0x88..8 : digit_w = nibble_w(h') - 8 in [-8, 7]
  u32 h[8];
  load_le<8>(h, hb + 32 * i);
  {
    const u32 off[8] = {0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u};
    add_n<8>(h, h, off);
  }
  ed_ext acc = ed_identity();
  for (int w = 63; w >= 0; w--) {
    if (w != 63)
      for (int d = 0; d < 4; d++) acc = ed_dbl(acc);
    u32 word = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) word = (k == (w >> 3)) ? h[k] : word;
    int dg = (int)((word >> (4 * (w & 7))) & 15) - 8;
    bool neg = dg < 0;
    u32 idx = (u32)(neg ? -dg : dg);
    ed_cached c;
    c.ypx = f25_load(tab + 32 * idx); c.ymx = f25_load(tab + 32 * idx + 8);
    c.z = f25_load(tab + 32 * idx + 16); c.t2d = f25_load(tab + 32 * idx + 24);
    acc = ed_add_cached(acc, ed_cached_neg_if(c, neg));
  }
  // + S*G: S' = S + sum_{j<19} 2^(13j+12); digits j<19: chunk - 4096, top: chunk
  {
    const u32 c19[8] = {0x02001000u, 0x00080040u, 0x04002001u, 0x00100080u, 0x08004002u, 0x00200100u, 0x10008004u, 0x00400200u};
    add_n<8>(S, S, c19);
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
  // S*G - h*A == R as affine points  (edwards.js:409-413)
  bool ok = f25_eq(acc.x, f25_mul(rx, acc.z)) && f25_eq(acc.y, f25_mul(ry, acc.z));
  return ok ? 1 : 0;
}

// EDDSA.hashInt for verify (eddsa/index.js:59,65-70): h = SHA512(Rencoded || pubBytes || message) as a
// little-endian integer, mod n.  Writes 32 bytes little-endian.
EB_HD void ed25519_hash_item(size_t i, const uint8_t* Rb, const uint8_t* Ab, const uint8_t* msgs,
                             const u64* msg_off, uint8_t* h_out) {
  sha512_ctx c;
  sha512_init(&c);
  sha512_update(&c, Rb + 32 * i, 32);
  sha512_update(&c, Ab + 32 * i, 32);
  sha512_update(&c, msgs + msg_off[i], (size_t)(msg_off[i + 1] - msg_off[i]));
  uint8_t dg[64];
  sha512_final(&c, dg);
  typedef Fp<ED25519_FN> S;
  S::fe lo, hi;
  load_le<8>(lo.v, dg);
  load_le<8>(hi.v, dg + 32);
  S::fe r = S::add(S::from_mont(S::to_mont(lo)), S::to_mont(hi));   // lo mod n + hi * 2^256 mod n
  for (int k = 0; k < 8; k++) {
    h_out[32 * i + 4 * k] = (uint8_t)r.v[k]; h_out[32 * i + 4 * k + 1] = (uint8_t)(r.v[k] >> 8);
    h_out[32 * i + 4 * k + 2] = (uint8_t)(r.v[k] >> 16); h_out[32 * i + 4 * k + 3] = (uint8_t)(r.v[k] >> 24);
  }
}

// ---------------------------------------------------------------------------
// EDDSA.prototype.sign (eddsa/index.js:34-44) with KeyPair.fromSecret (eddsa/key.js:52-75):
//   hash = SHA512(secret);  a = clamp(hash[0..31]);  prefix = hash[32..63];  A = a*G
//   r = SHA512(prefix || M) mod n;  R = r*G;  S = (r + SHA512(Renc || Aenc || M) * a) mod n;  sig = Renc || S
// Both scalar multiplications are fixed-base (the verify kernel's 13-bit window table, 20 additions each).

// s * G for a 256-bit little-endian scalar s < 2^255 (signed 13-bit windows over the niels table)
EB_HD ed_ext ed_mul_base(const u32* s, const u32* gtab) {
  u32 S[8];
  {
    const u32 c19[8] = {0x02001000u, 0x00080040u, 0x04002001u, 0x00100080u, 0x08004002u, 0x00200100u, 0x10008004u, 0x00400200u};
    add_n<8>(S, s, c19);
  }
  ed_ext acc = ed_identity();
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
// EDDSA.encodePoint (eddsa/index.js:94-98) of the affine point (x, y), both fully reduced (f25_normalize):
// y little-endian, x parity in the top bit
EB_HD void ed_encode_affine(const f25& x, const f25& y, uint8_t* out32) {
  for (int k = 0; k < 8; k++) {
    out32[4 * k] = (uint8_t)y.v[k]; out32[4 * k + 1] = (uint8_t)(y.v[k] >> 8);
    out32[4 * k + 2] = (uint8_t)(y.v[k] >> 16); out32[4 * k + 3] = (uint8_t)(y.v[k] >> 24);
  }
  out32[31] |= (x.v[0] & 1) ? 0x80 : 0;
}
// the same for a point in extended coordinates: one inversion
EB_HD void ed_encode(const ed_ext& p, uint8_t* out32) {
  f25 zi = f25_inv(p.z);
  f25 x = f25_normalize(f25_mul(p.x, zi)), y = f25_normalize(f25_mul(p.y, zi));
  ed_encode_affine(x, y, out32);
}
// 64-byte digest as a little-endian integer mod n, Montgomery form of the scalar field
EB_HD Fp<ED25519_FN>::fe ed_digest_mod_n(const uint8_t* dg) {
  typedef Fp<ED25519_FN> S;
  S::fe lo, hi;
  load_le<8>(lo.v, dg);
  load_le<8>(hi.v, dg + 32);
  // to_mont(lo) = lo R ; to_mont(to_mont(hi)) = hi R^2 = (hi 2^256) R
  return S::add(S::to_mont(lo), S::to_mont(S::to_mont(hi)));
}
// secrets: N x 32 bytes; msgs + msg_off: concatenated messages; sig: N x 64 out; pub: N x 32 out or NULL
EB_HD uint8_t ed25519_sign_item(size_t i, const uint8_t* secrets, const uint8_t* msgs, const u64* msg_off,
                                const u32* gtab, uint8_t* sig, uint8_t* pub) {
  typedef Fp<ED25519_FN> S;
  uint8_t hash[64], dg[64], aenc[32];
  sha512_ctx c;
  sha512_init(&c);
  sha512_update(&c, secrets + 32 * i, 32);
  sha512_final(&c, hash);
  hash[0] &= 248; hash[31] &= 127; hash[31] |= 64;                  // eddsa/key.js:58-62
  u32 a[8];
  load_le<8>(a, hash);
  ed_encode(ed_mul_base(a, gtab), aenc);                            // pubBytes
  if (pub) for (int k = 0; k < 32; k++) pub[32 * i + k] = aenc[k];
  const uint8_t* m = msgs + msg_off[i];
  const size_t ml = (size_t)(msg_off[i + 1] - msg_off[i]);
  sha512_init(&c);
  sha512_update(&c, hash + 32, 32);                                 // messagePrefix
  sha512_update(&c, m, ml);
  sha512_final(&c, dg);
  S::fe r = ed_digest_mod_n(dg);
  S::fe rp = S::from_mont(r);                                       // r < n, plain
  uint8_t* renc = sig + 64 * i;
  ed_encode(ed_mul_base(rp.v, gtab), renc);
  sha512_init(&c);
  sha512_update(&c, renc, 32);
  sha512_update(&c, aenc, 32);
  sha512_update(&c, m, ml);
  sha512_final(&c, dg);
  S::fe h = ed_digest_mod_n(dg);
  S::fe am; for (int k = 0; k < 8; k++) am.v[k] = a[k];
  S::fe sv = S::from_mont(S::add(r, S::mul(h, S::to_mont(am))));    // (r + h a) mod n
  for (int k = 0; k < 8; k++) {
    sig[64 * i + 32 + 4 * k] = (uint8_t)sv.v[k]; sig[64 * i + 32 + 4 * k + 1] = (uint8_t)(sv.v[k] >> 8);
    sig[64 * i + 32 + 4 * k + 2] = (uint8_t)(sv.v[k] >> 16); sig[64 * i + 32 + 4 * k + 3] = (uint8_t)(sv.v[k] >> 24);
  }
  // the clamped key and the nonce must not stay in local memory beyond this call
  for (int k = 0; k < 64; k++) hash[k] = 0;
  return 1;
}

// ---------------------------------------------------------------------------
// curve25519 ECDH: KeyPair.derive (ec/key.js:102-107).  priv, pubx: 32 bytes big-endian
// (priv as held by the key pair, i.e. already reduced mod n at import, ec/key.js:76-82).
// out: 32-byte big-endian x.  Status 1 = value returned, 5 = the reference throws
// 'Assertion failed' (Red.sqrt on a non-residue inside MontCurve.validate, mont.js:21-28).
template <bool VALIDATE>
EB_HD uint8_t x25519_ladder_item(size_t i, const uint8_t* priv, const uint8_t* pubx, uint8_t* out) {
  u32 k[8];
  load_be<8>(k, priv + 32 * i);
  f25 x;
  load_be<8>(x.v, pubx + 32 * i);                     // toRed reduces mod p; weak form is fine here
  // validate (mont.js:21-28): rhs = x^3 + A x^2 + x must be a square (or 0).  The residue test is NOT done here:
  // it shares one exponentiation with the inversion of the ladder's z at the end (f25_pow_p32).
  f25 rhs = f25_zero();
  if (VALIDATE) {
    f25 x2 = f25_sqr(x);
    rhs = f25_add(f25_add(f25_mul(x2, x), f25_mul_small(x2, 486662u)), x);
  }
  // Montgomery ladder, MSB first (mont.js:130-153): (a, b) = ((m+1)P, mP), diff = P = (x : 1)
  f25 ax = x, az = f25_one(), bx = f25_one(), bz = f25_zero();
  for (int bit = 255; bit >= 0; bit--) {
    u32 word = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) word = (w == (bit >> 5)) ? k[w] : word;
    bool one = (word >> (bit & 31)) & 1;
    // diffAdd(a, b) and dbl of the selected one (mont.js:82-128)
    f25 sa = f25_add(ax, az), da_ = f25_sub(ax, az);
    f25 sb = f25_add(bx, bz), db = f25_sub(bx, bz);
    f25 t1 = f25_mul(db, sa);        // (xb - zb)(xa + za)
    f25 t2 = f25_mul(sb, da_);       // (xb + zb)(xa - za)
    f25 nx = f25_sqr_hot(f25_add(t1, t2));               // * diff.z (= 1)
    f25 nz = f25_mul(x, f25_sqr_hot(f25_sub(t1, t2)));   // * diff.x
    // dbl of a (bit 1) or b (bit 0)
    f25 s = f25_cmov(sb, sa, one), d = f25_cmov(db, da_, one);
    f25 aa = f25_sqr_hot(s), bb = f25_sqr_hot(d);
    f25 c = f25_sub(aa, bb);
    f25 dx = f25_mul(aa, bb);
    f25 dz = f25_mul(c, f25_add(bb, f25_mul_small(c, 121666u)));
    // bit 0: a = diffAdd, b = dbl(b);  bit 1: b = diffAdd, a = dbl(a)
    ax = f25_cmov(nx, dx, one); az = f25_cmov(nz, dz, one);
    bx = f25_cmov(dx, nx, one); bz = f25_cmov(dz, nz, one);
  }
  f25 zinv;
  if (VALIDATE) {
    // y = rhs z^2 has the Legendre symbol of rhs; e = y^((p-3)/2): y e = chi(y), chi e = 1 / y, 1 / z = rhs z / y
    f25 y = f25_mul(rhs, f25_sqr(bz));
    f25 e = f25_pow_p32(y);
    f25 chi = f25_normalize(f25_mul(y, e));
    bool chi_one = chi.v[0] == 1 && (chi.v[1] | chi.v[2] | chi.v[3] | chi.v[4] | chi.v[5] | chi.v[6] | chi.v[7]) == 0;
    bool is_qr = chi_one;
    if (is_zero_n<8>(chi.v)) {
      // rhs == 0 or z == 0 (low-order inputs): the two questions are answered separately, as the reference does
      f25 leg = f25_normalize(f25_legendre(rhs));
      is_qr = is_zero_n<8>(leg.v) || (leg.v[0] == 1 && (leg.v[1] | leg.v[2] | leg.v[3] | leg.v[4] | leg.v[5] | leg.v[6] | leg.v[7]) == 0);
      zinv = f25_inv(bz);
    } else {
      zinv = f25_mul(f25_mul(e, rhs), bz);
    }
    if (!is_qr) {
      for (int b = 0; b < 32; b++) out[32 * i + b] = 0;
      return 5;
    }
  } else {
    zinv = f25_inv(bz);
  }
  f25 r = f25_normalize(f25_mul(bx, zinv));           // getX: x * z^-1, with inv(0) = 0 (mont.js:167-178)
  store_be<8>(out + 32 * i, r.v);
  return 1;
}
EB_HD uint8_t x25519_derive_item(size_t i, const uint8_t* priv, const uint8_t* pubx, uint8_t* out) {
  return x25519_ladder_item<true>(i, priv, pubx, out);
}
// MontCurve Point.mul(k).getX() (mont.js:130-153, 173-178): the ladder over all 256 bits of k, no validation
EB_HD uint8_t x25519_mul_item(size_t i, const uint8_t* k, const uint8_t* px, uint8_t* out) {
  return x25519_ladder_item<false>(i, k, px, out);
}

}  // namespace eb
