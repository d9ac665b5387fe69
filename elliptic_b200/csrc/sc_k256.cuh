// sc_k256.cuh -- arithmetic modulo the secp256k1 group order n, GLV split and
// scalar recoding.
//
// Replaces, for whole batches, the scalar pre-processing of the reference's
// EC.verify (lib/elliptic/ec/index.js:199-207: range checks, s.invm(n),
// u1 = e*s^-1, u2 = r*s^-1) and ShortCurve._endoSplit (short.js:168-185,
// constants curves.js:187-198).  bn.js does s^-1 with a binary extended GCD
// per item (dist:6436-6516); here inversions are batched with Montgomery's
// trick and one Fermat exponentiation per 16 items, in CIOS Montgomery form.
//
// The recoding is NOT the reference's getNAF/getJSF (utils.js:15-101, data
// dependent => divergent): it is a regular signed-odd fixed-window form, so
// every lane runs the same double/add schedule.  Any (k1,k2) with
// k1 + k2*lambda = k (mod n) gives the same point for an on-curve key, which is
// all the reference's result depends on (off-curve keys: see ecdsa_k256.cu).
#pragma once
#include "limbs.cuh"
#include "fp_mont.cuh"

namespace eb {

// All constants are passed as immediates through small functions so that the
// same code compiles for host emulation and device.
struct K256N {
  static EB_HD void n(u32* r) {
    const u32 v[8] = {0xd0364141u, 0xbfd25e8cu, 0xaf48a03bu, 0xbaaedce6u, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
    for (int i = 0; i < 8; i++) r[i] = v[i];
  }
  static EB_HD void r2(u32* r) {  // 2^512 mod n
    const u32 v[8] = {0x67d7d140u, 0x896cf214u, 0x0e7cf878u, 0x741496c2u, 0x5bcd07c6u, 0xe697f5e4u, 0x81c69bc5u, 0x9d671cd5u};
    for (int i = 0; i < 8; i++) r[i] = v[i];
  }
  static EB_HD void r1(u32* r) {  // 2^256 mod n  (Montgomery one)
    const u32 v[8] = {0x2fc9bebfu, 0x402da173u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0, 0, 0};
    for (int i = 0; i < 8; i++) r[i] = v[i];
  }
  static constexpr u32 n0inv = 0x5588b13fu;  // -n^-1 mod 2^32
};

// the same constants in the shape fp_mont.cuh's generic field wants
struct K256_FN {
  static constexpr int N = 8;
  static constexpr u32 n0inv = K256N::n0inv;
  static EB_HD void mod(u32* r) { K256N::n(r); }
  static EB_HD void r1(u32* r) { K256N::r1(r); }
  static EB_HD void r2(u32* r) { K256N::r2(r); }
};

// Montgomery product a*b*2^-256 mod n (CIOS); a < 2^256, b < n -> result < n.
// Device: the out-of-line two-accumulator PTX multiplier of fp_mont.cuh; host: the portable loop below.
EB_HD void sc_mont_mul(u32* r, const u32* a, const u32* b) {
#if defined(__CUDA_ARCH__)
  typedef Fp<K256_FN> S;
  S::fe x, y;
#pragma unroll
  for (int i = 0; i < 8; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
  S::fe z = S::mul(x, y);
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
  return;
#endif
  u32 n[8]; K256N::n(n);
  u32 t[10];
#pragma unroll
  for (int i = 0; i < 10; i++) t[i] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    u64 c = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      c += (u64)a[j] * b[i] + t[j];
      t[j] = (u32)c; c >>= 32;
    }
    c += t[8];
    t[8] = (u32)c; t[9] = (u32)(c >> 32);
    u32 m = t[0] * K256N::n0inv;
    c = (u64)m * n[0] + t[0];
    c >>= 32;
#pragma unroll
    for (int j = 1; j < 8; j++) {
      c += (u64)m * n[j] + t[j];
      t[j - 1] = (u32)c; c >>= 32;
    }
    c += t[8];
    t[7] = (u32)c;
    t[8] = t[9] + (u32)(c >> 32);
    t[9] = 0;
  }
  u32 d[8];
  u32 bw = sub_n<8>(d, t, n);
  bool ge = t[8] != 0 || bw == 0;
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = ge ? d[i] : t[i];
}

// a^(n-2) in Montgomery form (a in Montgomery form).
EB_HD void sc_mont_inv(u32* r, const u32* a) {
  const u32 e[8] = {0xd036413fu, 0xbfd25e8cu, 0xaf48a03bu, 0xbaaedce6u, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
  u32 acc[8], base[8];
  copy_n<8>(base, a);
  copy_n<8>(acc, a);  // top bit (255) of n-2 is set
  for (int i = 254; i >= 0; i--) {
    u32 t[8];
    sc_mont_mul(t, acc, acc);
    copy_n<8>(acc, t);
    if ((e[i >> 5] >> (i & 31)) & 1) {
      sc_mont_mul(t, acc, base);
      copy_n<8>(acc, t);
    }
  }
  copy_n<8>(r, acc);
}

// 1 <= a < n ?
EB_HD bool sc_in_range(const u32* a) {
  u32 n[8]; K256N::n(n);
  return !is_zero_n<8>(a) && !geq_n<8>(a, n);
}

// two's-complement helpers on 8 limbs
EB_HD void neg256(u32* r, const u32* a) {
  u32 z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  sub_n<8>(r, z, a);
}

// GLV decomposition of k (< n): k = k1 + k2*lambda (mod n) with k1, k2 odd.
// Outputs m1 = (|k1|-1)/2, m2 = (|k2|-1)/2 (5 limbs each) and the signs.
// Rounded quotients use the 2^384-scaled constants g1 = round(2^384*b2/n),
// g2 = round(2^384*(-b1)/n) for the reference's own basis v1 = (a1, b1),
// v2 = (a2, b2) (curves.js:189-198); the parity fix adds +-v1 / +-v2.
//
// Bound: before the fix (k1, k2) = -(d1 v1 + d2 v2) with |d1|, |d2| <= 1/2 (up
// to k / 2^385 from the scaled constants).  The fix adds e1 v1, then e2 v2,
// e1, e2 in {-1, 0, 1}, their signs set by the sign of k1 at that point.  The
// largest |k1| and |k2| over all (d1, d2, e1, e2) are at vertices of the
// regions those signs cut out of the square: |k1| < 2^128.12, |k2| < 2^128.66
// (tests/test_glv_window5.py derives them), so m1, m2 < 2^GLV_M_BITS.
constexpr int GLV_M_BITS = 128;
EB_HD void glv_split_odd(const u32* k, u32* m1, bool* neg1, u32* m2, bool* neg2) {
  const u32 g1[8] = {0x45dbb031u, 0xe893209au, 0x71e8ca7fu, 0x3daa8a14u, 0x9284eb15u, 0xe86c90e4u, 0xa7d46bcdu, 0x3086d221u};
  const u32 g2[8] = {0x8ac47f71u, 0x1571b4aeu, 0x9df506c6u, 0x221208acu, 0x0abfe4c4u, 0x6f547fa9u, 0x010e8828u, 0xe4437ed6u};
  const u32 a1[8] = {0x9284eb15u, 0xe86c90e4u, 0xa7d46bcdu, 0x3086d221u, 0, 0, 0, 0};
  const u32 mb1[8] = {0x0abfe4c3u, 0x6f547fa9u, 0x010e8828u, 0xe4437ed6u, 0, 0, 0, 0};  // -b1
  const u32 a2[8] = {0x9d44cfd8u, 0x57c1108du, 0xa8e2f3f6u, 0x14ca50f7u, 0x00000001u, 0, 0, 0};
  const u32 b2[8] = {0x9284eb15u, 0xe86c90e4u, 0xa7d46bcdu, 0x3086d221u, 0, 0, 0, 0};
  u32 t[16], c1[4], c2[4];
  const u32 half[4] = {0, 0, 0, 0x80000000u};  // 2^383 at limbs 8..11
  mul_rect<8, 8>(t, k, g1);
  {
    u32 cy = add_n<4>(t + 8, t + 8, half);
    u32 one[4] = {cy, 0, 0, 0};
    add_n<4>(c1, t + 12, one);
  }
  mul_rect<8, 8>(t, k, g2);
  {
    u32 cy = add_n<4>(t + 8, t + 8, half);
    u32 one[4] = {cy, 0, 0, 0};
    add_n<4>(c2, t + 12, one);
  }
  // k1 = k - c1*a1 - c2*a2 ; k2 = c1*(-b1) - c2*b2   (mod 2^256, two's complement)
  u32 p[9], k1[8], k2[8], q[8];
  mul_rect<4, 4>(p, c1, a1);
  sub_n<8>(k1, k, p);
  mul_rect<5, 4>(p, a2, c2);  // 9 limbs; low 8 used
  sub_n<8>(k1, k1, p);
  mul_rect<4, 4>(k2, c1, mb1);
  mul_rect<4, 4>(q, c2, b2);
  sub_n<8>(k2, k2, q);
  // parity fix (a1, b1 odd; a2 even, b2 odd)
  bool k1neg = (k1[7] >> 31) != 0;
  if ((k1[0] & 1) == 0) {
    if (!k1neg) { sub_n<8>(k1, k1, a1); add_n<8>(k2, k2, mb1); }   // -= (a1, b1)
    else        { add_n<8>(k1, k1, a1); sub_n<8>(k2, k2, mb1); }   // += (a1, b1)
    k1neg = (k1[7] >> 31) != 0;
  }
  if ((k2[0] & 1) == 0) {
    if (!k1neg) { sub_n<8>(k1, k1, a2); sub_n<8>(k2, k2, b2); }
    else        { add_n<8>(k1, k1, a2); add_n<8>(k2, k2, b2); }
  }
  *neg1 = (k1[7] >> 31) != 0;
  *neg2 = (k2[7] >> 31) != 0;
  u32 a[8];
  neg256(a, k1); cmov_n<8>(k1, a, *neg1);
  neg256(a, k2); cmov_n<8>(k2, a, *neg2);
#pragma unroll
  for (int i = 0; i < 5; i++) {
    m1[i] = (k1[i] >> 1) | (k1[i + 1] << 31);
    m2[i] = (k2[i] >> 1) | (k2[i + 1] << 31);
  }
}

}  // namespace eb
