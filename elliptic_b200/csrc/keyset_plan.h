// keyset_plan.h -- geometry of a key set's per-key tables and the automatic choice of their window width.
// Plain C++ (no CUDA): included by eb200.cu, keyset.cu and the host test harness.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/elliptic_b200.h"

// A key's table has `windows` windows of 2^(W-1) affine entries: entry (j, i) = (2i+1) 2^(W j) Q, x then y, in the
// limbs the main loop consumes (8 words per coordinate on secp256k1 / p256 / p224, 6 on p192, 12 on p384, 18 on p521).
// The windows cover m = (k - 1) / 2 for the odd scalar k the prep kernels store: the 131 bits of a GLV half on
// secp256k1 (beta * x is recomputed per lookup, not stored), bits(n) - 1 otherwise.  windows = floor(mbits / W) + 1
// keeps the top digit 2 m_top + 1 below 2^W, i.e. positive, for every W.
struct KeysetGeom { int mbits, limbs; };
static constexpr KeysetGeom keyset_geom(int curve) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: return {131, 8};
    case EB200_CURVE_P256: return {255, 8};
    case EB200_CURVE_P384: return {383, 12};
    case EB200_CURVE_P521: return {520, 18};
    case EB200_CURVE_P192: return {191, 6};
    case EB200_CURVE_P224: return {223, 8};
    default: return {0, 0};
  }
}
static inline int keyset_windows(int curve, int W) { return keyset_geom(curve).mbits / W + 1; }
static inline size_t keyset_key_bytes(int curve, int W) {       // one key's table
  return (size_t)keyset_windows(curve, W) * ((size_t)1 << (W - 1)) * 2 * keyset_geom(curve).limbs * 4;
}

// table_bits = 0: the widest W in EB200_KEYSET_MIN_BITS..MAX_BITS whose m tables fit `budget` bytes on one device;
// 0 when not even the narrowest fits (the caller then gets EB200_ERR_ARG: a set is never silently left without tables).
static inline uint32_t keyset_choose_bits(int curve, size_t m, size_t budget) {
  if (!keyset_geom(curve).limbs) return 0;
  for (int W = EB200_KEYSET_MAX_BITS; W >= EB200_KEYSET_MIN_BITS; W--) {
    size_t per = keyset_key_bytes(curve, W);
    if (m <= budget / per) return (uint32_t)W;
  }
  return 0;
}

// ed25519 key sets (eb200_eddsa_keyset_create) have a geometry of their own: entry (j, i) = i 2^(W j) (-A) for
// i = 1 .. 2^(W-1), affine niels (y+x, y-x, 2d x y), 24 words.  The windows cover every h < n < 2^253 with signed
// digits in [-2^(W-1), 2^(W-1)) and an unsigned top digit, which stays <= 2^(W-1) for W = 4..8.
constexpr int ED_KS_ENTRY_WORDS = 24;
static inline int ed_keyset_windows(int W) { return (253 + W - 1) / W; }
static inline size_t ed_keyset_key_bytes(int W) {
  return (size_t)ed_keyset_windows(W) * ((size_t)1 << (W - 1)) * ED_KS_ENTRY_WORDS * 4;
}
static inline uint32_t ed_keyset_choose_bits(size_t m, size_t budget) {
  for (int W = EB200_KEYSET_MAX_BITS; W >= EB200_KEYSET_MIN_BITS; W--)
    if (m <= budget / ed_keyset_key_bytes(W)) return (uint32_t)W;
  return 0;
}
