// ed25519_keyset_body.cuh -- per-thread bodies of the EdDSA key-set kernels (eddsa_keyset.cu): the batch form of
// `key = eddsa.keyFromPublic(bytes)` once and `eddsa.verify(msg, sig, key)` many times (lib/elliptic/eddsa/index.js:52-63,
// eddsa/key.js:17-44).  Host+device like the other bodies, so that the host emulation runs them.
//
// Build, once per key: the verdict of decoding A (ed_decode: TRUE, or the throw 2 / 5); for a key that decodes, window
// bases 2^(W j) (-A) by one chain of doublings, then per (key, window) the multiples i 2^(W j) (-A), i = 1 .. 2^(W-1), by
// repeated addition, made affine with one inversion per ED_KS_CHUNK entries.  The raw 32 key bytes are kept: hashInt
// reads key.pubBytes(), which for a key made from bytes is those bytes, non-canonical y included (eddsa/key.js:17-24).
// Verify: S*G from the fixed table (ed_mul_base), then one table gather and one niels add per window of h, and the
// affine comparison with R.  No decompression of A, no doubling and no per-item table.  The twisted-Edwards formulas
// are complete, so small- and mixed-order keys need no special case.
#pragma once
#include "ed25519_body.cuh"
#include "keyset_plan.h"

namespace eb {

constexpr int ED_KS_CHUNK = 16;         // entries per inversion in the table build

// keyFromPublic's verdict for key k: 1 (decodes), else the status of the throw (ed_decode)
EB_HD uint8_t ed_ks_classify_item(size_t k, const uint8_t* A) {
  f25 x, y;
  uint8_t st = ed_decode(A + 32 * k, &x, &y);
  return st ? st : 1;
}

// bases[(k windows + j) 24 ..] = 2^(W j) (-A_k) as X, Y, Z (T is not needed by the doubling)
EB_HD void ed_ks_bases_item(size_t k, const uint8_t* A, const uint8_t* kst, int W, int windows, u32* bases) {
  if (kst[k] != 1) return;
  f25 ax, ay;
  ed_decode(A + 32 * k, &ax, &ay);
  ed_ext b;
  b.x = f25_neg(ax); b.y = ay; b.z = f25_one(); b.t = f25_mul(b.x, ay);
  for (int j = 0; j < windows; j++) {
    u32* o = bases + ((size_t)k * windows + j) * 24;
    f25_store(o, b.x); f25_store(o + 8, b.y); f25_store(o + 16, b.z);
    if (j + 1 < windows)
      for (int d = 0; d < W; d++) b = ed_dbl(b);
  }
}

// window t = k windows + j of the table: entries i B, i = 1 .. 2^(W-1), B = bases[t]; affine niels, normalised
EB_HD void ed_ks_window_item(size_t t, const uint8_t* kst, int W, int windows, const u32* bases, u32* tab) {
  if (kst[t / windows] != 1) return;
  const int entries = 1 << (W - 1);
  f25 X = f25_load(bases + t * 24), Y = f25_load(bases + t * 24 + 8), Z = f25_load(bases + t * 24 + 16);
  ed_ext B;                                  // (X Z, Y Z, Z^2, X Y): the same point with its T coordinate
  B.x = f25_mul(X, Z); B.y = f25_mul(Y, Z); B.z = f25_sqr(Z); B.t = f25_mul(X, Y);
  const ed_cached cb = ed_to_cached(B);
  u32* out = tab + t * entries * ED_KS_ENTRY_WORDS;
  ed_ext P = B;
  for (int c = 0; c < entries; c += ED_KS_CHUNK) {
    // entry slot u holds X_u, Y_u and the running product Z_0 .. Z_u until the backward pass makes it affine
    f25 z[ED_KS_CHUNK];
    int cnt = entries - c < ED_KS_CHUNK ? entries - c : ED_KS_CHUNK;
    f25 prod = f25_one();
    for (int u = 0; u < cnt; u++) {
      if (c + u) P = ed_add_cached(P, cb);
      u32* e = out + ED_KS_ENTRY_WORDS * (c + u);
      z[u] = P.z;
      prod = f25_mul(prod, P.z);
      f25_store(e, P.x); f25_store(e + 8, P.y); f25_store(e + 16, prod);
    }
    f25 inv = f25_inv(prod);                 // points on the curve never have Z = 0
    for (int u = cnt - 1; u >= 0; u--) {
      u32* e = out + ED_KS_ENTRY_WORDS * (c + u);
      f25 zi = u ? f25_mul(inv, f25_load(e - ED_KS_ENTRY_WORDS + 16)) : inv;
      inv = f25_mul(inv, z[u]);
      f25 x = f25_mul(f25_load(e), zi), y = f25_mul(f25_load(e + 8), zi);
      f25_store(e, f25_normalize(f25_add(y, x)));
      f25_store(e + 8, f25_normalize(f25_sub(y, x)));
      f25_store(e + 16, f25_normalize(f25_mul(f25_mul(x, y), f25_2d())));
    }
  }
}

// One 24-word niels entry as 128-bit read-only loads on the device.
EB_HD ed_niels ed_ks_load_niels(const u32* src) {
  u32 w[ED_KS_ENTRY_WORDS];
#if defined(__CUDA_ARCH__)
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
#pragma unroll
  for (int q = 0; q < ED_KS_ENTRY_WORDS / 4; q++) {
    uint4 v = __ldg(s4 + q);
    w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
  }
#else
  for (int q = 0; q < ED_KS_ENTRY_WORDS; q++) w[q] = src[q];
#endif
  ed_niels r;
  r.ypx = f25_load(w); r.ymx = f25_load(w + 8); r.t2d = f25_load(w + 16);
  return r;
}

// EDDSA.verify for item i against key key_idx[i] of the set: the byte ed25519_verify_item gives for the same R, S, h and
// that key, in the reference's order -- S >= n, then R's throw, then the key's, then R + h A == S G.
// h: 32 bytes little-endian, h < n (hashInt).
EB_HD uint8_t ed25519_verify_keyed_item(size_t i, const uint8_t* Rb, const uint8_t* Sb, const uint8_t* hb, const u32* key_idx,
                                        const uint8_t* kst, int W, int windows, const u32* ktab, const u32* gtab) {
  u32 S[8], n[8];
  load_le<8>(S, Sb + 32 * i);
  ed_n(n);
  if (geq_n<8>(S, n)) return 0;                                   // eddsa/index.js:55-57
  f25 rx, ry;
  uint8_t st = ed_decode(Rb + 32 * i, &rx, &ry);                  // sig.R()
  if (st) return st;
  const u32 k = key_idx[i];
  st = kst[k];                                                    // key.pub()
  if (st != 1) return st;
  const u32* tab = ktab + ((size_t)k * windows << (W - 1)) * ED_KS_ENTRY_WORDS;

  ed_ext acc = ed_mul_base(S, gtab);
  // - h A: digits low to high with a carry, d_j in [-2^(W-1), 2^(W-1)) and an unsigned top digit.  These are the digits
  // ed_mul_base's scheme gives (h + sum_j 2^(W j + W - 1), each chunk minus 2^(W-1)); the order of the additions is free.
  u32 h[8];
  load_le<8>(h, hb + 32 * i);
  const u32 half = 1u << (W - 1);
  u32 carry = 0;
  for (int j = 0; j < windows; j++) {
    int pos = W * j, wi = pos >> 5;
    u32 lo = 0, hi = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) { lo = (q == wi) ? h[q] : lo; hi = (q == wi + 1) ? h[q] : hi; }
    u32 c = (u32)((((u64)hi << 32) | lo) >> (pos & 31)) & ((1u << W) - 1);
    c += carry;
    bool top = j == windows - 1;
    bool neg = !top && c >= half;
    carry = neg;
    u32 idx = neg ? (1u << W) - c : c;                            // |d_j|, 0 .. 2^(W-1)
    ed_niels q = ed_ks_load_niels(tab + (((size_t)j << (W - 1)) + (idx ? idx - 1 : 0)) * ED_KS_ENTRY_WORDS);
    q.ypx = f25_cmov(q.ypx, f25_one(), idx == 0);                 // digit 0: the neutral niels (1, 1, 0)
    q.ymx = f25_cmov(q.ymx, f25_one(), idx == 0);
    q.t2d = f25_cmov(q.t2d, f25_zero(), idx == 0);
    acc = ed_add_niels(acc, ed_niels_neg_if(q, neg));
  }
  // S G - h A == R as affine points  (edwards.js:409-413)
  bool ok = f25_eq(acc.x, f25_mul(rx, acc.z)) && f25_eq(acc.y, f25_mul(ry, acc.z));
  return ok ? 1 : 0;
}

// The key bytes hashInt reads for item i: key key_idx[i]'s raw 32 bytes, as the caller gave them.
EB_HD void ed_ks_gather_item(size_t i, const u32* key_idx, const uint8_t* A, uint8_t* out) {
  const uint8_t* a = A + 32 * (size_t)key_idx[i];
  for (int b = 0; b < 32; b++) out[32 * i + b] = a[b];
}

}  // namespace eb
