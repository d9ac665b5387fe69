// x25519_keyset_body.cuh -- per-thread bodies of the curve25519 key-set kernels (x25519_keyset.cu): the batch form of
// `pub = ec.keyFromPublic(x)` once and `keyPair.derive(pub)` many times (lib/elliptic/ec/key.js:102-107) on curve25519.
// Host+device like the other bodies, so that the host emulation runs them.
//
// curve25519 and edwards25519 are birationally equivalent, y = (u - 1) / (u + 1), u = (1 + y) / (1 - y), and the map
// is a group isomorphism, torsion included.  So a key is imported as its Edwards image and gets the EdDSA key set's
// table (ed25519_keyset_body.cuh: i 2^(W j) (-P), affine niels), built by the same bodies.  k P is then read off the
// table as k (-P) with one niels add per window and no doubling, and u(k P) = u(-k P) = (Z + Y) / (Z - Y): u does not
// see the sign of x, so either square root of the Edwards image serves.
//
// Create, once per key: the verdict of MontCurve.validate (mont.js:21-28) on u mod p, as x25519_ladder_item decides
// it (TRUE if u^3 + A u^2 + u is 0 or a square, else THROW_ASSERT), and for a TRUE key the 32-byte ed25519 encoding of
// its image with x's sign bit clear.  u = 0 maps to (0, -1).  u = -1, the one value without an image, has
// u^3 + A u^2 + u = A - 2, a non-residue: it is always rejected, so it never reaches the map.
// Derive, per item, in two kernels:
//   main       the digits of priv (< n) over the key's table, from the identity; Z + Y and Z - Y into the workspace;
//   normalise  one thread per X25519_KS_BATCH items: Montgomery's trick over their Z - Y, one inversion, u big-endian.
// Z - Y = 0 is k P = O (priv = 0, small-order keys, k a multiple of the key's order): the ladder's getX gives
// x inv(0) = 0 there (mont.js:173-178), and the normalisation leaves such items out of the product and writes 0.
#pragma once
#include "ed25519_keyset_body.cuh"

namespace eb {

constexpr int X25519_KS_BATCH = 16;                             // items per normalisation thread
constexpr int X25519_KS_NORM_THREADS = 1024 / X25519_KS_BATCH;  // 1024 items per block, as ED_SS_NORM_THREADS
// Workspace, word-major (word w of item i at ws[w * ld + i]), per item: Z + Y, Z - Y, the running product of the
// batch's live Z - Y.
constexpr int X25519_KS_WS_ZPY = 0, X25519_KS_WS_ZMY = 8, X25519_KS_WS_PROD = 16, X25519_KS_WS_WORDS = 24;

EB_HD f25 x25519_ks_ws_load(const u32* ws, int w, size_t ld, size_t i) {
  f25 a;
  for (int q = 0; q < 8; q++) a.v[q] = ws[(size_t)(w + q) * ld + i];
  return a;
}
EB_HD void x25519_ks_ws_store(u32* ws, int w, size_t ld, size_t i, const f25& a) {
  for (int q = 0; q < 8; q++) ws[(size_t)(w + q) * ld + i] = a.v[q];
}

// Key k: its verdict (1 = TRUE, 5 = THROW_ASSERT) and, for a TRUE key, A[32 k ..] = the encoding of its Edwards image
// (zeros otherwise).  pubx: m x 32 bytes big-endian, any value below 2^256 (toRed reduces it mod p).
EB_HD uint8_t x25519_ks_classify_item(size_t k, const uint8_t* pubx, uint8_t* A) {
  f25 u;
  load_be<8>(u.v, pubx + 32 * k);
  const f25 u2 = f25_sqr(u);
  const f25 rhs = f25_add(f25_add(f25_mul(u2, u), f25_mul_small(u2, 486662u)), u);
  const f25 leg = f25_normalize(f25_legendre(rhs));
  const bool one = leg.v[0] == 1 && (leg.v[1] | leg.v[2] | leg.v[3] | leg.v[4] | leg.v[5] | leg.v[6] | leg.v[7]) == 0;
  uint8_t* a = A + 32 * k;
  if (!(one || is_zero_n<8>(leg.v))) {
    for (int b = 0; b < 32; b++) a[b] = 0;
    return 5;
  }
  const f25 y = f25_normalize(f25_mul(f25_sub(u, f25_one()), f25_inv(f25_add(u, f25_one()))));
  ed_encode_affine(f25_zero(), y, a);
  return 1;
}

// Item i against key key_idx[i]: the key's verdict into status[i] and, for a TRUE key, priv (P = the key's point)
// with the signed-digit scheme of ed25519_verify_keyed_item.  priv: 32 bytes big-endian, priv < n.  ld: the
// workspace's item stride.  Table gathers are indexed by the digits of priv.
EB_HD void x25519_derive_keyed_item(size_t i, size_t ld, const uint8_t* priv, const u32* key_idx, const uint8_t* kst, int W,
                                    int windows, const u32* ktab, u32* ws, uint8_t* status) {
  const u32 k = key_idx[i];
  const uint8_t st = kst[k];
  status[i] = st;
  if (st != 1) return;
  const u32* tab = ktab + ((size_t)k * windows << (W - 1)) * ED_KS_ENTRY_WORDS;
  u32 h[8];
  load_be<8>(h, priv + 32 * i);
  ed_ext acc = ed_identity();
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
  x25519_ks_ws_store(ws, X25519_KS_WS_ZPY, ld, i, f25_add(acc.z, acc.y));
  x25519_ks_ws_store(ws, X25519_KS_WS_ZMY, ld, i, f25_sub(acc.z, acc.y));
}

// Thread t of ceil(n / X25519_KS_BATCH) writes u = (Z + Y) / (Z - Y) big-endian for items t, t + T, t + 2 T, ... below
// n (T: the thread count; a strided batch, so that a warp's workspace loads are coalesced), with one inversion for the
// batch.  An item whose key is not TRUE, or whose Z - Y is 0, is left out of the product and gets 32 zero bytes; every
// other factor is nonzero, so the product is invertible and each 1 / (Z - Y) is exact.
EB_HD void x25519_keyed_norm_item(size_t t, size_t n, size_t ld, u32* ws, const uint8_t* status, uint8_t* out) {
  const size_t T = (n + X25519_KS_BATCH - 1) / X25519_KS_BATCH;
  int cnt = 0;
  f25 prod = f25_one();
  for (int u = 0; u < X25519_KS_BATCH; u++) {
    const size_t i = t + (size_t)u * T;
    if (i >= n) break;
    if (status[i] == 1) {
      const f25 d = x25519_ks_ws_load(ws, X25519_KS_WS_ZMY, ld, i);
      if (!f25_is_zero(d)) prod = f25_mul(prod, d);
    }
    x25519_ks_ws_store(ws, X25519_KS_WS_PROD, ld, i, prod);         // the live factors of items 0 .. u
    cnt++;
  }
  f25 inv = f25_inv(prod);
  for (int u = cnt - 1; u >= 0; u--) {
    const size_t i = t + (size_t)u * T;
    f25 r = f25_zero();
    if (status[i] == 1) {
      const f25 d = x25519_ks_ws_load(ws, X25519_KS_WS_ZMY, ld, i);
      if (!f25_is_zero(d)) {
        const f25 zi = u ? f25_mul(inv, x25519_ks_ws_load(ws, X25519_KS_WS_PROD, ld, i - T)) : inv;
        inv = f25_mul(inv, d);
        r = f25_normalize(f25_mul(x25519_ks_ws_load(ws, X25519_KS_WS_ZPY, ld, i), zi));
      }
    }
    store_be<8>(out + 32 * i, r.v);
  }
}

}  // namespace eb
