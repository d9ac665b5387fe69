// ecdsa_keyset_body.cuh -- per-thread bodies of the key-set kernels (keyset.cu): the batch form of
// `key = ec.keyFromPublic(pub)`, `key.getPublic().precompute()` and `key.verify(msg, sig)`
// (lib/elliptic/ec/key.js:20-28, 84-99, 114-116; curve/base.js:312-327).  Host+device like the other bodies, so that
// the host emulation runs them.
//
// Build, once per key Q that imported and lies on the curve: window bases 2^(W j) Q by one chain of doublings per key,
// then per (key, window) the odd multiples (2i+1) 2^(W j) Q by repeated addition of twice the base, made affine with
// one inversion per KS_CHUNK entries (Z_i = Z_{i-1} h_i, so the h_i of a chunk undo its Z's one by one).
// Verify: scalars as the unkeyed prep kernels store them; u2 Q is one mixed add per window from the key's table (both
// GLV halves on secp256k1, the second through x -> beta x), u1 G the fixed-base adds of k256_dsm / SW<C>::dsm, then the
// same x comparison.  No doubling and no per-item table.  The mixed adds resolve P + P, P - P and O + P exactly
// (jac_madd_inl / SW<C>::madd_inl), which keys such as G, -G or 2^k G do reach.
#pragma once
#include "ecdsa_k256_body.cuh"
#include "ecdsa_sw_body.cuh"
#include "keyset_plan.h"

namespace eb {

constexpr int KS_CHUNK = 16;            // entries per inversion in the table build

// One table entry (NW words, 16-byte aligned) as 128-bit read-only loads on the device.
template <int NW>
EB_HD void ks_load_entry(u32* dst, const u32* src) {
  static_assert(NW % 4 == 0, "entries are whole 16-byte words");
#if defined(__CUDA_ARCH__)
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
#pragma unroll
  for (int q = 0; q < NW / 4; q++) {
    uint4 v = __ldg(s4 + q);
    dst[4 * q] = v.x; dst[4 * q + 1] = v.y; dst[4 * q + 2] = v.z; dst[4 * q + 3] = v.w;
  }
#else
  for (int q = 0; q < NW; q++) dst[q] = src[q];
#endif
}

// keyFromPublic's verdict for key k: the decoder's throw, else pub.validate()
EB_HD uint8_t k256_ks_classify_item(size_t k, const uint8_t* xy, const uint8_t* pre) {
  if (pre && pre[k]) return pre[k];
  ge_aff Q;
  Q.x = fe_from_be(xy + 64 * k);
  Q.y = fe_from_be(xy + 64 * k + 32);
  return aff_on_curve(Q) ? ST_TRUE : ST_FALSE;
}

// bases[(k windows + j) 24 ..] = 2^(W j) Q_k, Jacobian
EB_HD void k256_ks_bases_item(size_t k, const uint8_t* xy, const uint8_t* kst, int W, int windows, u32* bases) {
  if (kst[k] != ST_TRUE) return;
  ge_aff Q;
  Q.x = fe_from_be(xy + 64 * k);
  Q.y = fe_from_be(xy + 64 * k + 32);
  ge_jac b = jac_from_aff(Q);
  for (int j = 0; j < windows; j++) {
    u32* o = bases + ((size_t)k * windows + j) * 24;
    store_fe(o, b.x); store_fe(o + 8, b.y); store_fe(o + 16, b.z);
    if (j + 1 < windows)
      for (int d = 0; d < W; d++) b = jac_dbl(b);
  }
}

// window t = k windows + j of the table: entries (2i+1) B, B = bases[t], affine and normalised
EB_HD void k256_ks_window_item(size_t t, const uint8_t* kst, int W, int windows, const u32* bases, u32* tab) {
  if (kst[t / windows] != ST_TRUE) return;
  const int entries = 1 << (W - 1);
  ge_jac bj;
  bj.x = load_fe(bases + t * 24); bj.y = load_fe(bases + t * 24 + 8); bj.z = load_fe(bases + t * 24 + 16);
  ge_aff B = jac_to_aff(bj);
  ge_aff D = jac_to_aff(jac_dbl(jac_from_aff(B)));
  u32* out = tab + t * entries * 16;
  ge_jac P = jac_from_aff(B);
  for (int c = 0; c < entries; c += KS_CHUNK) {
    fe h[KS_CHUNK];
    int cnt = entries - c < KS_CHUNK ? entries - c : KS_CHUNK;
    for (int u = 0; u < cnt; u++) {
      if (c + u == 0) h[u] = fe_one();
      else { madd_out o = jac_madd_h(P, D); P = o.r; h[u] = o.h; }     // odd multiples of a point of prime order: never exceptional
      store_fe(out + 16 * (c + u), P.x); store_fe(out + 16 * (c + u) + 8, P.y);
    }
    fe inv = fe_inv(P.z);
    for (int u = cnt - 1; u >= 0; u--) {
      u32* e = out + 16 * (c + u);
      fe zi2 = fe_sqr(inv);
      store_fe(e, fe_normalize(fe_mul(load_fe(e), zi2)));
      store_fe(e + 8, fe_normalize(fe_mul(fe_mul(load_fe(e + 8), zi2), inv)));
      inv = fe_mul(inv, h[u]);
    }
  }
}

// u2*Q = k1*Q + k2*(lambda*Q) from one key's table `tab`: one mixed add per window and half, regular signed-odd digits.
// The keyed mul body's accumulation; k256_verify_keyed_item keeps its own copy of these loops, because calling these
// force-inlined helpers from it changes the code generated for the keyed verify kernels.
EB_HD ge_jac k256_ks_key_part(size_t i, size_t N, u32 flags, int W, int windows, const u32* tab, const u32* ws) {
  const fe beta = fe_beta();
  ge_jac acc = jac_infinity();
  for (int w = windows - 1; w >= 0; w--) {
    for (int h = 0; h < 2; h++) {
      bool dneg;
      u32 idx = ks_digit(ks_chunk(ws, N, i, h ? 13 : 8, 5, W * w, W), w == windows - 1, W, &dneg);
      const bool neg = ((flags & (h ? FL_NEG2 : FL_NEG1)) != 0) != dneg;
      u32 ent[16];
      ks_load_entry<16>(ent, tab + (((size_t)w << (W - 1)) + idx) * 16);
      ge_aff P;
      P.x = load_fe(ent);
      P.y = load_fe(ent + 8);
      if (h) P.x = fe_mul(P.x, beta);
      P = aff_neg_if(P, neg);
      if (w == windows - 1 && h == 0) acc = jac_from_aff(P);   // the accumulator starts from the first entry
      else acc = jac_madd(acc, P);
    }
  }
  return acc;
}
// acc + u1*G from the fixed table, as k256_dsm
EB_HD ge_jac k256_ks_g_part(ge_jac acc, size_t i, size_t N, u32 flags, const u32* ws, const u32* gtab) {
  for (int j = 0; j < GTAB_WINDOWS; j++) {
    bool dneg;
    u32 idx = ks_digit(ks_chunk(ws, N, i, 0, 8, GTAB_W * j, GTAB_W), j == GTAB_WINDOWS - 1, GTAB_W, &dneg);
    bool neg = dneg != ((flags & FL_NEGG) != 0);
    const u32* ent = gtab + ((size_t)j * GTAB_ENTRIES + idx) * 16;
    ge_aff P;
    P.x = load_fe(ent);
    P.y = load_fe(ent + 8);
    acc = jac_madd(acc, aff_neg_if(P, neg));
  }
  return acc;
}

// key.verify for item i against key key_idx[i] of the set.  The status eb200_ecdsa_verify_batch gives with that key:
// the key's throw first, FALSE for r, s out of range, ST_NEEDS_HOST for an off-curve key (the keyed replay kernel
// then runs the reference's own schedule on the key's coordinates).
EB_HD uint8_t k256_verify_keyed_item(size_t i, size_t N, const u32* key_idx, const uint8_t* kst, int W, int windows,
                                     const u32* ktab, const uint8_t* r, const u32* ws, const u32* gtab) {
  const u32 k = key_idx[i];
  const uint8_t ks = kst[k];
  if (ks > ST_TRUE) return ks;
  u32 flags = ws[(size_t)18 * N + i];
  if (flags & FL_INVALID) return ST_FALSE;
  if (ks != ST_TRUE) return ST_NEEDS_HOST;
  const u32* tab = ktab + ((size_t)k * windows << (W - 1)) * 16;
  const fe beta = fe_beta();

  // ---- u2*Q = k1*Q + k2*(lambda*Q): one mixed add per window and half, regular signed-odd digits
  ge_jac acc = jac_infinity();
  for (int w = windows - 1; w >= 0; w--) {
    for (int h = 0; h < 2; h++) {
      bool dneg;
      u32 idx = ks_digit(ks_chunk(ws, N, i, h ? 13 : 8, 5, W * w, W), w == windows - 1, W, &dneg);
      bool neg = dneg != ((flags & (h ? FL_NEG2 : FL_NEG1)) != 0);
      u32 ent[16];
      ks_load_entry<16>(ent, tab + (((size_t)w << (W - 1)) + idx) * 16);
      ge_aff P;
      P.x = load_fe(ent);
      P.y = load_fe(ent + 8);
      if (h) P.x = fe_mul(P.x, beta);
      P = aff_neg_if(P, neg);
      if (w == windows - 1 && h == 0) acc = jac_from_aff(P);   // the accumulator starts from the first entry
      else acc = jac_madd(acc, P);
    }
  }
  // ---- u1*G from the fixed table, as k256_dsm
  for (int j = 0; j < GTAB_WINDOWS; j++) {
    bool dneg;
    u32 idx = ks_digit(ks_chunk(ws, N, i, 0, 8, GTAB_W * j, GTAB_W), j == GTAB_WINDOWS - 1, GTAB_W, &dneg);
    bool neg = dneg != ((flags & FL_NEGG) != 0);
    const u32* ent = gtab + ((size_t)j * GTAB_ENTRIES + idx) * 16;
    ge_aff P;
    P.x = load_fe(ent);
    P.y = load_fe(ent + 8);
    acc = jac_madd(acc, aff_neg_if(P, neg));
  }

  // ---- accept iff R != O and x(R) == r (mod n)   (ec/index.js:222-228, short.js:908-925)
  if (fe_is_zero(acc.z)) return ST_FALSE;
  fe z2 = fe_sqr(acc.z);
  fe rf = fe_from_be(r + 32 * i);
  if (fe_eq(acc.x, fe_mul(rf, z2))) return ST_TRUE;
  const u32 pmn[8] = {0x2fc9baeeu, 0x402da172u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0, 0, 0};  // p - n
  if (!geq_n<8>(rf.v, pmn)) {      // r + n < p: second candidate
    u32 nn[8]; K256N::n(nn);
    fe rn;
    add_n<8>(rn.v, rf.v, nn);
    if (fe_eq(acc.x, fe_mul(rn, z2))) return ST_TRUE;
  }
  return ST_FALSE;
}

// Point.mul / G.mulAdd for item i on key key_idx[i] (k2 Q, plus k1 G unless FL_NOG), scalars as
// k256_prep_scalars_kernel stores them.  The Jacobian result goes to jout word-major (coordinate c, word w at
// jout[(8 c + w) N + i]), Z = 0 for an item that has no result here.  Status: the key's throw, ST_NEEDS_HOST for an
// off-curve key (the keyed replay then runs the unkeyed call's schedule), else ST_TRUE; k256_ks_norm_thread turns
// ST_TRUE into the affine point or ST_INFINITY.
EB_HD uint8_t k256_mul_keyed_item(size_t i, size_t N, const u32* key_idx, const uint8_t* kst, int W, int windows,
                                  const u32* ktab, const u32* ws, const u32* gtab, u32* jout) {
  const u32 k = key_idx[i];
  const uint8_t ks = kst[k];
  ge_jac acc = jac_infinity();
  if (ks == ST_TRUE) {
    u32 flags = ws[(size_t)18 * N + i];
    acc = k256_ks_key_part(i, N, flags, W, windows, ktab + ((size_t)k * windows << (W - 1)) * 16, ws);
    if (!(flags & FL_NOG)) acc = k256_ks_g_part(acc, i, N, flags, ws, gtab);
  }
  for (int w = 0; w < 8; w++) {
    jout[(size_t)w * N + i] = acc.x.v[w];
    jout[(size_t)(8 + w) * N + i] = acc.y.v[w];
    jout[(size_t)(16 + w) * N + i] = acc.z.v[w];
  }
  return ks == ST_TRUE ? ST_TRUE : ks == ST_FALSE ? ST_NEEDS_HOST : ks;
}

// Jacobian -> affine big-endian for items tid, tid + T, ... (up to `batch` <= 64, T * batch >= N) with one inversion
// (Montgomery's trick): the items whose status is ST_TRUE and whose Z != 0 form the product chain; the others are
// skipped, their output zeroed, and a ST_TRUE item with Z = 0 becomes ST_INFINITY.  xonly: 32 bytes x per item (derive),
// else x || y.  scratch: 8 x N words (prefix products).
EB_HD void k256_ks_norm_thread(size_t tid, size_t T, size_t N, int batch, const u32* jac, u32* scratch, bool xonly,
                               uint8_t* out, uint8_t* status) {
  const size_t ob = xonly ? 32 : 64;
  fe prod = fe_one();
  u64 live = 0;
  int cnt = 0;
  for (int j = 0; j < batch; j++) {
    size_t i = tid + (size_t)j * T;
    if (i >= N) break;
    cnt = j + 1;
    fe z;
    for (int w = 0; w < 8; w++) z.v[w] = jac[(size_t)(16 + w) * N + i];
    if (status[i] != ST_TRUE || fe_is_zero(z)) continue;
    live |= (u64)1 << j;
    for (int w = 0; w < 8; w++) scratch[(size_t)w * N + i] = prod.v[w];
    prod = fe_mul(prod, z);
  }
  if (cnt == 0) return;
  fe inv = fe_inv(prod);
  for (int j = cnt - 1; j >= 0; j--) {
    size_t i = tid + (size_t)j * T;
    uint8_t* o = out + ob * i;
    if (!((live >> j) & 1)) {
      for (size_t b = 0; b < ob; b++) o[b] = 0;
      if (status[i] == ST_TRUE) status[i] = ST_INFINITY;
      continue;
    }
    fe x, y, z, pre;
    for (int w = 0; w < 8; w++) {
      x.v[w] = jac[(size_t)w * N + i];
      y.v[w] = jac[(size_t)(8 + w) * N + i];
      z.v[w] = jac[(size_t)(16 + w) * N + i];
      pre.v[w] = scratch[(size_t)w * N + i];
    }
    fe zi = fe_mul(inv, pre);          // Z_i^-1
    inv = fe_mul(inv, z);              // drop Z_i from the running inverse
    fe zi2 = fe_sqr(zi);
    fe ax = fe_normalize(fe_mul(x, zi2));
    store_be<8>(o, ax.v);
    if (!xonly) {
      fe ay = fe_normalize(fe_mul(fe_mul(y, zi2), zi));
      store_be<8>(o + 32, ay.v);
    }
  }
}

// The same three steps on the a = -3 presets, in SW<C>'s Montgomery form (entries canonical, like its G table).
template <class C>
struct SWKeyed {
  typedef SW<C> W_;
  typedef typename W_::F F;
  typedef typename W_::fe fe;
  typedef typename W_::jac jac;
  typedef typename W_::aff aff;
  static constexpr int N = C::N;
  static_assert(N % 2 == 0, "an entry of 2 N words is read as 16-byte words");
  static_assert(W_::MBITS == C::BITS - 1, "keyset_geom() states the same bit count");

  static EB_HD uint8_t classify_item(size_t k, const uint8_t* xy, const uint8_t* pre) {
    if (pre && pre[k]) return pre[k];
    return W_::on_curve(W_::load_point(xy, k)) ? 1 : 0;
  }

  static EB_HD void bases_item(size_t k, const uint8_t* xy, const uint8_t* kst, int W, int windows, u32* bases) {
    if (kst[k] != 1) return;
    jac b = W_::from_aff(W_::load_point(xy, k));
    for (int j = 0; j < windows; j++) {
      u32* o = bases + ((size_t)k * windows + j) * 3 * N;
      store_fe_n<N>(o, b.x); store_fe_n<N>(o + N, b.y); store_fe_n<N>(o + 2 * N, b.z);
      if (j + 1 < windows)
        for (int d = 0; d < W; d++) b = W_::dbl(b);
    }
  }

  // a + p with h = Z3 / Z1 (table build; inputs never exceptional)
  static EB_HD jac madd_h(const jac& a, const aff& p, fe* hout) {
    fe z2 = F::sqr(a.z);
    fe u2 = F::mul(p.x, z2);
    fe s2 = F::mul(F::mul(p.y, z2), a.z);
    fe h = F::sub(a.x, u2);
    fe rr = F::sub(a.y, s2);
    fe h2 = F::sqr(h);
    fe h3 = F::mul(h2, h);
    fe v = F::mul(a.x, h2);
    jac r;
    r.x = F::sub(F::sub(F::add(F::sqr(rr), h3), v), v);
    r.y = F::sub(F::mul(rr, F::sub(v, r.x)), F::mul(a.y, h3));
    r.z = F::mul(a.z, h);
    *hout = h;
    return r;
  }

  static EB_HD void window_item(size_t t, const uint8_t* kst, int W, int windows, const u32* bases, u32* tab) {
    if (kst[t / windows] != 1) return;
    const int entries = 1 << (W - 1);
    jac bj;
    bj.x = load_fe_n<N>(bases + t * 3 * N); bj.y = load_fe_n<N>(bases + t * 3 * N + N); bj.z = load_fe_n<N>(bases + t * 3 * N + 2 * N);
    aff B = W_::to_aff(bj);
    aff D = W_::to_aff(W_::dbl(W_::from_aff(B)));
    u32* out = tab + t * entries * 2 * N;
    jac P = W_::from_aff(B);
    for (int c = 0; c < entries; c += KS_CHUNK) {
      fe h[KS_CHUNK];
      int cnt = entries - c < KS_CHUNK ? entries - c : KS_CHUNK;
      for (int u = 0; u < cnt; u++) {
        if (c + u == 0) h[u] = F::one();
        else P = madd_h(P, D, &h[u]);
        store_fe_n<N>(out + 2 * N * (c + u), P.x); store_fe_n<N>(out + 2 * N * (c + u) + N, P.y);
      }
      fe inv = F::inv(P.z);
      for (int u = cnt - 1; u >= 0; u--) {
        u32* e = out + 2 * N * (c + u);
        fe zi2 = F::sqr(inv);
        store_fe_n<N>(e, F::canon(F::mul(load_fe_n<N>(e), zi2)));
        store_fe_n<N>(e + N, F::canon(F::mul(F::mul(load_fe_n<N>(e + N), zi2), inv)));
        inv = F::mul(inv, h[u]);
      }
    }
  }

  // u2*Q from one key's table `tab`: one mixed add per window.  The keyed mul body's accumulation (verify_keyed_item
  // keeps its own copy, as k256_verify_keyed_item does)
  static EB_HD jac key_part(size_t i, size_t cnt_items, u32 flags, int W, int windows, const u32* tab, const u32* ws) {
    jac acc = W_::infinity();
    for (int w = windows - 1; w >= 0; w--) {
      bool dneg;
      u32 idx = ks_digit(ks_chunk(ws, cnt_items, i, N, N, W * w, W), w == windows - 1, W, &dneg);
      const bool neg = ((flags & W_::FL_NEG2) != 0) != dneg;
      u32 ent[2 * N];
      ks_load_entry<2 * N>(ent, tab + (((size_t)w << (W - 1)) + idx) * 2 * N);
      aff P;
      P.x = load_fe_n<N>(ent);
      P.y = load_fe_n<N>(ent + N);
      P.y = F::cmov(P.y, F::neg(P.y), neg);
      if (w == windows - 1) acc = W_::from_aff(P);
      else acc = W_::madd(acc, P);
    }
    return acc;
  }
  // acc + u1*G, as SW<C>::dsm
  static EB_HD jac g_part(jac acc, size_t i, size_t cnt_items, u32 flags, const u32* ws, const u32* gtab) {
    for (int j = 0; j < W_::GWINDOWS; j++) {
      bool dneg;
      u32 idx = ks_digit(W_::extract(ws, cnt_items, i, 0, W_::GW * j, W_::GW), j == W_::GWINDOWS - 1, W_::GW, &dneg);
      bool neg = dneg != ((flags & W_::FL_NEGG) != 0);
      const u32* ent = gtab + ((size_t)j * W_::GENTRIES + idx) * 2 * N;
      aff P;
      P.x = load_fe_n<N>(ent);
      P.y = load_fe_n<N>(ent + N);
      P.y = F::cmov(P.y, F::neg(P.y), neg);
      acc = W_::madd(acc, P);
    }
    return acc;
  }

  static EB_HD uint8_t verify_keyed_item(size_t i, size_t cnt_items, const u32* key_idx, const uint8_t* kst, int W,
                                         int windows, const u32* ktab, const uint8_t* r, const u32* ws, const u32* gtab) {
    const size_t LEN = C::LEN;
    const u32 k = key_idx[i];
    const uint8_t ks = kst[k];
    if (ks > 1) return ks;
    u32 flags = ws[(size_t)(2 * N) * cnt_items + i];
    if (flags & W_::FL_INVALID) return 0;
    if (ks != 1) return 4;               // ST_NEEDS_HOST: off-curve key, replayed
    const u32* tab = ktab + ((size_t)k * windows << (W - 1)) * 2 * N;
    jac acc = W_::infinity();
    for (int w = windows - 1; w >= 0; w--) {
      bool dneg;
      u32 idx = ks_digit(ks_chunk(ws, cnt_items, i, N, N, W * w, W), w == windows - 1, W, &dneg);
      bool neg = dneg != ((flags & W_::FL_NEG2) != 0);
      u32 ent[2 * N];
      ks_load_entry<2 * N>(ent, tab + (((size_t)w << (W - 1)) + idx) * 2 * N);
      aff P;
      P.x = load_fe_n<N>(ent);
      P.y = load_fe_n<N>(ent + N);
      P.y = F::cmov(P.y, F::neg(P.y), neg);
      if (w == windows - 1) acc = W_::from_aff(P);
      else acc = W_::madd(acc, P);
    }
    for (int j = 0; j < W_::GWINDOWS; j++) {           // u1*G, as SW<C>::dsm
      bool dneg;
      u32 idx = ks_digit(W_::extract(ws, cnt_items, i, 0, W_::GW * j, W_::GW), j == W_::GWINDOWS - 1, W_::GW, &dneg);
      bool neg = dneg != ((flags & W_::FL_NEGG) != 0);
      const u32* ent = gtab + ((size_t)j * W_::GENTRIES + idx) * 2 * N;
      aff P;
      P.x = load_fe_n<N>(ent);
      P.y = load_fe_n<N>(ent + N);
      P.y = F::cmov(P.y, F::neg(P.y), neg);
      acc = W_::madd(acc, P);
    }
    // accept iff R != O and x(R) == r (mod n)  (ec/index.js:222-228, eqXToP short.js:908-925)
    if (F::is_zero(acc.z)) return 0;
    fe z2 = F::sqr(acc.z);
    fe rp;
    W_::ldb(rp.v, r + LEN * i);
    if (F::eq(acc.x, F::mul(F::to_mont(rp), z2))) return 1;
    u32 pmn[N]; C::p_minus_n(pmn);
    if (!geq_n<N>(rp.v, pmn)) {
      u32 nmod[N]; W_::n_limbs(nmod);
      fe rn;
      add_n<N>(rn.v, rp.v, nmod);
      if (F::eq(acc.x, F::mul(F::to_mont(rn), z2))) return 1;
    }
    return 0;
  }
  // k256_mul_keyed_item on this curve: Jacobian result word-major (coordinate c, word w at jout[(N c + w) cnt + i]),
  // Montgomery form; 1 = ST_TRUE, 4 = ST_NEEDS_HOST, or the key's throw.
  static EB_HD uint8_t mul_keyed_item(size_t i, size_t cnt_items, const u32* key_idx, const uint8_t* kst, int W, int windows,
                                      const u32* ktab, const u32* ws, const u32* gtab, u32* jout) {
    const u32 k = key_idx[i];
    const uint8_t ks = kst[k];
    jac acc = W_::infinity();
    if (ks == 1) {
      u32 flags = ws[(size_t)(2 * N) * cnt_items + i];
      acc = key_part(i, cnt_items, flags, W, windows, ktab + ((size_t)k * windows << (W - 1)) * 2 * N, ws);
      if (!(flags & W_::FL_NOG)) acc = g_part(acc, i, cnt_items, flags, ws, gtab);
    }
    for (int w = 0; w < N; w++) {
      jout[(size_t)w * cnt_items + i] = acc.x.v[w];
      jout[(size_t)(N + w) * cnt_items + i] = acc.y.v[w];
      jout[(size_t)(2 * N + w) * cnt_items + i] = acc.z.v[w];
    }
    return ks == 1 ? 1 : ks == 0 ? 4 : ks;
  }

  // k256_ks_norm_thread on this curve: LEN bytes x (xonly) or x || y per item, as SW<C>::store_point writes them.
  // scratch: N x cnt_items words.
  static EB_HD void norm_thread(size_t tid, size_t T, size_t cnt_items, const u32* jac_in, u32* scratch, bool xonly,
                                uint8_t* out, uint8_t* status) {
    const size_t LEN = C::LEN, ob = xonly ? LEN : 2 * LEN;
    fe prod = F::one();
    u32 live = 0;
    int cnt = 0;
    for (int j = 0; j < W_::BATCH; j++) {
      size_t i = tid + (size_t)j * T;
      if (i >= cnt_items) break;
      cnt = j + 1;
      fe z = load_soa(jac_in, 2, cnt_items, i);
      if (status[i] != 1 || F::is_zero(z)) continue;
      live |= 1u << j;
      for (int w = 0; w < N; w++) scratch[(size_t)w * cnt_items + i] = prod.v[w];
      prod = F::mul(prod, z);
    }
    if (cnt == 0) return;
    fe inv = F::inv(prod);
    for (int j = cnt - 1; j >= 0; j--) {
      size_t i = tid + (size_t)j * T;
      uint8_t* o = out + ob * i;
      if (!((live >> j) & 1)) {
        for (size_t b = 0; b < ob; b++) o[b] = 0;
        if (status[i] == 1) status[i] = 7;               // ST_INFINITY
        continue;
      }
      fe pre;
      for (int w = 0; w < N; w++) pre.v[w] = scratch[(size_t)w * cnt_items + i];
      fe zi = F::mul(inv, pre);                          // Z_i^-1
      inv = F::mul(inv, load_soa(jac_in, 2, cnt_items, i));
      fe zi2 = F::sqr(zi);
      W_::stb(o, F::from_mont(F::mul(load_soa(jac_in, 0, cnt_items, i), zi2)).v);
      if (!xonly) W_::stb(o + LEN, F::from_mont(F::mul(F::mul(load_soa(jac_in, 1, cnt_items, i), zi2), zi)).v);
    }
  }
  static EB_HD fe load_soa(const u32* jac_in, int c, size_t cnt_items, size_t i) {
    fe r;
    for (int w = 0; w < N; w++) r.v[w] = jac_in[(size_t)(c * N + w) * cnt_items + i];
    return r;
  }
};

}  // namespace eb
