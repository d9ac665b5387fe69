// ecdsa_keyset_rp_body.cuh -- per-thread bodies of the keyed getKeyRecoveryParam kernels (keyset_recovery_param.cu):
// `ec.getKeyRecoveryParam(msg, sig, key.getPublic())` (ec/index.js:261-278) with the key's precomputed table.
// Host+device like the other bodies, so that the host emulation runs them.
//
// The scalars are the unkeyed recovery-parameter prep's (u1 = e / s, u2 = (r mod n) / s, FL_INVALID for s = 0 mod n).
// Main: P = u1 G + u2 Q from the key's table and the fixed table (ecdsa_keyset_body.cuh's keyed mul loops: no doubling,
// no per-item table), then the x test of recovery_param_item without inverting Z: X = r Z^2 gives j = 0, X = (r + n) Z^2
// (r < p - n) gives j = 2, anything else or Z = 0 no j.  Only Y and Z are stored.  Normalisation: one inversion per
// batch of live items (Montgomery's trick) for the parity of y = Y / Z^3, which completes recid = j | parity.
#pragma once
#include "ecdsa_keyset_body.cuh"

namespace eb {

// Item i on key key_idx[i], scalars as k256_prep_recovery_param_kernel (prep_thread mode 2) stores them.  recid[i] = j
// (0 or 2) and ST_TRUE when P passes the x test, with P's Y and Z word-major in yz (Y word w at yz[w N + i], Z at
// yz[(8 + w) N + i]); else recid[i] = 0 and the key's throw, ST_THROW_NO_RECOVERY, or ST_NEEDS_HOST for s = 0 (mod n),
// which the cold kernel decides.  The status eb200_ecdsa_recovery_param_batch gives for the key's x || y: an off-curve
// key never equals a recovered point.
EB_HD uint8_t k256_recovery_param_keyed_item(size_t i, size_t N, const u32* key_idx, const uint8_t* kst, int W, int windows,
                                             const u32* ktab, const uint8_t* r, const u32* ws, const u32* gtab, u32* yz,
                                             uint8_t* recid) {
  recid[i] = 0;
  const u32 k = key_idx[i];
  const uint8_t ks = kst[k];
  if (ks > ST_TRUE) return ks;
  if (ks != ST_TRUE) return ST_THROW_NO_RECOVERY;
  u32 rv[8], nn[8];
  load_be<8>(rv, r + 32 * i);
  K256N::n(nn);
  if (is_zero_n<8>(rv) || eq_n<8>(rv, nn)) return ST_THROW_NO_RECOVERY;   // r = 0 (mod n): rInv = 0, every Q' is O
  const u32 flags = ws[(size_t)18 * N + i];
  if (flags & FL_INVALID) return ST_NEEDS_HOST;                          // s = 0 (mod n)
  ge_jac acc = k256_ks_key_part(i, N, flags, W, windows, ktab + ((size_t)k * windows << (W - 1)) * 16, ws);
  acc = k256_ks_g_part(acc, i, N, flags, ws, gtab);
  if (fe_is_zero(acc.z)) return ST_THROW_NO_RECOVERY;
  fe z2 = fe_sqr(acc.z);
  u32 j = 0;
  if (!fe_eq(acc.x, fe_mul(fe_from_be(r + 32 * i), z2))) {
    const u32 pmn[8] = {0x2fc9baeeu, 0x402da172u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0, 0, 0};  // p mod n = p - n
    if (geq_n<8>(rv, pmn)) return ST_THROW_NO_RECOVERY;    // no second candidate (ec/index.js:243)
    fe rn;
    add_n<8>(rn.v, rv, nn);
    if (!fe_eq(acc.x, fe_mul(rn, z2))) return ST_THROW_NO_RECOVERY;
    j = 2;
  }
  for (int w = 0; w < 8; w++) {
    yz[(size_t)w * N + i] = acc.y.v[w];
    yz[(size_t)(8 + w) * N + i] = acc.z.v[w];
  }
  recid[i] = (uint8_t)j;
  return ST_TRUE;
}

// recid |= parity(Y / Z^3) for the ST_TRUE items tid, tid + T, ... (up to `batch` <= 64, T * batch >= N), with one
// inversion over the live items (Montgomery's trick).  scratch: 8 x N words (prefix products).
EB_HD void k256_ks_recid_norm_thread(size_t tid, size_t T, size_t N, int batch, const u32* yz, u32* scratch,
                                     const uint8_t* status, uint8_t* recid) {
  fe prod = fe_one();
  u64 live = 0;
  int cnt = 0;
  for (int j = 0; j < batch; j++) {
    size_t i = tid + (size_t)j * T;
    if (i >= N) break;
    if (status[i] != ST_TRUE) continue;
    cnt = j + 1;
    live |= (u64)1 << j;
    fe z;
    for (int w = 0; w < 8; w++) z.v[w] = yz[(size_t)(8 + w) * N + i];
    for (int w = 0; w < 8; w++) scratch[(size_t)w * N + i] = prod.v[w];
    prod = fe_mul(prod, z);
  }
  if (cnt == 0) return;
  fe inv = fe_inv(prod);
  for (int j = cnt - 1; j >= 0; j--) {
    if (!((live >> j) & 1)) continue;
    size_t i = tid + (size_t)j * T;
    fe y, z, pre;
    for (int w = 0; w < 8; w++) {
      y.v[w] = yz[(size_t)w * N + i];
      z.v[w] = yz[(size_t)(8 + w) * N + i];
      pre.v[w] = scratch[(size_t)w * N + i];
    }
    fe zi = fe_mul(inv, pre);          // Z_i^-1
    inv = fe_mul(inv, z);              // drop Z_i from the running inverse
    if (fe_is_odd(fe_mul(fe_mul(y, fe_sqr(zi)), zi))) recid[i] |= 1;
  }
}

// The same two bodies on the a = -3 presets, in SW<C>'s Montgomery form (status bytes as SW<C>: 1 = ST_TRUE,
// 4 = ST_NEEDS_HOST, 11 = ST_THROW_NO_RECOVERY).  yz: Y word w at yz[w cnt + i], Z at yz[(N + w) cnt + i].
template <class C>
struct SWKeyedRP {
  typedef SW<C> W_;
  typedef SWKeyed<C> K;
  typedef typename W_::F F;
  typedef typename W_::fe fe;
  typedef typename W_::jac jac;
  static constexpr int N = C::N;

  static EB_HD uint8_t main_item(size_t i, size_t cnt_items, const u32* key_idx, const uint8_t* kst, int W, int windows,
                                 const u32* ktab, const uint8_t* r, const u32* ws, const u32* gtab, u32* yz, uint8_t* recid) {
    const size_t LEN = C::LEN;
    recid[i] = 0;
    const u32 k = key_idx[i];
    const uint8_t ks = kst[k];
    if (ks > 1) return ks;
    if (ks != 1) return 11;                              // a recovered point is always on the curve
    u32 rn[N];
    W_::ldb(rn, r + LEN * i);
    W_::reduce_scalar(rn);
    if (is_zero_n<N>(rn)) return 11;                     // r = 0 (mod n): rInv = 0, every Q' is the point at infinity
    const u32 flags = ws[(size_t)(2 * N) * cnt_items + i];
    if (flags & W_::FL_INVALID) return 4;
    jac acc = K::key_part(i, cnt_items, flags, W, windows, ktab + ((size_t)k * windows << (W - 1)) * 2 * N, ws);
    acc = K::g_part(acc, i, cnt_items, flags, ws, gtab);
    if (F::is_zero(acc.z)) return 11;
    fe z2 = F::sqr(acc.z);
    fe rp;
    W_::ldb(rp.v, r + LEN * i);
    u32 j = 0;
    if (!F::eq(acc.x, F::mul(F::to_mont(rp), z2))) {
      u32 pmn[N]; C::p_minus_n(pmn);
      if (geq_n<N>(rp.v, pmn)) return 11;                // no second candidate (ec/index.js:243)
      u32 nmod[N]; W_::n_limbs(nmod);
      add_n<N>(rp.v, rp.v, nmod);                        // r + n < p
      if (!F::eq(acc.x, F::mul(F::to_mont(rp), z2))) return 11;
      j = 2;
    }
    for (int w = 0; w < N; w++) {
      yz[(size_t)w * cnt_items + i] = acc.y.v[w];
      yz[(size_t)(N + w) * cnt_items + i] = acc.z.v[w];
    }
    recid[i] = (uint8_t)j;
    return 1;
  }

  // k256_ks_recid_norm_thread on this curve, W_::BATCH items per thread; scratch: N x cnt_items words.
  static EB_HD void recid_norm_thread(size_t tid, size_t T, size_t cnt_items, const u32* yz, u32* scratch,
                                      const uint8_t* status, uint8_t* recid) {
    fe prod = F::one();
    u32 live = 0;
    int cnt = 0;
    for (int j = 0; j < W_::BATCH; j++) {
      size_t i = tid + (size_t)j * T;
      if (i >= cnt_items) break;
      if (status[i] != 1) continue;
      cnt = j + 1;
      live |= 1u << j;
      for (int w = 0; w < N; w++) scratch[(size_t)w * cnt_items + i] = prod.v[w];
      prod = F::mul(prod, K::load_soa(yz, 1, cnt_items, i));
    }
    if (cnt == 0) return;
    fe inv = F::inv(prod);
    for (int j = cnt - 1; j >= 0; j--) {
      if (!((live >> j) & 1)) continue;
      size_t i = tid + (size_t)j * T;
      fe pre;
      for (int w = 0; w < N; w++) pre.v[w] = scratch[(size_t)w * cnt_items + i];
      fe zi = F::mul(inv, pre);                          // Z_i^-1
      inv = F::mul(inv, K::load_soa(yz, 1, cnt_items, i));
      fe y = F::from_mont(F::mul(F::mul(K::load_soa(yz, 0, cnt_items, i), F::sqr(zi)), zi));
      recid[i] |= (uint8_t)(y.v[0] & 1);
    }
  }
};

}  // namespace eb
