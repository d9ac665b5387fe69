// eb200.cu -- CUDA kernels (sm_90a) and the C ABI of libelliptic_b200.so.
// See include/elliptic_b200.h for the boundary, ecdsa_k256_body.cuh (secp256k1) and
// ecdsa_sw_body.cuh (p256 / p384) for the algorithms.  No CPU fallback exists in this
// library by design: without a CUDA device every compute entry point fails.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <condition_variable>
#include <cstdlib>
#include <mutex>
#include <thread>
#include <type_traits>
#include <vector>
#include "../../include/elliptic_b200.h"
#include "ecdsa_k256_body.cuh"
#include "ecdsa_k256_replay.cuh"
#include "ecdsa_sw_replay.cuh"
#include "ecdsa_k256_sign_fast.cuh"
#include "der_sig.cuh"
#include "ecdsa_sw_sign.cuh"
#include "ecdsa_k256_sign.cuh"
#include "ecdsa_sw_body.cuh"
#include "ed25519_body.cuh"
#include "ed25519_ec.cuh"
#include "sw_runtime.cuh"
#include "kernel_bounds.h"
#include "recovery_param.h"
#include "keyset.h"
#include "unkeyed_forms.h"

using namespace eb;

// ---------------------------------------------------------------------------
// secp256k1 kernels
__global__ void __launch_bounds__(128) k256_gtab_kernel(u32* gtab) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)GTAB_WINDOWS * GTAB_ENTRIES) return;
  int j = (int)(t / GTAB_ENTRIES), idx = (int)(t % GTAB_ENTRIES);
  gtab_entry(j, idx, gtab + t * 16);
}

__global__ void __launch_bounds__(128) k256_prep_kernel(size_t N, const uint8_t* __restrict__ e,
                                                        const uint8_t* __restrict__ r,
                                                        const uint8_t* __restrict__ s,
                                                        u32* __restrict__ ws, u32* __restrict__ scratch, int batch) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  prep_thread(tid, T, N, e, r, s, ws, scratch, 0, batch);
}

__global__ void __launch_bounds__(EB_VERIFY_BLOCK, EB_K256_VERIFY_MINBLOCKS)
k256_verify_kernel(size_t N, const uint8_t* __restrict__ pub, const uint8_t* __restrict__ r,
                   const u32* __restrict__ ws, const u32* __restrict__ gtab,
                   u32* __restrict__ qtab, const uint8_t* __restrict__ pre, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (pre && pre[i]) { status[i] = pre[i]; return; }   // the reference throws while importing the key
  status[i] = verify_item(i, N, pub, r, ws, gtab, qtab);
}

__global__ void __launch_bounds__(128) k256_prep_recover_kernel(size_t N, const uint8_t* __restrict__ e,
                                                                const uint8_t* __restrict__ r,
                                                                const uint8_t* __restrict__ s,
                                                                u32* __restrict__ ws, u32* __restrict__ scratch) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  prep_thread(tid, T, N, e, r, s, ws, scratch, 1);
}
__global__ void __launch_bounds__(EB_VERIFY_BLOCK, EB_VERIFY_MINBLOCKS)
k256_recover_kernel(size_t N, const uint8_t* __restrict__ r, const uint8_t* __restrict__ recid,
                    const u32* __restrict__ ws, const u32* __restrict__ gtab, u32* __restrict__ qtab,
                    uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = recover_item(i, N, r, recid, ws, gtab, qtab, out);
}

// Two-kernel signing pipeline (ecdsa_k256_sign_fast.cuh); k256_sign_slow_kernel redoes flagged items with
// the literal retry loop of k256_sign_item.
__global__ void __launch_bounds__(128)
k256_sign_nonce_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv,
                       const u32* __restrict__ gtab, u32* __restrict__ ws, uint8_t* __restrict__ status,
                       const uint8_t* __restrict__ kgiven) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) k256_sign_nonce_item(i, N, e, priv, gtab, ws, status, kgiven);
}
__global__ void __launch_bounds__(128)
k256_sign_finish_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv, u32 canonical,
                        const u32* __restrict__ ws, u32* __restrict__ scratch, uint8_t* __restrict__ r,
                        uint8_t* __restrict__ s, uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  k256_sign_finish_thread(tid, T, N, e, priv, canonical, ws, scratch, r, s, recid, status);
}
__global__ void __launch_bounds__(128)
k256_sign_slow_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv, u32 canonical,
                      const u32* __restrict__ gtab, uint8_t* __restrict__ r, uint8_t* __restrict__ s,
                      uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = k256_sign_item(i, e, priv, canonical, gtab, r, s, recid);
}

// Exact replay of the reference's own GLV/JSF/wNAF schedule for the items the fast kernel flagged
// (un-validated off-curve keys, SURVEY 8a Q1).  Divergent by nature; flagged items are rare.
__global__ void __launch_bounds__(128) k256_replay_tab_kernel(u32* tab) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < 2 * REPLAY_NAF_PTS) rp_tab_entry(t, tab + 16 * t);
}
__global__ void __launch_bounds__(128)
k256_replay_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s,
                   const uint8_t* __restrict__ pub, const u32* __restrict__ tab, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = rp_verify_item(i, e, r, s, pub, tab);
}

// Point.mul / Point.mulAdd batches (short.js:422-441): k1*G + k2*P, k2*P, or k*G
__global__ void __launch_bounds__(128)
k256_prep_scalars_kernel(size_t N, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ k2, u32* __restrict__ ws) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) prep_scalars_item(i, N, k1, k2, ws);
}
__global__ void __launch_bounds__(EB_VERIFY_BLOCK, EB_VERIFY_MINBLOCKS)
k256_mul_add_kernel(size_t N, const uint8_t* __restrict__ pts, const u32* __restrict__ ws, const u32* __restrict__ gtab,
                    u32* __restrict__ qtab, uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = mul_add_item(i, N, pts, ws, gtab, qtab, out);
}
__global__ void __launch_bounds__(128)
k256_mul_add_replay_kernel(size_t N, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ k2,
                           const uint8_t* __restrict__ pts, const u32* __restrict__ tab, uint8_t* __restrict__ out,
                           uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = rp_mul_add_item(i, k1, k2, pts, tab, out);
}
__global__ void __launch_bounds__(128)
k256_mul_g_kernel(size_t N, const uint8_t* __restrict__ k, const u32* __restrict__ gtab, uint8_t* __restrict__ out,
                  uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = k256_mul_g_item(i, k, gtab, out);
}

__global__ void status_map_kernel(size_t N, uint8_t* __restrict__ status, uint8_t from, uint8_t to) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N && status[i] == from) status[i] = to;
}

// DER signatures -> fixed-width r, s (Signature._importDER, ec/signature.js:73-134).  `pre` carries the
// key-decoding verdict when there is one: a key that throws wins, as keyFromPublic runs first
// (ec/index.js:194-195).
__global__ void __launch_bounds__(128)
der_decode_kernel(size_t N, u32 len, const uint8_t* __restrict__ der, const unsigned long long* __restrict__ off,
                  uint8_t* __restrict__ r, uint8_t* __restrict__ s, uint8_t* __restrict__ pre, int pre_valid) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  bool ok = der_import(der + off[i], (size_t)(off[i + 1] - off[i]), len, r + (size_t)len * i, s + (size_t)len * i);
  uint8_t st = pre_valid ? pre[i] : 0;
  if (!st && !ok) st = ST_THROW_SIG_FORMAT;
  pre[i] = st;
}

// SEC1 decode (BaseCurve.decodePoint, lib/elliptic/curve/base.js:270-292; pointFromX short.js:187-204)
// fmt 1: 65-byte 04|06|07 || x || y ; fmt 2: 33-byte 02|03 || x.  Writes x||y (64 B) + a pre-status.
__global__ void __launch_bounds__(128) k256_decode_pub_kernel(size_t N, const uint8_t* __restrict__ in, u32 fmt,
                                                              uint8_t* __restrict__ xy, uint8_t* __restrict__ pre) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  uint8_t st = 0;
  if (fmt == EB200_PUB_SEC1_65) {
    const uint8_t* p = in + 65 * i;
    uint8_t tag = p[0];
    if (tag != 4 && tag != 6 && tag != 7) st = ST_THROW_POINT_FORMAT;
    else if ((tag == 6 && (p[64] & 1)) || (tag == 7 && !(p[64] & 1))) st = ST_THROW_ASSERT;   // base.js:278-281
    for (int k = 0; k < 64; k++) xy[64 * i + k] = p[1 + k];
  } else {
    const uint8_t* p = in + 33 * i;
    uint8_t tag = p[0];
    if (tag != 2 && tag != 3) st = ST_THROW_POINT_FORMAT;
    fe x = fe_from_be(p + 1);
    fe seven = fe_zero(); seven.v[0] = 7;
    fe y2 = fe_add(fe_mul(fe_sqr(x), x), seven);
    fe y = fe_sqrt_candidate(y2);
    if (!st && !fe_eq(fe_sqr(y), y2)) st = ST_THROW_INVALID_POINT;       // short.js:194-195
    y = fe_normalize(y);
    bool odd = tag == 3;
    if (((y.v[0] & 1) != 0) != odd) y = fe_normalize(fe_neg(y));
    x = fe_normalize(x);
    store_be<8>(xy + 64 * i, x.v);
    store_be<8>(xy + 64 * i + 32, y.v);
  }
  pre[i] = st;
}

// Scalar-field ops 16..21 of the self-test hook (eb200_selftest_fe, include/elliptic_b200.h) on the plain words
// a, b: the raw Montgomery product takes them as given, so a = R - 1 reaches the multiplier.  Returns false
// for any other op.
template <class S>
__device__ bool selftest_sc(int op, const u32* a, const u32* b, u32* out) {
  typedef typename S::fe fe_t;
  fe_t A = load_fe_n<S::N>(a), B = load_fe_n<S::N>(b), R;
  switch (op) {
    case 16: R = S::mul(A, B); break;
    case 17: R = S::to_mont(A); break;
    case 18: R = S::from_mont(A); break;
    case 19: R = S::add(A, B); break;
    case 20: R = S::sub(A, B); break;
    case 21: R = S::inv(A); break;
    default: return false;
  }
  store_fe_n<S::N>(out, R);
  return true;
}

__global__ void k256_selftest_fe_kernel(int op, size_t n, const u32* a, const u32* b, u32* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // mod n: the product, Montgomery conversion and inversion as prep_thread calls them
  if (op == 16 || op == 17 || op == 18) {
    u32 m[8] = {1, 0, 0, 0, 0, 0, 0, 0};            // from_mont: times a plain 1
    if (op == 16) copy_n<8>(m, b + 8 * i);
    if (op == 17) K256N::r2(m);
    sc_mont_mul(out + 8 * i, a + 8 * i, m);
    return;
  }
  if (op == 21) { sc_mont_inv(out + 8 * i, a + 8 * i); return; }
  if (op == 24 || op == 25) {                       // glv_split_odd: m1 (24) or m2 (25), then neg1, neg2
    u32 m1[5], m2[5];
    bool n1, n2;
    glv_split_odd(a + 8 * i, m1, &n1, m2, &n2);
    for (int w = 0; w < 5; w++) out[8 * i + w] = op == 24 ? m1[w] : m2[w];
    out[8 * i + 5] = n1; out[8 * i + 6] = n2; out[8 * i + 7] = 0;
    return;
  }
  if (selftest_sc<Fp<K256_FN>>(op, a + 8 * i, b + 8 * i, out + 8 * i)) return;
  fe A = load_fe(a + 8 * i), B = load_fe(b + 8 * i), R;
  switch (op) {
    case 0: R = fe_mul(A, B); break;
    case 1: R = fe_sqr(A); break;
    case 2: R = fe_add(A, B); break;
    case 3: R = fe_sub(A, B); break;
    case 4: R = fe_neg(A); break;
    case 5: R = fe_mul_small(A, b[8 * i]); break;
    case 6: R = fe_normalize(A); break;
    case 7: R = fe_inv(A); break;
    case 8: R = fe_sqrt_candidate(A); break;
    default: R = fe_zero();
  }
  store_fe(out + 8 * i, R);
}

// ---------------------------------------------------------------------------
// generic short-Weierstrass (a = -3) kernels
template <class C>
__global__ void __launch_bounds__(128) sw_gtab_kernel(u32* gtab) {
  typedef SW<C> W;
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)W::GWINDOWS * W::GENTRIES) return;
  int j = (int)(t / W::GENTRIES), idx = (int)(t % W::GENTRIES);
  W::gtab_entry(j, idx, gtab + t * 2 * W::N);
}
template <class C>
__global__ void __launch_bounds__(128) sw_prep_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                                                      const uint8_t* __restrict__ s, u32* __restrict__ ws,
                                                      u32* __restrict__ scratch) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  SW<C>::prep_thread(tid, T, N, e, r, s, ws, scratch);
}
template <class C>
__global__ void __launch_bounds__(128, (C::N <= 8) ? EB_SW_MINBLOCKS8 : EB_SW_MINBLOCKS_BIG)
sw_verify_kernel(size_t N, const uint8_t* __restrict__ pub, const uint8_t* __restrict__ r, const u32* __restrict__ ws,
                 const u32* __restrict__ gtab, u32* __restrict__ qtab, const uint8_t* __restrict__ pre,
                 uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (pre && pre[i]) { status[i] = pre[i]; return; }
  status[i] = SW<C>::verify_item(i, N, pub, r, ws, gtab, qtab);
}
// Exact replay of the reference's wNAF schedule for off-curve keys (ecdsa_sw_replay.cuh)
template <class C>
__global__ void __launch_bounds__(128) sw_replay_tab_kernel(u32* tab) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < SWReplay<C>::NAF_PTS) SWReplay<C>::tab_entry(t, tab + 2 * C::N * t);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_replay_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s,
                 const uint8_t* __restrict__ pub, const u32* __restrict__ tab, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = SWReplay<C>::verify_item(i, e, r, s, pub, tab);
}
// EC.recoverPubKey on the non-GLV curves
template <class C>
__global__ void __launch_bounds__(128)
sw_prep_recover_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s,
                       u32* __restrict__ ws) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) SW<C>::prep_recover_item(i, N, e, r, s, ws);
}
template <class C>
__global__ void __launch_bounds__(128, 2)
sw_recover_kernel(size_t N, const uint8_t* __restrict__ r, const uint8_t* __restrict__ recid, const u32* __restrict__ ws,
                  const u32* __restrict__ gtab, u32* __restrict__ qtab, uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = SW<C>::recover_item(i, N, r, recid, ws, gtab, qtab, out);
}

// EC.sign on p256 / p384 (ecdsa_sw_sign.cuh)
template <class SG>
__global__ void __launch_bounds__(128)
sw_sign_nonce_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv,
                     const u32* __restrict__ gtab, u32* __restrict__ ws, uint8_t* __restrict__ status,
                     const uint8_t* __restrict__ kgiven) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) SG::nonce_item(i, N, e, priv, gtab, ws, status, kgiven);
}
// EC.sign with the `pers` option and EC.genKeyPair({entropy, pers}): literal per-item loops on the byte-stream DRBG
template <class SG>
__global__ void __launch_bounds__(128)
sw_sign_pers_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv, const uint8_t* __restrict__ pers,
                    u32 np, u32 canonical, const u32* __restrict__ gtab, uint8_t* __restrict__ r, uint8_t* __restrict__ s,
                    uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = SG::slow_item_pers(i, e, priv, pers, (int)np, canonical, gtab, r, s, recid);
}
template <class SG>
__global__ void __launch_bounds__(128)
sw_keygen_kernel(size_t N, const uint8_t* __restrict__ entropy, u32 ne, const uint8_t* __restrict__ pers, u32 np,
                 uint8_t* __restrict__ out_priv, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = SG::keygen_item(i, entropy, (int)ne, pers, (int)np, out_priv);
}
__global__ void __launch_bounds__(128)
k256_sign_pers_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv, const uint8_t* __restrict__ pers,
                      u32 np, u32 canonical, const u32* __restrict__ gtab, uint8_t* __restrict__ r, uint8_t* __restrict__ s,
                      uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = k256_sign_item_pers(i, e, priv, pers, (int)np, canonical, gtab, r, s, recid);
}
__global__ void __launch_bounds__(128)
k256_keygen_kernel(size_t N, const uint8_t* __restrict__ entropy, u32 ne, const uint8_t* __restrict__ pers, u32 np,
                   uint8_t* __restrict__ out_priv, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = k256_keygen_item(i, entropy, (int)ne, pers, (int)np, out_priv);
}
template <class SG>
__global__ void __launch_bounds__(128)
sw_sign_finish_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv, u32 canonical,
                      const u32* __restrict__ ws, u32* __restrict__ scratch, uint8_t* __restrict__ r,
                      uint8_t* __restrict__ s, uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  SG::finish_thread(tid, T, N, e, priv, canonical, ws, scratch, r, s, recid, status);
}
template <class SG>
__global__ void __launch_bounds__(128)
sw_sign_slow_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv, u32 canonical,
                    const u32* __restrict__ gtab, uint8_t* __restrict__ r, uint8_t* __restrict__ s,
                    uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = SG::slow_item(i, e, priv, canonical, gtab, r, s, recid);
}

// Point.mul / mulAdd batches on the non-GLV short curves
template <class C>
__global__ void __launch_bounds__(128)
sw_prep_scalars_kernel(size_t N, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ k2, u32* __restrict__ ws) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) SW<C>::prep_scalars_item(i, N, k1, k2, ws);
}
template <class C>
__global__ void __launch_bounds__(128, 2)
sw_mul_add_kernel(size_t N, const uint8_t* __restrict__ pts, const u32* __restrict__ ws, const u32* __restrict__ gtab,
                  u32* __restrict__ qtab, uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = SW<C>::mul_add_item(i, N, pts, ws, gtab, qtab, out);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_mul_add_replay_kernel(size_t N, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ k2,
                         const uint8_t* __restrict__ pts, const u32* __restrict__ tab, uint8_t* __restrict__ out,
                         uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = SWReplay<C>::mul_add_item(i, k1, k2, pts, tab, out);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_mul_g_kernel(size_t N, const uint8_t* __restrict__ k, const u32* __restrict__ gtab, uint8_t* __restrict__ out,
                uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = SW<C>::mul_g_item(i, k, gtab, out);
}
template <class C>
__global__ void __launch_bounds__(128) sw_decode_pub_kernel(size_t N, const uint8_t* __restrict__ in, u32 fmt,
                                                            uint8_t* __restrict__ xy, uint8_t* __restrict__ pre) {
  typedef SW<C> W;
  typedef typename W::F F;
  constexpr size_t LEN = C::LEN;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  uint8_t st = 0;
  if (fmt == EB200_PUB_SEC1_65) {
    const uint8_t* p = in + (1 + 2 * LEN) * i;
    uint8_t tag = p[0];
    if (tag != 4 && tag != 6 && tag != 7) st = ST_THROW_POINT_FORMAT;
    else if ((tag == 6 && (p[2 * LEN] & 1)) || (tag == 7 && !(p[2 * LEN] & 1))) st = ST_THROW_ASSERT;
    for (size_t k = 0; k < 2 * LEN; k++) xy[2 * LEN * i + k] = p[1 + k];
  } else {
    const uint8_t* p = in + (1 + LEN) * i;
    uint8_t tag = p[0];
    if (tag != 2 && tag != 3) st = ST_THROW_POINT_FORMAT;
    typename F::fe t;
    W::ldb(t.v, p + 1);
    typename F::fe x = F::to_mont(t);
    typename F::fe y2 = F::add(F::sub(F::mul(F::sqr(x), x), F::add(F::dbl(x), x)), C::b());
    typename F::fe y = F::zero();
    uint8_t ss = W::sqrt_ref(y2, &y);                 // Red.sqrt: a^((p+1)/4), or Tonelli-Shanks on p224
    if (!st && ss) st = ss;
    if (!st && !F::eq(F::sqr(y), y2)) st = ST_THROW_INVALID_POINT;
    typename F::fe yp = F::from_mont(y);
    bool odd = tag == 3;
    if (((yp.v[0] & 1) != 0) != odd) yp = F::from_mont(F::neg(y));
    typename F::fe xp = F::from_mont(x);
    W::stb(xy + 2 * LEN * i, xp.v);
    W::stb(xy + 2 * LEN * i + LEN, yp.v);
  }
  pre[i] = st;
}
template <class C>
__global__ void sw_selftest_fe_kernel(int op, size_t n, const u32* a, const u32* b, u32* out) {
  typedef typename SW<C>::F F;
  constexpr int NL = SW<C>::N;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  typename F::fe A = F::to_mont(load_fe_n<NL>(a + NL * i)), B = F::to_mont(load_fe_n<NL>(b + NL * i)), R;
  switch (op) {
    case 0: R = F::mul(A, B); break;
    case 1: R = F::sqr(A); break;
    case 2: R = F::add(A, B); break;
    case 3: R = F::sub(A, B); break;
    case 4: R = F::neg(A); break;
    case 7: R = F::inv(A); break;
    default: R = A;
  }
  store_fe_n<NL>(out + NL * i, F::from_mont(R));
}
// The short curves' other self-test ops: the doubling's scaled products (8..11) and the scalar field (16..21).  A
// kernel of its own, first named by eb200_selftest_fe at the end of this file: instantiating this code inside
// sw_selftest_fe_kernel, which sw_kernel_order names early, changed the inlining in sw_mul_add_kernel<P384>.
template <class C>
__global__ void sw_selftest_ext_kernel(int op, size_t n, const u32* a, const u32* b, u32* out) {
  typedef typename SW<C>::F F;
  constexpr int NL = SW<C>::N;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (selftest_sc<typename C::S>(op, a + NL * i, b + NL * i, out + NL * i)) return;
  typename F::fe A = F::to_mont(load_fe_n<NL>(a + NL * i)), B = F::to_mont(load_fe_n<NL>(b + NL * i)), R;
  switch (op) {            // called as SW::dbl_inl calls them
    case 8: R = F::template mul_k<3>(A, B); break;
    case 9: R = F::template mul_k<4>(A, B); break;
    case 10: R = F::template sqr_k<8>(A); break;
    case 11: R = F::dbl(A); break;
    default: R = A;
  }
  store_fe_n<NL>(out + NL * i, F::from_mont(R));
}

// ---------------------------------------------------------------------------
// ed25519 / curve25519 kernels
__global__ void __launch_bounds__(128) ed_gtab_kernel(u32* gtab) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)ED_GWINDOWS * ED_GENTRIES) return;
  ed_gtab_entry((int)(t / ED_GENTRIES), (int)(t % ED_GENTRIES), gtab + t * 24);
}
__global__ void __launch_bounds__(128, 3)
ed25519_verify_kernel(size_t N, const uint8_t* __restrict__ R, const uint8_t* __restrict__ S,
                      const uint8_t* __restrict__ A, const uint8_t* __restrict__ h,
                      const u32* __restrict__ gtab, u32* __restrict__ atab, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = ed25519_verify_item(i, R, S, A, h, gtab, atab);
}
__global__ void f25_selftest_kernel(int op, size_t n, const u32* a, const u32* b, u32* out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (selftest_sc<Fp<ED25519_FN>>(op, a + 8 * i, b + 8 * i, out + 8 * i)) return;   // mod l (ed25519_ec.cuh)
  f25 A = f25_load(a + 8 * i), B = f25_load(b + 8 * i), R;
  switch (op) {
    case 0: R = f25_mul(A, B); break;
    case 1: R = f25_sqr(A); break;
    case 2: R = f25_add(A, B); break;
    case 3: R = f25_sub(A, B); break;
    case 4: R = f25_neg(A); break;
    case 5: R = f25_mul_small(A, b[8 * i]); break;
    case 6: R = f25_normalize(A); break;
    case 7: R = f25_inv(A); break;
    case 8: R = f25_pow_p58(A); break;
    default: R = f25_zero();
  }
  f25_store(out + 8 * i, R);
}
__global__ void __launch_bounds__(128)
ed25519_hash_kernel(size_t N, const uint8_t* __restrict__ R, const uint8_t* __restrict__ A,
                    const uint8_t* __restrict__ msgs, const u64* __restrict__ msg_off, uint8_t* __restrict__ h) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  ed25519_hash_item(i, R, A, msgs, msg_off, h);
}
__global__ void __launch_bounds__(128)
ed25519_sign_kernel(size_t N, const uint8_t* __restrict__ secrets, const uint8_t* __restrict__ msgs,
                    const u64* __restrict__ msg_off, const u32* __restrict__ gtab, uint8_t* __restrict__ sig,
                    uint8_t* __restrict__ pub, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = ed25519_sign_item(i, secrets, msgs, msg_off, gtab, sig, pub);
}
// the `ec` API over ed25519 (ed25519_ec.cuh)
__global__ void __launch_bounds__(128) ed_ec_decode_pub_kernel(size_t N, const uint8_t* __restrict__ in, u32 fmt,
                                                               uint8_t* __restrict__ xy, uint8_t* __restrict__ pre) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) pre[i] = ed_ec_decode_pub(in + (fmt == EB200_PUB_SEC1_65 ? 65 : 33) * i, fmt, xy + 64 * i);
}
__global__ void __launch_bounds__(128, 3)
ed_ec_verify_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s,
                    const uint8_t* __restrict__ xy, const uint8_t* __restrict__ pre, const u32* __restrict__ gtab,
                    u32* __restrict__ atab, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = ed_ec_verify_item(i, e, r, s, xy, pre, gtab, atab);
}
__global__ void __launch_bounds__(128)
ed_ec_sign_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ priv, const uint8_t* __restrict__ kgiven,
                  const uint8_t* __restrict__ pers, u32 np, u32 canonical, const u32* __restrict__ gtab,
                  uint8_t* __restrict__ r, uint8_t* __restrict__ s, uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = ed_ec_sign_item(i, e, priv, kgiven, pers, (int)np, canonical, gtab, r, s, recid);
}
__global__ void __launch_bounds__(128)
ed_ec_keygen_kernel(size_t N, const uint8_t* __restrict__ entropy, u32 ne, const uint8_t* __restrict__ pers, u32 np,
                    uint8_t* __restrict__ out_priv, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = ed_ec_keygen_item(i, entropy, (int)ne, pers, (int)np, out_priv);
}
__global__ void __launch_bounds__(128, 3)
ed_ec_mul_add_kernel(size_t N, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ k2, const uint8_t* __restrict__ pts,
                     u32 derive, const u32* __restrict__ gtab, u32* __restrict__ atab, uint8_t* __restrict__ out,
                     uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = ed_ec_mul_add_item(i, k1, k2, pts, derive != 0, gtab, atab, out);
}
// Montgomery-curve Point.mul (mont.js:130-153): the ladder alone, no validation (derive = validate + this)
__global__ void __launch_bounds__(128, 4)
x25519_mul_kernel(size_t N, const uint8_t* __restrict__ k, const uint8_t* __restrict__ px, uint8_t* __restrict__ out,
                  uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = x25519_mul_item(i, k, px, out);
}
__global__ void __launch_bounds__(128, 4)
x25519_derive_kernel(size_t N, const uint8_t* __restrict__ priv, const uint8_t* __restrict__ pubx,
                     uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = x25519_derive_item(i, priv, pubx, out);
}

// run-time short curves (sw_runtime.cuh): one thread per item; op 0 mul / mulAdd, 1 add, 2 dbl, 3 validate
template <int NL>
__global__ void __launch_bounds__(128)
rt_curve_kernel(int op, size_t N, RtCurve<NL> C, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ p1,
                const uint8_t* __restrict__ k2, const uint8_t* __restrict__ p2, u32 klen, uint8_t* __restrict__ out,
                uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = RtG<NL>::item(op, i, k1, p1, k2, p2, klen, out, C);
}

// ---------------------------------------------------------------------------
// contexts: one per CUDA device, created by eb200_init(devices, ndev, flags).  Host-pointer calls are
// sharded over the initialised devices in contiguous blocks (SURVEY 8e), each block driven by its own host
// thread on its own device; device-pointer calls run on the device that owns the pointers.
#include "chunk_plan.h"
namespace {
constexpr int MAX_CHUNKS = EB_MAX_CHUNKS;
constexpr int MAX_CURVES = 16;                       // curve ids index the per-context table arrays
constexpr int MAX_DEV = 16;
constexpr int STAGE_SLOTS = 8;                       // pinned staging ring for pageable caller buffers
constexpr size_t STAGE_BYTES = (size_t)4 << 20;
constexpr size_t SHARD_MIN_ITEMS = (size_t)1 << 14;  // below this per device a second GPU does not pay

// ---- parallel host memcpy (pageable caller buffers -> pinned staging slots) ----------------------------
struct CopyJob { void* dst; const void* src; size_t bytes; };
class CopyPool {
 public:
  void run(const CopyJob* j, int n) {
    if (n <= 0) return;
    std::lock_guard<std::mutex> one(call_mu_);
    if (n == 1) { memcpy(j[0].dst, j[0].src, j[0].bytes); return; }
    {
      std::lock_guard<std::mutex> lk(m_);
      if (workers_.empty()) for (int t = 0; t < 3; t++) workers_.emplace_back([this] { loop(); });
      jobs_.store(j); njobs_.store(n); next_.store(0); pending_ = n; gen_++;
    }
    cv_work_.notify_all();
    work();
    std::unique_lock<std::mutex> lk(m_);
    cv_done_.wait(lk, [&] { return pending_ == 0; });
  }
  ~CopyPool() {
    { std::lock_guard<std::mutex> lk(m_); stop_ = true; }
    cv_work_.notify_all();
    for (auto& t : workers_) t.join();
  }
 private:
  void loop() {
    unsigned long long seen = 0;
    for (;;) {
      { std::unique_lock<std::mutex> lk(m_); cv_work_.wait(lk, [&] { return stop_ || gen_ != seen; }); if (stop_) return; seen = gen_; }
      work();
    }
  }
  void work() {
    for (;;) {
      int i = next_.fetch_add(1);
      if (i >= njobs_.load()) break;
      const CopyJob* j = jobs_.load();
      memcpy(j[i].dst, j[i].src, j[i].bytes);
      std::lock_guard<std::mutex> lk(m_);
      if (--pending_ == 0) cv_done_.notify_all();
    }
  }
  std::mutex m_, call_mu_;
  std::condition_variable cv_work_, cv_done_;
  std::vector<std::thread> workers_;
  std::atomic<const CopyJob*> jobs_{nullptr};
  std::atomic<int> njobs_{0}, next_{0};
  int pending_ = 0;
  unsigned long long gen_ = 0;
  bool stop_ = false;
};

// Ctx::ev slots of the single-stream and device-pointer calls: h2d_ms = START..INPUTS_RESIDENT,
// kernel_ms = INPUTS_RESIDENT..KERNELS_DONE, d2h_ms = KERNELS_DONE..OUTPUTS_HOME, main_kernel_ms = MAIN_BEGIN..MAIN_END.
enum { EV_START, EV_INPUTS_RESIDENT, EV_KERNELS_DONE, EV_OUTPUTS_HOME, EV_MAIN_BEGIN, EV_MAIN_END, EV_SLOTS };

struct Ctx {
  std::mutex mu;                      // serialises the calls that use this device's buffers / events
  bool ready = false;
  int device = -1;
  cudaStream_t stream = nullptr, stream2 = nullptr, copy_stream = nullptr;
  u32* gtab[MAX_CURVES] = {};
  u32* sw_replay_tab[MAX_CURVES] = {}; // p256/p384: the reference's wnd-8 NAF table of G
  u32* replay_tab = nullptr;          // secp256k1: the reference's wnd-7 NAF table of G and its beta image
  uint8_t* d_in = nullptr; size_t d_in_cap = 0;
  uint8_t* d_ws = nullptr; size_t d_ws_cap = 0;
  uint8_t* d_status = nullptr; size_t d_status_cap = 0;
  cudaEvent_t ev[EV_SLOTS] = {};
  cudaEvent_t ev_in[MAX_CHUNKS] = {}, ev_k0[MAX_CHUNKS] = {}, ev_k1[MAX_CHUNKS] = {}, ev_done[MAX_CHUNKS] = {};
  uint8_t* h_stage[STAGE_SLOTS] = {};
  cudaEvent_t ev_stage[STAGE_SLOTS] = {};
  bool stage_used[STAGE_SLOTS] = {};
  unsigned stage_next = 0;
  CopyPool pool;                                       // this device's staging copies (one pool per device: no cross-device serialisation)
  eb200_timing timing = {};
};
Ctx g_ctx[MAX_DEV];
int g_devs[MAX_DEV];
int g_ndev = 0;
std::atomic<unsigned> g_rr{0};
std::mutex g_mu;                                     // init / shutdown / the device list
thread_local char g_err[256] = "";
thread_local eb200_timing t_timing = {};             // timing of this thread's last host-pointer call
thread_local Ctx* t_pending = nullptr;               // device-pointer call whose events have not been read yet
thread_local unsigned t_pending_launches = 0;

int cuda_fail(cudaError_t e, const char* what) {
  snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
  return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? EB200_ERR_NO_DEVICE : EB200_ERR_CUDA;
}
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return cuda_fail(e_, #call); } while (0)

// Launches kernels on one stream and counts them for eb200_timing.launches.  After a failed launch it launches
// nothing more and keeps the error in `rc` for the caller to return.
struct Launch {
  cudaStream_t st;
  unsigned count = 0;
  int rc = EB200_OK;
  template <class... P, class... A>
  void operator()(void (*kernel)(P...), unsigned grid, unsigned block, A... args) {
    if (rc) return;
    kernel<<<grid, block, 0, st>>>(args...);
    count++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = cuda_fail(e, "cudaGetLastError()");
  }
};
unsigned blocks128(size_t threads) { return (unsigned)((threads + 127) / 128); }
// grid of a prep / finish kernel whose threads each take up to `batch` items
unsigned batch_blocks(size_t n, int batch) { return blocks128((n + batch - 1) / batch); }
// Items per thread of the secp256k1 verify prep.  Each thread pays one inversion (~300 products mod n) for its
// batch, so a larger batch amortises it, as long as the grid still fills the GPU: 2^20 items at 32 per thread are
// 256 blocks of 128.  Smaller calls (and the pipelined host calls' 2^18-item chunks) keep PREP_BATCH.
int k256_prep_batch(size_t n) { return n >= ((size_t)1 << 20) ? 32 : PREP_BATCH; }

// Which kernels serve a curve id: secp256k1 and ed25519 have their own, the other short curves share the SW<C>
// templates and sign with their curves.js hash (p384: SHA-384, p521: SHA-512, the rest: SHA-256).
struct K256Curve {};
struct Ed25519Curve {};
template <class C_> struct SwCurve {
  typedef C_ C;
  typedef SWSign<C, std::conditional_t<std::is_same<C, P384>::value, Sha384W,
                                       std::conditional_t<std::is_same<C, P521>::value, Sha512W, Sha256W>>> SG;
};
template <class T> constexpr bool is_k256 = std::is_same<T, K256Curve>::value;
template <class T> constexpr bool is_ed25519 = std::is_same<T, Ed25519Curve>::value;

// Calls f(tag) with the tag type of `curve` (f returns an int status); EB200_ERR_UNSUPPORTED for other ids.
template <class F>
int with_curve(int curve, F&& f) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: return f(K256Curve{});
    case EB200_CURVE_ED25519: return f(Ed25519Curve{});
    case EB200_CURVE_P256: return f(SwCurve<P256>{});
    case EB200_CURVE_P384: return f(SwCurve<P384>{});
    case EB200_CURVE_P521: return f(SwCurve<P521>{});
    case EB200_CURVE_P192: return f(SwCurve<P192>{});
    case EB200_CURVE_P224: return f(SwCurve<P224>{});
    default: return EB200_ERR_UNSUPPORTED;
  }
}

// nvcc emits kernel templates in the order in which it first needs them, and NVVM's inlining into the 255-register
// p521 kernels (their registers and spills) depends on that order.  The dispatch above reaches every short-curve
// kernel through nested templates; naming these four families first keeps the module order their code was tuned in.
[[maybe_unused]] const void* const sw_kernel_order[] = {
    (const void*)sw_decode_pub_kernel<P256>, (const void*)sw_decode_pub_kernel<P384>, (const void*)sw_decode_pub_kernel<P521>,
    (const void*)sw_decode_pub_kernel<P192>, (const void*)sw_decode_pub_kernel<P224>,
    (const void*)sw_keygen_kernel<SwCurve<P256>::SG>, (const void*)sw_keygen_kernel<SwCurve<P384>::SG>,
    (const void*)sw_keygen_kernel<SwCurve<P521>::SG>, (const void*)sw_keygen_kernel<SwCurve<P192>::SG>,
    (const void*)sw_keygen_kernel<SwCurve<P224>::SG>,
    (const void*)sw_mul_g_kernel<P256>, (const void*)sw_mul_g_kernel<P384>, (const void*)sw_mul_g_kernel<P521>,
    (const void*)sw_mul_g_kernel<P192>, (const void*)sw_mul_g_kernel<P224>,
    (const void*)sw_selftest_fe_kernel<P256>, (const void*)sw_selftest_fe_kernel<P384>, (const void*)sw_selftest_fe_kernel<P521>,
    (const void*)sw_selftest_fe_kernel<P192>, (const void*)sw_selftest_fe_kernel<P224>,
};

int grow(uint8_t** p, size_t* cap, size_t need) {
  if (*cap >= need) return EB200_OK;
  if (*p) { cudaFree(*p); *p = nullptr; *cap = 0; }
  CK(cudaMalloc(p, need));
  *cap = need;
  return EB200_OK;
}
size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t fe_len(int curve) {   // field-element bytes for the selftest hooks (also the 25519 curves)
  if (curve == EB200_CURVE_P192) return 24;
  return (curve == EB200_CURVE_P384) ? 48 : (curve == EB200_CURVE_P521) ? 72 :     // 18 limbs; p224 = 8 limbs
         ((curve >= EB200_CURVE_SECP256K1 && curve <= EB200_CURVE_CURVE25519) || curve == EB200_CURVE_P224) ? 32 : 0;
}
constexpr size_t curve_len(int curve) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: case EB200_CURVE_P256: case EB200_CURVE_ED25519: return 32;
    case EB200_CURVE_P384: return 48;
    case EB200_CURVE_P521: return 66;
    case EB200_CURVE_P192: return 24;
    case EB200_CURVE_P224: return 28;
    default: return 0;
  }
}
size_t pub_item_bytes(size_t len, u32 fmt) {
  return fmt == EB200_PUB_XY ? 2 * len : fmt == EB200_PUB_SEC1_65 ? 1 + 2 * len : fmt == EB200_PUB_SEC1_33 ? 1 + len : 0;
}

// workspace: [ws words | scratch words | qtab words | decoded xy | pre-status]
struct WsLayout { size_t ws, scratch, qtab, xy, pre, total; };
WsLayout ws_layout(int curve, size_t n) {
  size_t prep_words = 0, scratch_words = 0, qtab_words = 0, len = curve_len(curve);
  with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    if constexpr (is_k256<T>) { prep_words = PREP_WORDS; scratch_words = 8; qtab_words = QTAB_WORDS; }
    else if constexpr (is_ed25519<T>) qtab_words = ED_ATAB_WORDS;
    else { typedef SW<typename T::C> W; prep_words = W::PREP_WORDS; scratch_words = W::N; qtab_words = W::QTAB_WORDS; }
    return EB200_OK;
  });
  WsLayout L;
  L.ws = 0;
  L.scratch = align256(L.ws + prep_words * n * 4);
  L.qtab = align256(L.scratch + scratch_words * n * 4);
  L.xy = align256(L.qtab + qtab_words * n * 4);
  L.pre = align256(L.xy + 2 * len * n);
  L.total = align256(L.pre + n);
  return L;
}


bool is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

struct Seg { void* dst; const void* src; size_t bytes; };
// Host -> device copies of `k` segments on stream st.  Pinned (or tiny) sources are copied directly;
// pageable ones go through the context's pinned ring, four pieces at a time with a parallel memcpy, so that
// a caller who did not pin its buffers (a Node.js Buffer) gets the pinned transfer rate (SURVEY 8b).
int h2d(Ctx& c, const Seg* seg, int k, cudaStream_t st) {
  size_t total = 0;
  for (int i = 0; i < k; i++) total += seg[i].bytes;
  bool direct = total < ((size_t)256 << 10);
  if (!direct) { direct = true; for (int i = 0; i < k; i++) if (seg[i].bytes && !is_pinned(seg[i].src)) { direct = false; break; } }
  if (direct) {
    for (int i = 0; i < k; i++) if (seg[i].bytes) CK(cudaMemcpyAsync(seg[i].dst, seg[i].src, seg[i].bytes, cudaMemcpyHostToDevice, st));
    return EB200_OK;
  }
  for (int s = 0; s < STAGE_SLOTS; s++) {
    if (!c.h_stage[s]) CK(cudaHostAlloc(&c.h_stage[s], STAGE_BYTES, cudaHostAllocDefault));
    if (!c.ev_stage[s]) CK(cudaEventCreateWithFlags(&c.ev_stage[s], cudaEventDisableTiming));
  }
  CopyJob jobs[4];
  void* dsts[4];
  int nj = 0;
  int slots[4];
  for (int i = 0; i < k; i++) {
    size_t off = 0;
    while (off < seg[i].bytes) {
      size_t m = seg[i].bytes - off < STAGE_BYTES ? seg[i].bytes - off : STAGE_BYTES;
      int slot = (int)(c.stage_next++ % STAGE_SLOTS);
      if (c.stage_used[slot]) CK(cudaEventSynchronize(c.ev_stage[slot]));
      jobs[nj] = CopyJob{c.h_stage[slot], (const uint8_t*)seg[i].src + off, m};
      dsts[nj] = (uint8_t*)seg[i].dst + off;
      slots[nj] = slot;
      nj++;
      off += m;
      if (nj == 4) {
        c.pool.run(jobs, nj);
        for (int j = 0; j < nj; j++) {
          CK(cudaMemcpyAsync(dsts[j], jobs[j].dst, jobs[j].bytes, cudaMemcpyHostToDevice, st));
          CK(cudaEventRecord(c.ev_stage[slots[j]], st));
          c.stage_used[slots[j]] = true;
        }
        nj = 0;
      }
    }
  }
  if (nj) {
    c.pool.run(jobs, nj);
    for (int j = 0; j < nj; j++) {
      CK(cudaMemcpyAsync(dsts[j], jobs[j].dst, jobs[j].bytes, cudaMemcpyHostToDevice, st));
      CK(cudaEventRecord(c.ev_stage[slots[j]], st));
      c.stage_used[slots[j]] = true;
    }
  }
  return EB200_OK;
}

// Builds the fixed-base table of `curve` (and the replay table of the curves that have one) on first use.
int ensure_table(Ctx& c, int curve) {
  return with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    if (c.gtab[curve]) return EB200_OK;
    if constexpr (is_k256<T>) {
      size_t entries = (size_t)GTAB_WINDOWS * GTAB_ENTRIES;
      CK(cudaMalloc(&c.gtab[curve], entries * 16 * 4));
      k256_gtab_kernel<<<blocks128(entries), 128, 0, c.stream>>>(c.gtab[curve]);
      CK(cudaGetLastError());
      CK(cudaMalloc(&c.replay_tab, (size_t)REPLAY_TAB_WORDS * 4));
      k256_replay_tab_kernel<<<2, 128, 0, c.stream>>>(c.replay_tab);
    } else if constexpr (is_ed25519<T>) {
      size_t entries = (size_t)ED_GWINDOWS * ED_GENTRIES;
      CK(cudaMalloc(&c.gtab[curve], entries * 24 * 4));
      ed_gtab_kernel<<<blocks128(entries), 128, 0, c.stream>>>(c.gtab[curve]);
    } else {
      typedef typename T::C C;
      typedef SW<C> W;
      size_t entries = (size_t)W::GWINDOWS * W::GENTRIES;
      CK(cudaMalloc(&c.gtab[curve], entries * 2 * W::N * 4));
      sw_gtab_kernel<C><<<blocks128(entries), 128, 0, c.stream>>>(c.gtab[curve]);
      CK(cudaGetLastError());
      CK(cudaMalloc(&c.sw_replay_tab[curve], (size_t)SWReplay<C>::TAB_WORDS * 4));
      sw_replay_tab_kernel<C><<<1, 128, 0, c.stream>>>(c.sw_replay_tab[curve]);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c.stream));
    return EB200_OK;
  });
}

// Launches decode (if needed) + prep + verify for n items on L's stream, recording ev_main0 / ev_main1 around the
// main kernel.  All pointers are device pointers.  der_verdict: a range screen's verdicts, for which the screened DER
// decode (unkeyed_forms.cu) takes der_decode_kernel's place.
int launch_verify(Ctx& c, int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r, const uint8_t* d_s,
                  const uint8_t* d_pub, u32 pub_fmt, uint8_t* d_status, uint8_t* d_workspace, Launch& L,
                  cudaEvent_t ev_main0, cudaEvent_t ev_main1,
                  const uint8_t* d_der = nullptr, const unsigned long long* d_der_off = nullptr,
                  const uint8_t* der_verdict = nullptr) {
  if (n == 0) return EB200_OK;
  const WsLayout W = ws_layout(curve, n);
  u32* ws = (u32*)(d_workspace + W.ws);
  u32* scratch = (u32*)(d_workspace + W.scratch);
  u32* qtab = (u32*)(d_workspace + W.qtab);
  uint8_t* dxy = d_workspace + W.xy;
  uint8_t* dpre = d_workspace + W.pre;
  const uint8_t* xy = d_pub;
  const uint8_t* pre = nullptr;
  const unsigned nb = blocks128(n);
  const u32* gt = c.gtab[curve];
  return with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    if (pub_fmt != EB200_PUB_XY) {
      if constexpr (is_k256<T>) L(k256_decode_pub_kernel, nb, 128, n, d_pub, pub_fmt, dxy, dpre);
      else if constexpr (is_ed25519<T>) L(ed_ec_decode_pub_kernel, nb, 128, n, d_pub, pub_fmt, dxy, dpre);
      else L(sw_decode_pub_kernel<typename T::C>, nb, 128, n, d_pub, pub_fmt, dxy, dpre);
      xy = dxy; pre = dpre;
    }
    if (d_der && der_verdict) {     // d_r / d_s are then scratch the decoder fills
      if (L.rc) return L.rc;
      cudaError_t err = unkeyed_der_decode_screened_launch(n, (u32)curve_len(curve), der_verdict, d_der, d_der_off,
                                                           (uint8_t*)d_r, (uint8_t*)d_s, dpre, (int)(pre != nullptr), L.st,
                                                           &L.count);
      if (err != cudaSuccess) return cuda_fail(err, "unkeyed_der_decode_screened_launch");
      pre = dpre;
    } else if (d_der) {
      L(der_decode_kernel, nb, 128, n, (u32)curve_len(curve), d_der, d_der_off, (uint8_t*)d_r, (uint8_t*)d_s, dpre,
        (int)(pre != nullptr));
      pre = dpre;
    }
    if constexpr (is_ed25519<T>) {     // the `ec` API over the Edwards preset: one kernel, per-item scalar inversion
      CK(cudaEventRecord(ev_main0, L.st));
      L(ed_ec_verify_kernel, nb, 128, n, d_e, d_r, d_s, xy, pre, gt, qtab, d_status);
      CK(cudaEventRecord(ev_main1, L.st));
    } else if constexpr (is_k256<T>) {
      L(k256_prep_kernel, batch_blocks(n, k256_prep_batch(n)), 128, n, d_e, d_r, d_s, ws, scratch, k256_prep_batch(n));
      CK(cudaEventRecord(ev_main0, L.st));
      L(k256_verify_kernel, (unsigned)((n + EB_VERIFY_BLOCK - 1) / EB_VERIFY_BLOCK), EB_VERIFY_BLOCK, n, xy, d_r, ws, gt,
        qtab, pre, d_status);
      CK(cudaEventRecord(ev_main1, L.st));
      L(k256_replay_kernel, nb, 128, n, d_e, d_r, d_s, xy, c.replay_tab, d_status);
    } else {
      typedef typename T::C C;
      L(sw_prep_kernel<C>, batch_blocks(n, SW<C>::BATCH), 128, n, d_e, d_r, d_s, ws, scratch);
      CK(cudaEventRecord(ev_main0, L.st));
      L(sw_verify_kernel<C>, nb, 128, n, xy, d_r, ws, gt, qtab, pre, d_status);
      CK(cudaEventRecord(ev_main1, L.st));
      L(sw_replay_kernel<C>, nb, 128, n, d_e, d_r, d_s, xy, c.sw_replay_tab[curve], d_status);
    }
    return L.rc;
  });
}

bool curve_ok(int curve) { return curve_len(curve) != 0; }
bool fmt_ok(u32 fmt) { return fmt == EB200_PUB_XY || fmt == EB200_PUB_SEC1_65 || fmt == EB200_PUB_SEC1_33; }

int ctx_create(Ctx& c, int device) {
  CK(cudaSetDevice(device));
  c.device = device;
  CK(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c.copy_stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c.stream2, cudaStreamNonBlocking));
  for (int i = 0; i < EV_SLOTS; i++) CK(cudaEventCreate(&c.ev[i]));
  for (int i = 0; i < MAX_CHUNKS; i++) {
    CK(cudaEventCreate(&c.ev_in[i]));
    CK(cudaEventCreate(&c.ev_k0[i]));
    CK(cudaEventCreate(&c.ev_k1[i]));
    CK(cudaEventCreate(&c.ev_done[i]));
  }
  c.ready = true;
  return EB200_OK;
}
void ctx_destroy(Ctx& c) {
  if (c.device < 0) return;
  cudaSetDevice(c.device);
  if (c.stream) cudaStreamSynchronize(c.stream);
  for (int k = 0; k < MAX_CURVES; k++) if (c.gtab[k]) { cudaFree(c.gtab[k]); c.gtab[k] = nullptr; }
  for (int k = 0; k < MAX_CURVES; k++) if (c.sw_replay_tab[k]) { cudaFree(c.sw_replay_tab[k]); c.sw_replay_tab[k] = nullptr; }
  if (c.replay_tab) { cudaFree(c.replay_tab); c.replay_tab = nullptr; }
  // the staging buffers may hold private keys or nonces of a signing call: wipe before release
  if (c.d_in) { cudaMemset(c.d_in, 0, c.d_in_cap); cudaFree(c.d_in); } c.d_in = nullptr; c.d_in_cap = 0;
  if (c.d_ws) { cudaMemset(c.d_ws, 0, c.d_ws_cap); cudaFree(c.d_ws); } c.d_ws = nullptr; c.d_ws_cap = 0;
  cudaFree(c.d_status); c.d_status = nullptr; c.d_status_cap = 0;
  for (int i = 0; i < EV_SLOTS; i++) if (c.ev[i]) { cudaEventDestroy(c.ev[i]); c.ev[i] = nullptr; }
  for (int i = 0; i < MAX_CHUNKS; i++) {
    if (c.ev_in[i]) { cudaEventDestroy(c.ev_in[i]); c.ev_in[i] = nullptr; }
    if (c.ev_k0[i]) { cudaEventDestroy(c.ev_k0[i]); c.ev_k0[i] = nullptr; }
    if (c.ev_k1[i]) { cudaEventDestroy(c.ev_k1[i]); c.ev_k1[i] = nullptr; }
    if (c.ev_done[i]) { cudaEventDestroy(c.ev_done[i]); c.ev_done[i] = nullptr; }
  }
  for (int s = 0; s < STAGE_SLOTS; s++) {
    if (c.h_stage[s]) { memset(c.h_stage[s], 0, STAGE_BYTES); cudaFreeHost(c.h_stage[s]); c.h_stage[s] = nullptr; }
    if (c.ev_stage[s]) { cudaEventDestroy(c.ev_stage[s]); c.ev_stage[s] = nullptr; }
    c.stage_used[s] = false;
  }
  if (c.stream) { cudaStreamDestroy(c.stream); c.stream = nullptr; }
  if (c.copy_stream) { cudaStreamDestroy(c.copy_stream); c.copy_stream = nullptr; }
  if (c.stream2) { cudaStreamDestroy(c.stream2); c.stream2 = nullptr; }
  c.ready = false;
  c.device = -1;
}

// The context that owns a device pointer (device-pointer entry points).
Ctx* ctx_of(const void* dptr) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, dptr) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) return nullptr;
  if (a.device < 0 || a.device >= MAX_DEV || !g_ctx[a.device].ready) return nullptr;
  return &g_ctx[a.device];
}

void merge_timing(eb200_timing& a, const eb200_timing& b) {
  if (b.h2d_ms > a.h2d_ms) a.h2d_ms = b.h2d_ms;
  if (b.kernel_ms > a.kernel_ms) a.kernel_ms = b.kernel_ms;
  if (b.d2h_ms > a.d2h_ms) a.d2h_ms = b.d2h_ms;
  if (b.main_kernel_ms > a.main_kernel_ms) a.main_kernel_ms = b.main_kernel_ms;
  a.launches += b.launches;
}

// Runs fn(ctx, lo, m) over contiguous blocks of [0, n): one block per listed device (run_sharded: per initialised device) when the batch is
// large enough, each on its own host thread (the blocks never exchange data; results land in the caller's
// buffers at their own offsets).  A single-block call rotates over the devices so that concurrent callers
// spread out.  Timing: the slowest block, launches summed.
template <class F>
int run_sharded_on(const int* devs, int nd, size_t n, F&& fn) {
  if (nd == 0) return EB200_ERR_NOT_INIT;
  int use = (int)(n / SHARD_MIN_ITEMS);
  if (use > nd) use = nd;
  if (use < 1) use = 1;
  t_pending = nullptr;
  if (use == 1) {
    Ctx& c = g_ctx[devs[nd > 1 ? g_rr.fetch_add(1) % (unsigned)nd : 0]];
    std::lock_guard<std::mutex> lk(c.mu);
    CK(cudaSetDevice(c.device));
    c.timing = eb200_timing{};
    int rc = fn(c, (size_t)0, n);
    t_timing = c.timing;
    return rc;
  }
  int rcs[MAX_DEV];
  eb200_timing tms[MAX_DEV];
  char errs[MAX_DEV][256];
  std::thread th[MAX_DEV];
  size_t per = ((n + use - 1) / use + 127) & ~(size_t)127;
  for (int k = 0; k < use; k++) {
    size_t lo = (size_t)k * per, m = lo >= n ? 0 : (lo + per <= n ? per : n - lo);
    th[k] = std::thread([&, k, lo, m] {
      errs[k][0] = 0;
      rcs[k] = EB200_OK;
      tms[k] = eb200_timing{};
      if (!m) return;
      Ctx& c = g_ctx[devs[k]];
      std::lock_guard<std::mutex> lk(c.mu);
      cudaError_t e = cudaSetDevice(c.device);
      if (e != cudaSuccess) { rcs[k] = cuda_fail(e, "cudaSetDevice"); }
      else { c.timing = eb200_timing{}; rcs[k] = fn(c, lo, m); tms[k] = c.timing; }
      if (rcs[k]) snprintf(errs[k], sizeof errs[k], "device %d: %s", c.device, g_err);
    });
  }
  int rc = EB200_OK;
  eb200_timing tm = {};
  for (int k = 0; k < use; k++) {
    th[k].join();
    if (rcs[k] && !rc) { rc = rcs[k]; snprintf(g_err, sizeof g_err, "%s", errs[k]); }
    merge_timing(tm, tms[k]);
  }
  t_timing = tm;
  return rc;
}

template <class F>
int run_sharded(size_t n, F&& fn) {
  int devs[MAX_DEV], nd;
  { std::lock_guard<std::mutex> lk(g_mu); nd = g_ndev; for (int i = 0; i < nd; i++) devs[i] = g_devs[i]; }
  return run_sharded_on(devs, nd, n, fn);
}

// Item i's range [off[i], off[i + 1]) of a variable-length input: not decreasing, and empty when the input is NULL.
bool range_ok(const uint8_t* bytes, const uint64_t* off, size_t i) { return off[i + 1] >= off[i] && (bytes || !off[i + 1]); }
// An address the staging copies can take for an input that is NULL because it is empty.
const uint8_t* or_empty(const uint8_t* bytes) {
  static const uint8_t none = 0;
  return bytes ? bytes : &none;
}
constexpr auto every_item = [](size_t) { return true; };

// The checks of an unkeyed host call, in order: a device, `supported` (the curve and public-key format; true for the
// 25519 calls), n = 0, ptrs_ok, `unaccelerated` (a curve the call refuses after its pointer checks), item_ok(i) for
// every item.  Then fn(c, lo, m) over the initialised devices (run_sharded).
template <class ItemOk, class Fn>
int host_run(bool supported, size_t n, bool ptrs_ok, ItemOk&& item_ok, Fn&& fn, bool unaccelerated = false) {
  if (!eb200_device_count()) return EB200_ERR_NOT_INIT;
  if (!supported) return EB200_ERR_UNSUPPORTED;
  if (n == 0) return EB200_OK;
  if (!ptrs_ok) return EB200_ERR_ARG;
  if (unaccelerated) return EB200_ERR_UNSUPPORTED;
  for (size_t i = 0; i < n; i++) if (!item_ok(i)) return EB200_ERR_ARG;
  return run_sharded(n, fn);
}

// A device -> host copy; rows > 1: `rows` rows of `bytes`, `pitch` bytes apart on the device, packed on the host.
// A NULL destination (an output the caller did not ask for) is skipped.
struct OutSeg { void* dst; const void* src; size_t bytes; size_t rows = 1, pitch = 0; };
struct Wipe { void* dst; size_t bytes; };

// Single-stream host call on c.stream: the inputs go up, run(L) launches the kernels, the outputs come home, and
// the device ranges in `wipe` (private keys, nonces) are cleared before the call returns.  kernel_ms covers the
// kernels only; main_kernel_ms is the same span when main_is_total, else the MAIN_BEGIN..MAIN_END events run records.
template <class Run>
int run_single(Ctx& c, std::initializer_list<Seg> in, Run&& run, std::initializer_list<OutSeg> out,
               std::initializer_list<Wipe> wipe, bool main_is_total) {
  cudaStream_t st = c.stream;
  Launch L{st};
  int rc;
  CK(cudaEventRecord(c.ev[EV_START], st));
  if ((rc = h2d(c, in.begin(), (int)in.size(), st))) return rc;
  CK(cudaEventRecord(c.ev[EV_INPUTS_RESIDENT], st));
  if ((rc = run(L)) || (rc = L.rc)) return rc;
  CK(cudaEventRecord(c.ev[EV_KERNELS_DONE], st));
  for (const OutSeg& o : out) {
    if (!o.dst || !o.bytes) continue;
    if (o.rows > 1) CK(cudaMemcpy2DAsync(o.dst, o.bytes, o.src, o.pitch, o.bytes, o.rows, cudaMemcpyDeviceToHost, st));
    else CK(cudaMemcpyAsync(o.dst, o.src, o.bytes, cudaMemcpyDeviceToHost, st));
  }
  for (const Wipe& w : wipe) if (w.bytes) CK(cudaMemsetAsync(w.dst, 0, w.bytes, st));
  CK(cudaEventRecord(c.ev[EV_OUTPUTS_HOME], st));
  CK(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&c.timing.h2d_ms, c.ev[EV_START], c.ev[EV_INPUTS_RESIDENT]);
  cudaEventElapsedTime(&c.timing.kernel_ms, c.ev[EV_INPUTS_RESIDENT], c.ev[EV_KERNELS_DONE]);
  cudaEventElapsedTime(&c.timing.d2h_ms, c.ev[EV_KERNELS_DONE], c.ev[EV_OUTPUTS_HOME]);
  if (main_is_total) c.timing.main_kernel_ms = c.timing.kernel_ms;
  else cudaEventElapsedTime(&c.timing.main_kernel_ms, c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
  c.timing.launches = L.count;
  return EB200_OK;
}

// Two-stream chunk pipeline of the fixed-stride host calls: chunk k's inputs go up on the copy stream, its kernels
// run on stream (k & 1) (so the grid tail of one chunk is filled by the next), its outputs come home on the copy
// stream behind them.  in(lo, m, seg) / out(lo, m, seg) fill up to 8 segments (out: dst = host, src = device);
// run(lo, m, L, slot, k) launches the kernels through L and records ev_k0[k] / ev_k1[k] around the main one.
// kernel_ms is the whole call on the GPU timeline; main_kernel_ms the span of the main kernels.
template <class In, class Run, class Out>
int run_chunked(Ctx& c, const ChunkPlan& P, In&& in, Run&& run, Out&& out) {
  int rc;
  cudaStream_t cs = c.copy_stream;
  unsigned launches = 0;
  CK(cudaEventRecord(c.ev[EV_START], cs));
  int used = 0;
  for (int k = 0; k < P.chunks; k++) {
    size_t lo = P.lo[k];
    size_t m = P.lo[k + 1] - lo;
    used = k + 1;
    Seg seg[8];
    int cnt = in(lo, m, seg);
    if ((rc = h2d(c, seg, cnt, cs))) return rc;
    CK(cudaEventRecord(c.ev_in[k], cs));
    Launch L{(k & 1) ? c.stream2 : c.stream};
    CK(cudaStreamWaitEvent(L.st, c.ev_in[k], 0));
    if ((rc = run(lo, m, L, k & 1, k)) || (rc = L.rc)) return rc;
    launches += L.count;
    CK(cudaEventRecord(c.ev_done[k], L.st));
  }
  for (int k = 0; k < used; k++) {
    size_t lo = P.lo[k];
    size_t m = P.lo[k + 1] - lo;
    CK(cudaStreamWaitEvent(cs, c.ev_done[k], 0));
    Seg seg[8];
    int cnt = out(lo, m, seg);
    for (int j = 0; j < cnt; j++)
      if (seg[j].dst && seg[j].bytes) CK(cudaMemcpyAsync(seg[j].dst, seg[j].src, seg[j].bytes, cudaMemcpyDeviceToHost, cs));
  }
  CK(cudaEventRecord(c.ev[EV_OUTPUTS_HOME], cs));
  CK(cudaStreamSynchronize(cs));
  CK(cudaStreamSynchronize(c.stream));
  CK(cudaStreamSynchronize(c.stream2));
  float total = 0, t = 0;
  cudaEventElapsedTime(&total, c.ev[EV_START], c.ev[EV_OUTPUTS_HOME]);
  cudaEventElapsedTime(&c.timing.h2d_ms, c.ev[EV_START], c.ev_in[used - 1]);       // all inputs resident
  for (int k = 0; k < used; k++) {       // chunks overlap on two streams: report the span of the main kernels
    cudaEventElapsedTime(&t, c.ev_k0[0], c.ev_k1[k]);
    if (t > c.timing.main_kernel_ms) c.timing.main_kernel_ms = t;
  }
  cudaEventElapsedTime(&t, c.ev_done[used - 1], c.ev[EV_OUTPUTS_HOME]);
  c.timing.d2h_ms = t;                                                              // exposed tail copy
  c.timing.kernel_ms = total;
  c.timing.launches = launches;
  return EB200_OK;
}

// Device-pointer call on the context that owns d_status (and the fixed-base table of `table_curve`, 0 = none): the
// kernels go on the caller's stream between the INPUTS_RESIDENT and KERNELS_DONE events, which
// eb200_last_timing() reads once the caller has synchronised that stream.
template <class Run>
int run_dev(const void* d_status, int table_curve, void* stream, Run&& run) {
  Ctx* cp = ctx_of(d_status);
  if (!cp) return EB200_ERR_NOT_INIT;
  Ctx& c = *cp;
  std::lock_guard<std::mutex> lk(c.mu);
  CK(cudaSetDevice(c.device));
  int rc;
  if (table_curve && (rc = ensure_table(c, table_curve))) return rc;
  Launch L{(cudaStream_t)stream};   // NULL is the CUDA default stream, as everywhere in CUDA
  CK(cudaEventRecord(c.ev[EV_INPUTS_RESIDENT], L.st));
  if ((rc = run(c, L)) || (rc = L.rc)) return rc;
  CK(cudaEventRecord(c.ev[EV_KERNELS_DONE], L.st));
  t_pending = &c;
  t_pending_launches = L.count;
  return EB200_OK;
}
}  // namespace

static void keysets_release_all();     // key sets (end of this file): eb200_shutdown frees their device memory

extern "C" {

const char* eb200_strerror(int code) {
  switch (code) {
    case EB200_OK: return "ok";
    case EB200_ERR_NO_DEVICE: return "no CUDA device available (this library has no CPU fallback)";
    case EB200_ERR_CUDA: return "CUDA error (see eb200_last_error)";
    case EB200_ERR_ARG: return "invalid argument";
    case EB200_ERR_NOT_INIT: return "eb200_init has not been called (or not for the device that owns these pointers)";
    case EB200_ERR_UNSUPPORTED: return "curve or format not supported by this build";
    default: return "unknown error";
  }
}

const char* eb200_last_error(void) { return g_err; }

int eb200_init(const int* devices, int ndev, uint32_t flags) {
  std::lock_guard<std::mutex> lk(g_mu);
  int cnt = 0;
  cudaError_t e = cudaGetDeviceCount(&cnt);
  if (e != cudaSuccess) { cuda_fail(e, "cudaGetDeviceCount"); return EB200_ERR_NO_DEVICE; }
  if (cnt == 0) { snprintf(g_err, sizeof g_err, "no CUDA devices"); return EB200_ERR_NO_DEVICE; }
  int all[MAX_DEV];
  if (!devices || ndev <= 0) {                       // NULL / 0: every visible device
    ndev = cnt < MAX_DEV ? cnt : MAX_DEV;
    for (int i = 0; i < ndev; i++) all[i] = i;
    devices = all;
  }
  if (ndev > MAX_DEV) return EB200_ERR_ARG;
  for (int i = 0; i < ndev; i++) if (devices[i] < 0 || devices[i] >= cnt || devices[i] >= MAX_DEV) return EB200_ERR_ARG;
  for (int i = 0; i < ndev; i++) {
    Ctx& c = g_ctx[devices[i]];
    std::lock_guard<std::mutex> lc(c.mu);
    if (!c.ready) {
      int rc = ctx_create(c, devices[i]);
      if (rc) { ctx_destroy(c); return rc; }
      g_devs[g_ndev++] = devices[i];
    }
    CK(cudaSetDevice(c.device));
    // the headline curve's table is built eagerly; the others on first use (or now, with EB200_INIT_ALL_TABLES)
    int rc = ensure_table(c, EB200_CURVE_SECP256K1);
    if (!rc && (flags & EB200_INIT_ALL_TABLES))
      for (int cv = EB200_CURVE_P256; cv <= EB200_CURVE_P224 && !rc; cv++)
        if (cv != EB200_CURVE_CURVE25519) rc = ensure_table(c, cv);
    if (rc) return rc;
  }
  return EB200_OK;
}

int eb200_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  keysets_release_all();
  for (int i = 0; i < g_ndev; i++) {
    Ctx& c = g_ctx[g_devs[i]];
    std::lock_guard<std::mutex> lc(c.mu);
    ctx_destroy(c);
  }
  g_ndev = 0;
  t_pending = nullptr;
  return EB200_OK;
}

int eb200_device_count(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  return g_ndev;
}

int eb200_last_timing(eb200_timing* out) {
  if (!out) return EB200_ERR_ARG;
  if (t_pending) {
    // device-pointer call made by this thread: the caller has synchronised its stream by now
    Ctx& c = *t_pending;
    std::lock_guard<std::mutex> lk(c.mu);
    t_timing = eb200_timing{};
    if (cudaEventElapsedTime(&t_timing.kernel_ms, c.ev[EV_INPUTS_RESIDENT], c.ev[EV_KERNELS_DONE]) != cudaSuccess)
      return EB200_ERR_CUDA;
    if (cudaEventElapsedTime(&t_timing.main_kernel_ms, c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]) != cudaSuccess)
      return EB200_ERR_CUDA;
    t_timing.launches = t_pending_launches;
    t_pending = nullptr;
  }
  *out = t_timing;
  return EB200_OK;
}

size_t eb200_ecdsa_verify_workspace_bytes(int curve, size_t n) {
  if (!curve_ok(curve)) return 0;
  return ws_layout(curve, n).total;
}

int eb200_ecdsa_verify_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r,
                                 const uint8_t* d_s, const uint8_t* d_pub, uint32_t pub_fmt,
                                 uint8_t* d_status, void* d_workspace, void* stream) {
  if (!curve_ok(curve) || !fmt_ok(pub_fmt)) return EB200_ERR_UNSUPPORTED;
  if (n == 0) return eb200_device_count() ? EB200_OK : EB200_ERR_NOT_INIT;
  if (!d_e || !d_r || !d_s || !d_pub || !d_status || !d_workspace) return EB200_ERR_ARG;
  return run_dev(d_status, curve, stream, [&](Ctx& c, Launch& L) {
    return launch_verify(c, curve, n, d_e, d_r, d_s, d_pub, pub_fmt, d_status, (uint8_t*)d_workspace, L,
                         c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
  });
}
}  // extern "C"

// Host-pointer verify on one device.  Large batches are cut into chunks: chunk k+1 is copied host->device on a
// copy stream while chunk k is being verified, and results stream back as each chunk finishes.
// chunk boundaries: chunk_plan.h (make_plan), unit-tested on the CPU through tests/hostemu
static int verify_on(Ctx& c, int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s, const uint8_t* pub,
                     uint32_t pub_fmt, uint8_t* status) {
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  const size_t len = curve_len(curve), pb = pub_item_bytes(len, pub_fmt);
  const ChunkPlan P = make_plan(n);
  if ((rc = grow(&c.d_in, &c.d_in_cap, align256(n * (3 * len + pb)) + 1024))) return rc;
  // two chunks in flight (alternating compute streams, so the grid tail of chunk k is filled by chunk k+1)
  const size_t ws_slot = ws_layout(curve, P.max_m).total;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (P.chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *d_e = c.d_in, *d_r = d_e + n * len, *d_s = d_r + n * len, *d_pub = d_s + n * len;
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {d_e + lo * len, e + lo * len, m * len};
      seg[1] = {d_r + lo * len, r + lo * len, m * len};
      seg[2] = {d_s + lo * len, s + lo * len, m * len};
      seg[3] = {d_pub + lo * pb, pub + lo * pb, m * pb};
      return 4;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      return launch_verify(c, curve, m, d_e + lo * len, d_r + lo * len, d_s + lo * len, d_pub + lo * pb, pub_fmt,
                           c.d_status + lo, c.d_ws + (size_t)slot * ws_slot, L, c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {status + lo, c.d_status + lo, m};
      return 1;
    });
}

// DER-encoded signatures, parsed on the GPU (variable length: concatenated bytes + offsets; sig_off points at
// this block's first offset, all offsets are absolute into `sigs`)
static int verify_der_on(Ctx& c, int curve, size_t n, const uint8_t* e, const uint8_t* sigs, const uint64_t* sig_off,
                         const uint8_t* pub, uint32_t pub_fmt, uint8_t* status) {
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  const size_t len = curve_len(curve), pb = pub_item_bytes(len, pub_fmt);
  const size_t sig_bytes = (size_t)(sig_off[n] - sig_off[0]);
  const size_t off_bytes = align256((n + 1) * 8);
  if ((rc = grow(&c.d_in, &c.d_in_cap, off_bytes + align256(n * (3 * len + pb)) + align256(sig_bytes) + 1024))) return rc;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, ws_layout(curve, n).total))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  unsigned long long* d_off = (unsigned long long*)c.d_in;
  uint8_t* d_e = c.d_in + off_bytes;
  uint8_t* d_r = d_e + n * len;
  uint8_t* d_s = d_r + n * len;
  uint8_t* d_pub = d_s + n * len;
  uint8_t* d_sig = d_pub + align256(n * pb);
  return run_single(c, {{d_off, sig_off, (n + 1) * 8}, {d_e, e, n * len}, {d_pub, pub, n * pb}, {d_sig, sigs + sig_off[0], sig_bytes}},
    [&](Launch& L) {     // offsets are used relative to sig_off[0] on the device
      return launch_verify(c, curve, n, d_e, d_r, d_s, d_pub, pub_fmt, c.d_status, c.d_ws, L, c.ev[EV_MAIN_BEGIN],
                           c.ev[EV_MAIN_END], d_sig - sig_off[0], d_off);
    },
    {{status, c.d_status, n}}, {}, false);
}

extern "C" {

int eb200_ecdsa_verify_batch(int curve, size_t n, const uint8_t* e, const uint8_t* r,
                             const uint8_t* s, const uint8_t* pub, uint32_t pub_fmt,
                             uint8_t* status) {
  const size_t len = curve_len(curve), pb = pub_item_bytes(len, pub_fmt);
  return host_run(curve_ok(curve) && fmt_ok(pub_fmt), n, e && r && s && pub && status, every_item, [&](Ctx& c, size_t lo, size_t m) {
    return verify_on(c, curve, m, e + lo * len, r + lo * len, s + lo * len, pub + lo * pb, pub_fmt, status + lo);
  });
}

int eb200_ecdsa_verify_batch_der(int curve, size_t n, const uint8_t* e, const uint8_t* sigs, const uint64_t* sig_off,
                                 const uint8_t* pub, uint32_t pub_fmt, uint8_t* status) {
  const size_t len = curve_len(curve), pb = pub_item_bytes(len, pub_fmt);
  return host_run(curve_ok(curve) && fmt_ok(pub_fmt), n, e && sigs && sig_off && pub && status,
    [&](size_t i) { return range_ok(sigs, sig_off, i); },
    [&](Ctx& c, size_t lo, size_t m) {
      return verify_der_on(c, curve, m, e + lo * len, sigs, sig_off + lo, pub + lo * pb, pub_fmt, status + lo);
    });
}

// ---- ECDSA public-key recovery ------------------------------------------------------------
}  // extern "C"

// The launches of one recoverPubKey block whose inputs are on the device: prep, then the recovery kernel between ev0 and
// ev1.  base: ws_layout(curve, n).total bytes of workspace.
static int recover_launches(Ctx& c, int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r, const uint8_t* d_s,
                            const uint8_t* d_id, uint8_t* base, uint8_t* d_out, uint8_t* d_status, Launch& L, cudaEvent_t ev0,
                            cudaEvent_t ev1) {
  const WsLayout W = ws_layout(curve, n);
  u32 *ws = (u32*)(base + W.ws), *qtab = (u32*)(base + W.qtab);
  return with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    if constexpr (is_ed25519<T>) return EB200_ERR_UNSUPPORTED;     // the entry points refuse it first
    else {
      if constexpr (is_k256<T>) {
        L(k256_prep_recover_kernel, batch_blocks(n, PREP_BATCH), 128, n, d_e, d_r, d_s, ws, (u32*)(base + W.scratch));
        CK(cudaEventRecord(ev0, L.st));
        L(k256_recover_kernel, (unsigned)((n + EB_VERIFY_BLOCK - 1) / EB_VERIFY_BLOCK), EB_VERIFY_BLOCK, n, d_r, d_id, ws,
          c.gtab[curve], qtab, d_out, d_status);
      } else {
        L(sw_prep_recover_kernel<typename T::C>, blocks128(n), 128, n, d_e, d_r, d_s, ws);
        CK(cudaEventRecord(ev0, L.st));
        L(sw_recover_kernel<typename T::C>, blocks128(n), 128, n, d_r, d_id, ws, c.gtab[curve], qtab, d_out, d_status);
      }
      CK(cudaEventRecord(ev1, L.st));
      return EB200_OK;
    }
  });
}

static int recover_on(Ctx& c, int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                      const uint8_t* recid, uint8_t* out_xy, uint8_t* status) {
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  const size_t len = curve_len(curve);
  const WsLayout W = ws_layout(curve, n);
  if ((rc = grow(&c.d_in, &c.d_in_cap, n * (5 * len + 1) + 256))) return rc;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, W.total))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *d_e = c.d_in, *d_r = d_e + len * n, *d_s = d_r + len * n, *d_out = d_s + len * n, *d_id = d_out + 2 * len * n;
  return run_single(c, {{d_e, e, len * n}, {d_r, r, len * n}, {d_s, s, len * n}, {d_id, recid, n}},
    [&](Launch& L) {
      return recover_launches(c, curve, n, d_e, d_r, d_s, d_id, c.d_ws, d_out, c.d_status, L, c.ev[EV_MAIN_BEGIN],
                              c.ev[EV_MAIN_END]);
    },
    {{out_xy, d_out, 2 * len * n}, {status, c.d_status, n}}, {}, false);
}

// The launches of one mul / mulAdd / derive block whose inputs are on the device (dk1 == NULL: no base-point term;
// d_pts == NULL: k2 G): the main kernel between ev0 and ev1, with the scalar prep in front of it and the replay (derive:
// the status map) behind it for an arbitrary point.  Writes x || y to d_out also for derive.  base: ws_layout(curve,
// n).total bytes of workspace, of which the scalar prep's digit words and the per-item tables are used.
static int mul_add_launches(Ctx& c, int curve, size_t n, const uint8_t* dk1, const uint8_t* d_k2, const uint8_t* d_pts,
                            uint8_t* base, uint8_t* d_out, uint8_t* d_status, bool derive, Launch& L, cudaEvent_t ev0,
                            cudaEvent_t ev1) {
  const WsLayout W = ws_layout(curve, n);
  u32 *ws = (u32*)(base + W.ws), *qtab = (u32*)(base + W.qtab);
  const unsigned nb = blocks128(n);
  return with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    const u32* gt = c.gtab[curve];
    if constexpr (is_ed25519<T>) {
      CK(cudaEventRecord(ev0, L.st));
      L(ed_ec_mul_add_kernel, nb, 128, n, dk1, d_k2, d_pts, derive ? 1u : 0u, gt, qtab, d_out, d_status);
      CK(cudaEventRecord(ev1, L.st));
    } else if (!d_pts) {
      CK(cudaEventRecord(ev0, L.st));
      if constexpr (is_k256<T>) L(k256_mul_g_kernel, nb, 128, n, d_k2, gt, d_out, d_status);
      else L(sw_mul_g_kernel<typename T::C>, nb, 128, n, d_k2, gt, d_out, d_status);
      CK(cudaEventRecord(ev1, L.st));
    } else {
      if constexpr (is_k256<T>) {
        L(k256_prep_scalars_kernel, nb, 128, n, dk1, d_k2, ws);
        CK(cudaEventRecord(ev0, L.st));
        L(k256_mul_add_kernel, (unsigned)((n + EB_VERIFY_BLOCK - 1) / EB_VERIFY_BLOCK), EB_VERIFY_BLOCK, n, d_pts, ws, gt,
          qtab, d_out, d_status);
      } else {
        L(sw_prep_scalars_kernel<typename T::C>, nb, 128, n, dk1, d_k2, ws);
        CK(cudaEventRecord(ev0, L.st));
        L(sw_mul_add_kernel<typename T::C>, nb, 128, n, d_pts, ws, gt, qtab, d_out, d_status);
      }
      CK(cudaEventRecord(ev1, L.st));
      if (derive) L(status_map_kernel, nb, 128, n, d_status, (uint8_t)ST_NEEDS_HOST, (uint8_t)ST_THROW_NOT_VALIDATED);
      else if constexpr (is_k256<T>) L(k256_mul_add_replay_kernel, nb, 128, n, dk1, d_k2, d_pts, c.replay_tab, d_out, d_status);
      else L(sw_mul_add_replay_kernel<typename T::C>, nb, 128, n, dk1, d_k2, d_pts, c.sw_replay_tab[curve], d_out, d_status);
    }
    return EB200_OK;
  });
}

// ---- Point.mul / Point.mulAdd batches ---------------------------------------------------------------
// k1 == NULL: k2*P;  pts == NULL: k2*G;  both given: k1*G + k2*P.
// derive: KeyPair.derive (ec/key.js:102-107) -- an off-curve point is the reference's
// 'public point not validated' throw instead of a replayed multiplication, and only x is returned.
static int mul_add_on(Ctx& c, int curve, size_t n, const uint8_t* k1, const uint8_t* k2, const uint8_t* pts,
                      uint8_t* out_xy, uint8_t* status, bool derive) {
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  const size_t len = curve_len(curve);
  const WsLayout W = ws_layout(curve, n);
  if ((rc = grow(&c.d_in, &c.d_in_cap, n * 6 * len + 256))) return rc;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, W.total))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *d_k1 = c.d_in, *d_k2 = d_k1 + len * n, *d_pts = d_k2 + len * n, *d_out = d_pts + 2 * len * n;
  return run_single(c, {{d_k1, k1, k1 ? len * n : 0}, {d_k2, k2, len * n}, {d_pts, pts, pts ? 2 * len * n : 0}},
    [&](Launch& L) {
      return mul_add_launches(c, curve, n, k1 ? d_k1 : nullptr, d_k2, pts ? d_pts : nullptr, c.d_ws, d_out, c.d_status, derive,
                              L, c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
    },
    // derive: x only; its scalars are private keys, which do not stay in the shared staging buffer
    {{out_xy, d_out, derive ? len : 2 * len * n, derive ? n : 1, 2 * len}, {status, c.d_status, n}},
    {{d_k2, derive ? len * n : 0}}, false);
}

static int mul_add_common(int curve, size_t n, const uint8_t* k1, const uint8_t* k2, const uint8_t* pts,
                          uint8_t* out_xy, uint8_t* status, bool derive = false) {
  const size_t len = curve_len(curve), ol = derive ? len : 2 * len;
  return host_run(curve_ok(curve), n, k2 && out_xy && status && (!k1 || pts), every_item, [&](Ctx& c, size_t lo, size_t m) {
    return mul_add_on(c, curve, m, k1 ? k1 + lo * len : nullptr, k2 + lo * len, pts ? pts + lo * 2 * len : nullptr,
                      out_xy + lo * ol, status + lo, derive);
  });
}

// ---- ECDSA sign (RFC 6979 nonces on the GPU) ---------------------------------------------------------
// Workspace of one sign block of n items: the nonce kernel's X, Y, Z and k words | the finish kernel's inversion scratch.
struct SignWs { size_t scr, total; };
static SignWs sign_ws(int curve, size_t n) {
  const size_t limbs = fe_len(curve) / 4;
  SignWs W;
  W.scr = align256(4 * limbs * 4 * n);                                // X, Y, Z, k
  W.total = W.scr + 2 * limbs * 4 * n;
  return W;
}

// The launches of one sign block whose inputs are on the device.  mode: kg != NULL -> the caller's nonces, one attempt
// (items the reference would `continue` on come back as EB200_ST_RETRY); pp != NULL -> the literal loop on the
// byte-stream DRBG (np bytes of pers; np = 0: none read); neither -> RFC 6979 fast pipeline.  The first kernel (the
// nonce kernel, or the whole loop) runs between ev0 and ev1.  base: sign_ws(curve, n).total bytes of workspace, which
// then holds nonces and k G.
static int sign_launches(Ctx& c, int curve, size_t n, const uint8_t* d_e, const uint8_t* d_k, const uint8_t* kg,
                         const uint8_t* pp, size_t np, u32 canonical, uint8_t* base, uint8_t* d_r, uint8_t* d_s, uint8_t* d_id,
                         uint8_t* d_status, Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  u32 *d_sws = (u32*)base, *d_scr = (u32*)(base + sign_ws(curve, n).scr);
  const unsigned nb = blocks128(n);
  return with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    const u32* gt = c.gtab[curve];
    CK(cudaEventRecord(ev0, L.st));
    if constexpr (is_ed25519<T>) {
      L(ed_ec_sign_kernel, nb, 128, n, d_e, d_k, kg, pp, (u32)np, canonical, gt, d_r, d_s, d_id, d_status);
      CK(cudaEventRecord(ev1, L.st));
    } else if constexpr (is_k256<T>) {
      if (pp) {
        L(k256_sign_pers_kernel, nb, 128, n, d_e, d_k, pp, (u32)np, canonical, gt, d_r, d_s, d_id, d_status);
        CK(cudaEventRecord(ev1, L.st));
      } else {
        L(k256_sign_nonce_kernel, nb, 128, n, d_e, d_k, gt, d_sws, d_status, kg);
        CK(cudaEventRecord(ev1, L.st));
        L(k256_sign_finish_kernel, batch_blocks(n, PREP_BATCH), 128, n, d_e, d_k, canonical, d_sws, d_scr, d_r, d_s, d_id, d_status);
        if (kg) L(status_map_kernel, nb, 128, n, d_status, (uint8_t)ST_NEEDS_HOST, (uint8_t)EB200_ST_RETRY);
        else L(k256_sign_slow_kernel, nb, 128, n, d_e, d_k, canonical, gt, d_r, d_s, d_id, d_status);
      }
    } else {
      typedef typename T::SG SG;
      if (pp) {
        L(sw_sign_pers_kernel<SG>, nb, 128, n, d_e, d_k, pp, (u32)np, canonical, gt, d_r, d_s, d_id, d_status);
        CK(cudaEventRecord(ev1, L.st));
      } else {
        L(sw_sign_nonce_kernel<SG>, nb, 128, n, d_e, d_k, gt, d_sws, d_status, kg);
        CK(cudaEventRecord(ev1, L.st));
        L(sw_sign_finish_kernel<SG>, batch_blocks(n, SG::BATCH), 128, n, d_e, d_k, canonical, d_sws, d_scr, d_r, d_s, d_id, d_status);
        if (kg) L(status_map_kernel, nb, 128, n, d_status, (uint8_t)ST_NEEDS_HOST, (uint8_t)EB200_ST_RETRY);
        else L(sw_sign_slow_kernel<SG>, nb, 128, n, d_e, d_k, canonical, gt, d_r, d_s, d_id, d_status);
      }
    }
    return EB200_OK;
  });
}

static int sign_on(Ctx& c, int curve, size_t n, const uint8_t* e, const uint8_t* priv, uint32_t flags,
                   uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid, uint8_t* status,
                   const uint8_t* kgiven = nullptr, const uint8_t* pers = nullptr, size_t np = 0) {
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  const size_t len = curve_len(curve);
  if ((rc = grow(&c.d_in, &c.d_in_cap, n * (5 * len + 1) + align256(np + 1) + 512))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  const SignWs W = sign_ws(curve, n);
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, W.total))) return rc;
  uint8_t *d_e = c.d_in, *d_k = d_e + len * n, *d_r = d_k + len * n, *d_s = d_r + len * n, *d_kg = d_s + len * n, *d_id = d_kg + len * n;
  uint8_t* d_pers = (uint8_t*)(((uintptr_t)(d_id + n) + 255) & ~(uintptr_t)255);
  const u32 canonical = flags & EB200_SIGN_CANONICAL;
  const uint8_t* kg = kgiven ? d_kg : nullptr;
  const uint8_t* pp = pers ? d_pers : nullptr;
  return run_single(c, {{d_e, e, len * n}, {d_k, priv, len * n}, {d_kg, kgiven, kgiven ? len * n : 0}, {d_pers, pers, pers ? np : 0}},
    [&](Launch& L) {
      return sign_launches(c, curve, n, d_e, d_k, kg, pp, np, canonical, c.d_ws, d_r, d_s, d_id, c.d_status, L,
                           c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
    },
    {{out_r, d_r, len * n}, {out_s, d_s, len * n}, {out_recid, d_id, n}, {status, c.d_status, n}},
    // private keys, nonces k and k*G live in buffers that later calls reuse: wipe them before returning
    {{d_k, len * n}, {d_kg, kgiven ? len * n : 0}, {c.d_ws, W.total}}, true);
}

// The launches of one genKeyPair block whose inputs are on the device: the keygen kernel (private keys to d_priv, its
// verdicts to d_status) between ev0 and ev1, then k G to d_pub with the multiplication's statuses in mul_status.
static int keygen_launches(Ctx& c, int curve, size_t n, const uint8_t* d_ent, size_t ne, const uint8_t* pp, size_t np,
                           uint8_t* d_priv, uint8_t* d_pub, uint8_t* d_status, uint8_t* mul_status, Launch& L, cudaEvent_t ev0,
                           cudaEvent_t ev1) {
  const unsigned nb = blocks128(n);
  return with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    const u32* gt = c.gtab[curve];
    CK(cudaEventRecord(ev0, L.st));
    if constexpr (is_k256<T>) L(k256_keygen_kernel, nb, 128, n, d_ent, (u32)ne, pp, (u32)np, d_priv, d_status);
    else if constexpr (is_ed25519<T>) L(ed_ec_keygen_kernel, nb, 128, n, d_ent, (u32)ne, pp, (u32)np, d_priv, d_status);
    else L(sw_keygen_kernel<typename T::SG>, nb, 128, n, d_ent, (u32)ne, pp, (u32)np, d_priv, d_status);
    CK(cudaEventRecord(ev1, L.st));
    if constexpr (is_k256<T>) L(k256_mul_g_kernel, nb, 128, n, d_priv, gt, d_pub, mul_status);
    else if constexpr (is_ed25519<T>) L(ed_ec_mul_add_kernel, nb, 128, n, nullptr, d_priv, nullptr, 0u, gt, nullptr, d_pub, mul_status);
    else L(sw_mul_g_kernel<typename T::C>, nb, 128, n, d_priv, gt, d_pub, mul_status);
    return EB200_OK;
  });
}

// EC.genKeyPair({entropy, pers}) (ec/index.js:55-79): private keys from HMAC-DRBG(entropy_i, nonce = n, pers), then
// the public points k*G.  entropy: n x ne bytes.
static int keygen_on(Ctx& c, int curve, size_t n, const uint8_t* entropy, size_t ne, const uint8_t* pers, size_t np,
                     uint8_t* out_priv, uint8_t* out_pub, uint8_t* status) {
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  const size_t len = curve_len(curve);
  if ((rc = grow(&c.d_in, &c.d_in_cap, align256(n * ne) + align256(np + 1) + n * 3 * len + n + 512))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t* d_ent = c.d_in;
  uint8_t* d_pers = d_ent + align256(n * ne);
  uint8_t* d_priv = d_pers + align256(np + 1);
  uint8_t* d_pub = d_priv + len * n;
  uint8_t* d_mst = d_pub + 2 * len * n;               // the multiplication's statuses (not returned)
  const uint8_t* pp = pers ? d_pers : nullptr;
  return run_single(c, {{d_ent, entropy, n * ne}, {d_pers, pers, pers ? np : 0}},
    [&](Launch& L) {
      return keygen_launches(c, curve, n, d_ent, ne, pp, np, d_priv, d_pub, c.d_status, d_mst, L, c.ev[EV_MAIN_BEGIN],
                             c.ev[EV_MAIN_END]);
    },
    {{out_priv, d_priv, len * n}, {out_pub, d_pub, 2 * len * n}, {status, c.d_status, n}},
    {{d_ent, n * ne}, {d_priv, len * n}}, true);
}

extern "C" {

int eb200_ecdsa_recover_batch(int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                              const uint8_t* recid, uint8_t* out_xy, uint8_t* status) {
  const size_t len = curve_len(curve);
  return host_run(curve_ok(curve), n, e && r && s && recid && out_xy && status, every_item, [&](Ctx& c, size_t lo, size_t m) {
    return recover_on(c, curve, m, e + lo * len, r + lo * len, s + lo * len, recid + lo, out_xy + lo * 2 * len, status + lo);
  }, curve == EB200_CURVE_ED25519);      // recoverPubKey over the Edwards preset is not accelerated
}

int eb200_scalar_mul_batch(int curve, size_t n, const uint8_t* k, const uint8_t* points_xy, uint8_t* out_xy,
                           uint8_t* status) {
  return mul_add_common(curve, n, nullptr, k, points_xy, out_xy, status);
}

int eb200_ecdh_derive_batch(int curve, size_t n, const uint8_t* priv, const uint8_t* pub_xy, uint8_t* out_x,
                            uint8_t* status) {
  if (n && !pub_xy) return EB200_ERR_ARG;
  return mul_add_common(curve, n, nullptr, priv, pub_xy, out_x, status, true);
}

int eb200_mul_add_batch(int curve, size_t n, const uint8_t* k1, const uint8_t* k2, const uint8_t* p2_xy,
                        uint8_t* out_xy, uint8_t* status) {
  if (n && (!k1 || !p2_xy)) return EB200_ERR_ARG;
  return mul_add_common(curve, n, k1, k2, p2_xy, out_xy, status);
}

int eb200_ecdsa_sign_batch(int curve, size_t n, const uint8_t* e, const uint8_t* priv, uint32_t flags,
                           uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid, uint8_t* status) {
  const size_t len = curve_len(curve);
  return host_run(curve_ok(curve), n, e && priv && out_r && out_s && out_recid && status, every_item,
    [&](Ctx& c, size_t lo, size_t m) {
      return sign_on(c, curve, m, e + lo * len, priv + lo * len, flags, out_r + lo * len, out_s + lo * len, out_recid + lo,
                     status + lo);
    });
}

// EC.sign with options.k (ec/index.js:154-157): one attempt with the caller's nonces
int eb200_ecdsa_sign_batch_k(int curve, size_t n, const uint8_t* e, const uint8_t* priv, const uint8_t* k, uint32_t flags,
                             uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid, uint8_t* status) {
  const size_t len = curve_len(curve);
  return host_run(curve_ok(curve), n, e && priv && k && out_r && out_s && out_recid && status, every_item,
    [&](Ctx& c, size_t lo, size_t m) {
      return sign_on(c, curve, m, e + lo * len, priv + lo * len, flags, out_r + lo * len, out_s + lo * len, out_recid + lo,
                     status + lo, k + lo * len);
    });
}

// EC.sign with options.pers (ec/index.js:143-151; the bytes after persEnc decoding, shared by the batch)
int eb200_ecdsa_sign_batch_pers(int curve, size_t n, const uint8_t* e, const uint8_t* priv, const uint8_t* pers, size_t pers_len,
                                uint32_t flags, uint8_t* out_r, uint8_t* out_s, uint8_t* out_recid, uint8_t* status) {
  const uint8_t* pp = or_empty(pers_len ? pers : nullptr);
  const size_t len = curve_len(curve);
  return host_run(curve_ok(curve), n,
    e && priv && out_r && out_s && out_recid && status && (pers || !pers_len) && pers_len <= (1u << 20), every_item,
    [&](Ctx& c, size_t lo, size_t m) {
      return sign_on(c, curve, m, e + lo * len, priv + lo * len, flags, out_r + lo * len, out_s + lo * len, out_recid + lo,
                     status + lo, nullptr, pp, pers_len);
    });
}

// EC.genKeyPair({entropy, pers}) (ec/index.js:55-79)
int eb200_ec_keygen_batch(int curve, size_t n, const uint8_t* entropy, size_t entropy_len, const uint8_t* pers, size_t pers_len,
                          uint8_t* out_priv, uint8_t* out_pub_xy, uint8_t* status) {
  const size_t len = curve_len(curve);
  return host_run(curve_ok(curve), n,
    entropy && entropy_len && out_priv && status && (pers || !pers_len) && pers_len <= (1u << 20) && entropy_len <= (1u << 16),
    every_item, [&](Ctx& c, size_t lo, size_t m) {
      return keygen_on(c, curve, m, entropy + lo * entropy_len, entropy_len, pers_len ? pers : nullptr, pers_len,
                       out_priv + lo * len, out_pub_xy ? out_pub_xy + lo * 2 * len : nullptr, status + lo);
    });
}

// ---- EdDSA (ed25519) verify ---------------------------------------------------------------
size_t eb200_eddsa_verify_workspace_bytes(size_t n) { return align256((size_t)ED_ATAB_WORDS * 4 * n); }

int eb200_eddsa_verify_batch_dev(size_t n, const uint8_t* d_R, const uint8_t* d_S, const uint8_t* d_A,
                                 const uint8_t* d_h, uint8_t* d_status, void* d_workspace, void* stream) {
  if (n == 0) return eb200_device_count() ? EB200_OK : EB200_ERR_NOT_INIT;
  if (!d_R || !d_S || !d_A || !d_h || !d_status || !d_workspace) return EB200_ERR_ARG;
  return run_dev(d_status, EB200_CURVE_ED25519, stream, [&](Ctx& c, Launch& L) {
    CK(cudaEventRecord(c.ev[EV_MAIN_BEGIN], L.st));
    L(ed25519_verify_kernel, blocks128(n), 128, n, d_R, d_S, d_A, d_h, c.gtab[EB200_CURVE_ED25519], (u32*)d_workspace, d_status);
    CK(cudaEventRecord(c.ev[EV_MAIN_END], L.st));
    return EB200_OK;
  });
}
}  // extern "C"

// The launches of one EdDSA verify block whose inputs are on the device.  msg_off != NULL: h = SHA512(R || A || M) mod n
// into dh first (msg_off: n + 1 offsets relative to msgs), by the screened hash (keyset_forms.cu) when verdict != NULL;
// then the verify kernel between ev0 and ev1.  atab: eb200_eddsa_verify_workspace_bytes(n) bytes of workspace.
static int eddsa_verify_launches(Ctx& c, size_t n, const uint8_t* dR, const uint8_t* dS, const uint8_t* dA, uint8_t* dh,
                                 const uint8_t* msgs, const u64* msg_off, const uint8_t* verdict, u32* atab, uint8_t* d_status,
                                 Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  const unsigned nb = blocks128(n);
  if (msg_off && verdict) {
    if (L.rc) return L.rc;
    cudaError_t err = keyset_ed_hash_screened_launch(n, verdict, dR, dA, msgs, msg_off, dh, L.st, &L.count);
    if (err != cudaSuccess) return cuda_fail(err, "keyset_ed_hash_screened_launch");
  } else if (msg_off) {
    L(ed25519_hash_kernel, nb, 128, n, dR, dA, msgs, msg_off, dh);
  }
  CK(cudaEventRecord(ev0, L.st));
  L(ed25519_verify_kernel, nb, 128, n, dR, dS, dA, (const uint8_t*)dh, c.gtab[EB200_CURVE_ED25519], atab, d_status);
  CK(cudaEventRecord(ev1, L.st));
  return L.rc;
}

// h == NULL: raw messages (msgs + offsets; msg_off points at this block's first offset, offsets absolute), SHA-512 on the GPU
static int eddsa_on(Ctx& c, size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* A, const uint8_t* h,
                    const uint8_t* msgs, const uint64_t* msg_off, uint8_t* status) {
  int rc = ensure_table(c, EB200_CURVE_ED25519);
  if (rc) return rc;
  const ChunkPlan P = make_plan(n);
  const int chunks = P.chunks;
  const size_t per = P.max_m;
  size_t mbytes = h ? 0 : (size_t)(msg_off[n] - msg_off[0]);
  size_t off_bytes = h ? 0 : (n + 1) * sizeof(uint64_t);
  size_t base = align256(n * 128);
  const size_t ws_slot = eb200_eddsa_verify_workspace_bytes(per < n ? per : n);
  if ((rc = grow(&c.d_in, &c.d_in_cap, base + align256(off_bytes) + align256(mbytes + 1)))) return rc;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *dR = c.d_in, *dS = dR + 32 * n, *dA = dS + 32 * n, *dh = dA + 32 * n;
  uint64_t* doff = (uint64_t*)(c.d_in + base);
  uint8_t* dm = c.d_in + base + align256(off_bytes);
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {dR + 32 * lo, R + 32 * lo, 32 * m};
      seg[1] = {dS + 32 * lo, S + 32 * lo, 32 * m};
      seg[2] = {dA + 32 * lo, A + 32 * lo, 32 * m};
      if (h) { seg[3] = {dh + 32 * lo, h + 32 * lo, 32 * m}; return 4; }
      seg[3] = {doff + lo, msg_off + lo, (m + 1) * sizeof(uint64_t)};
      seg[4] = {dm + (msg_off[lo] - msg_off[0]), msgs + msg_off[lo], (size_t)(msg_off[lo + m] - msg_off[lo])};
      return 5;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      return eddsa_verify_launches(c, m, dR + 32 * lo, dS + 32 * lo, dA + 32 * lo, dh + 32 * lo, h ? nullptr : dm - msg_off[0],
                                   h ? nullptr : doff + lo, nullptr, (u32*)(c.d_ws + (size_t)slot * ws_slot), c.d_status + lo, L,
                                   c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {status + lo, c.d_status + lo, m};
      return 1;
    });
}

// The sign kernel of one EDDSA.sign block whose inputs are on the device (msg_off: n + 1 offsets relative to msgs), or its
// screened form (unkeyed_forms.cu) when verdict != NULL, between ev0 and ev1.  pub may be NULL.
static int eddsa_sign_launches(Ctx& c, size_t n, const uint8_t* dsec, const uint8_t* msgs, const u64* msg_off,
                               const uint8_t* verdict, uint8_t* dsig, uint8_t* dpub, uint8_t* d_status, Launch& L,
                               cudaEvent_t ev0, cudaEvent_t ev1) {
  const u32* gt = c.gtab[EB200_CURVE_ED25519];
  CK(cudaEventRecord(ev0, L.st));
  if (verdict) {
    if (L.rc) return L.rc;
    cudaError_t err = unkeyed_ed25519_sign_screened_launch(n, verdict, dsec, msgs, msg_off, gt, dsig, dpub, d_status, L.st,
                                                           &L.count);
    if (err != cudaSuccess) return cuda_fail(err, "unkeyed_ed25519_sign_screened_launch");
  } else {
    L(ed25519_sign_kernel, blocks128(n), 128, n, dsec, msgs, msg_off, gt, dsig, dpub, d_status);
  }
  CK(cudaEventRecord(ev1, L.st));
  return L.rc;
}

// EDDSA.sign batch: secrets n x 32, raw messages (offsets absolute, msg_off points at this block's first one)
static int eddsa_sign_on(Ctx& c, size_t n, const uint8_t* secrets, const uint8_t* msgs, const uint64_t* msg_off,
                         uint8_t* sig, uint8_t* pub, uint8_t* status) {
  int rc = ensure_table(c, EB200_CURVE_ED25519);
  if (rc) return rc;
  size_t mbytes = (size_t)(msg_off[n] - msg_off[0]);
  size_t off_bytes = (n + 1) * sizeof(uint64_t);
  size_t base = align256(n * 128);                       // secrets | sig | pub
  if ((rc = grow(&c.d_in, &c.d_in_cap, base + align256(off_bytes) + align256(mbytes + 1)))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *dsec = c.d_in, *dsig = dsec + 32 * n, *dpub = dsig + 64 * n;
  uint64_t* doff = (uint64_t*)(c.d_in + base);
  uint8_t* dm = c.d_in + base + align256(off_bytes);
  return run_single(c, {{dsec, secrets, 32 * n}, {doff, msg_off, off_bytes}, {dm, msgs + msg_off[0], mbytes}},
    [&](Launch& L) {
      return eddsa_sign_launches(c, n, dsec, dm - msg_off[0], doff, nullptr, dsig, dpub, c.d_status, L, c.ev[EV_MAIN_BEGIN],
                                 c.ev[EV_MAIN_END]);
    },
    {{sig, dsig, 64 * n}, {pub, dpub, 32 * n}, {status, c.d_status, n}},
    {{dsec, 32 * n}}, true);             // secrets do not stay in the shared buffer
}

// The curve25519 kernel of one block whose inputs are on the device, between ev0 and ev1: the ladder with MontCurve.validate
// (KeyPair.derive) or without it (Point.mul).
static int x25519_launches(size_t n, const uint8_t* dk, const uint8_t* dx, uint8_t* dout, uint8_t* d_status, bool validate,
                           Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  CK(cudaEventRecord(ev0, L.st));
  L(validate ? x25519_derive_kernel : x25519_mul_kernel, blocks128(n), 128, n, dk, dx, dout, d_status);
  CK(cudaEventRecord(ev1, L.st));
  return L.rc;
}

static int x25519_on(Ctx& c, size_t n, const uint8_t* priv, const uint8_t* pubx, uint8_t* out, uint8_t* status, bool validate) {
  int rc;
  const ChunkPlan P = make_plan(n);
  if ((rc = grow(&c.d_in, &c.d_in_cap, n * 96))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *dk = c.d_in, *dx = dk + 32 * n, *dout = dx + 32 * n;
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {dk + 32 * lo, priv + 32 * lo, 32 * m};
      seg[1] = {dx + 32 * lo, pubx + 32 * lo, 32 * m};
      return 2;
    },
    [&](size_t lo, size_t m, Launch& L, int, int k) {
      int rc2 = x25519_launches(m, dk + 32 * lo, dx + 32 * lo, dout + 32 * lo, c.d_status + lo, validate, L, c.ev_k0[k],
                                c.ev_k1[k]);
      if (rc2) return rc2;
      CK(cudaMemsetAsync(dk + 32 * lo, 0, 32 * m, L.st));   // private scalars do not stay in the shared buffer
      return EB200_OK;
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {out + 32 * lo, dout + 32 * lo, 32 * m};
      seg[1] = {status + lo, c.d_status + lo, m};
      return 2;
    });
}

extern "C" {

int eb200_eddsa_verify_batch(size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* A, const uint8_t* h,
                             uint8_t* status) {
  return host_run(true, n, R && S && A && h && status, every_item, [&](Ctx& c, size_t lo, size_t m) {
    return eddsa_on(c, m, R + 32 * lo, S + 32 * lo, A + 32 * lo, h + 32 * lo, nullptr, nullptr, status + lo);
  });
}

// EdDSA verify from raw messages: SHA-512 on the GPU (SURVEY 8f row 3), then the same verify kernel.
int eb200_eddsa_verify_batch_msgs(size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* A,
                                  const uint8_t* msgs, const uint64_t* msg_off, uint8_t* status) {
  return host_run(true, n, R && S && A && msg_off && status, [&](size_t i) { return range_ok(msgs, msg_off, i); },
    [&](Ctx& c, size_t lo, size_t m) {
      return eddsa_on(c, m, R + 32 * lo, S + 32 * lo, A + 32 * lo, nullptr, or_empty(msgs), msg_off + lo, status + lo);
    });
}

// EDDSA.prototype.sign (eddsa/index.js:34-44) for keys given as 32-byte secrets (eddsa.keyFromSecret)
int eb200_eddsa_sign_batch(size_t n, const uint8_t* secrets, const uint8_t* msgs, const uint64_t* msg_off,
                           uint8_t* out_sig, uint8_t* out_pub, uint8_t* status) {
  return host_run(true, n, secrets && msg_off && out_sig && status, [&](size_t i) { return range_ok(msgs, msg_off, i); },
    [&](Ctx& c, size_t lo, size_t m) {
      return eddsa_sign_on(c, m, secrets + 32 * lo, or_empty(msgs), msg_off + lo, out_sig + 64 * lo,
                           out_pub ? out_pub + 32 * lo : nullptr, status + lo);
    });
}

// ---- curve25519 ECDH derive -------------------------------------------------------------------
int eb200_x25519_derive_batch_dev(size_t n, const uint8_t* d_priv, const uint8_t* d_pubx, uint8_t* d_out,
                                  uint8_t* d_status, void* stream) {
  if (n == 0) return eb200_device_count() ? EB200_OK : EB200_ERR_NOT_INIT;
  if (!d_priv || !d_pubx || !d_out || !d_status) return EB200_ERR_ARG;
  return run_dev(d_status, 0, stream, [&](Ctx& c, Launch& L) {
    return x25519_launches(n, d_priv, d_pubx, d_out, d_status, true, L, c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
  });
}

int eb200_x25519_derive_batch(size_t n, const uint8_t* priv, const uint8_t* pubx, uint8_t* out, uint8_t* status) {
  return host_run(true, n, priv && pubx && out && status, every_item, [&](Ctx& c, size_t lo, size_t m) {
    return x25519_on(c, m, priv + 32 * lo, pubx + 32 * lo, out + 32 * lo, status + lo, true);
  });
}

// Montgomery-curve Point.mul (mont.js:130-153): x(k * P) for x-only points, k any 256-bit integer, no validation
int eb200_x25519_mul_batch(size_t n, const uint8_t* k, const uint8_t* px, uint8_t* out_x, uint8_t* status) {
  return host_run(true, n, k && px && out_x && status, every_item, [&](Ctx& c, size_t lo, size_t m) {
    return x25519_on(c, m, k + 32 * lo, px + 32 * lo, out_x + 32 * lo, status + lo, false);
  });
}

// ---- run-time short curves (the generic .curve API, SURVEY 8f-4) ------------------------------------------------
}  // extern "C"

namespace {
// big-endian bytes -> little-endian limbs (zero-extended); false if the value does not fit
template <int NL> bool rt_limbs(u32* r, const uint8_t* be, size_t len) {
  for (int i = 0; i < NL; i++) r[i] = 0;
  for (size_t b = 0; b < len; b++) {
    size_t bit = 8 * (len - 1 - b);
    if (bit / 32 >= (size_t)NL) { if (be[b]) return false; continue; }
    r[bit / 32] |= (u32)be[b] << (bit % 32);
  }
  return true;
}
// r = 2 r mod p
template <int NL> void rt_dbl_mod(u32* r, const u32* p) {
  u32 hi = r[NL - 1] >> 31;
  for (int i = NL - 1; i > 0; i--) r[i] = (r[i] << 1) | (r[i - 1] >> 31);
  r[0] <<= 1;
  u32 d[NL];
  u64 bw = 0;
  for (int i = 0; i < NL; i++) { u64 t = (u64)r[i] - p[i] - bw; d[i] = (u32)t; bw = (t >> 32) & 1; }
  if (hi || !bw) for (int i = 0; i < NL; i++) r[i] = d[i];
}
template <int NL> int rt_make(RtCurve<NL>& C, const eb200_short_curve* c) {
  if (!rt_limbs<NL>(C.p, c->p, c->len)) return EB200_ERR_ARG;
  u32 a[NL], b[NL];
  if (!rt_limbs<NL>(a, c->a, c->len) || !rt_limbs<NL>(b, c->b, c->len)) return EB200_ERR_ARG;
  if (!(C.p[0] & 1)) return EB200_ERR_ARG;                        // Montgomery arithmetic needs an odd modulus
  bool gt3 = false;
  for (int i = 1; i < NL; i++) gt3 = gt3 || C.p[i];
  if (!gt3 && C.p[0] <= 3) return EB200_ERR_ARG;
  u32 inv = 1;                                                     // -p^-1 mod 2^32 by Newton iteration
  for (int i = 0; i < 5; i++) inv *= 2 - C.p[0] * inv;
  C.n0inv = 0u - inv;
  // R mod p and R^2 mod p by repeated doubling of 1
  u32 r[NL];
  for (int i = 0; i < NL; i++) r[i] = i == 0;
  for (int i = 0; i < 32 * NL; i++) rt_dbl_mod<NL>(r, C.p);
  for (int i = 0; i < NL; i++) C.r1[i] = r[i];
  for (int i = 0; i < 32 * NL; i++) rt_dbl_mod<NL>(r, C.p);
  for (int i = 0; i < NL; i++) C.r2[i] = r[i];
  // a, b reduced and in Montgomery form: x R mod p by doubling x 32 NL times (host side, once per call)
  auto to_mont = [&](u32* x) {
    for (;;) {                                                    // reduce x below p first
      u32 d[NL]; u64 bw = 0;
      for (int i = 0; i < NL; i++) { u64 t = (u64)x[i] - C.p[i] - bw; d[i] = (u32)t; bw = (t >> 32) & 1; }
      if (bw) break;
      for (int i = 0; i < NL; i++) x[i] = d[i];
    }
    for (int i = 0; i < 32 * NL; i++) rt_dbl_mod<NL>(x, C.p);
  };
  bool az = true;
  to_mont(a); to_mont(b);
  for (int i = 0; i < NL; i++) { C.a[i] = a[i]; C.b[i] = b[i]; az = az && a[i] == 0; }
  C.a_is_zero = az;
  C.len = c->len;
  return EB200_OK;
}
template <int NL>
int rt_on(Ctx& c, const RtCurve<NL>& C, int op, size_t n, const uint8_t* k1, const uint8_t* p1, const uint8_t* k2, const uint8_t* p2,
          size_t klen, uint8_t* out, uint8_t* status) {
  int rc;
  const size_t pl = 2 * (size_t)C.len;
  if ((rc = grow(&c.d_in, &c.d_in_cap, n * (2 * klen + 3 * pl) + 1024))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *dk1 = c.d_in, *dk2 = dk1 + klen * n, *dp1 = dk2 + klen * n, *dp2 = dp1 + pl * n, *dout = dp2 + pl * n;
  return run_single(c, {{dk1, k1, k1 ? klen * n : 0}, {dk2, k2, k2 ? klen * n : 0}, {dp1, p1, pl * n}, {dp2, p2, p2 ? pl * n : 0}},
    [&](Launch& L) {
      L(rt_curve_kernel<NL>, blocks128(n), 128, op, n, C, k1 ? dk1 : nullptr, dp1, k2 ? dk2 : nullptr, p2 ? dp2 : nullptr,
        (u32)klen, dout, c.d_status);
      return EB200_OK;
    },
    {{op != 3 ? out : nullptr, dout, pl * n}, {status, c.d_status, n}}, {}, true);
}
template <int NL>
int rt_call(const eb200_short_curve* cv, int op, size_t n, const uint8_t* k1, const uint8_t* p1, const uint8_t* k2, const uint8_t* p2,
            size_t klen, uint8_t* out, uint8_t* status) {
  RtCurve<NL> C;
  int rc = rt_make<NL>(C, cv);
  if (rc) return rc;
  const size_t pl = 2 * (size_t)cv->len;
  return run_sharded(n, [&](Ctx& c, size_t lo, size_t m) {
    return rt_on<NL>(c, C, op, m, k1 ? k1 + lo * klen : nullptr, p1 + lo * pl, k2 ? k2 + lo * klen : nullptr, p2 ? p2 + lo * pl : nullptr,
                     klen, out ? out + lo * pl : nullptr, status + lo);
  });
}
int rt_dispatch(const eb200_short_curve* cv, int op, size_t n, const uint8_t* k1, const uint8_t* p1, const uint8_t* k2, const uint8_t* p2,
                size_t klen, uint8_t* out, uint8_t* status) {
  if (!eb200_device_count()) return EB200_ERR_NOT_INIT;
  if (!cv || !cv->p || !cv->a || !cv->b || cv->len == 0 || cv->len > 72 || klen > 128) return EB200_ERR_ARG;
  if (n == 0) return EB200_OK;
  if (!p1 || !status || (op != 3 && !out)) return EB200_ERR_ARG;
  if (cv->len <= 32) return rt_call<8>(cv, op, n, k1, p1, k2, p2, klen, out, status);
  if (cv->len <= 48) return rt_call<12>(cv, op, n, k1, p1, k2, p2, klen, out, status);
  return rt_call<18>(cv, op, n, k1, p1, k2, p2, klen, out, status);
}
}  // namespace

extern "C" {

int eb200_curve_mul_batch(const eb200_short_curve* curve, size_t n, const uint8_t* k, size_t klen, const uint8_t* points_xy,
                          uint8_t* out_xy, uint8_t* status) {
  if (n && (!k || !klen)) return EB200_ERR_ARG;
  return rt_dispatch(curve, 0, n, k, points_xy, nullptr, nullptr, klen, out_xy, status);
}
int eb200_curve_mul_add_batch(const eb200_short_curve* curve, size_t n, const uint8_t* k1, const uint8_t* p1_xy, const uint8_t* k2,
                              const uint8_t* p2_xy, size_t klen, uint8_t* out_xy, uint8_t* status) {
  if (n && (!k1 || !k2 || !p2_xy || !klen)) return EB200_ERR_ARG;
  return rt_dispatch(curve, 0, n, k1, p1_xy, k2, p2_xy, klen, out_xy, status);
}
int eb200_curve_add_batch(const eb200_short_curve* curve, size_t n, const uint8_t* p1_xy, const uint8_t* p2_xy, uint8_t* out_xy,
                          uint8_t* status) {
  if (n && !p2_xy) return EB200_ERR_ARG;
  return rt_dispatch(curve, 1, n, nullptr, p1_xy, nullptr, p2_xy, 0, out_xy, status);
}
int eb200_curve_dbl_batch(const eb200_short_curve* curve, size_t n, const uint8_t* p_xy, uint8_t* out_xy, uint8_t* status) {
  return rt_dispatch(curve, 2, n, nullptr, p_xy, nullptr, nullptr, 0, out_xy, status);
}
int eb200_curve_validate_batch(const eb200_short_curve* curve, size_t n, const uint8_t* p_xy, uint8_t* status) {
  return rt_dispatch(curve, 3, n, nullptr, p_xy, nullptr, nullptr, 0, nullptr, status);
}

// ---- self-test hooks (first initialised device) ------------------------------------------------------
static Ctx* first_ctx() {
  std::lock_guard<std::mutex> lk(g_mu);
  return g_ndev ? &g_ctx[g_devs[0]] : nullptr;
}

int eb200_selftest_fe(int curve, int op, size_t n, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  Ctx* cp = first_ctx();
  if (!cp) return EB200_ERR_NOT_INIT;
  if (!fe_len(curve)) return EB200_ERR_UNSUPPORTED;
  if (n == 0) return EB200_OK;
  Ctx& c = *cp;
  std::lock_guard<std::mutex> lk(c.mu);
  CK(cudaSetDevice(c.device));
  size_t bytes = n * fe_len(curve);
  u32 *da, *db, *dout;
  CK(cudaMalloc(&da, bytes)); CK(cudaMalloc(&db, bytes)); CK(cudaMalloc(&dout, bytes));
  // stream-ordered copies: a synchronous cudaMemcpy from pageable memory may return before its DMA lands,
  // and c.stream (non-blocking) does not wait for the legacy default stream
  CK(cudaMemcpyAsync(da, a, bytes, cudaMemcpyHostToDevice, c.stream));
  CK(cudaMemcpyAsync(db, b, bytes, cudaMemcpyHostToDevice, c.stream));
  const unsigned nb = blocks128(n);
  if (curve == EB200_CURVE_ED25519 || curve == EB200_CURVE_CURVE25519) f25_selftest_kernel<<<nb, 128, 0, c.stream>>>(op, n, da, db, dout);
  else with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    if constexpr (is_k256<T>) k256_selftest_fe_kernel<<<nb, 128, 0, c.stream>>>(op, n, da, db, dout);
    else if constexpr (!is_ed25519<T>) {
      if (op >= 8) sw_selftest_ext_kernel<typename T::C><<<nb, 128, 0, c.stream>>>(op, n, da, db, dout);
      else sw_selftest_fe_kernel<typename T::C><<<nb, 128, 0, c.stream>>>(op, n, da, db, dout);
    }
    return EB200_OK;
  });
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, dout, bytes, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  cudaFree(da); cudaFree(db); cudaFree(dout);
  return EB200_OK;
}

int eb200_selftest_gtab_dims(int curve, int* windows, int* entries, int* wbits) {
  if (!windows || !entries || !wbits) return EB200_ERR_ARG;
  // ed25519 answers with the p224 geometry, as it always has (its own table is not in this layout)
  return with_curve(curve == EB200_CURVE_ED25519 ? EB200_CURVE_P224 : curve, [&](auto cv) {
    typedef decltype(cv) T;
    if constexpr (is_k256<T>) { *windows = GTAB_WINDOWS; *entries = GTAB_ENTRIES; *wbits = GTAB_W; }
    else if constexpr (!is_ed25519<T>) { typedef SW<typename T::C> W; *windows = W::GWINDOWS; *entries = W::GENTRIES; *wbits = W::GW; }
    return EB200_OK;
  });
}

int eb200_selftest_gtab(int curve, uint32_t* out, size_t n_words) {
  Ctx* cp = first_ctx();
  if (!cp) return EB200_ERR_NOT_INIT;
  int w, en, b;
  int rc = eb200_selftest_gtab_dims(curve, &w, &en, &b);
  if (rc) return rc;
  size_t words = (size_t)w * en * 2 * (fe_len(curve) / 4);
  if (!out || n_words < words) return EB200_ERR_ARG;
  Ctx& c = *cp;
  std::lock_guard<std::mutex> lk(c.mu);
  CK(cudaSetDevice(c.device));
  if ((rc = ensure_table(c, curve))) return rc;
  CK(cudaMemcpyAsync(out, c.gtab[curve], words * 4, cudaMemcpyDeviceToHost, c.stream));
  CK(cudaStreamSynchronize(c.stream));
  return EB200_OK;
}

}  // extern "C"

// ---- EC.getKeyRecoveryParam ----------------------------------------------------------------------------------------
// The kernels are in recovery_param.cu (see there why); this side stages the buffers and runs them like recover_on.
// The launches of one block whose inputs are on the device; base: ws_layout(curve, n).total bytes of workspace.
static int recovery_param_launches(Ctx& c, int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r, const uint8_t* d_s,
                                   const uint8_t* d_q, uint8_t* d_id, uint8_t* d_status, uint8_t* base, Launch& L,
                                   cudaEvent_t ev0, cudaEvent_t ev1) {
  const WsLayout W = ws_layout(curve, n);
  const RecoveryParamArgs a{d_e, d_r, d_s, d_q, d_id, d_status, c.gtab[curve], (u32*)(base + W.ws), (u32*)(base + W.scratch),
                            (u32*)(base + W.qtab)};
  cudaError_t err = recovery_param_launch(curve, n, a, L.st, ev0, ev1, &L.count);
  return err == cudaSuccess ? EB200_OK : cuda_fail(err, "recovery_param_launch");
}

static int recovery_param_on(Ctx& c, int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                             const uint8_t* q_xy, uint8_t* out_recid, uint8_t* status) {
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  const size_t len = curve_len(curve);
  const WsLayout W = ws_layout(curve, n);
  if ((rc = grow(&c.d_in, &c.d_in_cap, n * (5 * len + 1) + 256))) return rc;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, W.total))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *d_e = c.d_in, *d_r = d_e + len * n, *d_s = d_r + len * n, *d_q = d_s + len * n, *d_id = d_q + 2 * len * n;
  return run_single(c, {{d_e, e, len * n}, {d_r, r, len * n}, {d_s, s, len * n}, {d_q, q_xy, 2 * len * n}},
    [&](Launch& L) {
      return recovery_param_launches(c, curve, n, d_e, d_r, d_s, d_q, d_id, c.d_status, c.d_ws, L, c.ev[EV_MAIN_BEGIN],
                                     c.ev[EV_MAIN_END]);
    },
    {{out_recid, d_id, n}, {status, c.d_status, n}}, {}, false);     // nothing secret: no wipe
}

extern "C" {

int eb200_ecdsa_recovery_param_batch(int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                                     const uint8_t* q_xy, uint8_t* out_recid, uint8_t* status) {
  const size_t len = curve_len(curve);
  return host_run(curve_ok(curve), n, e && r && s && q_xy && out_recid && status, every_item, [&](Ctx& c, size_t lo, size_t m) {
    return recovery_param_on(c, curve, m, e + lo * len, r + lo * len, s + lo * len, q_xy + lo * 2 * len, out_recid + lo,
                             status + lo);
  }, curve == EB200_CURVE_ED25519);      // cofactor 8: the one-multiplication identity fails
}

}  // extern "C"

// ---- key sets ---------------------------------------------------------------------------------------------------------
// The kernels are in keyset.cu (see there why); this side owns the handles, stages the buffers and launches the unchanged
// decode and prep kernels of this file around them.
enum KeysetKind { KS_PUBLIC, KS_SIGNING };      // public keys (verify, mul) or ed25519 secrets (eb200_eddsa_sign_batch_keyed)
struct eb200_keyset {
  int curve = 0;
  int kind = KS_PUBLIC;
  size_t m = 0;
  u32 W = 0, fmt = 0;
  size_t device_bytes = 0;
  bool live = false;                  // false once eb200_shutdown has freed the device copies
  int ndev = 0;
  int devs[MAX_DEV] = {};             // the devices that hold a copy: keyed calls are sharded over these only
  KeysetDev dev[MAX_DEV] = {};        // indexed by CUDA ordinal, like g_ctx
};

namespace {
std::mutex g_ks_mu;                   // the list of live sets (taken inside g_mu by shutdown, never the other way round)
std::vector<eb200_keyset*> g_keysets;

// frees the device copies; the caller holds whatever keeps the set's devices from being used
void keyset_free_device(eb200_keyset* ks) {
  for (int i = 0; i < ks->ndev; i++) {
    KeysetDev& d = ks->dev[ks->devs[i]];
    if (cudaSetDevice(ks->devs[i]) != cudaSuccess) { cudaGetLastError(); continue; }
    if (ks->kind == KS_SIGNING && d.tab) cudaMemset(d.tab, 0, ED_SIGNSET_KEY_BYTES * ks->m);   // the secret words
    cudaFree(d.xy); cudaFree(d.kst); cudaFree(d.tab);
    d = KeysetDev{};
  }
  ks->ndev = 0;
  ks->live = false;
}

// One device's copy of the set: keys up, decode (this file's kernels), classify + tables (keyset.cu), verdicts home.
int keyset_build_on(Ctx& c, eb200_keyset* ks, const uint8_t* pub, uint8_t* key_status) {
  const int curve = ks->curve;
  const size_t m = ks->m, len = curve_len(curve), pb = pub_item_bytes(len, ks->fmt);
  const int windows = keyset_windows(curve, (int)ks->W);
  int rc = ensure_table(c, curve);
  if (rc) return rc;
  KeysetDev& d = ks->dev[c.device];
  d.W = (int)ks->W;
  CK(cudaMalloc(&d.xy, 2 * len * m));
  CK(cudaMalloc(&d.kst, m));
  CK(cudaMalloc(&d.tab, keyset_key_bytes(curve, (int)ks->W) * m));
  if ((rc = grow(&c.d_in, &c.d_in_cap, align256(m * pb) + m))) return rc;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, m * windows * 3 * keyset_geom(curve).limbs * 4))) return rc;
  uint8_t *d_pub = c.d_in, *d_pre = c.d_in + align256(m * pb);
  return run_single(c, {{d_pub, pub, m * pb}},
    [&](Launch& L) {
      const uint8_t* pre = nullptr;
      if (ks->fmt == EB200_PUB_XY) CK(cudaMemcpyAsync(d.xy, d_pub, 2 * len * m, cudaMemcpyDeviceToDevice, L.st));
      else {
        pre = d_pre;
        int rc2 = with_curve(curve, [&](auto cv) {
          typedef decltype(cv) T;
          if constexpr (is_k256<T>) L(k256_decode_pub_kernel, blocks128(m), 128, m, d_pub, ks->fmt, d.xy, d_pre);
          else if constexpr (is_ed25519<T>) return EB200_ERR_UNSUPPORTED;
          else L(sw_decode_pub_kernel<typename T::C>, blocks128(m), 128, m, d_pub, ks->fmt, d.xy, d_pre);
          return L.rc;
        });
        if (rc2) return rc2;
      }
      cudaError_t err = keyset_build_launch(curve, m, d, pre, (u32*)c.d_ws, L.st, &L.count);
      return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_build_launch");
    },
    {{key_status, d.kst, m}}, {}, true);
}

// Workspace of one keyed_verify_launches block of n items: the prep words and the inversion scratch, as ws_layout places
// them (no per-item table).
size_t keyed_verify_ws_bytes(int curve, size_t n) { return ws_layout(curve, n).qtab; }

// The launches of one keyed verify block whose inputs are on the device: the unchanged prep kernel of the set's curve,
// then keyed main (between ev0 and ev1) and keyed replay.  base: keyed_verify_ws_bytes(curve, m) of workspace.
int keyed_verify_launches(Ctx& c, int curve, size_t m, const KeysetDev& d, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                          const u32* idx, uint8_t* base, uint8_t* status, Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  const WsLayout W = ws_layout(curve, m);
  u32 *ws = (u32*)(base + W.ws), *scratch = (u32*)(base + W.scratch);
  const u32* replay = nullptr;
  int rc = with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    if constexpr (is_ed25519<T>) return EB200_ERR_UNSUPPORTED;
    else if constexpr (is_k256<T>) {
      L(k256_prep_kernel, batch_blocks(m, k256_prep_batch(m)), 128, m, e, r, s, ws, scratch, k256_prep_batch(m));
      replay = c.replay_tab;
    } else {
      typedef typename T::C C;
      L(sw_prep_kernel<C>, batch_blocks(m, SW<C>::BATCH), 128, m, e, r, s, ws, scratch);
      replay = c.sw_replay_tab[curve];
    }
    return L.rc;
  });
  if (rc) return rc;
  const KeyedVerifyArgs a{e, r, s, idx, status, ws, c.gtab[curve], replay};
  cudaError_t err = keyset_verify_launch(curve, m, d, a, L.st, ev0, ev1, &L.count);
  return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_verify_launch");
}

// Keyed verify of one block on one device of the set, chunked like verify_on.  Launches per chunk: keyed_verify_launches.
int verify_keyed_on(Ctx& c, const KeysetDev& d, int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                    const u32* key_idx, uint8_t* status) {
  int rc;
  const size_t len = curve_len(curve);
  const ChunkPlan P = make_plan(n);
  const size_t idx_bytes = align256(n * 4);
  if ((rc = grow(&c.d_in, &c.d_in_cap, idx_bytes + align256(n * 3 * len) + 1024))) return rc;
  const size_t ws_slot = keyed_verify_ws_bytes(curve, P.max_m);
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (P.chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  u32* d_idx = (u32*)c.d_in;
  uint8_t *d_e = c.d_in + idx_bytes, *d_r = d_e + n * len, *d_s = d_r + n * len;
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {d_e + lo * len, e + lo * len, m * len};
      seg[1] = {d_r + lo * len, r + lo * len, m * len};
      seg[2] = {d_s + lo * len, s + lo * len, m * len};
      seg[3] = {d_idx + lo, key_idx + lo, m * 4};
      return 4;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      return keyed_verify_launches(c, curve, m, d, d_e + lo * len, d_r + lo * len, d_s + lo * len, d_idx + lo,
                                   c.d_ws + (size_t)slot * ws_slot, c.d_status + lo, L, c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {status + lo, c.d_status + lo, m};
      return 1;
    });
}

// The launches of one keyed DER verify block whose inputs are on the device: the keyed DER decode (der + off[i] is item
// i's encoding), or with `pre` the screened one (pre: the index-and-range screen's verdicts), then keyed_verify_launches
// and the verdict merge.  idx: the key indices the set may be addressed with; r, s (m x len) and vd (m bytes) the decoded
// halves and verdicts; base: keyed_verify_ws_bytes(curve, m) of workspace.
int keyed_der_launches(Ctx& c, int curve, size_t m, const KeysetDev& d, const uint8_t* e, const uint8_t* der,
                       const unsigned long long* off, const u32* idx, const uint8_t* pre, uint8_t* r, uint8_t* s, uint8_t* vd,
                       uint8_t* base, uint8_t* status, Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  const u32 len = (u32)curve_len(curve);
  cudaError_t err = pre ? keyset_der_decode_screened_launch(m, len, pre, der, off, idx, d, r, s, vd, L.st, &L.count)
                        : keyset_der_decode_launch(m, len, der, off, idx, d, r, s, vd, L.st, &L.count);
  if (err != cudaSuccess) return cuda_fail(err, pre ? "keyset_der_decode_screened_launch" : "keyset_der_decode_launch");
  int rc = keyed_verify_launches(c, curve, m, d, e, r, s, idx, base, status, L, ev0, ev1);
  if (rc) return rc;
  if ((err = keyset_verdict_merge_launch(m, vd, status, L.st, &L.count)) != cudaSuccess)
    return cuda_fail(err, "keyset_verdict_merge_launch");
  return EB200_OK;
}

// Keyed verify of DER signatures, one block on one device of the set, chunked like verify_keyed_on; the variable-length
// segments as eddsa_sign_keyed_on stages them (sig_off points at this block's first offset, offsets absolute).
// Launches per chunk: keyed_der_launches without a screen.
int verify_keyed_der_on(Ctx& c, const KeysetDev& d, int curve, size_t n, const uint8_t* e, const uint8_t* sigs,
                        const uint64_t* sig_off, const u32* key_idx, uint8_t* status) {
  int rc;
  const size_t len = curve_len(curve);
  const ChunkPlan P = make_plan(n);
  const size_t sig_bytes = (size_t)(sig_off[n] - sig_off[0]);
  const size_t off_bytes = align256((n + 1) * 8);
  const size_t base = align256(n * 4) + align256(n * 3 * len) + align256(n);   // key_idx | e, r, s | verdicts
  if ((rc = grow(&c.d_in, &c.d_in_cap, base + off_bytes + align256(sig_bytes + 1)))) return rc;
  const size_t ws_slot = keyed_verify_ws_bytes(curve, P.max_m);
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (P.chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  u32* d_idx = (u32*)c.d_in;
  uint8_t *d_e = c.d_in + align256(n * 4), *d_r = d_e + n * len, *d_s = d_r + n * len;
  uint8_t* d_vd = d_e + align256(n * 3 * len);
  unsigned long long* d_off = (unsigned long long*)(c.d_in + base);
  uint8_t* d_sig = c.d_in + base + off_bytes;
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {d_e + lo * len, e + lo * len, m * len};
      seg[1] = {d_idx + lo, key_idx + lo, m * 4};
      seg[2] = {d_off + lo, sig_off + lo, (m + 1) * 8};
      seg[3] = {d_sig + (sig_off[lo] - sig_off[0]), sigs + sig_off[lo], (size_t)(sig_off[lo + m] - sig_off[lo])};
      return 4;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      return keyed_der_launches(c, curve, m, d, d_e + lo * len, d_sig - sig_off[0], d_off + lo, d_idx + lo, nullptr,
                                d_r + lo * len, d_s + lo * len, d_vd + lo, c.d_ws + (size_t)slot * ws_slot, c.d_status + lo, L,
                                c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {status + lo, c.d_status + lo, m};
      return 1;
    });
}

// workspace of the keyed device-pointer calls: [screened key_idx (n words) | verdicts (n bytes) | body bytes], the body
// as each call places it (eb200_ecdsa_verify_batch_keyed_dev: prep words and the inversion scratch, as ws_layout
// places them)
struct KeyedDevWs { size_t idx, verdict, prep, total; };
KeyedDevWs keyed_dev_ws(size_t n, size_t body) {
  KeyedDevWs L;
  L.idx = 0;
  L.verdict = align256(n * 4);
  L.prep = L.verdict + align256(n);
  L.total = L.prep + body;
  return L;
}

// Workspace of one keyed_mul_launches or keyed_rp_launches block of n items: prep words | inversion scratch (as
// ws_layout places them) | Jacobian results (3 x limbs x n words; recovery parameter: Y, Z, 2 x limbs x n).
size_t keyed_mul_ws_bytes(int curve, size_t n) {
  return align256(keyed_verify_ws_bytes(curve, n) + 3 * (size_t)keyset_geom(curve).limbs * n * 4);
}

// eb200_ecdsa_verify_batch_keyed_der_dev keeps the decoded r, s (len bytes each) and the index-and-range screen's verdict
// of every item in the Jacobian-result region of keyed_mul_ws_bytes (3 x limbs words per item), which starts behind the
// prep words and inversion scratch that the unchanged prep writes; so the keyed workspace size serves it unchanged.
constexpr bool keyed_der_fits_jacobian(int curve) { return 2 * curve_len(curve) + 1 <= 3 * (size_t)keyset_geom(curve).limbs * 4; }
static_assert(keyed_der_fits_jacobian(EB200_CURVE_SECP256K1) && keyed_der_fits_jacobian(EB200_CURVE_P256) &&
              keyed_der_fits_jacobian(EB200_CURVE_P384) && keyed_der_fits_jacobian(EB200_CURVE_P521) &&
              keyed_der_fits_jacobian(EB200_CURVE_P192) && keyed_der_fits_jacobian(EB200_CURVE_P224),
              "r, s and the screen verdicts of the keyed DER device form must fit the keyed workspace's Jacobian region");

// The launches of one keyed mul / mulAdd / derive block whose inputs are on the device (k1 == NULL: no base-point term):
// prep_scalars, keyed main (between ev0 and ev1), normalisation, then the keyed replay (derive: the status map).
// base: keyed_mul_ws_bytes(curve, m) of workspace.
int keyed_mul_launches(Ctx& c, int curve, size_t m, const KeysetDev& d, const uint8_t* k1, const uint8_t* k2, const u32* idx,
                       uint8_t* base, uint8_t* out, uint8_t* status, bool derive, Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  const WsLayout W = ws_layout(curve, m);
  u32 *ws = (u32*)(base + W.ws), *scratch = (u32*)(base + W.scratch), *jac = (u32*)(base + W.qtab);
  const u32* replay = nullptr;
  int batch = 0;
  int rc = with_curve(curve, [&](auto cv) {
    typedef decltype(cv) T;
    if constexpr (is_ed25519<T>) return EB200_ERR_UNSUPPORTED;
    else if constexpr (is_k256<T>) {
      L(k256_prep_scalars_kernel, blocks128(m), 128, m, k1, k2, ws);
      replay = c.replay_tab;
      batch = k256_prep_batch(m);
    } else {
      L(sw_prep_scalars_kernel<typename T::C>, blocks128(m), 128, m, k1, k2, ws);
      replay = c.sw_replay_tab[curve];
    }
    return L.rc;
  });
  if (rc) return rc;
  const KeyedMulArgs a{k1, k2, idx, ws, jac, scratch, c.gtab[curve], replay, out, status, batch, derive};
  cudaError_t err = keyset_mul_launch(curve, m, d, a, L.st, ev0, ev1, &L.count);
  if (err != cudaSuccess) return cuda_fail(err, "keyset_mul_launch");
  if (derive) L(status_map_kernel, blocks128(m), 128, m, status, (uint8_t)ST_NEEDS_HOST, (uint8_t)ST_THROW_NOT_VALIDATED);
  return L.rc;
}

// Keyed Point.mul / G.mulAdd / KeyPair.derive of one block on one device of the set, chunked like verify_keyed_on.
// k1 == NULL: k2 times the key (derive: x only, and an off-curve key is THROW_NOT_VALIDATED instead of replayed);
// else k1 G + k2 times the key.  Launches per chunk: keyed_mul_launches.  derive: the private scalars, their digit
// words and the Jacobian results are cleared on the chunk's stream behind its kernels, as x25519_on does.
int mul_keyed_on(Ctx& c, const KeysetDev& d, int curve, size_t n, const uint8_t* k1, const uint8_t* k2, const u32* key_idx,
                 uint8_t* out, uint8_t* status, bool derive) {
  int rc;
  const size_t len = curve_len(curve), ol = derive ? len : 2 * len;
  const ChunkPlan P = make_plan(n);
  const size_t idx_bytes = align256(n * 4), k_bytes = align256(n * len);
  if ((rc = grow(&c.d_in, &c.d_in_cap, idx_bytes + 2 * k_bytes + n * ol + 256))) return rc;
  const size_t ws_slot = keyed_mul_ws_bytes(curve, P.max_m);
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (P.chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  u32* d_idx = (u32*)c.d_in;
  uint8_t *d_k1 = c.d_in + idx_bytes, *d_k2 = d_k1 + k_bytes, *d_out = d_k2 + k_bytes;
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {d_k2 + lo * len, k2 + lo * len, m * len};
      seg[1] = {d_idx + lo, key_idx + lo, m * 4};
      seg[2] = {d_k1 + lo * len, k1 ? k1 + lo * len : nullptr, k1 ? m * len : 0};
      return 3;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      uint8_t* base = c.d_ws + (size_t)slot * ws_slot;
      int rc2 = keyed_mul_launches(c, curve, m, d, k1 ? d_k1 + lo * len : nullptr, d_k2 + lo * len, d_idx + lo, base,
                                   d_out + lo * ol, c.d_status + lo, derive, L, c.ev_k0[k], c.ev_k1[k]);
      if (rc2) return rc2;
      if (derive) {
        CK(cudaMemsetAsync(d_k2 + lo * len, 0, m * len, L.st));     // the private scalars
        CK(cudaMemsetAsync(base, 0, ws_slot, L.st));                 // their digit words and the Jacobian results
      }
      return L.rc;
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {out + lo * ol, d_out + lo * ol, m * ol};
      seg[1] = {status + lo, c.d_status + lo, m};
      return 2;
    });
}

// The launches of one keyed getKeyRecoveryParam block whose inputs are on the device: the unkeyed recovery-parameter
// prep (recovery_param.cu), keyed main (between ev0 and ev1), recid normalisation, cold (keyset_recovery_param.cu).
// base: keyed_mul_ws_bytes(curve, m) of workspace (Y, Z in its Jacobian-result region).
int keyed_rp_launches(Ctx& c, int curve, size_t m, const KeysetDev& d, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                      const u32* idx, uint8_t* base, uint8_t* recid, uint8_t* status, Launch& L, cudaEvent_t ev0,
                      cudaEvent_t ev1) {
  const WsLayout W = ws_layout(curve, m);
  u32 *ws = (u32*)(base + W.ws), *scratch = (u32*)(base + W.scratch), *yz = (u32*)(base + W.qtab);
  cudaError_t err = recovery_param_prep_launch(curve, m, e, r, s, ws, scratch, L.st, &L.count);
  if (err != cudaSuccess) return cuda_fail(err, "recovery_param_prep_launch");
  const KeyedRecoveryParamArgs a{e, r, idx, ws, yz, scratch, c.gtab[curve], recid, status,
                                 curve == EB200_CURVE_SECP256K1 ? k256_prep_batch(m) : 0};
  err = keyset_recovery_param_launch(curve, m, d, a, L.st, ev0, ev1, &L.count);
  return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_recovery_param_launch");
}

// Keyed getKeyRecoveryParam of one block on one device of the set, chunked like mul_keyed_on.  Launches per chunk:
// keyed_rp_launches.
int recovery_param_keyed_on(Ctx& c, const KeysetDev& d, int curve, size_t n, const uint8_t* e, const uint8_t* r,
                            const uint8_t* s, const u32* key_idx, uint8_t* out_recid, uint8_t* status) {
  int rc;
  const size_t len = curve_len(curve);
  const ChunkPlan P = make_plan(n);
  const size_t idx_bytes = align256(n * 4);
  if ((rc = grow(&c.d_in, &c.d_in_cap, idx_bytes + align256(n * 3 * len) + n + 256))) return rc;
  const size_t ws_slot = keyed_mul_ws_bytes(curve, P.max_m);
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (P.chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  u32* d_idx = (u32*)c.d_in;
  uint8_t *d_e = c.d_in + idx_bytes, *d_r = d_e + n * len, *d_s = d_r + n * len, *d_id = c.d_in + idx_bytes + align256(n * 3 * len);
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {d_e + lo * len, e + lo * len, m * len};
      seg[1] = {d_r + lo * len, r + lo * len, m * len};
      seg[2] = {d_s + lo * len, s + lo * len, m * len};
      seg[3] = {d_idx + lo, key_idx + lo, m * 4};
      return 4;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      return keyed_rp_launches(c, curve, m, d, d_e + lo * len, d_r + lo * len, d_s + lo * len, d_idx + lo,
                               c.d_ws + (size_t)slot * ws_slot, d_id + lo, c.d_status + lo, L, c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {out_recid + lo, d_id + lo, m};
      seg[1] = {status + lo, c.d_status + lo, m};
      return 2;
    });
}

// ---- EdDSA (ed25519) key sets: kernels in eddsa_keyset.cu, the hash kernel of this file --------------------------------
// One device's copy: raw keys up, classify + tables, verdicts home.
int ed_keyset_build_on(Ctx& c, eb200_keyset* ks, const uint8_t* A, uint8_t* key_status) {
  const size_t m = ks->m;
  const int W = (int)ks->W;
  int rc;
  KeysetDev& d = ks->dev[c.device];
  d.W = W;
  CK(cudaMalloc(&d.xy, 32 * m));
  CK(cudaMalloc(&d.kst, m));
  CK(cudaMalloc(&d.tab, ed_keyset_key_bytes(W) * m));
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, m * ed_keyset_windows(W) * 24 * 4))) return rc;
  return run_single(c, {{d.xy, A, 32 * m}},
    [&](Launch& L) {
      cudaError_t err = ed_keyset_build_launch(m, d, (u32*)c.d_ws, L.st, &L.count);
      return err == cudaSuccess ? EB200_OK : cuda_fail(err, "ed_keyset_build_launch");
    },
    {{key_status, d.kst, m}}, {}, true);
}

// The launches of one keyed EdDSA verify block whose inputs are on the device.  msg_off != NULL (raw messages, m + 1
// offsets relative to msgs): the keys' raw bytes gathered into A and h = SHA512(R || A || M) mod n into h first, by the
// screened hash (keyset_forms.cu) when verdict != NULL; then the keyed verify between ev0 and ev1.
int keyed_eddsa_verify_launches(Ctx& c, size_t m, const KeysetDev& d, const uint8_t* R, const uint8_t* S, uint8_t* h,
                                uint8_t* A, const uint8_t* msgs, const u64* msg_off, const u32* idx, const uint8_t* verdict,
                                uint8_t* status, Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  cudaError_t err;
  if (msg_off) {
    if ((err = ed_keyset_gather_launch(m, d, idx, A, L.st, &L.count)) != cudaSuccess) return cuda_fail(err, "ed_keyset_gather_launch");
    if (verdict) {
      if ((err = keyset_ed_hash_screened_launch(m, verdict, R, A, msgs, msg_off, h, L.st, &L.count)) != cudaSuccess)
        return cuda_fail(err, "keyset_ed_hash_screened_launch");
    } else {
      L(ed25519_hash_kernel, blocks128(m), 128, m, R, A, msgs, msg_off, h);
      if (L.rc) return L.rc;
    }
  }
  CK(cudaEventRecord(ev0, L.st));
  if ((err = ed_keyset_verify_launch(m, d, R, S, h, idx, c.gtab[EB200_CURVE_ED25519], status, L.st, &L.count)) != cudaSuccess)
    return cuda_fail(err, "ed_keyset_verify_launch");
  CK(cudaEventRecord(ev1, L.st));
  return EB200_OK;
}

// Keyed EdDSA verify of one block on one device of the set, chunked like eddsa_on.  h == NULL: raw messages (msg_off
// points at this block's first offset, offsets absolute).  Launches per chunk: keyed_eddsa_verify_launches.
int eddsa_keyed_on(Ctx& c, const KeysetDev& d, size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* h,
                   const uint8_t* msgs, const uint64_t* msg_off, const u32* key_idx, uint8_t* status) {
  int rc;
  const ChunkPlan P = make_plan(n);
  size_t mbytes = h ? 0 : (size_t)(msg_off[n] - msg_off[0]);
  size_t off_bytes = h ? 0 : (n + 1) * sizeof(uint64_t);
  size_t base = align256(n * 132);                 // R | S | h | gathered keys | key_idx
  if ((rc = grow(&c.d_in, &c.d_in_cap, base + align256(off_bytes) + align256(mbytes + 1)))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  uint8_t *dR = c.d_in, *dS = dR + 32 * n, *dh = dS + 32 * n, *dA = dh + 32 * n;
  u32* didx = (u32*)(dA + 32 * n);
  uint64_t* doff = (uint64_t*)(c.d_in + base);
  uint8_t* dm = c.d_in + base + align256(off_bytes);
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {dR + 32 * lo, R + 32 * lo, 32 * m};
      seg[1] = {dS + 32 * lo, S + 32 * lo, 32 * m};
      seg[2] = {didx + lo, key_idx + lo, 4 * m};
      if (h) { seg[3] = {dh + 32 * lo, h + 32 * lo, 32 * m}; return 4; }
      seg[3] = {doff + lo, msg_off + lo, (m + 1) * sizeof(uint64_t)};
      seg[4] = {dm + (msg_off[lo] - msg_off[0]), msgs + msg_off[lo], (size_t)(msg_off[lo + m] - msg_off[lo])};
      return 5;
    },
    [&](size_t lo, size_t m, Launch& L, int, int k) {
      return keyed_eddsa_verify_launches(c, m, d, dR + 32 * lo, dS + 32 * lo, dh + 32 * lo, dA + 32 * lo,
                                         h ? nullptr : dm - msg_off[0], h ? nullptr : doff + lo, didx + lo, nullptr,
                                         c.d_status + lo, L, c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {status + lo, c.d_status + lo, m};
      return 1;
    });
}

// ---- EdDSA (ed25519) signing sets: kernels in eddsa_signset.cu -----------------------------------------------------------
// One device's copy: secrets up, a, prefix and A derived on the GPU, A home; the staged secrets are wiped.
int ed_signset_build_on(Ctx& c, eb200_keyset* ks, const uint8_t* secrets, uint8_t* out_pub) {
  const size_t m = ks->m;
  int rc = ensure_table(c, EB200_CURVE_ED25519);
  if (rc) return rc;
  KeysetDev& d = ks->dev[c.device];
  CK(cudaMalloc(&d.xy, 32 * m));
  CK(cudaMalloc(&d.tab, ED_SIGNSET_KEY_BYTES * m));
  if ((rc = grow(&c.d_in, &c.d_in_cap, 32 * m))) return rc;
  uint8_t* dsec = c.d_in;
  return run_single(c, {{dsec, secrets, 32 * m}},
    [&](Launch& L) {
      cudaError_t err = ed_signset_create_launch(m, d, dsec, c.gtab[EB200_CURVE_ED25519], L.st, &L.count);
      return err == cudaSuccess ? EB200_OK : cuda_fail(err, "ed_signset_create_launch");
    },
    {{out_pub, d.xy, 32 * m}}, {{dsec, 32 * m}}, true);   // secrets do not stay in the shared buffer
}

// The launches of one keyed EdDSA sign block whose inputs are on the device (msg_off: m + 1 offsets relative to msgs):
// ed_signset_sign_launch, or its screened form (keyset_forms.cu) when verdict != NULL, with the main kernels between ev0
// and ev1; then the nonces r are cleared from ws (ed_signset_ws_bytes(m) bytes).
int keyed_eddsa_sign_launches(Ctx& c, size_t m, const KeysetDev& d, const uint8_t* msgs, const u64* msg_off, const u32* idx,
                              const uint8_t* verdict, uint8_t* ws, uint8_t* sig, Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  const u32* gt = c.gtab[EB200_CURVE_ED25519];
  cudaError_t err =
      verdict ? keyset_ss_sign_screened_launch(m, verdict, d, msgs, msg_off, idx, gt, (u32*)ws, sig, L.st, ev0, ev1, &L.count)
              : ed_signset_sign_launch(m, d, msgs, msg_off, idx, gt, (u32*)ws, sig, L.st, ev0, ev1, &L.count);
  if (err != cudaSuccess) return cuda_fail(err, verdict ? "keyset_ss_sign_screened_launch" : "ed_signset_sign_launch");
  CK(cudaMemsetAsync(ws + ed_signset_nonce_offset(m), 0, ed_signset_nonce_bytes(m), L.st));   // the nonces r
  return EB200_OK;
}

// Keyed EdDSA sign of one block on one device of the set, chunked like eddsa_keyed_on (msg_off points at this block's
// first offset, offsets absolute).  Launches per chunk: keyed_eddsa_sign_launches.
int eddsa_sign_keyed_on(Ctx& c, const KeysetDev& d, size_t n, const uint8_t* msgs, const uint64_t* msg_off,
                        const u32* key_idx, uint8_t* sig) {
  int rc;
  const ChunkPlan P = make_plan(n);
  const size_t mbytes = (size_t)(msg_off[n] - msg_off[0]);
  const size_t off_bytes = (n + 1) * sizeof(uint64_t);
  const size_t base = align256(n * 68);            // sig | key_idx
  if ((rc = grow(&c.d_in, &c.d_in_cap, base + align256(off_bytes) + align256(mbytes + 1)))) return rc;
  const size_t ws_slot = align256(ed_signset_ws_bytes(P.max_m));
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (P.chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  uint8_t* dsig = c.d_in;
  u32* didx = (u32*)(dsig + 64 * n);
  uint64_t* doff = (uint64_t*)(c.d_in + base);
  uint8_t* dm = c.d_in + base + align256(off_bytes);
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {didx + lo, key_idx + lo, 4 * m};
      seg[1] = {doff + lo, msg_off + lo, (m + 1) * sizeof(uint64_t)};
      seg[2] = {dm + (msg_off[lo] - msg_off[0]), msgs + msg_off[lo], (size_t)(msg_off[lo + m] - msg_off[lo])};
      return 3;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      return keyed_eddsa_sign_launches(c, m, d, dm - msg_off[0], doff + lo, didx + lo, nullptr, c.d_ws + (size_t)slot * ws_slot,
                                       dsig + 64 * lo, L, c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {sig + 64 * lo, dsig + 64 * lo, 64 * m};
      return 1;
    });
}

// ---- curve25519 key sets: kernels in x25519_keyset.cu ------------------------------------------------------------------
// One device's copy: keys up, verdicts, Edwards images and tables, verdicts home.
int x25519_keyset_build_on(Ctx& c, eb200_keyset* ks, const uint8_t* pubx, uint8_t* key_status) {
  const size_t m = ks->m;
  const int W = (int)ks->W;
  int rc;
  KeysetDev& d = ks->dev[c.device];
  d.W = W;
  CK(cudaMalloc(&d.xy, 32 * m));
  CK(cudaMalloc(&d.kst, m));
  CK(cudaMalloc(&d.tab, ed_keyset_key_bytes(W) * m));
  if ((rc = grow(&c.d_in, &c.d_in_cap, 32 * m))) return rc;
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, m * ed_keyset_windows(W) * 24 * 4))) return rc;
  uint8_t* dx = c.d_in;
  return run_single(c, {{dx, pubx, 32 * m}},
    [&](Launch& L) {
      cudaError_t err = x25519_keyset_build_launch(m, d, dx, (u32*)c.d_ws, L.st, &L.count);
      return err == cudaSuccess ? EB200_OK : cuda_fail(err, "x25519_keyset_build_launch");
    },
    {{key_status, d.kst, m}}, {}, true);
}

// The launches of one keyed curve25519 derive block whose inputs are on the device: keyed main (between ev0 and ev1) and
// normalisation; then the private scalars k and the per-item results in ws (x25519_keyset_ws_bytes(m) bytes) are cleared.
int keyed_x25519_launches(size_t m, const KeysetDev& d, uint8_t* k, const u32* idx, uint8_t* ws, uint8_t* out, uint8_t* status,
                          Launch& L, cudaEvent_t ev0, cudaEvent_t ev1) {
  cudaError_t err = x25519_keyset_derive_launch(m, d, k, idx, (u32*)ws, out, status, L.st, ev0, ev1, &L.count);
  if (err != cudaSuccess) return cuda_fail(err, "x25519_keyset_derive_launch");
  CK(cudaMemsetAsync(k, 0, 32 * m, L.st));                           // the private scalars
  CK(cudaMemsetAsync(ws, 0, x25519_keyset_ws_bytes(m), L.st));       // the per-item results
  return EB200_OK;
}

// Keyed curve25519 derive of one block on one device of the set, chunked like mul_keyed_on.  Launches per chunk:
// keyed_x25519_launches.
int x25519_derive_keyed_on(Ctx& c, const KeysetDev& d, size_t n, const uint8_t* priv, const u32* key_idx, uint8_t* out,
                           uint8_t* status) {
  int rc;
  const ChunkPlan P = make_plan(n);
  const size_t idx_bytes = align256(n * 4), k_bytes = align256(n * 32);
  if ((rc = grow(&c.d_in, &c.d_in_cap, idx_bytes + k_bytes + n * 32))) return rc;
  const size_t ws_slot = align256(x25519_keyset_ws_bytes(P.max_m));
  if ((rc = grow(&c.d_ws, &c.d_ws_cap, (P.chunks > 1 ? 2 : 1) * ws_slot))) return rc;
  if ((rc = grow(&c.d_status, &c.d_status_cap, n))) return rc;
  u32* d_idx = (u32*)c.d_in;
  uint8_t *d_k = c.d_in + idx_bytes, *d_out = d_k + k_bytes;
  return run_chunked(c, P,
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {d_k + 32 * lo, priv + 32 * lo, 32 * m};
      seg[1] = {d_idx + lo, key_idx + lo, 4 * m};
      return 2;
    },
    [&](size_t lo, size_t m, Launch& L, int slot, int k) {
      return keyed_x25519_launches(m, d, d_k + 32 * lo, d_idx + lo, c.d_ws + (size_t)slot * ws_slot, d_out + 32 * lo,
                                   c.d_status + lo, L, c.ev_k0[k], c.ev_k1[k]);
    },
    [&](size_t lo, size_t m, Seg* seg) {
      seg[0] = {out + 32 * lo, d_out + 32 * lo, 32 * m};
      seg[1] = {status + lo, c.d_status + lo, m};
      return 2;
    });
}

// h < n for a 32-byte little-endian h (the keyed tables cover 253 bits)
bool ed_scalar_below_n(const uint8_t* h) {
  static const uint8_t n_le[32] = {0xed, 0xd3, 0xf5, 0x5c, 0x1a, 0x63, 0x12, 0x58, 0xd6, 0x9c, 0xf7, 0xa2, 0xde, 0xf9, 0xde, 0x14,
                                   0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x10};
  for (int b = 31; b >= 0; b--)
    if (h[b] != n_le[b]) return h[b] < n_le[b];
  return false;
}
// priv < n for a 32-byte big-endian curve25519 private key (the keyed tables cover 253 bits); most keys are decided by
// their first byte
bool x25519_priv_below_n(const uint8_t* k) {
  static const uint8_t n_be[32] = {0x10, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                   0x14, 0xde, 0xf9, 0xde, 0xa2, 0xf7, 0x9c, 0xd6, 0x58, 0x12, 0x63, 0x1a, 0x5c, 0xf5, 0xd3, 0xed};
  for (int b = 0; b < 32; b++)
    if (k[b] != n_be[b]) return k[b] < n_be[b];
  return false;
}

// Builds the set on every initialised device (build(ctx) per device) and registers it; on failure frees what was
// allocated and deletes ks.  eb200_last_timing: the slowest device's build, launches summed.
template <class Build>
int keyset_create_on_devices(eb200_keyset* ks, eb200_keyset** out, Build&& build) {
  int devs[MAX_DEV], nd;
  { std::lock_guard<std::mutex> lk(g_mu); nd = g_ndev; for (int i = 0; i < nd; i++) devs[i] = g_devs[i]; }
  if (nd == 0) { delete ks; return EB200_ERR_NOT_INIT; }
  t_pending = nullptr;
  eb200_timing tm = {};
  int rc = EB200_OK;
  for (int i = 0; i < nd && !rc; i++) {
    Ctx& c = g_ctx[devs[i]];
    std::lock_guard<std::mutex> lk(c.mu);
    cudaError_t e = cudaSetDevice(c.device);
    if (e != cudaSuccess) { rc = cuda_fail(e, "cudaSetDevice"); break; }
    ks->devs[ks->ndev++] = c.device;                 // listed first, so that a failed build frees what it allocated
    c.timing = eb200_timing{};
    rc = build(c);
    merge_timing(tm, c.timing);
  }
  t_timing = tm;
  if (rc) {
    keyset_free_device(ks);
    delete ks;
    return rc;
  }
  ks->live = true;
  { std::lock_guard<std::mutex> lk(g_ks_mu); g_keysets.push_back(ks); }
  *out = ks;
  return EB200_OK;
}
// ---- argument checks and dispatch of the keyed calls -------------------------------------------------------------------
// The kinds of set the keyed calls take.
enum KeyedKind { KK_ECDSA, KK_ED_PUBLIC, KK_ED_SIGNING, KK_X25519 };
bool keyed_kind_is(const eb200_keyset* ks, KeyedKind k) {
  switch (k) {
    case KK_ECDSA: return keyset_geom(ks->curve).limbs != 0;
    case KK_ED_PUBLIC: return ks->curve == EB200_CURVE_ED25519 && ks->kind == KS_PUBLIC;
    case KK_ED_SIGNING: return ks->curve == EB200_CURVE_ED25519 && ks->kind == KS_SIGNING;
    default: return ks->curve == EB200_CURVE_CURVE25519;
  }
}
// The fixed-base table the calls on a set of this kind use (0: none).
int keyed_table_curve(const eb200_keyset* ks, KeyedKind kind) {
  return kind == KK_ECDSA ? ks->curve : kind == KK_X25519 ? 0 : EB200_CURVE_ED25519;
}

// The checks of a keyed host call, in order: the set's kind, its lifetime, n = 0, ptrs_ok, then for every item its key
// index and item_ok(i).  Then fn(c, d, lo, m) for the blocks of the batch, sharded over the set's devices, with d the
// set's copy on c's device and the kind's fixed-base table loaded.
template <class ItemOk, class Fn>
int keyed_host_run(const eb200_keyset* ks, KeyedKind kind, size_t n, const u32* key_idx, bool ptrs_ok, ItemOk&& item_ok,
                   Fn&& fn) {
  if (!ks || !keyed_kind_is(ks, kind)) return EB200_ERR_ARG;
  if (!ks->live || !eb200_device_count()) return EB200_ERR_NOT_INIT;
  if (n == 0) return EB200_OK;
  if (!ptrs_ok || !key_idx) return EB200_ERR_ARG;
  for (size_t i = 0; i < n; i++) if (key_idx[i] >= ks->m || !item_ok(i)) return EB200_ERR_ARG;
  const int table = keyed_table_curve(ks, kind);
  return run_sharded_on(ks->devs, ks->ndev, n, [&](Ctx& c, size_t lo, size_t m) {
    const KeysetDev& d = ks->dev[c.device];
    if (!d.tab) return EB200_ERR_NOT_INIT;           // never a table pointer of another device
    int rc;
    if (table && (rc = ensure_table(c, table))) return rc;
    return fn(c, d, lo, m);
  });
}

// Body bytes of the workspace (keyed_dev_ws) of the device-pointer calls a set takes, n items:
//   ECDSA sets: keyed_mul_ws_bytes -- mul / mulAdd / derive and getKeyRecoveryParam as their host forms place it in
//     each chunk's slot, the keyed verify its keyed_verify_ws_bytes at the start;
//   EdDSA sets: gathered key bytes (32 n, raw messages only) | h (32 n: the hash, or the screened copies of h);
//   signing sets: ed_signset_ws_bytes, the sign launch's workspace;
//   curve25519 sets: screened private scalars (32 n) | x25519_keyset_ws_bytes, the derive launch's workspace.
size_t keyed_dev_body_bytes(const eb200_keyset* ks, size_t n) {
  if (keyset_geom(ks->curve).limbs) return keyed_mul_ws_bytes(ks->curve, n);
  if (ks->curve == EB200_CURVE_CURVE25519) return align256(32 * n) + x25519_keyset_ws_bytes(n);
  if (ks->kind == KS_SIGNING) return ed_signset_ws_bytes(n);
  return align256(32 * n) + 32 * n;
}

// The checks of a keyed device-pointer call, in order: the set's kind, its lifetime, n = 0, the pointers, the device
// that owns d_status.  Then run(c, L, d, idx, verdict, body) on the caller's stream, with d the set's copy on that
// device and the workspace's regions as keyed_dev_ws places them.
template <class Run>
int keyed_dev_run(const eb200_keyset* ks, KeyedKind kind, size_t n, bool ptrs_ok, uint8_t* d_status, void* d_workspace,
                  void* stream, Run&& run) {
  if (!ks || !keyed_kind_is(ks, kind)) return EB200_ERR_ARG;
  if (!ks->live || !eb200_device_count()) return EB200_ERR_NOT_INIT;
  if (n == 0) return EB200_OK;
  if (!ptrs_ok || !d_status || !d_workspace) return EB200_ERR_ARG;
  const Ctx* owner = ctx_of(d_status);
  if (!owner) return EB200_ERR_NOT_INIT;
  const KeysetDev& d = ks->dev[owner->device];
  if (!d.tab) return EB200_ERR_ARG;                // an initialised device that does not hold this set
  const KeyedDevWs Lw = keyed_dev_ws(n, 0);
  uint8_t* base = (uint8_t*)d_workspace;
  return run_dev(d_status, keyed_table_curve(ks, kind), stream, [&](Ctx& c, Launch& L) {
    return run(c, L, d, (u32*)(base + Lw.idx), base + Lw.verdict, base + Lw.prep);
  });
}

// The keyed device-pointer calls put a screen in front of their host form's launch function and a verdict merge behind
// it; these return the CUDA error of a failed one.
int index_screen(const eb200_keyset* ks, size_t n, const uint32_t* d_key_idx, u32* idx, uint8_t* vd, Launch& L) {
  cudaError_t err = keyset_index_screen_launch(n, d_key_idx, ks->m, idx, vd, L.st, &L.count);
  return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_index_screen_launch");
}
int range_screen(const eb200_keyset* ks, size_t n, const uint32_t* d_key_idx, const uint64_t* d_off, uint64_t len, u32* idx,
                 uint8_t* vd, Launch& L) {
  cudaError_t err = keyset_index_range_screen_launch(n, d_key_idx, ks->m, d_off, len, idx, vd, L.st, &L.count);
  return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_index_range_screen_launch");
}
int scalar_screen(const eb200_keyset* ks, size_t n, const uint32_t* d_key_idx, const uint8_t* d_k, bool big_endian, u32* idx,
                  uint8_t* k, uint8_t* vd, Launch& L) {
  cudaError_t err = keyset_index_scalar_screen_launch(n, d_key_idx, ks->m, d_k, big_endian, idx, k, vd, L.st, &L.count);
  return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_index_scalar_screen_launch");
}
// ol == 0: the verdicts replace the statuses; else they also zero the screened items' ol-byte rows of out.
int verdict_merge(size_t n, const uint8_t* vd, uint8_t* d_status, uint8_t* out, u32 ol, Launch& L) {
  cudaError_t err = ol ? keyset_verdict_merge_out_launch(n, vd, d_status, out, ol, L.st, &L.count)
                       : keyset_verdict_merge_launch(n, vd, d_status, L.st, &L.count);
  return err == cudaSuccess ? EB200_OK : cuda_fail(err, ol ? "keyset_verdict_merge_out_launch" : "keyset_verdict_merge_launch");
}

// Keyed mul / mulAdd / derive with device pointers: index screen, keyed_mul_launches, merge; derive clears the digit
// words and Jacobian results behind them.
int mul_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_k1, const uint8_t* d_k2, const uint32_t* d_key_idx,
                  uint8_t* d_out, uint8_t* d_status, void* d_workspace, void* stream, bool need_k1, bool derive) {
  return keyed_dev_run(ks, KK_ECDSA, n, d_k2 && (d_k1 || !need_k1) && d_key_idx && d_out, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      const int curve = ks->curve;
      const size_t ol = derive ? curve_len(curve) : 2 * curve_len(curve);
      int rc;
      if ((rc = index_screen(ks, n, d_key_idx, idx, vd, L)) ||
          (rc = keyed_mul_launches(c, curve, n, d, d_k1, d_k2, idx, body, d_out, d_status, derive, L, c.ev[EV_MAIN_BEGIN],
                                   c.ev[EV_MAIN_END])) ||
          (rc = verdict_merge(n, vd, d_status, d_out, (u32)ol, L)))
        return rc;
      if (derive) CK(cudaMemsetAsync(body, 0, keyed_mul_ws_bytes(curve, n), L.st));   // digit words, Jacobian results
      return EB200_OK;
    });
}

// The three keyed multiplication calls on host buffers: k1 == NULL (need_k1 false) is k2 times the key.
int mul_keyed_host(const eb200_keyset* ks, size_t n, const uint8_t* k1, const uint8_t* k2, const uint32_t* key_idx,
                   uint8_t* out, uint8_t* status, bool need_k1, bool derive) {
  return keyed_host_run(ks, KK_ECDSA, n, key_idx, k2 && (k1 || !need_k1) && out && status, every_item,
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      const size_t len = curve_len(ks->curve), ol = derive ? len : 2 * len;
      return mul_keyed_on(c, d, ks->curve, m, k1 ? k1 + lo * len : nullptr, k2 + lo * len, key_idx + lo, out + lo * ol,
                          status + lo, derive);
    });
}
}  // namespace

static void keysets_release_all() {
  std::lock_guard<std::mutex> lk(g_ks_mu);
  for (eb200_keyset* ks : g_keysets) keyset_free_device(ks);
  g_keysets.clear();
}

extern "C" {

int eb200_keyset_create(int curve, size_t m, const uint8_t* pub, uint32_t pub_fmt, uint32_t table_bits,
                        uint8_t* key_status, eb200_keyset** out) {
  if (out) *out = nullptr;
  if (!out || !pub || !key_status || m == 0 || m > 0xffffffffull || !fmt_ok(pub_fmt)) return EB200_ERR_ARG;
  if (table_bits && (table_bits < EB200_KEYSET_MIN_BITS || table_bits > EB200_KEYSET_MAX_BITS)) return EB200_ERR_ARG;
  if (!keyset_geom(curve).limbs) return EB200_ERR_UNSUPPORTED;      // the 25519 curves, and unknown ids as elsewhere
  if (!table_bits && !(table_bits = keyset_choose_bits(curve, m, EB200_KEYSET_DEFAULT_BUDGET))) {
    snprintf(g_err, sizeof g_err, "the tables of %zu keys do not fit the default budget at any width: pass table_bits", m);
    return EB200_ERR_ARG;
  }
  eb200_keyset* ks = new eb200_keyset;
  ks->curve = curve; ks->m = m; ks->W = table_bits; ks->fmt = pub_fmt;
  ks->device_bytes = 2 * curve_len(curve) * m + m + keyset_key_bytes(curve, (int)table_bits) * m;
  return keyset_create_on_devices(ks, out, [&](Ctx& c) { return keyset_build_on(c, ks, pub, key_status); });
}

int eb200_keyset_info(const eb200_keyset* ks, int* curve, size_t* m, uint32_t* table_bits, size_t* device_bytes) {
  if (!ks) return EB200_ERR_ARG;
  if (curve) *curve = ks->curve;
  if (m) *m = ks->m;
  if (table_bits) *table_bits = ks->W;
  if (device_bytes) *device_bytes = ks->device_bytes;
  return EB200_OK;
}

int eb200_keyset_destroy(eb200_keyset* ks) {
  if (!ks) return EB200_OK;
  {
    std::lock_guard<std::mutex> lk(g_ks_mu);
    for (size_t i = 0; i < g_keysets.size(); i++)
      if (g_keysets[i] == ks) { g_keysets.erase(g_keysets.begin() + i); break; }
    if (ks->live) keyset_free_device(ks);
  }
  delete ks;
  return EB200_OK;
}

int eb200_ecdsa_verify_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* e, const uint8_t* r,
                                   const uint8_t* s, const uint32_t* key_idx, uint8_t* status) {
  return keyed_host_run(ks, KK_ECDSA, n, key_idx, e && r && s && status, every_item,
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      const size_t len = curve_len(ks->curve);
      return verify_keyed_on(c, d, ks->curve, m, e + lo * len, r + lo * len, s + lo * len, key_idx + lo, status + lo);
    });
}

int eb200_ecdsa_verify_batch_keyed_der(const eb200_keyset* ks, size_t n, const uint8_t* e, const uint8_t* sigs,
                                       const uint64_t* sig_off, const uint32_t* key_idx, uint8_t* status) {
  return keyed_host_run(ks, KK_ECDSA, n, key_idx, e && sigs && sig_off && status,
    [&](size_t i) { return range_ok(sigs, sig_off, i); },
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      return verify_keyed_der_on(c, d, ks->curve, m, e + lo * curve_len(ks->curve), sigs, sig_off + lo, key_idx + lo,
                                 status + lo);
    });
}

size_t eb200_ecdsa_verify_keyed_workspace_bytes(const eb200_keyset* ks, size_t n) {
  if (!ks || !keyset_geom(ks->curve).limbs) return 0;
  return keyed_dev_ws(n, keyed_verify_ws_bytes(ks->curve, n)).total;
}

int eb200_ecdsa_verify_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_e, const uint8_t* d_r,
                                       const uint8_t* d_s, const uint32_t* d_key_idx, uint8_t* d_status,
                                       void* d_workspace, void* stream) {
  return keyed_dev_run(ks, KK_ECDSA, n, d_e && d_r && d_s && d_key_idx, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      int rc;
      if ((rc = index_screen(ks, n, d_key_idx, idx, vd, L)) ||
          (rc = keyed_verify_launches(c, ks->curve, n, d, d_e, d_r, d_s, idx, body, d_status, L, c.ev[EV_MAIN_BEGIN],
                                      c.ev[EV_MAIN_END])))
        return rc;
      return verdict_merge(n, vd, d_status, nullptr, 0, L);
    });
}

// workspace body (keyed_mul_ws_bytes): [keyed_verify_ws_bytes | r (n x len) | s (n x len) | screen verdicts (n)], the last
// three inside the Jacobian-result region (keyed_der_fits_jacobian)
int eb200_ecdsa_verify_batch_keyed_der_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_e, const uint8_t* d_sigs,
                                           uint64_t sigs_len, const uint64_t* d_sig_off, const uint32_t* d_key_idx,
                                           uint8_t* d_status, void* d_workspace, void* stream) {
  return keyed_dev_run(ks, KK_ECDSA, n, d_e && d_sig_off && d_key_idx && (d_sigs || !sigs_len), d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      const int curve = ks->curve;
      const size_t len = curve_len(curve);
      uint8_t *r = body + keyed_verify_ws_bytes(curve, n), *s = r + len * n, *pre = s + len * n;
      int rc = range_screen(ks, n, d_key_idx, d_sig_off, sigs_len, idx, pre, L);
      if (rc) return rc;
      return keyed_der_launches(c, curve, n, d, d_e, d_sigs, (const unsigned long long*)d_sig_off, idx, pre, r, s, vd, body,
                                d_status, L, c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
    });
}

int eb200_scalar_mul_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* k, const uint32_t* key_idx, uint8_t* out_xy,
                                 uint8_t* status) {
  return mul_keyed_host(ks, n, nullptr, k, key_idx, out_xy, status, false, false);
}

int eb200_mul_add_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* k1, const uint8_t* k2, const uint32_t* key_idx,
                              uint8_t* out_xy, uint8_t* status) {
  return mul_keyed_host(ks, n, k1, k2, key_idx, out_xy, status, true, false);
}

int eb200_ecdh_derive_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* priv, const uint32_t* key_idx, uint8_t* out_x,
                                  uint8_t* status) {
  return mul_keyed_host(ks, n, nullptr, priv, key_idx, out_x, status, false, true);
}

int eb200_ecdsa_recovery_param_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* e, const uint8_t* r,
                                           const uint8_t* s, const uint32_t* key_idx, uint8_t* out_recid, uint8_t* status) {
  return keyed_host_run(ks, KK_ECDSA, n, key_idx, e && r && s && out_recid && status, every_item,
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      const size_t len = curve_len(ks->curve);
      return recovery_param_keyed_on(c, d, ks->curve, m, e + lo * len, r + lo * len, s + lo * len, key_idx + lo,
                                     out_recid + lo, status + lo);
    });
}

int eb200_eddsa_keyset_create(size_t m, const uint8_t* A, uint32_t table_bits, uint8_t* key_status, eb200_keyset** out) {
  if (out) *out = nullptr;
  if (!out || !A || !key_status || m == 0 || m > 0xffffffffull) return EB200_ERR_ARG;
  if (table_bits && (table_bits < EB200_KEYSET_MIN_BITS || table_bits > EB200_KEYSET_MAX_BITS)) return EB200_ERR_ARG;
  if (!table_bits && !(table_bits = ed_keyset_choose_bits(m, EB200_KEYSET_DEFAULT_BUDGET))) {
    snprintf(g_err, sizeof g_err, "the tables of %zu keys do not fit the default budget at any width: pass table_bits", m);
    return EB200_ERR_ARG;
  }
  eb200_keyset* ks = new eb200_keyset;
  ks->curve = EB200_CURVE_ED25519; ks->m = m; ks->W = table_bits;
  ks->device_bytes = 32 * m + m + ed_keyset_key_bytes((int)table_bits) * m;
  return keyset_create_on_devices(ks, out, [&](Ctx& c) { return ed_keyset_build_on(c, ks, A, key_status); });
}

int eb200_eddsa_verify_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* R, const uint8_t* S, const uint8_t* h,
                                   const uint32_t* key_idx, uint8_t* status) {
  return keyed_host_run(ks, KK_ED_PUBLIC, n, key_idx, R && S && h && status,
    [&](size_t i) { return ed_scalar_below_n(h + 32 * i); },
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      return eddsa_keyed_on(c, d, m, R + 32 * lo, S + 32 * lo, h + 32 * lo, nullptr, nullptr, key_idx + lo, status + lo);
    });
}

int eb200_eddsa_verify_batch_keyed_msgs(const eb200_keyset* ks, size_t n, const uint8_t* R, const uint8_t* S,
                                        const uint8_t* msgs, const uint64_t* msg_off, const uint32_t* key_idx,
                                        uint8_t* status) {
  return keyed_host_run(ks, KK_ED_PUBLIC, n, key_idx, R && S && msg_off && status,
    [&](size_t i) { return range_ok(msgs, msg_off, i); },
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      return eddsa_keyed_on(c, d, m, R + 32 * lo, S + 32 * lo, nullptr, or_empty(msgs), msg_off + lo, key_idx + lo, status + lo);
    });
}

int eb200_eddsa_signing_set_create(size_t m, const uint8_t* secrets, uint8_t* out_pub, eb200_keyset** out) {
  if (out) *out = nullptr;
  if (!out || !secrets || m == 0 || m > 0xffffffffull) return EB200_ERR_ARG;
  eb200_keyset* ks = new eb200_keyset;
  ks->curve = EB200_CURVE_ED25519; ks->kind = KS_SIGNING; ks->m = m;
  ks->device_bytes = (32 + ED_SIGNSET_KEY_BYTES) * m;
  return keyset_create_on_devices(ks, out, [&](Ctx& c) { return ed_signset_build_on(c, ks, secrets, out_pub); });
}

int eb200_eddsa_sign_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* msgs, const uint64_t* msg_off,
                                 const uint32_t* key_idx, uint8_t* out_sig, uint8_t* status) {
  int rc = keyed_host_run(ks, KK_ED_SIGNING, n, key_idx, msg_off && out_sig && status,
    [&](size_t i) { return range_ok(msgs, msg_off, i); },
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      return eddsa_sign_keyed_on(c, d, m, or_empty(msgs), msg_off + lo, key_idx + lo, out_sig + 64 * lo);
    });
  if (rc == EB200_OK && n) memset(status, EB200_ST_TRUE, n);         // the reference cannot fail here
  return rc;
}

int eb200_x25519_keyset_create(size_t m, const uint8_t* pubx, uint32_t table_bits, uint8_t* key_status, eb200_keyset** out) {
  if (out) *out = nullptr;
  if (!out || !pubx || !key_status || m == 0 || m > 0xffffffffull) return EB200_ERR_ARG;
  if (table_bits && (table_bits < EB200_KEYSET_MIN_BITS || table_bits > EB200_KEYSET_MAX_BITS)) return EB200_ERR_ARG;
  if (!table_bits && !(table_bits = ed_keyset_choose_bits(m, EB200_KEYSET_DEFAULT_BUDGET))) {
    snprintf(g_err, sizeof g_err, "the tables of %zu keys do not fit the default budget at any width: pass table_bits", m);
    return EB200_ERR_ARG;
  }
  eb200_keyset* ks = new eb200_keyset;
  ks->curve = EB200_CURVE_CURVE25519; ks->m = m; ks->W = table_bits;
  ks->device_bytes = 32 * m + m + ed_keyset_key_bytes((int)table_bits) * m;
  return keyset_create_on_devices(ks, out, [&](Ctx& c) { return x25519_keyset_build_on(c, ks, pubx, key_status); });
}

int eb200_x25519_derive_batch_keyed(const eb200_keyset* ks, size_t n, const uint8_t* priv, const uint32_t* key_idx,
                                    uint8_t* out_x, uint8_t* status) {
  return keyed_host_run(ks, KK_X25519, n, key_idx, priv && out_x && status,
    [&](size_t i) { return x25519_priv_below_n(priv + 32 * i); },
    [&](Ctx& c, const KeysetDev& d, size_t lo, size_t m) {
      return x25519_derive_keyed_on(c, d, m, priv + 32 * lo, key_idx + lo, out_x + 32 * lo, status + lo);
    });
}

size_t eb200_keyset_dev_workspace_bytes(const eb200_keyset* ks, size_t n) {
  if (!ks) return 0;
  return keyed_dev_ws(n, keyed_dev_body_bytes(ks, n)).total;
}

int eb200_scalar_mul_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_k, const uint32_t* d_key_idx,
                                     uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace, void* stream) {
  return mul_keyed_dev(ks, n, nullptr, d_k, d_key_idx, d_out_xy, d_status, d_workspace, stream, false, false);
}

int eb200_mul_add_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_k1, const uint8_t* d_k2,
                                  const uint32_t* d_key_idx, uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace,
                                  void* stream) {
  return mul_keyed_dev(ks, n, d_k1, d_k2, d_key_idx, d_out_xy, d_status, d_workspace, stream, true, false);
}

int eb200_ecdh_derive_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_priv, const uint32_t* d_key_idx,
                                      uint8_t* d_out_x, uint8_t* d_status, void* d_workspace, void* stream) {
  return mul_keyed_dev(ks, n, nullptr, d_priv, d_key_idx, d_out_x, d_status, d_workspace, stream, false, true);
}

int eb200_ecdsa_recovery_param_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_e, const uint8_t* d_r,
                                               const uint8_t* d_s, const uint32_t* d_key_idx, uint8_t* d_out_recid,
                                               uint8_t* d_status, void* d_workspace, void* stream) {
  return keyed_dev_run(ks, KK_ECDSA, n, d_e && d_r && d_s && d_key_idx && d_out_recid, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      int rc;
      if ((rc = index_screen(ks, n, d_key_idx, idx, vd, L)) ||
          (rc = keyed_rp_launches(c, ks->curve, n, d, d_e, d_r, d_s, idx, body, d_out_recid, d_status, L, c.ev[EV_MAIN_BEGIN],
                                  c.ev[EV_MAIN_END])))
        return rc;
      return verdict_merge(n, vd, d_status, d_out_recid, 1, L);
    });
}

// workspace body: [unused (32 n) | screened h (32 n)]
int eb200_eddsa_verify_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_R, const uint8_t* d_S,
                                       const uint8_t* d_h, const uint32_t* d_key_idx, uint8_t* d_status, void* d_workspace,
                                       void* stream) {
  return keyed_dev_run(ks, KK_ED_PUBLIC, n, d_R && d_S && d_h && d_key_idx, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      uint8_t* h = body + align256(32 * n);
      int rc;
      if ((rc = scalar_screen(ks, n, d_key_idx, d_h, false, idx, h, vd, L)) ||
          (rc = keyed_eddsa_verify_launches(c, n, d, d_R, d_S, h, nullptr, nullptr, nullptr, idx, nullptr, d_status, L,
                                            c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END])))
        return rc;
      return verdict_merge(n, vd, d_status, nullptr, 0, L);
    });
}

// workspace body: [gathered key bytes (32 n) | h (32 n)]
int eb200_eddsa_verify_batch_keyed_msgs_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_R, const uint8_t* d_S,
                                            const uint8_t* d_msgs, uint64_t msgs_len, const uint64_t* d_msg_off,
                                            const uint32_t* d_key_idx, uint8_t* d_status, void* d_workspace, void* stream) {
  return keyed_dev_run(ks, KK_ED_PUBLIC, n, d_R && d_S && d_msg_off && d_key_idx && (d_msgs || !msgs_len), d_status,
                       d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      int rc;
      if ((rc = range_screen(ks, n, d_key_idx, d_msg_off, msgs_len, idx, vd, L)) ||
          (rc = keyed_eddsa_verify_launches(c, n, d, d_R, d_S, body + align256(32 * n), body, d_msgs, d_msg_off, idx, vd,
                                            d_status, L, c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END])))
        return rc;
      return verdict_merge(n, vd, d_status, nullptr, 0, L);
    });
}

// workspace body: the sign launch's (ed_signset_ws_bytes)
int eb200_eddsa_sign_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_msgs, uint64_t msgs_len,
                                     const uint64_t* d_msg_off, const uint32_t* d_key_idx, uint8_t* d_out_sig,
                                     uint8_t* d_status, void* d_workspace, void* stream) {
  return keyed_dev_run(ks, KK_ED_SIGNING, n, d_msg_off && d_key_idx && d_out_sig && (d_msgs || !msgs_len), d_status,
                       d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      int rc;
      if ((rc = range_screen(ks, n, d_key_idx, d_msg_off, msgs_len, idx, vd, L)) ||
          (rc = keyed_eddsa_sign_launches(c, n, d, d_msgs, d_msg_off, idx, vd, body, d_out_sig, L, c.ev[EV_MAIN_BEGIN],
                                          c.ev[EV_MAIN_END])))
        return rc;
      CK(cudaMemsetAsync(d_status, EB200_ST_TRUE, n, L.st));          // the reference cannot fail here
      return verdict_merge(n, vd, d_status, d_out_sig, 64, L);
    });
}

// workspace body: [screened private scalars (32 n) | the derive launch's (x25519_keyset_ws_bytes)]
int eb200_x25519_derive_batch_keyed_dev(const eb200_keyset* ks, size_t n, const uint8_t* d_priv, const uint32_t* d_key_idx,
                                        uint8_t* d_out_x, uint8_t* d_status, void* d_workspace, void* stream) {
  return keyed_dev_run(ks, KK_X25519, n, d_priv && d_key_idx && d_out_x, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, const KeysetDev& d, u32* idx, uint8_t* vd, uint8_t* body) {
      uint8_t* k = body;
      int rc;
      if ((rc = scalar_screen(ks, n, d_key_idx, d_priv, true, idx, k, vd, L)) ||
          (rc = keyed_x25519_launches(n, d, k, idx, body + align256(32 * n), d_out_x, d_status, L, c.ev[EV_MAIN_BEGIN],
                                      c.ev[EV_MAIN_END])))
        return rc;
      return verdict_merge(n, vd, d_status, d_out_x, 32, L);
    });
}

}  // extern "C"

// ---- device-pointer forms of the unkeyed calls ---------------------------------------------------------------------------
// Each runs its host form's launch sequence (the *_launches functions above) on the caller's stream through run_dev, with
// the workspace regions as dev_ws places them, and the calls with variable-length ranges put a range screen in front and
// a verdict merge behind it.
namespace {
// The workspace of the unkeyed device-pointer calls on `curve`, n items.  Every call places its regions from the start:
//   verify, recover, getKeyRecoveryParam, mul / mulAdd / derive, ed25519 verify: ws_layout(curve, n) (on ed25519 its
//     first region is the verify kernel's per-item tables);
//   then [verdict, rows): per-item bytes -- range verdicts (DER verify, ed25519 messages, EdDSA sign) or keygen's
//     multiplication statuses;
//   then [rows, total): 2 len bytes per item -- decoded r, s (DER verify), x || y (derive), k G (keygen without
//     d_out_pub_xy), h (ed25519 messages, 32 bytes per item);
//   sign alone places sign_ws(curve, n) from the start.
struct DevWs { size_t verdict, rows, total; };
DevWs dev_ws(int curve, size_t n) {
  DevWs D;
  D.verdict = ws_layout(curve, n).total;
  D.rows = D.verdict + align256(n);
  D.total = D.rows + align256(2 * curve_len(curve) * n);
  const size_t sign = sign_ws(curve, n).total;
  if (sign > D.total) D.total = sign;
  return D;
}

// n = 0 and the argument checks of an unkeyed device-pointer call, after its curve check: DEV_GO to go on, else what to
// return -- EB200_OK (n = 0 with a device) or EB200_ERR_NOT_INIT (without), EB200_ERR_ARG for a refused argument.
constexpr int DEV_GO = 1;
int dev_checks(size_t n, bool args_ok) {
  if (n == 0) return eb200_device_count() ? EB200_OK : EB200_ERR_NOT_INIT;
  return args_ok ? DEV_GO : EB200_ERR_ARG;
}

int sign_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_priv, const uint8_t* d_k, const uint8_t* d_pers,
             size_t pers_len, bool pers, uint32_t flags, uint8_t* d_out_r, uint8_t* d_out_s, uint8_t* d_out_recid,
             uint8_t* d_status, void* d_workspace, void* stream, bool need_k) {
  if (!curve_ok(curve)) return EB200_ERR_UNSUPPORTED;
  int rc = dev_checks(n, d_e && d_priv && (d_k || !need_k) && d_out_r && d_out_s && d_out_recid && d_status && d_workspace &&
                             (!pers || ((d_pers || !pers_len) && pers_len <= (1u << 20))));
  if (rc != DEV_GO) return rc;
  return run_dev(d_status, curve, stream, [&](Ctx& c, Launch& L) {
    // pers with pers_len = 0: the kernel reads no byte of it, but a non-NULL pointer selects the pers loop
    const uint8_t* pp = !pers ? nullptr : pers_len ? d_pers : d_status;
    uint8_t* base = (uint8_t*)d_workspace;
    int rc2 = sign_launches(c, curve, n, d_e, d_priv, need_k ? d_k : nullptr, pp, pers ? pers_len : 0,
                            flags & EB200_SIGN_CANONICAL, base, d_out_r, d_out_s, d_out_recid, d_status, L,
                            c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
    if (rc2) return rc2;
    CK(cudaMemsetAsync(base, 0, sign_ws(curve, n).total, L.st));     // nonces, k G, the finish kernel's scratch
    return EB200_OK;
  });
}

int mul_add_dev(int curve, size_t n, const uint8_t* d_k1, const uint8_t* d_k2, const uint8_t* d_pts, uint8_t* d_out,
                uint8_t* d_status, void* d_workspace, void* stream, bool args_ok, bool derive) {
  if (!curve_ok(curve)) return EB200_ERR_UNSUPPORTED;
  int rc = dev_checks(n, args_ok && d_k2 && d_out && d_status && d_workspace);
  if (rc != DEV_GO) return rc;
  return run_dev(d_status, curve, stream, [&](Ctx& c, Launch& L) {
    const size_t len = curve_len(curve);
    const DevWs D = dev_ws(curve, n);
    uint8_t* base = (uint8_t*)d_workspace;
    int rc2 = mul_add_launches(c, curve, n, d_k1, d_k2, d_pts, base, derive ? base + D.rows : d_out, d_status, derive, L,
                               c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
    if (rc2 || !derive) return rc2;
    CK(cudaMemcpy2DAsync(d_out, len, base + D.rows, 2 * len, len, n, cudaMemcpyDeviceToDevice, L.st));   // x of x || y
    CK(cudaMemsetAsync(base, 0, D.total, L.st));     // the scalars' digit words, the per-item tables, x || y
    return EB200_OK;
  });
}

// The range-screened calls: the range screen into the verdicts at dev_ws's `verdict`, then run(c, L, verdict, base).
template <class Run>
int range_screened_dev(int table_curve, size_t n, const uint64_t* d_off, uint64_t len, uint8_t* d_status, void* d_workspace,
                       void* stream, Run&& run) {
  return run_dev(d_status, table_curve, stream, [&](Ctx& c, Launch& L) {
    uint8_t* base = (uint8_t*)d_workspace;
    uint8_t* verdict = base + dev_ws(table_curve, n).verdict;
    cudaError_t err = unkeyed_range_screen_launch(n, d_off, len, verdict, L.st, &L.count);
    if (err != cudaSuccess) return cuda_fail(err, "unkeyed_range_screen_launch");
    return run(c, L, verdict, base);
  });
}
}  // namespace

extern "C" {

size_t eb200_dev_workspace_bytes(int curve, size_t n) {
  if (!curve_ok(curve)) return 0;
  return dev_ws(curve, n).total;
}

int eb200_ecdsa_sign_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_priv, uint32_t flags, uint8_t* d_out_r,
                               uint8_t* d_out_s, uint8_t* d_out_recid, uint8_t* d_status, void* d_workspace, void* stream) {
  return sign_dev(curve, n, d_e, d_priv, nullptr, nullptr, 0, false, flags, d_out_r, d_out_s, d_out_recid, d_status,
                  d_workspace, stream, false);
}

int eb200_ecdsa_sign_batch_k_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_priv, const uint8_t* d_k,
                                 uint32_t flags, uint8_t* d_out_r, uint8_t* d_out_s, uint8_t* d_out_recid, uint8_t* d_status,
                                 void* d_workspace, void* stream) {
  return sign_dev(curve, n, d_e, d_priv, d_k, nullptr, 0, false, flags, d_out_r, d_out_s, d_out_recid, d_status, d_workspace,
                  stream, true);
}

int eb200_ecdsa_sign_batch_pers_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_priv, const uint8_t* d_pers,
                                    size_t pers_len, uint32_t flags, uint8_t* d_out_r, uint8_t* d_out_s, uint8_t* d_out_recid,
                                    uint8_t* d_status, void* d_workspace, void* stream) {
  return sign_dev(curve, n, d_e, d_priv, nullptr, d_pers, pers_len, true, flags, d_out_r, d_out_s, d_out_recid, d_status,
                  d_workspace, stream, false);
}

// workspace: the multiplication's statuses at dev_ws's `verdict`, k G at `rows` when d_out_pub_xy is NULL; both cleared
int eb200_ec_keygen_batch_dev(int curve, size_t n, const uint8_t* d_entropy, size_t entropy_len, const uint8_t* d_pers,
                              size_t pers_len, uint8_t* d_out_priv, uint8_t* d_out_pub_xy, uint8_t* d_status, void* d_workspace,
                              void* stream) {
  if (!curve_ok(curve)) return EB200_ERR_UNSUPPORTED;
  int rc = dev_checks(n, d_entropy && entropy_len && d_out_priv && d_status && d_workspace && (d_pers || !pers_len) &&
                             pers_len <= (1u << 20) && entropy_len <= (1u << 16));
  if (rc != DEV_GO) return rc;
  return run_dev(d_status, curve, stream, [&](Ctx& c, Launch& L) {
    const DevWs D = dev_ws(curve, n);
    uint8_t* base = (uint8_t*)d_workspace;
    int rc2 = keygen_launches(c, curve, n, d_entropy, entropy_len, pers_len ? d_pers : nullptr, pers_len, d_out_priv,
                              d_out_pub_xy ? d_out_pub_xy : base + D.rows, d_status, base + D.verdict, L, c.ev[EV_MAIN_BEGIN],
                              c.ev[EV_MAIN_END]);
    if (rc2) return rc2;
    CK(cudaMemsetAsync(base + D.verdict, 0, D.total - D.verdict, L.st));
    return EB200_OK;
  });
}

int eb200_ecdsa_recover_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r, const uint8_t* d_s,
                                  const uint8_t* d_recid, uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace, void* stream) {
  if (!curve_ok(curve)) return EB200_ERR_UNSUPPORTED;
  int rc = dev_checks(n, d_e && d_r && d_s && d_recid && d_out_xy && d_status && d_workspace);
  if (rc != DEV_GO) return rc;
  if (curve == EB200_CURVE_ED25519) return EB200_ERR_UNSUPPORTED;      // as eb200_ecdsa_recover_batch
  return run_dev(d_status, curve, stream, [&](Ctx& c, Launch& L) {
    return recover_launches(c, curve, n, d_e, d_r, d_s, d_recid, (uint8_t*)d_workspace, d_out_xy, d_status, L,
                            c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
  });
}

int eb200_ecdsa_recovery_param_batch_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_r, const uint8_t* d_s,
                                         const uint8_t* d_q_xy, uint8_t* d_out_recid, uint8_t* d_status, void* d_workspace,
                                         void* stream) {
  if (!curve_ok(curve)) return EB200_ERR_UNSUPPORTED;
  int rc = dev_checks(n, d_e && d_r && d_s && d_q_xy && d_out_recid && d_status && d_workspace);
  if (rc != DEV_GO) return rc;
  if (curve == EB200_CURVE_ED25519) return EB200_ERR_UNSUPPORTED;      // as eb200_ecdsa_recovery_param_batch
  return run_dev(d_status, curve, stream, [&](Ctx& c, Launch& L) {
    return recovery_param_launches(c, curve, n, d_e, d_r, d_s, d_q_xy, d_out_recid, d_status, (uint8_t*)d_workspace, L,
                                   c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
  });
}

int eb200_scalar_mul_batch_dev(int curve, size_t n, const uint8_t* d_k, const uint8_t* d_points_xy, uint8_t* d_out_xy,
                               uint8_t* d_status, void* d_workspace, void* stream) {
  return mul_add_dev(curve, n, nullptr, d_k, d_points_xy, d_out_xy, d_status, d_workspace, stream, true, false);
}

int eb200_mul_add_batch_dev(int curve, size_t n, const uint8_t* d_k1, const uint8_t* d_k2, const uint8_t* d_p2_xy,
                            uint8_t* d_out_xy, uint8_t* d_status, void* d_workspace, void* stream) {
  return mul_add_dev(curve, n, d_k1, d_k2, d_p2_xy, d_out_xy, d_status, d_workspace, stream, d_k1 && d_p2_xy, false);
}

int eb200_ecdh_derive_batch_dev(int curve, size_t n, const uint8_t* d_priv, const uint8_t* d_pub_xy, uint8_t* d_out_x,
                                uint8_t* d_status, void* d_workspace, void* stream) {
  return mul_add_dev(curve, n, nullptr, d_priv, d_pub_xy, d_out_x, d_status, d_workspace, stream, d_pub_xy != nullptr, true);
}

int eb200_x25519_mul_batch_dev(size_t n, const uint8_t* d_k, const uint8_t* d_px, uint8_t* d_out_x, uint8_t* d_status,
                               void* stream) {
  int rc = dev_checks(n, d_k && d_px && d_out_x && d_status);
  if (rc != DEV_GO) return rc;
  return run_dev(d_status, 0, stream, [&](Ctx& c, Launch& L) {
    return x25519_launches(n, d_k, d_px, d_out_x, d_status, false, L, c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
  });
}

// workspace: launch_verify's (ws_layout), the range verdicts, the decoded r and s
int eb200_ecdsa_verify_batch_der_dev(int curve, size_t n, const uint8_t* d_e, const uint8_t* d_sigs, uint64_t sigs_len,
                                     const uint64_t* d_sig_off, const uint8_t* d_pub, uint32_t pub_fmt, uint8_t* d_status,
                                     void* d_workspace, void* stream) {
  if (!curve_ok(curve) || !fmt_ok(pub_fmt)) return EB200_ERR_UNSUPPORTED;
  int rc = dev_checks(n, d_e && (d_sigs || !sigs_len) && d_sig_off && d_pub && d_status && d_workspace);
  if (rc != DEV_GO) return rc;
  return range_screened_dev(curve, n, d_sig_off, sigs_len, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, uint8_t* verdict, uint8_t* base) {
      const size_t len = curve_len(curve);
      uint8_t* r = base + dev_ws(curve, n).rows;
      int rc2 = launch_verify(c, curve, n, d_e, r, r + len * n, d_pub, pub_fmt, d_status, base, L, c.ev[EV_MAIN_BEGIN],
                              c.ev[EV_MAIN_END], d_sigs, (const unsigned long long*)d_sig_off, verdict);
      if (rc2) return rc2;
      cudaError_t err = keyset_verdict_merge_launch(n, verdict, d_status, L.st, &L.count);
      return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_verdict_merge_launch");
    });
}

// workspace: the verify kernel's tables (ws_layout), the range verdicts, h
int eb200_eddsa_verify_batch_msgs_dev(size_t n, const uint8_t* d_R, const uint8_t* d_S, const uint8_t* d_A,
                                      const uint8_t* d_msgs, uint64_t msgs_len, const uint64_t* d_msg_off, uint8_t* d_status,
                                      void* d_workspace, void* stream) {
  int rc = dev_checks(n, d_R && d_S && d_A && (d_msgs || !msgs_len) && d_msg_off && d_status && d_workspace);
  if (rc != DEV_GO) return rc;
  return range_screened_dev(EB200_CURVE_ED25519, n, d_msg_off, msgs_len, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, uint8_t* verdict, uint8_t* base) {
      uint8_t* h = base + dev_ws(EB200_CURVE_ED25519, n).rows;
      int rc2 = eddsa_verify_launches(c, n, d_R, d_S, d_A, h, d_msgs, d_msg_off, verdict, (u32*)base, d_status, L,
                                      c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
      if (rc2) return rc2;
      cudaError_t err = keyset_verdict_merge_launch(n, verdict, d_status, L.st, &L.count);
      return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_verdict_merge_launch");
    });
}

// workspace: the range verdicts alone (the sign kernel keeps its secrets in registers and local memory)
int eb200_eddsa_sign_batch_dev(size_t n, const uint8_t* d_secrets, const uint8_t* d_msgs, uint64_t msgs_len,
                               const uint64_t* d_msg_off, uint8_t* d_out_sig, uint8_t* d_out_pub, uint8_t* d_status,
                               void* d_workspace, void* stream) {
  int rc = dev_checks(n, d_secrets && (d_msgs || !msgs_len) && d_msg_off && d_out_sig && d_status && d_workspace);
  if (rc != DEV_GO) return rc;
  return range_screened_dev(EB200_CURVE_ED25519, n, d_msg_off, msgs_len, d_status, d_workspace, stream,
    [&](Ctx& c, Launch& L, uint8_t* verdict, uint8_t*) {
      int rc2 = eddsa_sign_launches(c, n, d_secrets, d_msgs, d_msg_off, verdict, d_out_sig, d_out_pub, d_status, L,
                                    c.ev[EV_MAIN_BEGIN], c.ev[EV_MAIN_END]);
      if (rc2) return rc2;
      cudaError_t err = keyset_verdict_merge_out_launch(n, verdict, d_status, d_out_sig, 64, L.st, &L.count);
      return err == cudaSuccess ? EB200_OK : cuda_fail(err, "keyset_verdict_merge_out_launch");
    });
}

}  // extern "C"
