// keyset.cu -- kernels of eb200_keyset_create (classify -> window bases -> table windows) and of
// eb200_ecdsa_verify_batch_keyed (main: one table lookup and mixed add per window, no doubling; replay: the items
// whose key is off the curve, through the reference's own schedule).  Bodies: ecdsa_keyset_body.cuh.
//
// A translation unit of its own for the reason recovery_param.cu gives: kernels added to eb200.cu's module change
// NVVM's inlining into the 255-register p384 / p521 kernels there.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include "../../include/elliptic_b200.h"
#include "kernel_bounds.h"
#include "keyset.h"

// The bodies' out-of-line helpers are external functions that eb200.cu defines too: the unnamed namespace keeps this
// unit's copies to itself.
namespace {
#include "ecdsa_k256_body.cuh"
#include "ecdsa_k256_replay.cuh"
#include "ecdsa_sw_body.cuh"
#include "ecdsa_sw_replay.cuh"
#include "ecdsa_keyset_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(128)
k256_keyset_classify_kernel(size_t m, const uint8_t* __restrict__ xy, const uint8_t* __restrict__ pre, uint8_t* __restrict__ kst) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) kst[k] = k256_ks_classify_item(k, xy, pre);
}
__global__ void __launch_bounds__(128)
k256_keyset_bases_kernel(size_t m, const uint8_t* __restrict__ xy, const uint8_t* __restrict__ kst, int W, int windows,
                         u32* __restrict__ bases) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) k256_ks_bases_item(k, xy, kst, W, windows, bases);
}
__global__ void __launch_bounds__(128)
k256_keyset_window_kernel(size_t m, const uint8_t* __restrict__ kst, int W, int windows, const u32* __restrict__ bases,
                          u32* __restrict__ tab) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m * windows) k256_ks_window_item(t, kst, W, windows, bases, tab);
}
__global__ void __launch_bounds__(EB_VERIFY_BLOCK, EB_VERIFY_MINBLOCKS)
k256_verify_keyed_kernel(size_t N, const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, int W, int windows,
                         const u32* __restrict__ ktab, const uint8_t* __restrict__ r, const u32* __restrict__ ws,
                         const u32* __restrict__ gtab, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = k256_verify_keyed_item(i, N, key_idx, kst, W, windows, ktab, r, ws, gtab);
}
__global__ void __launch_bounds__(128)
k256_replay_keyed_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s,
                         const u32* __restrict__ key_idx, const uint8_t* __restrict__ xy, const u32* __restrict__ tab,
                         uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = rp_verify_item(0, e + 32 * i, r + 32 * i, s + 32 * i, xy + 64 * (size_t)key_idx[i], tab);
}

template <class C>
__global__ void __launch_bounds__(128)
sw_keyset_classify_kernel(size_t m, const uint8_t* __restrict__ xy, const uint8_t* __restrict__ pre, uint8_t* __restrict__ kst) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) kst[k] = SWKeyed<C>::classify_item(k, xy, pre);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_keyset_bases_kernel(size_t m, const uint8_t* __restrict__ xy, const uint8_t* __restrict__ kst, int W, int windows,
                       u32* __restrict__ bases) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) SWKeyed<C>::bases_item(k, xy, kst, W, windows, bases);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_keyset_window_kernel(size_t m, const uint8_t* __restrict__ kst, int W, int windows, const u32* __restrict__ bases,
                        u32* __restrict__ tab) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m * windows) SWKeyed<C>::window_item(t, kst, W, windows, bases, tab);
}
template <class C>
__global__ void __launch_bounds__(128, (C::N <= 8) ? EB_SW_MINBLOCKS8 : EB_SW_MINBLOCKS_BIG)
sw_verify_keyed_kernel(size_t N, const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, int W, int windows,
                       const u32* __restrict__ ktab, const uint8_t* __restrict__ r, const u32* __restrict__ ws,
                       const u32* __restrict__ gtab, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = SWKeyed<C>::verify_keyed_item(i, N, key_idx, kst, W, windows, ktab, r, ws, gtab);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_replay_keyed_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r, const uint8_t* __restrict__ s,
                       const u32* __restrict__ key_idx, const uint8_t* __restrict__ xy, const u32* __restrict__ tab,
                       uint8_t* __restrict__ status) {
  constexpr size_t LEN = C::LEN;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = SWReplay<C>::verify_item(0, e + LEN * i, r + LEN * i, s + LEN * i, xy + 2 * LEN * (size_t)key_idx[i], tab);
}

namespace {
// launch, check, count
#define KS_LAUNCH(...)                                        \
  do {                                                        \
    __VA_ARGS__;                                              \
    cudaError_t err_ = cudaGetLastError();                    \
    if (err_ != cudaSuccess) return err_;                     \
    ++*launches;                                              \
  } while (0)

unsigned blocks128(size_t threads) { return (unsigned)((threads + 127) / 128); }

template <class C>
cudaError_t sw_build(int curve, size_t m, const KeysetDev& k, const uint8_t* pre, u32* bases, cudaStream_t st, unsigned* launches) {
  const int windows = keyset_windows(curve, k.W);
  KS_LAUNCH((sw_keyset_classify_kernel<C><<<blocks128(m), 128, 0, st>>>(m, k.xy, pre, k.kst)));
  KS_LAUNCH((sw_keyset_bases_kernel<C><<<blocks128(m), 128, 0, st>>>(m, k.xy, k.kst, k.W, windows, bases)));
  KS_LAUNCH((sw_keyset_window_kernel<C><<<blocks128(m * windows), 128, 0, st>>>(m, k.kst, k.W, windows, bases, k.tab)));
  return cudaSuccess;
}
template <class C>
cudaError_t sw_verify(int curve, size_t n, const KeysetDev& k, const KeyedVerifyArgs& a, cudaStream_t st, cudaEvent_t main_begin,
                      cudaEvent_t main_end, unsigned* launches) {
  const int windows = keyset_windows(curve, k.W);
  cudaError_t err;
  if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
  KS_LAUNCH((sw_verify_keyed_kernel<C><<<blocks128(n), 128, 0, st>>>(n, a.key_idx, k.kst, k.W, windows, k.tab, a.r, a.ws, a.gtab,
                                                                   a.status)));
  if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
  KS_LAUNCH((sw_replay_keyed_kernel<C><<<blocks128(n), 128, 0, st>>>(n, a.e, a.r, a.s, a.key_idx, k.xy, a.replay_tab, a.status)));
  return cudaSuccess;
}
}  // namespace

cudaError_t keyset_build_launch(int curve, size_t m, const KeysetDev& k, const uint8_t* pre, uint32_t* bases, cudaStream_t st,
                                unsigned* launches) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: {
      const int windows = keyset_windows(curve, k.W);
      KS_LAUNCH((k256_keyset_classify_kernel<<<blocks128(m), 128, 0, st>>>(m, k.xy, pre, k.kst)));
      KS_LAUNCH((k256_keyset_bases_kernel<<<blocks128(m), 128, 0, st>>>(m, k.xy, k.kst, k.W, windows, bases)));
      KS_LAUNCH((k256_keyset_window_kernel<<<blocks128(m * windows), 128, 0, st>>>(m, k.kst, k.W, windows, bases, k.tab)));
      return cudaSuccess;
    }
    case EB200_CURVE_P256: return sw_build<P256>(curve, m, k, pre, bases, st, launches);
    case EB200_CURVE_P384: return sw_build<P384>(curve, m, k, pre, bases, st, launches);
    case EB200_CURVE_P521: return sw_build<P521>(curve, m, k, pre, bases, st, launches);
    case EB200_CURVE_P192: return sw_build<P192>(curve, m, k, pre, bases, st, launches);
    case EB200_CURVE_P224: return sw_build<P224>(curve, m, k, pre, bases, st, launches);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t keyset_verify_launch(int curve, size_t n, const KeysetDev& k, const KeyedVerifyArgs& a, cudaStream_t st,
                                 cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: {
      const int windows = keyset_windows(curve, k.W);
      cudaError_t err;
      if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
      KS_LAUNCH((k256_verify_keyed_kernel<<<(unsigned)((n + EB_VERIFY_BLOCK - 1) / EB_VERIFY_BLOCK), EB_VERIFY_BLOCK, 0, st>>>(
          n, a.key_idx, k.kst, k.W, windows, k.tab, a.r, a.ws, a.gtab, a.status)));
      if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
      KS_LAUNCH((k256_replay_keyed_kernel<<<blocks128(n), 128, 0, st>>>(n, a.e, a.r, a.s, a.key_idx, k.xy, a.replay_tab, a.status)));
      return cudaSuccess;
    }
    case EB200_CURVE_P256: return sw_verify<P256>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P384: return sw_verify<P384>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P521: return sw_verify<P521>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P192: return sw_verify<P192>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P224: return sw_verify<P224>(curve, n, k, a, st, main_begin, main_end, launches);
    default: return cudaErrorInvalidValue;
  }
}
