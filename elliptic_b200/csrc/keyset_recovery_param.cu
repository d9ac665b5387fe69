// keyset_recovery_param.cu -- kernels of eb200_ecdsa_recovery_param_batch_keyed (getKeyRecoveryParam against the
// tables eb200_keyset_create builds): main (the keyed mul loops into P = u1 G + u2 Q, the x test on Jacobian P, Y and Z
// stored), recid normalisation (one inversion per batch of live items for the parity of y) and cold (the s = 0 (mod n)
// items, recovery_param_cold_item on the key's coordinates).  The scalar prep is recovery_param.cu's, unchanged.
// Bodies: ecdsa_keyset_rp_body.cuh.
//
// A translation unit of its own for the reason keyset_mul.cu gives: in one module with the other key-set kernels these
// change NVVM's code for them (their out-of-line group-law helpers gain callers).
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
#include "ecdsa_k256_sign.cuh"
#include "ecdsa_sw_body.cuh"
#include "ecdsa_keyset_body.cuh"
#include "ecdsa_keyset_rp_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(EB_VERIFY_BLOCK, EB_VERIFY_MINBLOCKS)
k256_recovery_param_keyed_kernel(size_t N, const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, int W, int windows,
                                 const u32* __restrict__ ktab, const uint8_t* __restrict__ r, const u32* __restrict__ ws,
                                 const u32* __restrict__ gtab, u32* __restrict__ yz, uint8_t* __restrict__ recid,
                                 uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = k256_recovery_param_keyed_item(i, N, key_idx, kst, W, windows, ktab, r, ws, gtab, yz, recid);
}
__global__ void __launch_bounds__(128)
k256_recid_norm_kernel(size_t N, int batch, const u32* __restrict__ yz, u32* __restrict__ scratch,
                       const uint8_t* __restrict__ status, uint8_t* __restrict__ recid) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  k256_ks_recid_norm_thread(tid, T, N, batch, yz, scratch, status, recid);
}
__global__ void __launch_bounds__(128)
k256_recovery_param_cold_keyed_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                                      const u32* __restrict__ key_idx, const uint8_t* __restrict__ xy,
                                      const u32* __restrict__ gtab, uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = recovery_param_cold_item(0, e + 32 * i, r + 32 * i, xy + 64 * (size_t)key_idx[i], gtab, recid + i);
}

template <class C>
__global__ void __launch_bounds__(128, (C::N <= 8) ? EB_SW_MINBLOCKS8 : EB_SW_MINBLOCKS_BIG)
sw_recovery_param_keyed_kernel(size_t N, const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, int W, int windows,
                               const u32* __restrict__ ktab, const uint8_t* __restrict__ r, const u32* __restrict__ ws,
                               const u32* __restrict__ gtab, u32* __restrict__ yz, uint8_t* __restrict__ recid,
                               uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = SWKeyedRP<C>::main_item(i, N, key_idx, kst, W, windows, ktab, r, ws, gtab, yz, recid);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_recid_norm_kernel(size_t N, const u32* __restrict__ yz, u32* __restrict__ scratch, const uint8_t* __restrict__ status,
                     uint8_t* __restrict__ recid) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  SWKeyedRP<C>::recid_norm_thread(tid, T, N, yz, scratch, status, recid);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_recovery_param_cold_keyed_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                                    const u32* __restrict__ key_idx, const uint8_t* __restrict__ xy,
                                    const u32* __restrict__ gtab, uint8_t* __restrict__ recid, uint8_t* __restrict__ status) {
  constexpr size_t LEN = C::LEN;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = SW<C>::recovery_param_cold_item(0, e + LEN * i, r + LEN * i, xy + 2 * LEN * (size_t)key_idx[i], gtab, recid + i);
}

namespace {
// launch, check, count
#define KRP_LAUNCH(...)                                       \
  do {                                                        \
    __VA_ARGS__;                                              \
    cudaError_t err_ = cudaGetLastError();                    \
    if (err_ != cudaSuccess) return err_;                     \
    ++*launches;                                              \
  } while (0)

unsigned blocks128(size_t threads) { return (unsigned)((threads + 127) / 128); }

template <class C>
cudaError_t sw_rp(int curve, size_t n, const KeysetDev& k, const KeyedRecoveryParamArgs& a, cudaStream_t st,
                  cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches) {
  const int windows = keyset_windows(curve, k.W);
  cudaError_t err;
  if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
  KRP_LAUNCH((sw_recovery_param_keyed_kernel<C><<<blocks128(n), 128, 0, st>>>(n, a.key_idx, k.kst, k.W, windows, k.tab, a.r,
                                                                            a.ws, a.gtab, a.yz, a.recid, a.status)));
  if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
  KRP_LAUNCH((sw_recid_norm_kernel<C><<<blocks128((n + SW<C>::BATCH - 1) / SW<C>::BATCH), 128, 0, st>>>(n, a.yz, a.scratch,
                                                                                                      a.status, a.recid)));
  KRP_LAUNCH((sw_recovery_param_cold_keyed_kernel<C><<<blocks128(n), 128, 0, st>>>(n, a.e, a.r, a.key_idx, k.xy, a.gtab,
                                                                                 a.recid, a.status)));
  return cudaSuccess;
}
}  // namespace

cudaError_t keyset_recovery_param_launch(int curve, size_t n, const KeysetDev& k, const KeyedRecoveryParamArgs& a,
                                         cudaStream_t st, cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: {
      const int windows = keyset_windows(curve, k.W);
      cudaError_t err;
      if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
      KRP_LAUNCH((k256_recovery_param_keyed_kernel<<<(unsigned)((n + EB_VERIFY_BLOCK - 1) / EB_VERIFY_BLOCK), EB_VERIFY_BLOCK, 0,
                                                     st>>>(n, a.key_idx, k.kst, k.W, windows, k.tab, a.r, a.ws, a.gtab, a.yz,
                                                           a.recid, a.status)));
      if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
      KRP_LAUNCH((k256_recid_norm_kernel<<<blocks128((n + a.batch - 1) / a.batch), 128, 0, st>>>(n, a.batch, a.yz, a.scratch,
                                                                                               a.status, a.recid)));
      KRP_LAUNCH((k256_recovery_param_cold_keyed_kernel<<<blocks128(n), 128, 0, st>>>(n, a.e, a.r, a.key_idx, k.xy, a.gtab,
                                                                                     a.recid, a.status)));
      return cudaSuccess;
    }
    case EB200_CURVE_P256: return sw_rp<P256>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P384: return sw_rp<P384>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P521: return sw_rp<P521>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P192: return sw_rp<P192>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P224: return sw_rp<P224>(curve, n, k, a, st, main_begin, main_end, launches);
    default: return cudaErrorInvalidValue;
  }
}
