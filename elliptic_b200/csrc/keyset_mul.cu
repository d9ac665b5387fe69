// keyset_mul.cu -- kernels of the keyed Point.mul / mulAdd / derive calls (eb200_scalar_mul_batch_keyed,
// eb200_mul_add_batch_keyed, eb200_ecdh_derive_batch_keyed) on the tables eb200_keyset_create builds: main (one table
// lookup and mixed add per window into a Jacobian point, then the fixed-base adds unless FL_NOG), normalisation (one
// inversion per prep-sized batch of items) and the replay of off-curve-key items through the unkeyed call's schedule.
// Bodies: ecdsa_keyset_body.cuh.
//
// A translation unit of its own, apart from keyset.cu: in one module with the build and verify kernels these kernels
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
#include "ecdsa_k256_replay.cuh"
#include "ecdsa_sw_body.cuh"
#include "ecdsa_sw_replay.cuh"
#include "ecdsa_keyset_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(EB_VERIFY_BLOCK, EB_VERIFY_MINBLOCKS)
k256_mul_keyed_kernel(size_t N, const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, int W, int windows,
                      const u32* __restrict__ ktab, const u32* __restrict__ ws, const u32* __restrict__ gtab,
                      u32* __restrict__ jout, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = k256_mul_keyed_item(i, N, key_idx, kst, W, windows, ktab, ws, gtab, jout);
}
__global__ void __launch_bounds__(128)
k256_keyed_norm_kernel(size_t N, int batch, const u32* __restrict__ jac, u32* __restrict__ scratch, int xonly,
                       uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  k256_ks_norm_thread(tid, T, N, batch, jac, scratch, xonly != 0, out, status);
}
__global__ void __launch_bounds__(128)
k256_mul_replay_keyed_kernel(size_t N, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ k2,
                             const u32* __restrict__ key_idx, const uint8_t* __restrict__ xy, const u32* __restrict__ tab,
                             uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = rp_mul_add_item(0, k1 ? k1 + 32 * i : nullptr, k2 + 32 * i, xy + 64 * (size_t)key_idx[i], tab, out + 64 * i);
}

template <class C>
__global__ void __launch_bounds__(128, (C::N <= 8) ? EB_SW_MINBLOCKS8 : EB_SW_MINBLOCKS_BIG)
sw_mul_keyed_kernel(size_t N, const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, int W, int windows,
                    const u32* __restrict__ ktab, const u32* __restrict__ ws, const u32* __restrict__ gtab,
                    u32* __restrict__ jout, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = SWKeyed<C>::mul_keyed_item(i, N, key_idx, kst, W, windows, ktab, ws, gtab, jout);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_keyed_norm_kernel(size_t N, const u32* __restrict__ jac, u32* __restrict__ scratch, int xonly, uint8_t* __restrict__ out,
                     uint8_t* __restrict__ status) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  SWKeyed<C>::norm_thread(tid, T, N, jac, scratch, xonly != 0, out, status);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_mul_replay_keyed_kernel(size_t N, const uint8_t* __restrict__ k1, const uint8_t* __restrict__ k2,
                           const u32* __restrict__ key_idx, const uint8_t* __restrict__ xy, const u32* __restrict__ tab,
                           uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  constexpr size_t LEN = C::LEN;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = SWReplay<C>::mul_add_item(0, k1 ? k1 + LEN * i : nullptr, k2 + LEN * i, xy + 2 * LEN * (size_t)key_idx[i], tab,
                                        out + 2 * LEN * i);
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
cudaError_t sw_mul(int curve, size_t n, const KeysetDev& k, const KeyedMulArgs& a, cudaStream_t st, cudaEvent_t main_begin,
                   cudaEvent_t main_end, unsigned* launches) {
  const int windows = keyset_windows(curve, k.W);
  cudaError_t err;
  if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
  KS_LAUNCH((sw_mul_keyed_kernel<C><<<blocks128(n), 128, 0, st>>>(n, a.key_idx, k.kst, k.W, windows, k.tab, a.ws, a.gtab, a.jac,
                                                                 a.status)));
  if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
  KS_LAUNCH((sw_keyed_norm_kernel<C><<<blocks128((n + SW<C>::BATCH - 1) / SW<C>::BATCH), 128, 0, st>>>(
      n, a.jac, a.scratch, a.derive ? 1 : 0, a.out, a.status)));
  if (!a.derive)
    KS_LAUNCH((sw_mul_replay_keyed_kernel<C><<<blocks128(n), 128, 0, st>>>(n, a.k1, a.k2, a.key_idx, k.xy, a.replay_tab, a.out,
                                                                         a.status)));
  return cudaSuccess;
}
}  // namespace

cudaError_t keyset_mul_launch(int curve, size_t n, const KeysetDev& k, const KeyedMulArgs& a, cudaStream_t st,
                              cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: {
      const int windows = keyset_windows(curve, k.W);
      cudaError_t err;
      if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
      KS_LAUNCH((k256_mul_keyed_kernel<<<(unsigned)((n + EB_VERIFY_BLOCK - 1) / EB_VERIFY_BLOCK), EB_VERIFY_BLOCK, 0, st>>>(
          n, a.key_idx, k.kst, k.W, windows, k.tab, a.ws, a.gtab, a.jac, a.status)));
      if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
      KS_LAUNCH((k256_keyed_norm_kernel<<<blocks128((n + a.batch - 1) / a.batch), 128, 0, st>>>(n, a.batch, a.jac, a.scratch,
                                                                                             a.derive ? 1 : 0, a.out, a.status)));
      if (!a.derive)
        KS_LAUNCH((k256_mul_replay_keyed_kernel<<<blocks128(n), 128, 0, st>>>(n, a.k1, a.k2, a.key_idx, k.xy, a.replay_tab, a.out,
                                                                             a.status)));
      return cudaSuccess;
    }
    case EB200_CURVE_P256: return sw_mul<P256>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P384: return sw_mul<P384>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P521: return sw_mul<P521>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P192: return sw_mul<P192>(curve, n, k, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P224: return sw_mul<P224>(curve, n, k, a, st, main_begin, main_end, launches);
    default: return cudaErrorInvalidValue;
  }
}
