// recovery_param.cu -- kernels of eb200_ecdsa_recovery_param_batch (EC.getKeyRecoveryParam, ec/index.js:261-278):
// prep -> main (one u1 G + u2 Q per item: recovery_param_item in ecdsa_k256_body.cuh / ecdsa_sw_body.cuh) -> cold (the
// s = 0 (mod n) items the main kernel flagged, launched every time like the replay kernels).  The keyed call
// (keyset_recovery_param.cu) runs the same prep through recovery_param_prep_launch.
//
// They live in a translation unit of their own.  In eb200.cu's module, even placed after every other kernel, they
// changed NVVM's inlining into the 255-register p384 / p521 verify, recover and mulAdd kernels (more p521 spills);
// here the existing kernels keep their code.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include "../../include/elliptic_b200.h"
#include "kernel_bounds.h"
#include "recovery_param.h"

// The bodies' out-of-line helpers (fe_mul, jac_dbl, ...) are external functions that eb200.cu defines too: the unnamed
// namespace keeps this unit's copies to itself.
namespace {
#include "ecdsa_k256_body.cuh"
#include "ecdsa_k256_sign.cuh"
#include "ecdsa_sw_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(128) k256_prep_recovery_param_kernel(size_t N, const uint8_t* __restrict__ e,
                                                                       const uint8_t* __restrict__ r,
                                                                       const uint8_t* __restrict__ s,
                                                                       u32* __restrict__ ws, u32* __restrict__ scratch) {
  size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t T = (size_t)gridDim.x * blockDim.x;
  prep_thread(tid, T, N, e, r, s, ws, scratch, 2);
}
__global__ void __launch_bounds__(EB_VERIFY_BLOCK, EB_VERIFY_MINBLOCKS)
k256_recovery_param_kernel(size_t N, const uint8_t* __restrict__ q, const uint8_t* __restrict__ r, const u32* __restrict__ ws,
                           const u32* __restrict__ gtab, u32* __restrict__ qtab, uint8_t* __restrict__ recid,
                           uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = recovery_param_item(i, N, q, r, ws, gtab, qtab, recid);
}
__global__ void __launch_bounds__(128)
k256_recovery_param_cold_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                                const uint8_t* __restrict__ q, const u32* __restrict__ gtab, uint8_t* __restrict__ recid,
                                uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = recovery_param_cold_item(i, e, r, q, gtab, recid);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_prep_recovery_param_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                              const uint8_t* __restrict__ s, u32* __restrict__ ws) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) SW<C>::prep_recovery_param_item(i, N, e, r, s, ws);
}
template <class C>
__global__ void __launch_bounds__(128, (C::N <= 8) ? EB_SW_MINBLOCKS8 : EB_SW_MINBLOCKS_BIG)
sw_recovery_param_kernel(size_t N, const uint8_t* __restrict__ q, const uint8_t* __restrict__ r, const u32* __restrict__ ws,
                         const u32* __restrict__ gtab, u32* __restrict__ qtab, uint8_t* __restrict__ recid,
                         uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = SW<C>::recovery_param_item(i, N, q, r, ws, gtab, qtab, recid);
}
template <class C>
__global__ void __launch_bounds__(128)
sw_recovery_param_cold_kernel(size_t N, const uint8_t* __restrict__ e, const uint8_t* __restrict__ r,
                              const uint8_t* __restrict__ q, const u32* __restrict__ gtab, uint8_t* __restrict__ recid,
                              uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || status[i] != ST_NEEDS_HOST) return;
  status[i] = SW<C>::recovery_param_cold_item(i, e, r, q, gtab, recid);
}

namespace {
// launch, check, count
#define RP_LAUNCH(...)                                        \
  do {                                                        \
    __VA_ARGS__;                                              \
    cudaError_t err_ = cudaGetLastError();                    \
    if (err_ != cudaSuccess) return err_;                     \
    ++*launches;                                              \
  } while (0)

unsigned blocks128(size_t threads) { return (unsigned)((threads + 127) / 128); }

template <class C>
cudaError_t sw_launch(size_t n, const RecoveryParamArgs& a, cudaStream_t st, cudaEvent_t main_begin, cudaEvent_t main_end,
                      unsigned* launches) {
  const unsigned nb = blocks128(n);
  cudaError_t err;
  RP_LAUNCH((sw_prep_recovery_param_kernel<C><<<nb, 128, 0, st>>>(n, a.e, a.r, a.s, a.ws)));
  if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
  RP_LAUNCH((sw_recovery_param_kernel<C><<<nb, 128, 0, st>>>(n, a.q, a.r, a.ws, a.gtab, a.qtab, a.recid, a.status)));
  if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
  RP_LAUNCH((sw_recovery_param_cold_kernel<C><<<nb, 128, 0, st>>>(n, a.e, a.r, a.q, a.gtab, a.recid, a.status)));
  return cudaSuccess;
}
}  // namespace

cudaError_t recovery_param_launch(int curve, size_t n, const RecoveryParamArgs& a, cudaStream_t st, cudaEvent_t main_begin,
                                  cudaEvent_t main_end, unsigned* launches) {
  switch (curve) {
    case EB200_CURVE_SECP256K1: {
      cudaError_t err;
      RP_LAUNCH((k256_prep_recovery_param_kernel<<<blocks128((n + PREP_BATCH - 1) / PREP_BATCH), 128, 0, st>>>(
          n, a.e, a.r, a.s, a.ws, a.scratch)));
      if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
      RP_LAUNCH((k256_recovery_param_kernel<<<(unsigned)((n + EB_VERIFY_BLOCK - 1) / EB_VERIFY_BLOCK), EB_VERIFY_BLOCK, 0, st>>>(
          n, a.q, a.r, a.ws, a.gtab, a.qtab, a.recid, a.status)));
      if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
      RP_LAUNCH((k256_recovery_param_cold_kernel<<<blocks128(n), 128, 0, st>>>(n, a.e, a.r, a.q, a.gtab, a.recid, a.status)));
      return cudaSuccess;
    }
    case EB200_CURVE_P256: return sw_launch<P256>(n, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P384: return sw_launch<P384>(n, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P521: return sw_launch<P521>(n, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P192: return sw_launch<P192>(n, a, st, main_begin, main_end, launches);
    case EB200_CURVE_P224: return sw_launch<P224>(n, a, st, main_begin, main_end, launches);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t recovery_param_prep_launch(int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s, u32* ws,
                                       u32* scratch, cudaStream_t st, unsigned* launches) {
  const unsigned nb = blocks128(n);
  switch (curve) {
    case EB200_CURVE_SECP256K1:
      RP_LAUNCH((k256_prep_recovery_param_kernel<<<blocks128((n + PREP_BATCH - 1) / PREP_BATCH), 128, 0, st>>>(n, e, r, s, ws,
                                                                                                               scratch)));
      return cudaSuccess;
    case EB200_CURVE_P256: RP_LAUNCH((sw_prep_recovery_param_kernel<P256><<<nb, 128, 0, st>>>(n, e, r, s, ws))); return cudaSuccess;
    case EB200_CURVE_P384: RP_LAUNCH((sw_prep_recovery_param_kernel<P384><<<nb, 128, 0, st>>>(n, e, r, s, ws))); return cudaSuccess;
    case EB200_CURVE_P521: RP_LAUNCH((sw_prep_recovery_param_kernel<P521><<<nb, 128, 0, st>>>(n, e, r, s, ws))); return cudaSuccess;
    case EB200_CURVE_P192: RP_LAUNCH((sw_prep_recovery_param_kernel<P192><<<nb, 128, 0, st>>>(n, e, r, s, ws))); return cudaSuccess;
    case EB200_CURVE_P224: RP_LAUNCH((sw_prep_recovery_param_kernel<P224><<<nb, 128, 0, st>>>(n, e, r, s, ws))); return cudaSuccess;
    default: return cudaErrorInvalidValue;
  }
}
