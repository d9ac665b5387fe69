// eddsa_keyset.cu -- kernels of eb200_eddsa_keyset_create (classify -> window bases -> table windows) and of
// eb200_eddsa_verify_batch_keyed[_msgs] (key-byte gather for the hash, keyed main).  Bodies: ed25519_keyset_body.cuh.
//
// A translation unit of its own for the reason recovery_param.cu gives: kernels added to eb200.cu's module change
// NVVM's inlining into the 255-register p384 / p521 kernels there.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/elliptic_b200.h"
#include "keyset.h"

// The bodies' out-of-line helpers are external functions that eb200.cu defines too: the unnamed namespace keeps this
// unit's copies to itself.
namespace {
#include "ed25519_keyset_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(128)
ed_keyset_classify_kernel(size_t m, const uint8_t* __restrict__ A, uint8_t* __restrict__ kst) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) kst[k] = ed_ks_classify_item(k, A);
}
__global__ void __launch_bounds__(128)
ed_keyset_bases_kernel(size_t m, const uint8_t* __restrict__ A, const uint8_t* __restrict__ kst, int W, int windows,
                       u32* __restrict__ bases) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) ed_ks_bases_item(k, A, kst, W, windows, bases);
}
__global__ void __launch_bounds__(128)
ed_keyset_window_kernel(size_t m, const uint8_t* __restrict__ kst, int W, int windows, const u32* __restrict__ bases,
                        u32* __restrict__ tab) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m * windows) ed_ks_window_item(t, kst, W, windows, bases, tab);
}
__global__ void __launch_bounds__(128)
ed_keyset_gather_kernel(size_t N, const u32* __restrict__ key_idx, const uint8_t* __restrict__ A, uint8_t* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ed_ks_gather_item(i, key_idx, A, out);
}
__global__ void __launch_bounds__(128, 3)
ed25519_verify_keyed_kernel(size_t N, const uint8_t* __restrict__ R, const uint8_t* __restrict__ S, const uint8_t* __restrict__ h,
                            const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, int W, int windows,
                            const u32* __restrict__ ktab, const u32* __restrict__ gtab, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  status[i] = ed25519_verify_keyed_item(i, R, S, h, key_idx, kst, W, windows, ktab, gtab);
}

namespace {
// launch, check, count
#define EKS_LAUNCH(...)                                       \
  do {                                                        \
    __VA_ARGS__;                                              \
    cudaError_t err_ = cudaGetLastError();                    \
    if (err_ != cudaSuccess) return err_;                     \
    ++*launches;                                              \
  } while (0)

unsigned blocks128(size_t threads) { return (unsigned)((threads + 127) / 128); }
}  // namespace

cudaError_t ed_keyset_build_launch(size_t m, const KeysetDev& k, uint32_t* bases, cudaStream_t st, unsigned* launches) {
  const int windows = ed_keyset_windows(k.W);
  EKS_LAUNCH((ed_keyset_classify_kernel<<<blocks128(m), 128, 0, st>>>(m, k.xy, k.kst)));
  EKS_LAUNCH((ed_keyset_bases_kernel<<<blocks128(m), 128, 0, st>>>(m, k.xy, k.kst, k.W, windows, bases)));
  EKS_LAUNCH((ed_keyset_window_kernel<<<blocks128(m * windows), 128, 0, st>>>(m, k.kst, k.W, windows, bases, k.tab)));
  return cudaSuccess;
}

cudaError_t ed_keyset_gather_launch(size_t n, const KeysetDev& k, const uint32_t* key_idx, uint8_t* A_out, cudaStream_t st,
                                    unsigned* launches) {
  EKS_LAUNCH((ed_keyset_gather_kernel<<<blocks128(n), 128, 0, st>>>(n, key_idx, k.xy, A_out)));
  return cudaSuccess;
}

cudaError_t ed_keyset_verify_launch(size_t n, const KeysetDev& k, const uint8_t* R, const uint8_t* S, const uint8_t* h,
                                    const uint32_t* key_idx, const uint32_t* gtab, uint8_t* status, cudaStream_t st,
                                    unsigned* launches) {
  EKS_LAUNCH((ed25519_verify_keyed_kernel<<<blocks128(n), 128, 0, st>>>(n, R, S, h, key_idx, k.kst, k.W, ed_keyset_windows(k.W),
                                                                       k.tab, gtab, status)));
  return cudaSuccess;
}
