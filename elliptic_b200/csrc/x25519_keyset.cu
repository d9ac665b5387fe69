// x25519_keyset.cu -- kernels of eb200_x25519_keyset_create (classify -> window bases -> table windows) and of
// eb200_x25519_derive_batch_keyed (keyed main -> normalise).  Bodies: x25519_keyset_body.cuh; the table bodies are the
// EdDSA key set's (ed25519_keyset_body.cuh).
//
// A translation unit of its own for the reason recovery_param.cu gives: kernels added to eb200.cu's module change
// NVVM's inlining into the unrelated kernels there.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/elliptic_b200.h"
#include "keyset.h"

// The bodies' out-of-line helpers are external functions that eb200.cu defines too: the unnamed namespace keeps this
// unit's copies to itself.
namespace {
#include "x25519_keyset_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(128)
x25519_keyset_classify_kernel(size_t m, const uint8_t* __restrict__ pubx, uint8_t* __restrict__ A, uint8_t* __restrict__ kst) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) kst[k] = x25519_ks_classify_item(k, pubx, A);
}
__global__ void __launch_bounds__(128)
x25519_keyset_bases_kernel(size_t m, const uint8_t* __restrict__ A, const uint8_t* __restrict__ kst, int W, int windows,
                           u32* __restrict__ bases) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) ed_ks_bases_item(k, A, kst, W, windows, bases);
}
__global__ void __launch_bounds__(128)
x25519_keyset_window_kernel(size_t m, const uint8_t* __restrict__ kst, int W, int windows, const u32* __restrict__ bases,
                            u32* __restrict__ tab) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < m * windows) ed_ks_window_item(t, kst, W, windows, bases, tab);
}
__global__ void __launch_bounds__(128)
x25519_derive_keyed_kernel(size_t N, const uint8_t* __restrict__ priv, const u32* __restrict__ key_idx,
                           const uint8_t* __restrict__ kst, int W, int windows, const u32* __restrict__ ktab,
                           u32* __restrict__ ws, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) x25519_derive_keyed_item(i, N, priv, key_idx, kst, W, windows, ktab, ws, status);
}
__global__ void __launch_bounds__(X25519_KS_NORM_THREADS)
x25519_keyed_norm_kernel(size_t N, u32* __restrict__ ws, const uint8_t* __restrict__ status, uint8_t* __restrict__ out) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < (N + X25519_KS_BATCH - 1) / X25519_KS_BATCH) x25519_keyed_norm_item(t, N, N, ws, status, out);
}

namespace {
// launch, check, count
#define XKS_LAUNCH(...)                                       \
  do {                                                        \
    __VA_ARGS__;                                              \
    cudaError_t err_ = cudaGetLastError();                    \
    if (err_ != cudaSuccess) return err_;                     \
    ++*launches;                                              \
  } while (0)

unsigned blocks_of(size_t threads, unsigned per) { return (unsigned)((threads + per - 1) / per); }
}  // namespace

cudaError_t x25519_keyset_build_launch(size_t m, const KeysetDev& k, const uint8_t* pubx, uint32_t* bases, cudaStream_t st,
                                       unsigned* launches) {
  const int windows = ed_keyset_windows(k.W);
  XKS_LAUNCH((x25519_keyset_classify_kernel<<<blocks_of(m, 128), 128, 0, st>>>(m, pubx, k.xy, k.kst)));
  XKS_LAUNCH((x25519_keyset_bases_kernel<<<blocks_of(m, 128), 128, 0, st>>>(m, k.xy, k.kst, k.W, windows, bases)));
  XKS_LAUNCH((x25519_keyset_window_kernel<<<blocks_of(m * windows, 128), 128, 0, st>>>(m, k.kst, k.W, windows, bases, k.tab)));
  return cudaSuccess;
}

size_t x25519_keyset_ws_bytes(size_t n) { return (size_t)X25519_KS_WS_WORDS * 4 * n; }

cudaError_t x25519_keyset_derive_launch(size_t n, const KeysetDev& k, const uint8_t* priv, const uint32_t* key_idx, uint32_t* ws,
                                        uint8_t* out, uint8_t* status, cudaStream_t st, cudaEvent_t main_begin,
                                        cudaEvent_t main_end, unsigned* launches) {
  cudaError_t err;
  if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
  XKS_LAUNCH((x25519_derive_keyed_kernel<<<blocks_of(n, 128), 128, 0, st>>>(n, priv, key_idx, k.kst, k.W,
                                                                             ed_keyset_windows(k.W), k.tab, ws, status)));
  if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
  XKS_LAUNCH((x25519_keyed_norm_kernel<<<blocks_of((n + X25519_KS_BATCH - 1) / X25519_KS_BATCH, X25519_KS_NORM_THREADS),
                                         X25519_KS_NORM_THREADS, 0, st>>>(n, ws, status, out)));
  return cudaSuccess;
}
