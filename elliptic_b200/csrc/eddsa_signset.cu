// eddsa_signset.cu -- kernels of eb200_eddsa_signing_set_create (create) and of eb200_eddsa_sign_batch_keyed (nonce ->
// normalise -> challenge).  Bodies: ed25519_signset_body.cuh.
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
#include "ed25519_signset_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(128)
ed_signset_create_kernel(size_t m, const uint8_t* __restrict__ secrets, const u32* __restrict__ gtab, u32* __restrict__ keys,
                         uint8_t* __restrict__ pub) {
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) ed_ss_create_item(k, secrets, gtab, keys, pub);
}
__global__ void __launch_bounds__(128)
ed_signset_nonce_kernel(size_t N, const uint8_t* __restrict__ msgs, const u64* __restrict__ msg_off,
                        const u32* __restrict__ key_idx, const u32* __restrict__ keys, const u32* __restrict__ gtab,
                        u32* __restrict__ ws) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ed_ss_nonce_item(i, N, msgs, msg_off, key_idx, keys, gtab, ws);
}
__global__ void __launch_bounds__(ED_SS_NORM_THREADS)
ed_signset_normalise_kernel(size_t N, u32* __restrict__ ws, uint8_t* __restrict__ sig) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < (N + ED_SS_BATCH - 1) / ED_SS_BATCH) ed_ss_normalise_item(t, N, N, ws, sig);
}
__global__ void __launch_bounds__(128)
ed_signset_challenge_kernel(size_t N, const uint8_t* __restrict__ msgs, const u64* __restrict__ msg_off,
                            const u32* __restrict__ key_idx, const u32* __restrict__ keys, const uint8_t* __restrict__ A,
                            const u32* __restrict__ ws, uint8_t* __restrict__ sig) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ed_ss_challenge_item(i, N, msgs, msg_off, key_idx, keys, A, ws, sig);
}

namespace {
// launch, check, count
#define ESS_LAUNCH(...)                                       \
  do {                                                        \
    __VA_ARGS__;                                              \
    cudaError_t err_ = cudaGetLastError();                    \
    if (err_ != cudaSuccess) return err_;                     \
    ++*launches;                                              \
  } while (0)

unsigned blocks_of(size_t threads, unsigned per) { return (unsigned)((threads + per - 1) / per); }
}  // namespace

cudaError_t ed_signset_create_launch(size_t m, const KeysetDev& k, const uint8_t* secrets, const uint32_t* gtab,
                                     cudaStream_t st, unsigned* launches) {
  ESS_LAUNCH((ed_signset_create_kernel<<<blocks_of(m, 128), 128, 0, st>>>(m, secrets, gtab, k.tab, k.xy)));
  return cudaSuccess;
}

cudaError_t ed_signset_normalise_launch(size_t n, uint32_t* ws, uint8_t* sig, cudaStream_t st, unsigned* launches) {
  ESS_LAUNCH((ed_signset_normalise_kernel<<<blocks_of((n + ED_SS_BATCH - 1) / ED_SS_BATCH, ED_SS_NORM_THREADS),
                                            ED_SS_NORM_THREADS, 0, st>>>(n, ws, sig)));
  return cudaSuccess;
}

size_t ed_signset_ws_bytes(size_t n) { return (size_t)ED_SS_WS_WORDS * 4 * n; }
size_t ed_signset_nonce_bytes(size_t n) { return (size_t)8 * 4 * n; }
size_t ed_signset_nonce_offset(size_t n) { return (size_t)ED_SS_WS_R * 4 * n; }

cudaError_t ed_signset_sign_launch(size_t n, const KeysetDev& k, const uint8_t* msgs, const uint64_t* msg_off,
                                   const uint32_t* key_idx, const uint32_t* gtab, uint32_t* ws, uint8_t* sig, cudaStream_t st,
                                   cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches) {
  cudaError_t err;
  if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
  ESS_LAUNCH((ed_signset_nonce_kernel<<<blocks_of(n, 128), 128, 0, st>>>(n, msgs, msg_off, key_idx, k.tab, gtab, ws)));
  if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
  if ((err = ed_signset_normalise_launch(n, ws, sig, st, launches)) != cudaSuccess) return err;
  ESS_LAUNCH((ed_signset_challenge_kernel<<<blocks_of(n, 128), 128, 0, st>>>(n, msgs, msg_off, key_idx, k.tab, k.xy, ws, sig)));
  return cudaSuccess;
}
