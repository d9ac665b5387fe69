// keyset_forms.cu -- the kernels that frame the unchanged keyed ECDSA verify (keyset.cu) for
// eb200_ecdsa_verify_batch_keyed_der (DER decode with the key's verdict, in front of the unchanged prep),
// eb200_ecdsa_verify_batch_keyed_dev (index screen in front of it) and eb200_ecdsa_verify_batch_keyed_der_dev (the same
// DER decode behind the index-and-range screen), and the verdict merge that all three run behind the keyed
// replay; and those that frame the unchanged keyed kernels of the other device-pointer keyed calls: the index, scalar
// and message-range screens, the merge that also zeroes outputs, and the screened hash and challenge kernels (the
// screened nonce kernel is in keyset_forms_nonce.cu).  Bodies: keyset_forms_body.cuh.
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
#include "keyset_forms_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(128)
keyset_der_decode_kernel(size_t N, u32 len, const uint8_t* __restrict__ der, const unsigned long long* __restrict__ off,
                         const u32* __restrict__ key_idx, const uint8_t* __restrict__ kst, uint8_t* __restrict__ r,
                         uint8_t* __restrict__ s, uint8_t* __restrict__ verdict) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) verdict[i] = ks_der_verdict_item(i, len, der, off, key_idx, kst, r, s);
}
__global__ void __launch_bounds__(128)
keyset_der_decode_screened_kernel(size_t N, u32 len, const uint8_t* __restrict__ pre, const uint8_t* __restrict__ der,
                                  const unsigned long long* __restrict__ off, const u32* __restrict__ idx,
                                  const uint8_t* __restrict__ kst, uint8_t* __restrict__ r, uint8_t* __restrict__ s,
                                  uint8_t* __restrict__ verdict) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) verdict[i] = ks_der_screened_item(i, len, pre, der, off, idx, kst, r, s);
}
__global__ void __launch_bounds__(128)
keyset_index_screen_kernel(size_t N, const u32* __restrict__ key_idx, size_t m, u32* __restrict__ idx_out,
                           uint8_t* __restrict__ verdict) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) verdict[i] = ks_index_screen_item(i, key_idx, m, idx_out);
}
__global__ void __launch_bounds__(128)
keyset_verdict_merge_kernel(size_t N, const uint8_t* __restrict__ verdict, uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ks_verdict_merge_item(i, verdict, status);
}

__global__ void __launch_bounds__(128)
keyset_index_scalar_screen_kernel(size_t N, const u32* __restrict__ key_idx, size_t m, const uint8_t* __restrict__ k,
                                  bool big_endian, u32* __restrict__ idx_out, uint8_t* __restrict__ k_out,
                                  uint8_t* __restrict__ verdict) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) verdict[i] = ks_index_scalar_screen_item(i, key_idx, m, k, big_endian, idx_out, k_out);
}
__global__ void __launch_bounds__(128)
keyset_index_range_screen_kernel(size_t N, const u32* __restrict__ key_idx, size_t m, const u64* __restrict__ off,
                                 u64 msgs_len, u32* __restrict__ idx_out, uint8_t* __restrict__ verdict) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) verdict[i] = ks_index_range_screen_item(i, key_idx, m, off, msgs_len, idx_out);
}
__global__ void __launch_bounds__(128)
keyset_verdict_merge_out_kernel(size_t N, const uint8_t* __restrict__ verdict, uint8_t* __restrict__ status,
                                uint8_t* __restrict__ out, u32 ol) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ks_verdict_merge_out_item(i, verdict, status, out, ol);
}
__global__ void __launch_bounds__(128)
keyset_ed_hash_screened_kernel(size_t N, const uint8_t* __restrict__ verdict, const uint8_t* __restrict__ R,
                               const uint8_t* __restrict__ A, const uint8_t* __restrict__ msgs, const u64* __restrict__ msg_off,
                               uint8_t* __restrict__ h) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ks_ed_hash_screened_item(i, verdict, R, A, msgs, msg_off, h);
}
__global__ void __launch_bounds__(128)
keyset_ss_challenge_screened_kernel(size_t N, const uint8_t* __restrict__ verdict, const uint8_t* __restrict__ msgs,
                                    const u64* __restrict__ msg_off, const u32* __restrict__ key_idx,
                                    const u32* __restrict__ keys, const uint8_t* __restrict__ A, const u32* __restrict__ ws,
                                    uint8_t* __restrict__ sig) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ks_ss_challenge_screened_item(i, N, verdict, msgs, msg_off, key_idx, keys, A, ws, sig);
}

namespace {
unsigned blocks128(size_t threads) { return (unsigned)((threads + 127) / 128); }

cudaError_t counted(unsigned* launches) {
  cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) ++*launches;
  return err;
}
}  // namespace

cudaError_t keyset_der_decode_launch(size_t n, uint32_t len, const uint8_t* der, const unsigned long long* off,
                                     const uint32_t* key_idx, const KeysetDev& k, uint8_t* r, uint8_t* s, uint8_t* verdict,
                                     cudaStream_t st, unsigned* launches) {
  keyset_der_decode_kernel<<<blocks128(n), 128, 0, st>>>(n, len, der, off, key_idx, k.kst, r, s, verdict);
  return counted(launches);
}

cudaError_t keyset_der_decode_screened_launch(size_t n, uint32_t len, const uint8_t* pre, const uint8_t* der,
                                              const unsigned long long* off, const uint32_t* idx, const KeysetDev& k,
                                              uint8_t* r, uint8_t* s, uint8_t* verdict, cudaStream_t st, unsigned* launches) {
  keyset_der_decode_screened_kernel<<<blocks128(n), 128, 0, st>>>(n, len, pre, der, off, idx, k.kst, r, s, verdict);
  return counted(launches);
}

cudaError_t keyset_index_screen_launch(size_t n, const uint32_t* key_idx, size_t m, uint32_t* idx_out, uint8_t* verdict,
                                       cudaStream_t st, unsigned* launches) {
  keyset_index_screen_kernel<<<blocks128(n), 128, 0, st>>>(n, key_idx, m, idx_out, verdict);
  return counted(launches);
}

cudaError_t keyset_verdict_merge_launch(size_t n, const uint8_t* verdict, uint8_t* status, cudaStream_t st, unsigned* launches) {
  keyset_verdict_merge_kernel<<<blocks128(n), 128, 0, st>>>(n, verdict, status);
  return counted(launches);
}

cudaError_t keyset_index_scalar_screen_launch(size_t n, const uint32_t* key_idx, size_t m, const uint8_t* k, bool big_endian,
                                              uint32_t* idx_out, uint8_t* k_out, uint8_t* verdict, cudaStream_t st,
                                              unsigned* launches) {
  keyset_index_scalar_screen_kernel<<<blocks128(n), 128, 0, st>>>(n, key_idx, m, k, big_endian, idx_out, k_out, verdict);
  return counted(launches);
}

cudaError_t keyset_index_range_screen_launch(size_t n, const uint32_t* key_idx, size_t m, const uint64_t* off,
                                             uint64_t msgs_len, uint32_t* idx_out, uint8_t* verdict, cudaStream_t st,
                                             unsigned* launches) {
  keyset_index_range_screen_kernel<<<blocks128(n), 128, 0, st>>>(n, key_idx, m, off, msgs_len, idx_out, verdict);
  return counted(launches);
}

cudaError_t keyset_verdict_merge_out_launch(size_t n, const uint8_t* verdict, uint8_t* status, uint8_t* out, uint32_t ol,
                                            cudaStream_t st, unsigned* launches) {
  keyset_verdict_merge_out_kernel<<<blocks128(n), 128, 0, st>>>(n, verdict, status, out, ol);
  return counted(launches);
}

cudaError_t keyset_ed_hash_screened_launch(size_t n, const uint8_t* verdict, const uint8_t* R, const uint8_t* A,
                                           const uint8_t* msgs, const uint64_t* msg_off, uint8_t* h, cudaStream_t st,
                                           unsigned* launches) {
  keyset_ed_hash_screened_kernel<<<blocks128(n), 128, 0, st>>>(n, verdict, R, A, msgs, msg_off, h);
  return counted(launches);
}

cudaError_t keyset_ss_sign_screened_launch(size_t n, const uint8_t* verdict, const KeysetDev& k, const uint8_t* msgs,
                                           const uint64_t* msg_off, const uint32_t* key_idx, const uint32_t* gtab, uint32_t* ws,
                                           uint8_t* sig, cudaStream_t st, cudaEvent_t main_begin, cudaEvent_t main_end,
                                           unsigned* launches) {
  cudaError_t err;
  if ((err = cudaEventRecord(main_begin, st)) != cudaSuccess) return err;
  if ((err = keyset_ss_nonce_screened_launch(n, verdict, k, msgs, msg_off, key_idx, gtab, ws, st, launches)) != cudaSuccess)
    return err;
  if ((err = cudaEventRecord(main_end, st)) != cudaSuccess) return err;
  if ((err = ed_signset_normalise_launch(n, ws, sig, st, launches)) != cudaSuccess) return err;
  keyset_ss_challenge_screened_kernel<<<blocks128(n), 128, 0, st>>>(n, verdict, msgs, msg_off, key_idx, k.tab, k.xy, ws, sig);
  return counted(launches);
}
