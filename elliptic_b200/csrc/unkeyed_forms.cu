// unkeyed_forms.cu -- the kernels that frame the unchanged unkeyed kernels of eb200.cu for the device-pointer forms of the
// calls with variable-length ranges: the index-free range screen, the screened DER decode that launch_verify runs in
// place of der_decode_kernel for eb200_ecdsa_verify_batch_der_dev, and the screened EdDSA sign kernel.  Bodies:
// unkeyed_forms_body.cuh.  The merges behind them are keyset_forms.cu's.
//
// A translation unit of its own for the reason recovery_param.cu gives: kernels added to eb200.cu's module change
// NVVM's inlining into the unrelated kernels there.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/elliptic_b200.h"
#include "unkeyed_forms.h"

// The bodies' out-of-line helpers are external functions that eb200.cu defines too: the unnamed namespace keeps this
// unit's copies to itself.
namespace {
#include "unkeyed_forms_body.cuh"
}  // namespace

using namespace eb;

__global__ void __launch_bounds__(128)
unkeyed_range_screen_kernel(size_t N, const u64* __restrict__ off, u64 len, uint8_t* __restrict__ verdict) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) verdict[i] = ud_range_screen_item(i, off, len);
}
__global__ void __launch_bounds__(128)
unkeyed_der_decode_screened_kernel(size_t N, u32 len, const uint8_t* __restrict__ verdict, const uint8_t* __restrict__ der,
                                   const unsigned long long* __restrict__ off, uint8_t* __restrict__ r, uint8_t* __restrict__ s,
                                   uint8_t* __restrict__ pre, int pre_valid) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ud_der_decode_screened_item(i, len, verdict, der, off, r, s, pre, pre_valid);
}
__global__ void __launch_bounds__(128)
unkeyed_ed25519_sign_screened_kernel(size_t N, const uint8_t* __restrict__ verdict, const uint8_t* __restrict__ secrets,
                                     const uint8_t* __restrict__ msgs, const u64* __restrict__ msg_off,
                                     const u32* __restrict__ gtab, uint8_t* __restrict__ sig, uint8_t* __restrict__ pub,
                                     uint8_t* __restrict__ status) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) status[i] = ud_ed25519_sign_screened_item(i, verdict, secrets, msgs, msg_off, gtab, sig, pub);
}

namespace {
unsigned blocks128(size_t threads) { return (unsigned)((threads + 127) / 128); }

cudaError_t counted(unsigned* launches) {
  cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) ++*launches;
  return err;
}
}  // namespace

cudaError_t unkeyed_range_screen_launch(size_t n, const uint64_t* off, uint64_t len, uint8_t* verdict, cudaStream_t st,
                                        unsigned* launches) {
  unkeyed_range_screen_kernel<<<blocks128(n), 128, 0, st>>>(n, off, len, verdict);
  return counted(launches);
}

cudaError_t unkeyed_der_decode_screened_launch(size_t n, uint32_t len, const uint8_t* verdict, const uint8_t* der,
                                               const unsigned long long* off, uint8_t* r, uint8_t* s, uint8_t* pre,
                                               int pre_valid, cudaStream_t st, unsigned* launches) {
  unkeyed_der_decode_screened_kernel<<<blocks128(n), 128, 0, st>>>(n, len, verdict, der, off, r, s, pre, pre_valid);
  return counted(launches);
}

cudaError_t unkeyed_ed25519_sign_screened_launch(size_t n, const uint8_t* verdict, const uint8_t* secrets, const uint8_t* msgs,
                                                 const uint64_t* msg_off, const uint32_t* gtab, uint8_t* sig, uint8_t* pub,
                                                 uint8_t* status, cudaStream_t st, unsigned* launches) {
  unkeyed_ed25519_sign_screened_kernel<<<blocks128(n), 128, 0, st>>>(n, verdict, secrets, msgs, msg_off, gtab, sig, pub,
                                                                      status);
  return counted(launches);
}
