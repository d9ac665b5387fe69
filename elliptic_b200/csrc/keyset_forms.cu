// keyset_forms.cu -- the kernels that frame the unchanged keyed ECDSA verify (keyset.cu) for
// eb200_ecdsa_verify_batch_keyed_der (DER decode with the key's verdict, in front of the unchanged prep) and
// eb200_ecdsa_verify_batch_keyed_dev (index screen in front of it), and the verdict merge that both run behind the keyed
// replay.  Bodies: keyset_forms_body.cuh.
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

cudaError_t keyset_index_screen_launch(size_t n, const uint32_t* key_idx, size_t m, uint32_t* idx_out, uint8_t* verdict,
                                       cudaStream_t st, unsigned* launches) {
  keyset_index_screen_kernel<<<blocks128(n), 128, 0, st>>>(n, key_idx, m, idx_out, verdict);
  return counted(launches);
}

cudaError_t keyset_verdict_merge_launch(size_t n, const uint8_t* verdict, uint8_t* status, cudaStream_t st, unsigned* launches) {
  keyset_verdict_merge_kernel<<<blocks128(n), 128, 0, st>>>(n, verdict, status);
  return counted(launches);
}
