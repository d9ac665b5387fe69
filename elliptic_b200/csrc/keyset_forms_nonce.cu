// keyset_forms_nonce.cu -- the screened nonce kernel of eb200_eddsa_sign_batch_keyed_dev (body:
// ks_ss_nonce_screened_item in keyset_forms_body.cuh), launched by keyset_ss_sign_screened_launch in keyset_forms.cu.
//
// A translation unit of its own: in keyset_forms.cu's module, next to the screened challenge kernel, ptxas (with
// -split-compile) gives the nonce kernel's out-of-line callees ed_add_niels and f25_mul 228 and 72 bytes of spills and
// the kernel a 688-byte stack, which made the device-pointer sign slower than its host form.  Alone, the kernel
// compiles as ed_signset_nonce_kernel does, with no spilling callee.
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
keyset_ss_nonce_screened_kernel(size_t N, const uint8_t* __restrict__ verdict, const uint8_t* __restrict__ msgs,
                                const u64* __restrict__ msg_off, const u32* __restrict__ key_idx, const u32* __restrict__ keys,
                                const u32* __restrict__ gtab, u32* __restrict__ ws) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ks_ss_nonce_screened_item(i, N, verdict, msgs, msg_off, key_idx, keys, gtab, ws);
}
cudaError_t keyset_ss_nonce_screened_launch(size_t n, const uint8_t* verdict, const KeysetDev& k, const uint8_t* msgs,
                                            const uint64_t* msg_off, const uint32_t* key_idx, const uint32_t* gtab,
                                            uint32_t* ws, cudaStream_t st, unsigned* launches) {
  keyset_ss_nonce_screened_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(n, verdict, msgs, msg_off, key_idx, k.tab,
                                                                               gtab, ws);
  cudaError_t err = cudaGetLastError();
  if (err == cudaSuccess) ++*launches;
  return err;
}
