// unkeyed_forms.h -- the kernels of unkeyed_forms.cu, launched by eb200.cu for the device-pointer forms of the unkeyed
// calls with variable-length ranges.  Each launches one kernel on `st` and adds it to *launches.  verdict: n bytes, 0 or
// EB200_ST_BAD_ITEM (unkeyed_forms_body.cuh).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

// Range screen: verdict[i] = EB200_ST_BAD_ITEM for off[i + 1] < off[i] or off[i + 1] > len, else 0.
cudaError_t unkeyed_range_screen_launch(size_t n, const uint64_t* off, uint64_t len, uint8_t* verdict, cudaStream_t st,
                                        unsigned* launches);
// der_decode_kernel with the range screen's verdicts: a screened item reads no byte of der; r = s = 0 for it and for a
// rejected encoding.  Arguments otherwise as der_decode_kernel's.
cudaError_t unkeyed_der_decode_screened_launch(size_t n, uint32_t len, const uint8_t* verdict, const uint8_t* der,
                                               const unsigned long long* off, uint8_t* r, uint8_t* s, uint8_t* pre,
                                               int pre_valid, cudaStream_t st, unsigned* launches);
// ed25519_sign_kernel with the range screen's verdicts: a screened item reads nothing, zeroes its pub row (pub may be
// NULL) and gets status 0.
cudaError_t unkeyed_ed25519_sign_screened_launch(size_t n, const uint8_t* verdict, const uint8_t* secrets, const uint8_t* msgs,
                                                 const uint64_t* msg_off, const uint32_t* gtab, uint8_t* sig, uint8_t* pub,
                                                 uint8_t* status, cudaStream_t st, unsigned* launches);
