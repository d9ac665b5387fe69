// recovery_param.h -- the EC.getKeyRecoveryParam kernels (recovery_param.cu), launched by eb200.cu
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

// Device buffers of one eb200_ecdsa_recovery_param_batch block: e, r, s (n x len) and q (n x 2 len) in; recid and
// status (n bytes) out; the curve's fixed-base table; ws / scratch / qtab as ws_layout places them.
struct RecoveryParamArgs {
  const uint8_t *e, *r, *s, *q;
  uint8_t *recid, *status;
  const uint32_t* gtab;
  uint32_t *ws, *scratch, *qtab;
};

// Launches prep, main and cold on `st` for a short preset, recording main_begin / main_end around the main kernel, and
// adds the kernels launched to *launches.  Other curve ids launch nothing and return cudaErrorInvalidValue.
cudaError_t recovery_param_launch(int curve, size_t n, const RecoveryParamArgs& a, cudaStream_t st, cudaEvent_t main_begin,
                                  cudaEvent_t main_end, unsigned* launches);

// The prep kernel alone (u1 = e / s, u2 = (r mod n) / s, FL_INVALID for s = 0 mod n into ws; scratch: the secp256k1
// inversion's prefix products), for eb200_ecdsa_recovery_param_batch_keyed: its words are laid out as the verify prep's.
// Adds one launch to *launches.
cudaError_t recovery_param_prep_launch(int curve, size_t n, const uint8_t* e, const uint8_t* r, const uint8_t* s, uint32_t* ws,
                                       uint32_t* scratch, cudaStream_t st, unsigned* launches);
