// keyset.h -- the key-set kernels (keyset.cu), launched by eb200.cu
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "keyset_plan.h"

// One device's copy of a key set: m keys decoded to x || y (2 len bytes each), keyFromPublic's verdict per key
// (a throw status, EB200_ST_TRUE = on the curve, EB200_ST_FALSE = imported but off the curve) and the tables of the
// on-curve keys, keyset_key_bytes() apart, W bits per window.
struct KeysetDev {
  uint8_t* xy;
  uint8_t* kst;
  uint32_t* tab;
  int W;
};

// Classifies the m keys (pre: the decoder's statuses, or NULL for {x, y} input) and builds their tables on `st`.
// bases: scratch of m * windows * 3 * limbs words.  Adds the kernels launched (three) to *launches.
cudaError_t keyset_build_launch(int curve, size_t m, const KeysetDev& k, const uint8_t* pre, uint32_t* bases, cudaStream_t st,
                                unsigned* launches);

// Device buffers of one eb200_ecdsa_verify_batch_keyed block: e, r, s (n x len) and key_idx (n words) in, status out;
// ws as the curve's unkeyed prep kernel left it; the curve's fixed-base and replay tables.
struct KeyedVerifyArgs {
  const uint8_t *e, *r, *s;
  const uint32_t* key_idx;
  uint8_t* status;
  const uint32_t *ws, *gtab, *replay_tab;
};

// Launches the keyed main kernel (between main_begin and main_end) and the keyed replay of off-curve-key items on `st`;
// adds the kernels launched (two) to *launches.  Other curve ids launch nothing and return cudaErrorInvalidValue.
cudaError_t keyset_verify_launch(int curve, size_t n, const KeysetDev& k, const KeyedVerifyArgs& a, cudaStream_t st,
                                 cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches);
