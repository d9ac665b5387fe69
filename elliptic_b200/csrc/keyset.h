// keyset.h -- the key-set kernels (keyset.cu, keyset_forms.cu, keyset_forms_nonce.cu, keyset_mul.cu,
// keyset_recovery_param.cu, eddsa_keyset.cu, eddsa_signset.cu, x25519_keyset.cu), launched by eb200.cu
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "keyset_plan.h"

// One device's copy of a key set: m keys decoded to x || y (2 len bytes each), keyFromPublic's verdict per key
// (a throw status, EB200_ST_TRUE = on the curve, EB200_ST_FALSE = imported but off the curve) and the tables of the
// on-curve keys, keyset_key_bytes() apart, W bits per window.  An ed25519 set (eddsa_keyset.cu) keeps the 32 raw bytes
// of each key in `xy`, its verdict (EB200_ST_TRUE or the decoder's throw) in `kst` and ed_keyset_key_bytes() per key.
// An ed25519 signing set (eddsa_signset.cu) keeps each key's encoded A in `xy` and its secret words in `tab`: a
// (Montgomery form mod n) then the 32-byte message prefix, ED_SIGNSET_KEY_BYTES per key; `kst` is NULL and W = 0.
// A curve25519 set (x25519_keyset.cu) keeps in `xy` the ed25519 encoding of each key's Edwards image (zeros for a key
// that is not TRUE), its verdict (EB200_ST_TRUE or EB200_ST_THROW_ASSERT) in `kst` and the ed25519 set's tables in
// `tab`, ed_keyset_key_bytes() per key.
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

// keyset_forms.cu: the kernels around keyset_verify_launch for the DER and device-pointer forms of the keyed verify.  Each
// launches one kernel on `st` and adds it to *launches.  verdict: n bytes, 0 = the keyed status stands, else the item's
// status (keyset_forms_body.cuh).
// DER decode: der / off as der_decode_kernel takes them (n + 1 offsets into der); writes r, s (n x len; zeros for a
// rejected encoding) for the unchanged prep kernel, and per item the key's import throw (k.kst[key_idx[i]]), else
// EB200_ST_THROW_SIG_FORMAT for a rejected encoding, else 0.
cudaError_t keyset_der_decode_launch(size_t n, uint32_t len, const uint8_t* der, const unsigned long long* off,
                                     const uint32_t* key_idx, const KeysetDev& k, uint8_t* r, uint8_t* s, uint8_t* verdict,
                                     cudaStream_t st, unsigned* launches);
// The DER decode behind the index-and-range screen: pre holds that screen's verdicts and idx its screened indices; an
// item with a non-zero pre reads nothing, gets r = s = 0 and verdict pre[i], any other is decoded as above.
cudaError_t keyset_der_decode_screened_launch(size_t n, uint32_t len, const uint8_t* pre, const uint8_t* der,
                                              const unsigned long long* off, const uint32_t* idx, const KeysetDev& k,
                                              uint8_t* r, uint8_t* s, uint8_t* verdict, cudaStream_t st, unsigned* launches);
// Index screen: idx_out[i] = key_idx[i] when it is below m, else 0 with verdict EB200_ST_BAD_KEY_INDEX.
cudaError_t keyset_index_screen_launch(size_t n, const uint32_t* key_idx, size_t m, uint32_t* idx_out, uint8_t* verdict,
                                       cudaStream_t st, unsigned* launches);
// Verdict merge, behind the keyed replay: status[i] = verdict[i] wherever that is not 0.
cudaError_t keyset_verdict_merge_launch(size_t n, const uint8_t* verdict, uint8_t* status, cudaStream_t st, unsigned* launches);
// The device-pointer forms of the other keyed calls (keyset_forms_body.cuh), one kernel each unless stated.
// Index and scalar screen: as the index screen, and k_out[32 i ..] = the 32-byte scalar k[32 i ..] (little-endian, or
// big_endian), zeros with verdict EB200_ST_BAD_ITEM when it is not below the ed25519 group order n.
cudaError_t keyset_index_scalar_screen_launch(size_t n, const uint32_t* key_idx, size_t m, const uint8_t* k, bool big_endian,
                                              uint32_t* idx_out, uint8_t* k_out, uint8_t* verdict, cudaStream_t st,
                                              unsigned* launches);
// Index and range screen: as the index screen, then verdict EB200_ST_BAD_ITEM for off[i + 1] < off[i] or > msgs_len.
cudaError_t keyset_index_range_screen_launch(size_t n, const uint32_t* key_idx, size_t m, const uint64_t* off,
                                             uint64_t msgs_len, uint32_t* idx_out, uint8_t* verdict, cudaStream_t st,
                                             unsigned* launches);
// Verdict merge of a call with outputs: as the verdict merge, and out[ol i .. ol i + ol) = 0 where the verdict is not 0.
cudaError_t keyset_verdict_merge_out_launch(size_t n, const uint8_t* verdict, uint8_t* status, uint8_t* out, uint32_t ol,
                                            cudaStream_t st, unsigned* launches);
// The keyed EdDSA hash (ed25519_hash_kernel) of the items whose verdict is 0; h = 0 for the others.
cudaError_t keyset_ed_hash_screened_launch(size_t n, const uint8_t* verdict, const uint8_t* R, const uint8_t* A,
                                           const uint8_t* msgs, const uint64_t* msg_off, uint8_t* h, cudaStream_t st,
                                           unsigned* launches);
// keyset_forms_nonce.cu: the screened nonce kernel alone (one kernel); the items whose verdict is not 0 read no message
// byte and leave R = the identity, r = 0 in ws.
cudaError_t keyset_ss_nonce_screened_launch(size_t n, const uint8_t* verdict, const KeysetDev& k, const uint8_t* msgs,
                                            const uint64_t* msg_off, const uint32_t* key_idx, const uint32_t* gtab,
                                            uint32_t* ws, cudaStream_t st, unsigned* launches);
// ed_signset_sign_launch with screened nonce and challenge kernels around the unchanged normalisation: the items whose
// verdict is not 0 read no message byte and leave R = the identity, r = 0 in ws.  Three kernels.
cudaError_t keyset_ss_sign_screened_launch(size_t n, const uint8_t* verdict, const KeysetDev& k, const uint8_t* msgs,
                                           const uint64_t* msg_off, const uint32_t* key_idx, const uint32_t* gtab, uint32_t* ws,
                                           uint8_t* sig, cudaStream_t st, cudaEvent_t main_begin, cudaEvent_t main_end,
                                           unsigned* launches);

// keyset_mul.cu.  Device buffers of one keyed mul / mulAdd / derive block: k1 (NULL: no base-point term), k2 (n x len, as the caller
// gave them: the replay uses them unreduced) and key_idx in; ws as the curve's unkeyed prep_scalars kernel left it;
// jac: 3 x limbs x n words and scratch: limbs x n words of workspace; out (n x 2 len, or n x len for derive) and status
// out.  batch: items per normalisation thread on secp256k1 (the other curves use SW<C>::BATCH).
struct KeyedMulArgs {
  const uint8_t *k1, *k2;
  const uint32_t* key_idx;
  const uint32_t* ws;
  uint32_t *jac, *scratch;
  const uint32_t *gtab, *replay_tab;
  uint8_t *out, *status;
  int batch;
  bool derive;
};

// Launches the keyed main kernel (between main_begin and main_end), the normalisation and, unless a.derive, the keyed
// replay of off-curve-key items on `st`; adds the kernels launched (three, or two for derive) to *launches.  For
// derive, the off-curve-key items are left as ST_NEEDS_HOST with zeroed output.  Other curve ids launch nothing and
// return cudaErrorInvalidValue.
cudaError_t keyset_mul_launch(int curve, size_t n, const KeysetDev& k, const KeyedMulArgs& a, cudaStream_t st,
                              cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches);

// keyset_recovery_param.cu.  Device buffers of one keyed getKeyRecoveryParam block: e, r (n x len) and key_idx in; ws as
// the curve's unkeyed recovery-parameter prep left it; yz: 2 x limbs x n words and scratch: limbs x n words of
// workspace; recid and status (n bytes) out.  batch: items per normalisation thread on secp256k1 (the other curves use
// SW<C>::BATCH).
struct KeyedRecoveryParamArgs {
  const uint8_t *e, *r;
  const uint32_t* key_idx;
  const uint32_t* ws;
  uint32_t *yz, *scratch;
  const uint32_t* gtab;
  uint8_t *recid, *status;
  int batch;
};

// Launches the keyed main kernel (between main_begin and main_end), the recid normalisation and the cold kernel for
// s = 0 (mod n) on `st`; adds the kernels launched (three) to *launches.  Other curve ids launch nothing and return
// cudaErrorInvalidValue.
cudaError_t keyset_recovery_param_launch(int curve, size_t n, const KeysetDev& k, const KeyedRecoveryParamArgs& a,
                                         cudaStream_t st, cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches);

// ed25519 (eddsa_keyset.cu).  Build: classifies the m raw keys in k.xy and builds their tables on `st`; bases: scratch of
// m * ed_keyset_windows(W) * 24 words.  Adds the kernels launched (three) to *launches.
cudaError_t ed_keyset_build_launch(size_t m, const KeysetDev& k, uint32_t* bases, cudaStream_t st, unsigned* launches);
// Writes the raw bytes of key key_idx[i] to A_out[32 i ..] for the hash kernel (one kernel).
cudaError_t ed_keyset_gather_launch(size_t n, const KeysetDev& k, const uint32_t* key_idx, uint8_t* A_out, cudaStream_t st,
                                    unsigned* launches);
// The keyed main kernel: R, S, h (n x 32, h < n) and key_idx in, status out; gtab: the ed25519 fixed-base table.
cudaError_t ed_keyset_verify_launch(size_t n, const KeysetDev& k, const uint8_t* R, const uint8_t* S, const uint8_t* h,
                                    const uint32_t* key_idx, const uint32_t* gtab, uint8_t* status, cudaStream_t st,
                                    unsigned* launches);

// ed25519 signing sets (eddsa_signset.cu).  Create: secrets (m x 32) in, k.tab and k.xy (the encoded A) out; gtab: the
// ed25519 fixed-base table.  One kernel.
constexpr size_t ED_SIGNSET_KEY_BYTES = 64;
cudaError_t ed_signset_create_launch(size_t m, const KeysetDev& k, const uint8_t* secrets, const uint32_t* gtab,
                                     cudaStream_t st, unsigned* launches);
// Workspace of a sign launch of n items, and the byte range [offset, offset + bytes) of it that holds the nonces r.
size_t ed_signset_ws_bytes(size_t n);
size_t ed_signset_nonce_offset(size_t n);
size_t ed_signset_nonce_bytes(size_t n);
// Sign: msgs / msg_off (offsets relative to msgs), key_idx in, sig (n x 64) out; ws: ed_signset_ws_bytes(n).  Launches
// nonce (between main_begin and main_end), normalise and challenge kernels on `st` and adds three to *launches.
cudaError_t ed_signset_sign_launch(size_t n, const KeysetDev& k, const uint8_t* msgs, const uint64_t* msg_off,
                                   const uint32_t* key_idx, const uint32_t* gtab, uint32_t* ws, uint8_t* sig, cudaStream_t st,
                                   cudaEvent_t main_begin, cudaEvent_t main_end, unsigned* launches);
// The normalisation kernel of a sign launch alone: R of the n items in ws encoded into sig[64 i ..].  One kernel.
cudaError_t ed_signset_normalise_launch(size_t n, uint32_t* ws, uint8_t* sig, cudaStream_t st, unsigned* launches);

// curve25519 key sets (x25519_keyset.cu).  Build: classifies the m keys (pubx: m x 32 big-endian, on the device), writes
// their Edwards images to k.xy and builds their tables on `st`; bases: scratch of m * ed_keyset_windows(W) * 24 words.
// Adds the kernels launched (three) to *launches.
cudaError_t x25519_keyset_build_launch(size_t m, const KeysetDev& k, const uint8_t* pubx, uint32_t* bases, cudaStream_t st,
                                       unsigned* launches);
// Workspace of a derive launch of n items.
size_t x25519_keyset_ws_bytes(size_t n);
// Derive: priv (n x 32 big-endian, each < n) and key_idx in, out (n x 32 big-endian u) and status out; ws:
// x25519_keyset_ws_bytes(n).  Launches the keyed main kernel (between main_begin and main_end) and the normalisation on
// `st` and adds two to *launches.
cudaError_t x25519_keyset_derive_launch(size_t n, const KeysetDev& k, const uint8_t* priv, const uint32_t* key_idx, uint32_t* ws,
                                        uint8_t* out, uint8_t* status, cudaStream_t st, cudaEvent_t main_begin,
                                        cudaEvent_t main_end, unsigned* launches);
