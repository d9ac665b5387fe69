// Host emulation of the keyed DER decode of eb200_ecdsa_verify_batch_keyed_der_dev -- TEST INFRASTRUCTURE ONLY.
// Runs keyset_forms_body.cuh's index-and-range screen and the screened keyed DER decode in the kernels' order, beside the
// unscreened keyed DER decode the host form launches.  The product library (libelliptic_b200.so) never contains or
// calls this code.
#include <vector>
#include "keyset_dev_emu.cpp"

extern "C" {

// keyset_index_range_screen_kernel then keyset_der_decode_screened_kernel over N items: off holds N + 1 offsets into the
// der_len bytes at der, kst the set's m verdicts.  idx_out, r, s (N x len) and verdict out.
void he_ks_der_screened(size_t N, u32 len, const u32* key_idx, size_t m, const uint8_t* der, u64 der_len, const u64* off,
                        const uint8_t* kst, u32* idx_out, uint8_t* r, uint8_t* s, uint8_t* verdict) {
  std::vector<uint8_t> pre(N, 0xA5);
  for (size_t i = 0; i < N; i++) pre[i] = ks_index_range_screen_item(i, key_idx, m, off, der_len, idx_out);
  for (size_t i = 0; i < N; i++)
    verdict[i] = ks_der_screened_item(i, len, pre.data(), der, (const unsigned long long*)off, idx_out, kst, r, s);
}

// keyset_der_decode_kernel over N items, as eb200_ecdsa_verify_batch_keyed_der launches it.
void he_ks_der_plain(size_t N, u32 len, const uint8_t* der, const u64* off, const u32* key_idx, const uint8_t* kst, uint8_t* r,
                     uint8_t* s, uint8_t* verdict) {
  for (size_t i = 0; i < N; i++)
    verdict[i] = ks_der_verdict_item(i, len, der, (const unsigned long long*)off, key_idx, kst, r, s);
}
}
