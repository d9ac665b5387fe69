// Host emulation of the bodies around the keyed verify for its DER and device-pointer forms -- TEST INFRASTRUCTURE ONLY.
// Compiles keyset_forms_body.cuh (the bodies keyset_forms.cu launches) with the keyed verify bodies of keyset_emu.cpp, so
// that a test can run keyed DER decode -> prep -> keyed main -> keyed replay -> verdict merge in the kernels' order.
// The product library (libelliptic_b200.so) never contains or calls this code.
#include "keyset_emu.cpp"
#include "../../elliptic_b200/csrc/keyset_forms_body.cuh"

extern "C" {

// keyset_der_decode_kernel over N items: der / off as eb200_ecdsa_verify_batch_der takes them, kst: the set's verdicts.
void he_ks_der_decode(size_t N, u32 len, const uint8_t* der, const unsigned long long* off, const u32* key_idx,
                      const uint8_t* kst, uint8_t* r, uint8_t* s, uint8_t* verdict) {
  for (size_t i = 0; i < N; i++) verdict[i] = ks_der_verdict_item(i, len, der, off, key_idx, kst, r, s);
}

// keyset_index_screen_kernel over N items.
void he_ks_index_screen(size_t N, const u32* key_idx, size_t m, u32* idx_out, uint8_t* verdict) {
  for (size_t i = 0; i < N; i++) verdict[i] = ks_index_screen_item(i, key_idx, m, idx_out);
}

// keyset_verdict_merge_kernel over N items.
void he_ks_verdict_merge(size_t N, const uint8_t* verdict, uint8_t* status) {
  for (size_t i = 0; i < N; i++) ks_verdict_merge_item(i, verdict, status);
}
}
