// Host emulation of the bodies around the unkeyed kernels for their device-pointer forms -- TEST INFRASTRUCTURE ONLY.
// Compiles unkeyed_forms_body.cuh (the bodies unkeyed_forms.cu launches) with the EdDSA bodies of ed_signset_emu.cpp, so
// that a test can run the range screen and the screened DER decode alone, and a screened EdDSA sign batch in the
// kernels' order: range screen -> screened sign -> merge.
// The product library (libelliptic_b200.so) never contains or calls this code.
#include "../../elliptic_b200/csrc/unkeyed_forms_body.cuh"
#include "ed_signset_emu.cpp"

extern "C" {

// unkeyed_range_screen_kernel over N items (off: N + 1 offsets).
void he_ud_range_screen(size_t N, const u64* off, u64 len, uint8_t* verdict) {
  for (size_t i = 0; i < N; i++) verdict[i] = ud_range_screen_item(i, off, len);
}

// unkeyed_der_decode_screened_kernel over N items.
void he_ud_der_decode_screened(size_t N, u32 len, const uint8_t* verdict, const uint8_t* der, const unsigned long long* off,
                               uint8_t* r, uint8_t* s, uint8_t* pre, int pre_valid) {
  for (size_t i = 0; i < N; i++) ud_der_decode_screened_item(i, len, verdict, der, off, r, s, pre, pre_valid);
}

// The screened sign of eb200_eddsa_sign_batch_dev over n items, from the range screen to the merge.  pub may be NULL.
void he_ud_sign_screened(size_t n, const uint8_t* secrets, const uint8_t* msgs, u64 msgs_len, const u64* off, uint8_t* sig,
                         uint8_t* pub, uint8_t* status) {
  const u32* gtab = ed_host_gtab().data();
  std::vector<uint8_t> vd(n, 0xA5);
  for (size_t i = 0; i < n; i++) vd[i] = ud_range_screen_item(i, off, msgs_len);
  for (size_t i = 0; i < n; i++) status[i] = ud_ed25519_sign_screened_item(i, vd.data(), secrets, msgs, off, gtab, sig, pub);
  for (size_t i = 0; i < n; i++) ks_verdict_merge_out_item(i, vd.data(), status, sig, 64);
}
}
