// Host emulation of the bodies around the keyed kernels for their device-pointer forms -- TEST INFRASTRUCTURE ONLY.
// Compiles keyset_forms_body.cuh (the bodies keyset_forms.cu launches) with the EdDSA signing-set bodies of
// ed_signset_emu.cpp, so that a test can run the screens and merges alone and a screened sign batch in the kernels'
// order: range screen -> screened nonce -> normalise -> screened challenge -> merge.
// The product library (libelliptic_b200.so) never contains or calls this code.
#include "../../elliptic_b200/csrc/keyset_forms_body.cuh"
#include "ed_signset_emu.cpp"

extern "C" {

// keyset_index_scalar_screen_kernel over N items.
void he_ks_index_scalar_screen(size_t N, const u32* key_idx, size_t m, const uint8_t* k, int big_endian, u32* idx_out,
                               uint8_t* k_out, uint8_t* verdict) {
  for (size_t i = 0; i < N; i++) verdict[i] = ks_index_scalar_screen_item(i, key_idx, m, k, big_endian != 0, idx_out, k_out);
}

// keyset_index_range_screen_kernel over N items (off: N + 1 offsets).
void he_ks_index_range_screen(size_t N, const u32* key_idx, size_t m, const u64* off, u64 msgs_len, u32* idx_out,
                              uint8_t* verdict) {
  for (size_t i = 0; i < N; i++) verdict[i] = ks_index_range_screen_item(i, key_idx, m, off, msgs_len, idx_out);
}

// keyset_verdict_merge_out_kernel over N items.
void he_ks_verdict_merge_out(size_t N, const uint8_t* verdict, uint8_t* status, uint8_t* out, u32 ol) {
  for (size_t i = 0; i < N; i++) ks_verdict_merge_out_item(i, verdict, status, out, ol);
}

// keyset_ed_hash_screened_kernel over N items.
void he_ks_ed_hash_screened(size_t N, const uint8_t* verdict, const uint8_t* R, const uint8_t* A, const uint8_t* msgs,
                            const u64* off, uint8_t* h) {
  for (size_t i = 0; i < N; i++) ks_ed_hash_screened_item(i, verdict, R, A, msgs, off, h);
}

// The screened sign of eb200_eddsa_sign_batch_keyed_dev over n items, from the range screen to the merge, on a
// workspace of stale words; keys / pub as he_ed_signset_create wrote them (m keys).  status: n out, sig: n x 64 out.
void he_ks_sign_screened(const u32* keys, const uint8_t* pub, size_t m, size_t n, const uint8_t* msgs, u64 msgs_len,
                         const u64* off, const u32* key_idx, uint8_t* sig, uint8_t* status) {
  const u32* gtab = ed_host_gtab().data();
  std::vector<u32> ws((size_t)ED_SS_WS_WORDS * n, 0xA5A5A5A5u), idx(n, 0xA5A5A5A5u);
  std::vector<uint8_t> vd(n, 0xA5);
  for (size_t i = 0; i < n; i++) vd[i] = ks_index_range_screen_item(i, key_idx, m, off, msgs_len, idx.data());
  for (size_t i = 0; i < n; i++) ks_ss_nonce_screened_item(i, n, vd.data(), msgs, off, idx.data(), keys, gtab, ws.data());
  for (size_t t = 0; t < (n + ED_SS_BATCH - 1) / ED_SS_BATCH; t++) ed_ss_normalise_item(t, n, n, ws.data(), sig);
  for (size_t i = 0; i < n; i++) ks_ss_challenge_screened_item(i, n, vd.data(), msgs, off, idx.data(), keys, pub, ws.data(), sig);
  for (size_t i = 0; i < n; i++) status[i] = EB200_ST_TRUE;
  for (size_t i = 0; i < n; i++) ks_verdict_merge_out_item(i, vd.data(), status, sig, 64);
}
}
