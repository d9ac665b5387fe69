// Host emulation of the curve25519 key-set kernel bodies -- TEST INFRASTRUCTURE ONLY.
// Compiles the same .cuh bodies x25519_keyset.cu launches, with their portable C++ fallbacks, and runs them in the
// kernels' order: classify -> window bases -> table windows, then the keyed main body and the batched normalisation.
// The unkeyed ladder body runs on the same items for comparison.  The product library never contains or calls this code.
#include <cstring>
#include <vector>
#include "../../elliptic_b200/csrc/x25519_keyset_body.cuh"
using namespace eb;

extern "C" {

// pubx: m x 32 keys; priv: N x 32 (each < n); key_idx: N.  key_status, A (the Edwards images): m, m x 32 out;
// out, status: N x 32, N out.
void he_x25519_keyset_derive(int W, size_t m, const uint8_t* pubx, size_t N, const uint8_t* priv, const u32* key_idx,
                             uint8_t* key_status, uint8_t* A, uint8_t* out, uint8_t* status) {
  const int windows = ed_keyset_windows(W);
  std::vector<u32> bases(m * windows * 24), tab(ed_keyset_key_bytes(W) / 4 * m), ws((size_t)X25519_KS_WS_WORDS * N);
  for (size_t k = 0; k < m; k++) key_status[k] = x25519_ks_classify_item(k, pubx, A);
  for (size_t k = 0; k < m; k++) ed_ks_bases_item(k, A, key_status, W, windows, bases.data());
  for (size_t t = 0; t < m * windows; t++) ed_ks_window_item(t, key_status, W, windows, bases.data(), tab.data());
  for (size_t i = 0; i < N; i++) x25519_derive_keyed_item(i, N, priv, key_idx, key_status, W, windows, tab.data(), ws.data(), status);
  for (size_t t = 0; t < (N + X25519_KS_BATCH - 1) / X25519_KS_BATCH; t++) x25519_keyed_norm_item(t, N, N, ws.data(), status, out);
}

// The unkeyed body (x25519_derive_item) on N items, pubx: N x 32.
void he_x25519_unkeyed_derive(size_t N, const uint8_t* priv, const uint8_t* pubx, uint8_t* out, uint8_t* status) {
  for (size_t i = 0; i < N; i++) status[i] = x25519_derive_item(i, priv, pubx, out);
}
}
