// Host emulation of the EdDSA signing-set kernel bodies -- TEST INFRASTRUCTURE ONLY.
// Compiles the same .cuh bodies eddsa_signset.cu launches, with their portable C++ fallbacks, and runs them in the
// kernels' order: create, then nonce -> normalise -> challenge over a whole batch.  The unkeyed body
// (ed25519_sign_item) runs on the same items for comparison.  The product library never contains or calls this code.
#include <cstring>
#include <vector>
#include "../../elliptic_b200/csrc/ed25519_signset_body.cuh"
#include "ed_keyset_emu.cpp"        // ed_host_gtab(): the fixed-base table, built incrementally
using namespace eb;

extern "C" {

int he_ed_signset_batch() { return ED_SS_BATCH; }

// create: m secrets (m x 32) -> key words (m x ED_SS_KEY_WORDS) and encoded public keys (m x 32)
void he_ed_signset_create(size_t m, const uint8_t* secrets, u32* keys, uint8_t* pub) {
  const u32* gtab = ed_host_gtab().data();
  for (size_t k = 0; k < m; k++) ed_ss_create_item(k, secrets, gtab, keys, pub);
}

// sign: n items, item i by key key_idx[i] of (keys, pub) as create wrote them; sig: n x 64
void he_ed_signset_sign(const u32* keys, const uint8_t* pub, size_t n, const uint8_t* msgs, const u64* off, const u32* key_idx,
                        uint8_t* sig) {
  const u32* gtab = ed_host_gtab().data();
  std::vector<u32> ws((size_t)ED_SS_WS_WORDS * n, 0xA5A5A5A5u);
  for (size_t i = 0; i < n; i++) ed_ss_nonce_item(i, n, msgs, off, key_idx, keys, gtab, ws.data());
  for (size_t t = 0; t < (n + ED_SS_BATCH - 1) / ED_SS_BATCH; t++) ed_ss_normalise_item(t, n, n, ws.data(), sig);
  for (size_t i = 0; i < n; i++) ed_ss_challenge_item(i, n, msgs, off, key_idx, keys, pub, ws.data(), sig);
}

// the unkeyed body: secrets n x 32; sig n x 64, pub n x 32
void he_ed_sign_unkeyed(size_t n, const uint8_t* secrets, const uint8_t* msgs, const u64* off, uint8_t* sig, uint8_t* pub) {
  const u32* gtab = ed_host_gtab().data();
  for (size_t i = 0; i < n; i++) ed25519_sign_item(i, secrets, msgs, off, gtab, sig, pub);
}

// The normalisation body alone on n points given item-major as X, Y, Z (n x 8 words each): Renc by the batched body
// into batched (n x 64, bytes 0..31 of each row) and by the per-item ed_encode into single (n x 32).
void he_ed_signset_normalise(size_t n, const u32* X, const u32* Y, const u32* Z, uint8_t* batched, uint8_t* single) {
  std::vector<u32> ws((size_t)ED_SS_WS_WORDS * n, 0xA5A5A5A5u);
  for (size_t i = 0; i < n; i++) {
    ed_ss_ws_store(ws.data(), ED_SS_WS_X, n, i, f25_load(X + 8 * i));
    ed_ss_ws_store(ws.data(), ED_SS_WS_Y, n, i, f25_load(Y + 8 * i));
    ed_ss_ws_store(ws.data(), ED_SS_WS_Z, n, i, f25_load(Z + 8 * i));
  }
  for (size_t t = 0; t < (n + ED_SS_BATCH - 1) / ED_SS_BATCH; t++) ed_ss_normalise_item(t, n, n, ws.data(), batched);
  for (size_t i = 0; i < n; i++) {
    ed_ext p;
    p.x = f25_load(X + 8 * i); p.y = f25_load(Y + 8 * i); p.z = f25_load(Z + 8 * i); p.t = f25_zero();
    ed_encode(p, single + 32 * i);
  }
}
}
