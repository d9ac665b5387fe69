// Host emulation of the EdDSA key-set kernel bodies -- TEST INFRASTRUCTURE ONLY.
// Compiles the same .cuh bodies eddsa_keyset.cu launches, with their portable C++ fallbacks, and runs them in the
// kernels' order: classify -> window bases -> table windows, then (raw messages) key gather -> hash, then the keyed main
// body.  The unkeyed body runs on the same items for comparison.  The product library never contains or calls this code.
#include <cstring>
#include <vector>
#include "../../elliptic_b200/csrc/ed25519_keyset_body.cuh"
using namespace eb;

// fixed-base table, built incrementally (entry (j, i) = i 2^(13 j) G, as ed_gtab_entry)
static const std::vector<u32>& ed_host_gtab() {
  static std::vector<u32> gtab;
  if (gtab.empty()) {
    gtab.resize((size_t)ED_GWINDOWS * ED_GENTRIES * 24);
    ed_ext base = ed_identity();
    ed_G(&base.x, &base.y);
    base.t = f25_mul(base.x, base.y);
    for (int j = 0; j < ED_GWINDOWS; j++) {
      ed_cached cb = ed_to_cached(base);
      ed_ext acc = ed_identity();
      for (int i = 0; i < ED_GENTRIES; i++) {
        f25 zi = f25_inv(acc.z);
        f25 x = f25_mul(acc.x, zi), y = f25_mul(acc.y, zi);
        u32* o = &gtab[((size_t)j * ED_GENTRIES + i) * 24];
        f25_store(o, f25_normalize(f25_add(y, x)));
        f25_store(o + 8, f25_normalize(f25_sub(y, x)));
        f25_store(o + 16, f25_normalize(f25_mul(f25_mul(x, y), f25_2d())));
        acc = ed_add_cached(acc, cb);
      }
      for (int k = 0; k < ED_GW; k++) base = ed_dbl(base);
    }
  }
  return gtab;
}

struct Set { std::vector<uint8_t> kst; std::vector<u32> tab; int W, windows; };

static void build(size_t m, const uint8_t* A, int W, Set& S) {
  S.W = W; S.windows = ed_keyset_windows(W);
  S.kst.resize(m);
  S.tab.assign(ed_keyset_key_bytes(W) / 4 * m, 0);
  std::vector<u32> bases(m * S.windows * 24);
  for (size_t k = 0; k < m; k++) S.kst[k] = ed_ks_classify_item(k, A);
  for (size_t k = 0; k < m; k++) ed_ks_bases_item(k, A, S.kst.data(), W, S.windows, bases.data());
  for (size_t t = 0; t < m * S.windows; t++) ed_ks_window_item(t, S.kst.data(), W, S.windows, bases.data(), S.tab.data());
}

extern "C" {

// A: m raw keys; R, S: N x 32; h: N x 32 (h < n), or NULL for msgs + off (hashed over the gathered key bytes).
// key_status: m bytes, status: N bytes.
void he_ed_keyset_verify(int W, size_t m, const uint8_t* A, size_t N, const uint8_t* R, const uint8_t* S, const uint8_t* h,
                         const uint8_t* msgs, const u64* off, const u32* key_idx, uint8_t* key_status, uint8_t* status) {
  const u32* gtab = ed_host_gtab().data();
  Set st;
  build(m, A, W, st);
  memcpy(key_status, st.kst.data(), m);
  std::vector<uint8_t> hh;
  if (!h) {
    std::vector<uint8_t> Ag(32 * N);
    hh.resize(32 * N);
    for (size_t i = 0; i < N; i++) ed_ks_gather_item(i, key_idx, A, Ag.data());
    for (size_t i = 0; i < N; i++) ed25519_hash_item(i, R, Ag.data(), msgs, off, hh.data());
    h = hh.data();
  }
  for (size_t i = 0; i < N; i++)
    status[i] = ed25519_verify_keyed_item(i, R, S, h, key_idx, st.kst.data(), W, st.windows, st.tab.data(), gtab);
}

// The unkeyed body (ed25519_verify_item) on N items, A: N x 32.
void he_ed_unkeyed_verify(size_t N, const uint8_t* R, const uint8_t* S, const uint8_t* A, const uint8_t* h, uint8_t* status) {
  const u32* gtab = ed_host_gtab().data();
  std::vector<u32> atab((size_t)ED_ATAB_WORDS * N);
  for (size_t i = 0; i < N; i++) status[i] = ed25519_verify_item(i, R, S, A, h, gtab, atab.data());
}

// One key's table as the main loop reads it (windows * 2^(W-1) entries of y+x, y-x, 2d x y; 24 words each).
void he_ed_keyset_table(int W, const uint8_t* A, u32* out) {
  Set st;
  build(1, A, W, st);
  memcpy(out, st.tab.data(), st.tab.size() * 4);
}

int he_ed_keyset_windows(int W) { return ed_keyset_windows(W); }
size_t he_ed_keyset_key_bytes(int W) { return ed_keyset_key_bytes(W); }
unsigned he_ed_keyset_choose_bits(size_t m, size_t budget) { return ed_keyset_choose_bits(m, budget); }
}
