// Host emulation of the key-set kernel bodies -- TEST INFRASTRUCTURE ONLY.
// Compiles the same .cuh bodies keyset.cu launches, with their portable C++ fallbacks, and runs them in the kernels'
// order: classify -> window bases -> table windows, then prep -> keyed main -> keyed replay of the off-curve-key items.
// The product library (libelliptic_b200.so) never contains or calls this code.
#include <cstring>
#include <vector>
#include "../../elliptic_b200/csrc/ecdsa_k256_body.cuh"
#include "../../elliptic_b200/csrc/ecdsa_k256_replay.cuh"
#include "../../elliptic_b200/csrc/ecdsa_sw_body.cuh"
#include "../../elliptic_b200/csrc/ecdsa_sw_replay.cuh"
#include "../../elliptic_b200/csrc/ecdsa_keyset_body.cuh"
using namespace eb;

// secp256k1 fixed-base table, built incrementally (entry (j, i) = (2i + 1) 2^(W j) G, as gtab_entry)
static const std::vector<u32>& k256_host_gtab() {
  static std::vector<u32> tab;
  if (tab.empty()) {
    tab.resize((size_t)GTAB_WINDOWS * GTAB_ENTRIES * 16);
    ge_jac base = jac_from_aff(k256_G());
    for (int j = 0; j < GTAB_WINDOWS; j++) {
      ge_aff b = jac_to_aff(base);
      ge_jac d = jac_dbl(jac_from_aff(b));
      ge_jac acc = jac_from_aff(b);
      for (int i = 0; i < GTAB_ENTRIES; i++) {
        ge_aff r = jac_to_aff(acc);
        store_fe(&tab[((size_t)j * GTAB_ENTRIES + i) * 16], fe_normalize(r.x));
        store_fe(&tab[((size_t)j * GTAB_ENTRIES + i) * 16 + 8], fe_normalize(r.y));
        acc = jac_add_inl(acc, d);
      }
      for (int k = 0; k < GTAB_W; k++) base = jac_dbl(base);
    }
  }
  return tab;
}

struct Set { std::vector<uint8_t> kst; std::vector<u32> tab; int W, windows; };

static void k256_build(size_t m, const uint8_t* xy, int W, Set& S) {
  S.W = W; S.windows = keyset_windows(EB200_CURVE_SECP256K1, W);
  S.kst.resize(m);
  S.tab.assign(keyset_key_bytes(EB200_CURVE_SECP256K1, W) / 4 * m, 0);
  std::vector<u32> bases(m * S.windows * 24);
  for (size_t k = 0; k < m; k++) S.kst[k] = k256_ks_classify_item(k, xy, nullptr);
  for (size_t k = 0; k < m; k++) k256_ks_bases_item(k, xy, S.kst.data(), W, S.windows, bases.data());
  for (size_t t = 0; t < m * S.windows; t++) k256_ks_window_item(t, S.kst.data(), W, S.windows, bases.data(), S.tab.data());
}

static void k256_keyed_host(int W, size_t m, const uint8_t* xy, size_t N, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                            const u32* key_idx, uint8_t* key_status, uint8_t* status) {
  const u32* gtab = k256_host_gtab().data();
  static std::vector<u32> rtab;
  if (rtab.empty()) {
    rtab.resize(REPLAY_TAB_WORDS);
    for (int t = 0; t < 2 * REPLAY_NAF_PTS; t++) rp_tab_entry(t, &rtab[16 * t]);
  }
  Set S;
  k256_build(m, xy, W, S);
  memcpy(key_status, S.kst.data(), m);
  std::vector<u32> ws((size_t)PREP_WORDS * N), scratch((size_t)8 * N);
  size_t T = (N + PREP_BATCH - 1) / PREP_BATCH;
  for (size_t t = 0; t < T; t++) prep_thread(t, T, N, e, r, s, ws.data(), scratch.data());
  for (size_t i = 0; i < N; i++)
    status[i] = k256_verify_keyed_item(i, N, key_idx, S.kst.data(), W, S.windows, S.tab.data(), r, ws.data(), gtab);
  for (size_t i = 0; i < N; i++)
    if (status[i] == ST_NEEDS_HOST)
      status[i] = rp_verify_item(0, e + 32 * i, r + 32 * i, s + 32 * i, xy + 64 * (size_t)key_idx[i], rtab.data());
}

template <class C>
static void sw_build(int curve, size_t m, const uint8_t* xy, int W, Set& S) {
  typedef SWKeyed<C> K;
  S.W = W; S.windows = keyset_windows(curve, W);
  S.kst.resize(m);
  S.tab.assign(keyset_key_bytes(curve, W) / 4 * m, 0);
  std::vector<u32> bases(m * S.windows * 3 * C::N);
  for (size_t k = 0; k < m; k++) S.kst[k] = K::classify_item(k, xy, nullptr);
  for (size_t k = 0; k < m; k++) K::bases_item(k, xy, S.kst.data(), W, S.windows, bases.data());
  for (size_t t = 0; t < m * S.windows; t++) K::window_item(t, S.kst.data(), W, S.windows, bases.data(), S.tab.data());
}

template <class C>
static void sw_keyed_host(int curve, int W, size_t m, const uint8_t* xy, size_t N, const uint8_t* e, const uint8_t* r,
                          const uint8_t* s, const u32* key_idx, uint8_t* key_status, uint8_t* status) {
  typedef SW<C> W_;
  typedef SWKeyed<C> K;
  const size_t LEN = C::LEN;
  static std::vector<u32> gtab, rtab;
  if (gtab.empty()) {
    gtab.resize((size_t)W_::GWINDOWS * W_::GENTRIES * 2 * W_::N);
    for (int j = 0; j < W_::GWINDOWS; j++)
      for (int i = 0; i < W_::GENTRIES; i++) W_::gtab_entry(j, i, &gtab[((size_t)j * W_::GENTRIES + i) * 2 * W_::N]);
    rtab.resize(SWReplay<C>::TAB_WORDS);
    for (int t = 0; t < SWReplay<C>::NAF_PTS; t++) SWReplay<C>::tab_entry(t, &rtab[2 * C::N * t]);
  }
  Set S;
  sw_build<C>(curve, m, xy, W, S);
  memcpy(key_status, S.kst.data(), m);
  std::vector<u32> ws((size_t)W_::PREP_WORDS * N), scratch((size_t)W_::N * N);
  size_t T = (N + W_::BATCH - 1) / W_::BATCH;
  for (size_t t = 0; t < T; t++) W_::prep_thread(t, T, N, e, r, s, ws.data(), scratch.data());
  for (size_t i = 0; i < N; i++)
    status[i] = K::verify_keyed_item(i, N, key_idx, S.kst.data(), W, S.windows, S.tab.data(), r, ws.data(), gtab.data());
  for (size_t i = 0; i < N; i++)
    if (status[i] == ST_NEEDS_HOST)
      status[i] = SWReplay<C>::verify_item(0, e + LEN * i, r + LEN * i, s + LEN * i, xy + 2 * LEN * (size_t)key_idx[i], rtab.data());
}

extern "C" {

// curve: the C-ABI id (1 secp256k1, 2 p256, 3 p384, 6 p521, 7 p192, 8 p224).  xy: m keys x || y; the other arguments as
// eb200_ecdsa_verify_batch_keyed takes them.  key_status: m bytes, status: N bytes.
void he_keyset_verify(int curve, int W, size_t m, const uint8_t* xy, size_t N, const uint8_t* e, const uint8_t* r,
                      const uint8_t* s, const u32* key_idx, uint8_t* key_status, uint8_t* status) {
  if (curve == 1) k256_keyed_host(W, m, xy, N, e, r, s, key_idx, key_status, status);
  else if (curve == 2) sw_keyed_host<P256>(curve, W, m, xy, N, e, r, s, key_idx, key_status, status);
  else if (curve == 3) sw_keyed_host<P384>(curve, W, m, xy, N, e, r, s, key_idx, key_status, status);
  else if (curve == 6) sw_keyed_host<P521>(curve, W, m, xy, N, e, r, s, key_idx, key_status, status);
  else if (curve == 7) sw_keyed_host<P192>(curve, W, m, xy, N, e, r, s, key_idx, key_status, status);
  else sw_keyed_host<P224>(curve, W, m, xy, N, e, r, s, key_idx, key_status, status);
}

// One key's table as the main loop reads it, with every coordinate converted to plain canonical limbs
// (out: windows * 2^(W-1) entries of x || y, 2 * limbs words each).
void he_keyset_table(int curve, int W, const uint8_t* xy, u32* out) {
  Set S;
  if (curve == 1) {
    k256_build(1, xy, W, S);
    memcpy(out, S.tab.data(), S.tab.size() * 4);
    return;
  }
  auto plain = [&](auto c) {
    typedef decltype(c) C;
    typedef typename SW<C>::F F;
    sw_build<C>(curve, 1, xy, W, S);
    for (size_t k = 0; k < S.tab.size(); k += C::N) {
      typename F::fe v = F::from_mont(load_fe_n<C::N>(&S.tab[k]));
      store_fe_n<C::N>(out + k, v);
    }
  };
  if (curve == 2) plain(P256{});
  else if (curve == 3) plain(P384{});
  else if (curve == 6) plain(P521{});
  else if (curve == 7) plain(P192{});
  else plain(P224{});
}

// beta * x of a secp256k1 entry, as the second GLV half of the main loop computes it
void he_k256_beta_x(const u32* x, u32* out) { store_fe(out, fe_normalize(fe_mul(load_fe(x), fe_beta()))); }

int he_keyset_windows(int curve, int W) { return keyset_windows(curve, W); }
size_t he_keyset_key_bytes(int curve, int W) { return keyset_key_bytes(curve, W); }
unsigned he_keyset_choose_bits(int curve, size_t m, size_t budget) { return keyset_choose_bits(curve, m, budget); }
}
