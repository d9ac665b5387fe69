// Host emulation of the EC.getKeyRecoveryParam kernel bodies -- TEST INFRASTRUCTURE ONLY.
// Compiles the same .cuh bodies recovery_param.cu launches, with their portable C++ fallbacks, and runs them in the
// kernels' order: prep -> main -> the items the main body flags through the cold body.  The product library
// (libelliptic_b200.so) never contains or calls this code.
#include <cstring>
#include <vector>
#include "../../elliptic_b200/csrc/ecdsa_k256_body.cuh"
#include "../../elliptic_b200/csrc/ecdsa_k256_sign.cuh"
#include "../../elliptic_b200/csrc/ecdsa_sw_body.cuh"
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

static void k256_recovery_param_host(size_t N, const uint8_t* e, const uint8_t* r, const uint8_t* s, const uint8_t* q,
                                     uint8_t* recid, uint8_t* status) {
  const u32* gtab = k256_host_gtab().data();
  std::vector<u32> ws((size_t)PREP_WORDS * N), scratch((size_t)8 * N), qtab((size_t)QTAB_WORDS * N);
  size_t T = (N + PREP_BATCH - 1) / PREP_BATCH;
  for (size_t t = 0; t < T; t++) prep_thread(t, T, N, e, r, s, ws.data(), scratch.data(), 2);
  for (size_t i = 0; i < N; i++) status[i] = recovery_param_item(i, N, q, r, ws.data(), gtab, qtab.data(), recid);
  for (size_t i = 0; i < N; i++)
    if (status[i] == ST_NEEDS_HOST) status[i] = recovery_param_cold_item(i, e, r, q, gtab, recid);
}

template <class C>
static void sw_recovery_param_host(size_t N, const uint8_t* e, const uint8_t* r, const uint8_t* s, const uint8_t* q,
                                   uint8_t* recid, uint8_t* status) {
  typedef SW<C> W;
  static std::vector<u32> gtab;
  if (gtab.empty()) {
    gtab.resize((size_t)W::GWINDOWS * W::GENTRIES * 2 * W::N);
    for (int j = 0; j < W::GWINDOWS; j++)
      for (int i = 0; i < W::GENTRIES; i++) W::gtab_entry(j, i, &gtab[((size_t)j * W::GENTRIES + i) * 2 * W::N]);
  }
  std::vector<u32> ws((size_t)W::PREP_WORDS * N), qtab((size_t)W::QTAB_WORDS * N);
  for (size_t i = 0; i < N; i++) W::prep_recovery_param_item(i, N, e, r, s, ws.data());
  for (size_t i = 0; i < N; i++) status[i] = W::recovery_param_item(i, N, q, r, ws.data(), gtab.data(), qtab.data(), recid);
  for (size_t i = 0; i < N; i++)
    if (status[i] == ST_NEEDS_HOST) status[i] = W::recovery_param_cold_item(i, e, r, q, gtab.data(), recid);
}

// curve: the C-ABI id (1 secp256k1, 2 p256, 3 p384, 6 p521, 7 p192, 8 p224); arguments as
// eb200_ecdsa_recovery_param_batch takes them
extern "C" void he_recovery_param(int curve, size_t N, const uint8_t* e, const uint8_t* r, const uint8_t* s, const uint8_t* q,
                                  uint8_t* recid, uint8_t* status) {
  if (curve == 1) k256_recovery_param_host(N, e, r, s, q, recid, status);
  else if (curve == 2) sw_recovery_param_host<P256>(N, e, r, s, q, recid, status);
  else if (curve == 6) sw_recovery_param_host<P521>(N, e, r, s, q, recid, status);
  else if (curve == 7) sw_recovery_param_host<P192>(N, e, r, s, q, recid, status);
  else if (curve == 8) sw_recovery_param_host<P224>(N, e, r, s, q, recid, status);
  else sw_recovery_param_host<P384>(N, e, r, s, q, recid, status);
}
