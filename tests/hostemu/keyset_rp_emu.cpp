// Host emulation of the keyed getKeyRecoveryParam bodies -- TEST INFRASTRUCTURE ONLY.
// Runs the same .cuh bodies keyset.cu, recovery_param.cu and keyset_recovery_param.cu launch, in the kernels' order:
// classify -> window bases -> table windows, then the unkeyed recovery-parameter prep -> keyed main -> recid
// normalisation -> cold for the s = 0 (mod n) items on the key's coordinates.  The set builders and fixed-base tables are
// keyset_emu.cpp's.  The product library never contains or calls this code.
#include "keyset_emu.cpp"
#include "../../elliptic_b200/csrc/ecdsa_k256_sign.cuh"
#include "../../elliptic_b200/csrc/ecdsa_keyset_rp_body.cuh"

// The decoder's throws (pre[k] != 0) override the set's verdicts, as k256_ks_classify_item / classify_item take them
static void take_throws(size_t m, const uint8_t* pre, Set& S) {
  for (size_t k = 0; pre && k < m; k++)
    if (pre[k]) S.kst[k] = pre[k];
}

static void k256_rp_host(int W, size_t m, const uint8_t* xy, const uint8_t* pre, size_t N, const uint8_t* e, const uint8_t* r,
                         const uint8_t* s, const u32* key_idx, int batch, uint8_t* key_status, uint8_t* recid, uint8_t* status) {
  const u32* gtab = k256_host_gtab().data();
  Set S;
  k256_build(m, xy, W, S);
  take_throws(m, pre, S);
  memcpy(key_status, S.kst.data(), m);
  std::vector<u32> ws((size_t)PREP_WORDS * N), yz((size_t)16 * N), scratch((size_t)8 * N);
  size_t T = (N + PREP_BATCH - 1) / PREP_BATCH;
  for (size_t t = 0; t < T; t++) prep_thread(t, T, N, e, r, s, ws.data(), scratch.data(), 2);
  for (size_t i = 0; i < N; i++)
    status[i] = k256_recovery_param_keyed_item(i, N, key_idx, S.kst.data(), W, S.windows, S.tab.data(), r, ws.data(), gtab,
                                               yz.data(), recid);
  T = (N + batch - 1) / batch;
  for (size_t t = 0; t < T; t++) k256_ks_recid_norm_thread(t, T, N, batch, yz.data(), scratch.data(), status, recid);
  for (size_t i = 0; i < N; i++)
    if (status[i] == ST_NEEDS_HOST)
      status[i] = recovery_param_cold_item(0, e + 32 * i, r + 32 * i, xy + 64 * (size_t)key_idx[i], gtab, recid + i);
}

template <class C>
static void sw_rp_host(int curve, int W, size_t m, const uint8_t* xy, const uint8_t* pre, size_t N, const uint8_t* e,
                       const uint8_t* r, const uint8_t* s, const u32* key_idx, uint8_t* key_status, uint8_t* recid,
                       uint8_t* status) {
  typedef SW<C> W_;
  typedef SWKeyedRP<C> K;
  const size_t LEN = C::LEN;
  static std::vector<u32> gtab;
  if (gtab.empty()) {
    gtab.resize((size_t)W_::GWINDOWS * W_::GENTRIES * 2 * W_::N);
    for (int j = 0; j < W_::GWINDOWS; j++)
      for (int i = 0; i < W_::GENTRIES; i++) W_::gtab_entry(j, i, &gtab[((size_t)j * W_::GENTRIES + i) * 2 * W_::N]);
  }
  Set S;
  sw_build<C>(curve, m, xy, W, S);
  take_throws(m, pre, S);
  memcpy(key_status, S.kst.data(), m);
  std::vector<u32> ws((size_t)W_::PREP_WORDS * N), yz((size_t)2 * C::N * N), scratch((size_t)C::N * N);
  for (size_t i = 0; i < N; i++) W_::prep_recovery_param_item(i, N, e, r, s, ws.data());
  for (size_t i = 0; i < N; i++)
    status[i] = K::main_item(i, N, key_idx, S.kst.data(), W, S.windows, S.tab.data(), r, ws.data(), gtab.data(), yz.data(), recid);
  size_t T = (N + W_::BATCH - 1) / W_::BATCH;
  for (size_t t = 0; t < T; t++) K::recid_norm_thread(t, T, N, yz.data(), scratch.data(), status, recid);
  for (size_t i = 0; i < N; i++)
    if (status[i] == ST_NEEDS_HOST)
      status[i] = W_::recovery_param_cold_item(0, e + LEN * i, r + LEN * i, xy + 2 * LEN * (size_t)key_idx[i], gtab.data(),
                                               recid + i);
}

extern "C" {

// curve: the C-ABI id; xy: m keys x || y; pre: m decoder statuses (0 = decoded) or NULL; e, r, s, key_idx as
// eb200_ecdsa_recovery_param_batch_keyed takes them; batch: items per normalisation thread on secp256k1 (the other curves
// use SW<C>::BATCH = 16).  key_status: m bytes, recid and status: N bytes.
void he_keyset_recovery_param(int curve, int W, size_t m, const uint8_t* xy, const uint8_t* pre, size_t N, const uint8_t* e,
                              const uint8_t* r, const uint8_t* s, const u32* key_idx, int batch, uint8_t* key_status,
                              uint8_t* recid, uint8_t* status) {
  if (curve == 1) k256_rp_host(W, m, xy, pre, N, e, r, s, key_idx, batch, key_status, recid, status);
  else if (curve == 2) sw_rp_host<P256>(curve, W, m, xy, pre, N, e, r, s, key_idx, key_status, recid, status);
  else if (curve == 3) sw_rp_host<P384>(curve, W, m, xy, pre, N, e, r, s, key_idx, key_status, recid, status);
  else if (curve == 6) sw_rp_host<P521>(curve, W, m, xy, pre, N, e, r, s, key_idx, key_status, recid, status);
  else if (curve == 7) sw_rp_host<P192>(curve, W, m, xy, pre, N, e, r, s, key_idx, key_status, recid, status);
  else sw_rp_host<P224>(curve, W, m, xy, pre, N, e, r, s, key_idx, key_status, recid, status);
}
}
