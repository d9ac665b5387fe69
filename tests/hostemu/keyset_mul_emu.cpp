// Host emulation of the keyed Point.mul / mulAdd / derive bodies -- TEST INFRASTRUCTURE ONLY.
// Runs the same .cuh bodies keyset.cu and eb200.cu launch, in the kernels' order: classify -> window bases -> table
// windows, then prep_scalars -> keyed main -> normalisation -> keyed replay of the off-curve-key items (derive: the
// status map).  The set builders and fixed-base tables are keyset_emu.cpp's.  The product library never contains or
// calls this code.
#include "keyset_emu.cpp"

// op: 0 = pub.mul(k2), 1 = G.mulAdd(k1, pub, k2), 2 = keyPair(k2).derive(pub)
static void k256_mul_host(int W, int op, size_t m, const uint8_t* xy, size_t N, const uint8_t* k1, const uint8_t* k2,
                          const u32* key_idx, int batch, uint8_t* key_status, uint8_t* out, uint8_t* status) {
  const u32* gtab = k256_host_gtab().data();
  static std::vector<u32> rtab;
  if (rtab.empty()) {
    rtab.resize(REPLAY_TAB_WORDS);
    for (int t = 0; t < 2 * REPLAY_NAF_PTS; t++) rp_tab_entry(t, &rtab[16 * t]);
  }
  Set S;
  k256_build(m, xy, W, S);
  memcpy(key_status, S.kst.data(), m);
  const uint8_t* kk1 = op == 1 ? k1 : nullptr;
  std::vector<u32> ws((size_t)PREP_WORDS * N), jac((size_t)24 * N), scratch((size_t)8 * N);
  for (size_t i = 0; i < N; i++) prep_scalars_item(i, N, kk1, k2, ws.data());
  for (size_t i = 0; i < N; i++)
    status[i] = k256_mul_keyed_item(i, N, key_idx, S.kst.data(), W, S.windows, S.tab.data(), ws.data(), gtab, jac.data());
  size_t T = (N + batch - 1) / batch;
  for (size_t t = 0; t < T; t++) k256_ks_norm_thread(t, T, N, batch, jac.data(), scratch.data(), op == 2, out, status);
  for (size_t i = 0; i < N; i++) {
    if (status[i] != ST_NEEDS_HOST) continue;
    if (op == 2) status[i] = ST_THROW_NOT_VALIDATED;
    else status[i] = rp_mul_add_item(0, kk1 ? kk1 + 32 * i : nullptr, k2 + 32 * i, xy + 64 * (size_t)key_idx[i], rtab.data(), out + 64 * i);
  }
}

template <class C>
static void sw_mul_host(int curve, int W, int op, size_t m, const uint8_t* xy, size_t N, const uint8_t* k1, const uint8_t* k2,
                        const u32* key_idx, uint8_t* key_status, uint8_t* out, uint8_t* status) {
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
  const uint8_t* kk1 = op == 1 ? k1 : nullptr;
  std::vector<u32> ws((size_t)W_::PREP_WORDS * N), jac((size_t)3 * C::N * N), scratch((size_t)C::N * N);
  for (size_t i = 0; i < N; i++) W_::prep_scalars_item(i, N, kk1, k2, ws.data());
  for (size_t i = 0; i < N; i++)
    status[i] = K::mul_keyed_item(i, N, key_idx, S.kst.data(), W, S.windows, S.tab.data(), ws.data(), gtab.data(), jac.data());
  size_t T = (N + W_::BATCH - 1) / W_::BATCH;
  for (size_t t = 0; t < T; t++) K::norm_thread(t, T, N, jac.data(), scratch.data(), op == 2, out, status);
  for (size_t i = 0; i < N; i++) {
    if (status[i] != ST_NEEDS_HOST) continue;
    if (op == 2) status[i] = ST_THROW_NOT_VALIDATED;
    else status[i] = SWReplay<C>::mul_add_item(0, kk1 ? kk1 + LEN * i : nullptr, k2 + LEN * i, xy + 2 * LEN * (size_t)key_idx[i],
                                               rtab.data(), out + 2 * LEN * i);
  }
}

extern "C" {

// curve: the C-ABI id; xy: m keys x || y; k1, k2: N x len scalars (k1 read for op 1 only); batch: items per
// normalisation thread on secp256k1 (the other curves use SW<C>::BATCH = 16).  out: N x 2 len (op 2: N x len).
void he_keyset_mul(int curve, int W, int op, size_t m, const uint8_t* xy, size_t N, const uint8_t* k1, const uint8_t* k2,
                   const u32* key_idx, int batch, uint8_t* key_status, uint8_t* out, uint8_t* status) {
  if (curve == 1) k256_mul_host(W, op, m, xy, N, k1, k2, key_idx, batch, key_status, out, status);
  else if (curve == 2) sw_mul_host<P256>(curve, W, op, m, xy, N, k1, k2, key_idx, key_status, out, status);
  else if (curve == 3) sw_mul_host<P384>(curve, W, op, m, xy, N, k1, k2, key_idx, key_status, out, status);
  else if (curve == 6) sw_mul_host<P521>(curve, W, op, m, xy, N, k1, k2, key_idx, key_status, out, status);
  else if (curve == 7) sw_mul_host<P192>(curve, W, op, m, xy, N, k1, k2, key_idx, key_status, out, status);
  else sw_mul_host<P224>(curve, W, op, m, xy, N, k1, k2, key_idx, key_status, out, status);
}
}
