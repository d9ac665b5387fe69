// Host emulation of the secp256k1 per-item table and prep batching -- TEST INFRASTRUCTURE ONLY.
// The kernel bodies (all of hostemu.cpp) plus the table build it replaced (a doubling, a rescale of Q to the
// doubling's Z, then seven 8M+3S mixed additions) kept as a reference body; the tests compare the co-Z build
// the kernels run with it on the same points.
#include "hostemu.cpp"

namespace ref {

fe qtab_build(const ge_aff& Q, u32* tab) {
  ge_jac D = jac_dbl(jac_from_aff(Q));
  fe C2 = fe_sqr(D.z);
  fe C3 = fe_mul(C2, D.z);
  ge_aff Dp; Dp.x = D.x; Dp.y = D.y;
  ge_jac P;
  P.x = fe_mul(Q.x, C2);
  P.y = fe_mul(Q.y, C3);
  P.z = fe_one();
  store_fe(tab + 0, P.x); store_fe(tab + 8, P.y);
  for (int k = 1; k < QTAB_ENTRIES; k++) {
    madd_out o = jac_madd_h(P, Dp);
    P = o.r;
    store_fe(tab + 24 * k, P.x); store_fe(tab + 24 * k + 8, P.y);
    store_fe(tab + 24 * k + 16, o.h);
  }
  fe zglobal = fe_mul(P.z, D.z);
  fe beta = fe_beta();
  fe zs = fe_one();
  for (int k = QTAB_ENTRIES - 1; k >= 0; k--) {
    fe X = load_fe(tab + 24 * k), Y = load_fe(tab + 24 * k + 8);
    fe hk = fe_one();
    if (k > 0) hk = load_fe(tab + 24 * k + 16);
    if (k < QTAB_ENTRIES - 1) {
      fe zs2 = fe_sqr(zs);
      fe zs3 = fe_mul(zs2, zs);
      X = fe_mul(X, zs2);
      Y = fe_mul(Y, zs3);
      store_fe(tab + 24 * k, X); store_fe(tab + 24 * k + 8, Y);
    }
    store_fe(tab + 24 * k + 16, fe_mul(X, beta));
    zs = fe_mul(zs, hk);
  }
  return zglobal;
}

}  // namespace ref

extern "C" {

// Per-item table of the affine Q (16 words) into tab (QTAB_WORDS words), its Zg into zg (8 words).
// which: 0 the kernels' body, 1 the reference body.
void fx_qtab(int which, const u32* q, u32* tab, u32* zg) {
  ge_aff Q; Q.x = load_fe(q); Q.y = load_fe(q + 8);
  store_fe(zg, which ? ref::qtab_build(Q, tab) : qtab_build(Q, tab));
}

int fx_qtab_words() { return QTAB_WORDS; }

// prep_thread over N items with `batch` items per thread on T threads (the caller picks T >= N / batch); ws gets
// PREP_WORDS x N words.
void fx_prep(size_t N, const uint8_t* e, const uint8_t* r, const uint8_t* s, int mode, int batch, size_t T, u32* ws) {
  std::vector<u32> scratch((size_t)8 * N);
  for (size_t t = 0; t < T; t++) prep_thread(t, T, N, e, r, s, ws, scratch.data(), mode, batch);
}
}
