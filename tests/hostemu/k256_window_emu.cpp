// Host emulation of the secp256k1 kernel bodies with their per-item window constants -- TEST INFRASTRUCTURE ONLY.
// Built with and without -DEB_K256_FQ=1, so the same extreme-scalar cases run through both field forms.
#include "hostemu.cpp"

extern "C" {

void fx_glv_windows(int* w, int* windows, int* entries, int* mbits) {
  *w = QTAB_W; *windows = QTAB_WINDOWS; *entries = QTAB_ENTRIES + QTAB_HI_ENTRIES; *mbits = GLV_M_BITS;
}

#if !EB_K256_FQ
// The table k256_dsm builds for the affine Q (16 words): the workspace part into tab (QTAB_WORDS words), the rest
// into hi (QTAB_HI_ENTRIES * 24 words), Zg into zg (8 words).
void fx_qtab_split(const u32* q, u32* tab, u32* hi, u32* zg) {
  ge_aff Q; Q.x = load_fe(q); Q.y = load_fe(q + 8);
  store_fe(zg, qtab_build<QTAB_HI_ENTRIES>(Q, tab, hi));
}
#endif
}
