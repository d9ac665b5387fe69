// ecdsa_k256_body.cuh -- per-thread bodies of the secp256k1 batch ECDSA-verify
// kernels (host+device so the logic can be unit-tested on a CPU-only box; the
// product only ever launches the __global__ wrappers in ecdsa_k256.cu).
//
// Path replaced (reference, lib/elliptic):
//   ec/index.js:188-229   EC.verify: range checks, s^-1, u1, u2, R = u1*G + u2*Q,
//                         reject infinity, compare x(R) with r ("Maxwell trick")
//   curve/short.js:218-249, 443-450   jmulAdd -> _endoWnafMulAdd (GLV)
//   curve/base.js:128-253             _wnafMulAdd (interleaved wNAF/JSF loop)
//   curve/short.js:908-925            JPoint.eqXToP
//
// GPU-first algorithm (same outputs, different schedule):
//   kernel 1 (prep): Montgomery-trick batch inversion of s over 16-32 items/thread,
//     u1 = e/s, u2 = r/s, GLV split of u2 into odd (k1,k2), regular recoding.
//   kernel 2 (main): one thread per signature.  Per-item table {1,3,..,31}*Q in
//     "effective affine" form on an isomorphic curve (shared Z), 26 windows of
//     5 doublings + 2 mixed adds (Q and beta*Q share the table: x -> beta*x),
//     then 13 mixed adds from a fixed 20-bit-window table of G (GTAB_W), then
//     the projective x comparison.  All lanes run the same double/add
//     schedule; exceptional group-law cases go to a cold path.
//
// Off-curve public keys (the reference does not validate uncompressed keys,
// ec/key.js:95; its output is then not a group-law function, SURVEY 8a Q1) are
// detected and reported as EB_NEEDS_HOST.
#pragma once
#include "ge_k256.cuh"
#include "sc_k256.cuh"
#ifndef EB_K256_FQ
#define EB_K256_FQ 0      // 1 = hot double/add loops on the carry-free 9 x 29-bit field (fq_pm.cuh / gq_k256.cuh); measured slower (DESIGN.md 4b), kept as a build option
#endif
#include "gq_k256.cuh"

namespace eb {

enum : uint8_t {
  ST_FALSE = 0, ST_TRUE = 1, ST_THROW_INVALID_POINT = 2, ST_THROW_NOT_VALIDATED = 3,
  ST_NEEDS_HOST = 4, ST_THROW_ASSERT = 5, ST_THROW_POINT_FORMAT = 6, ST_INFINITY = 7, ST_THROW_SECOND_KEY = 8, ST_THROW_SIG_FORMAT = 9,
  ST_THROW_NO_RECOVERY = 11,
};

// workspace layout (SoA, word-major so lanes are coalesced): PREP_WORDS words per item
//   [0..7]  mG = (u1' - 1)/2 where u1' = u1 or n-u1 made odd (8 limbs)
//   [8..12] m1 = (|k1|-1)/2, [13..17] m2 = (|k2|-1)/2
//   [18]    flags: bit0 sig invalid (-> FALSE), bit1 negG, bit2 neg1, bit3 neg2, bit4 no base-point term
constexpr int PREP_WORDS = 19;
constexpr u32 FL_INVALID = 1, FL_NEGG = 2, FL_NEG1 = 4, FL_NEG2 = 8, FL_NOG = 16;
constexpr int PREP_BATCH = 16;          // items per thread in the batched inversion
// Per-item windows of the GLV halves m1, m2 (< 2^GLV_M_BITS): 16 odd multiples 1,3,..,31 of Q cost 8 more table
// additions than 8 multiples, and save 3 doublings and 14 mixed adds over 4-bit windows.  The first QTAB_ENTRIES
// live in the item's table in the workspace (qtab), the other QTAB_HI_ENTRIES in thread-local memory, so the
// workspace a caller allocates keeps its size; all 16 share one Z.
constexpr int QTAB_W = 5;
constexpr int QTAB_ENTRIES = 8;                                // odd multiples 1,3,..,15: in the workspace
constexpr int QTAB_HI_ENTRIES = (1 << (QTAB_W - 1)) - QTAB_ENTRIES;   // 17,19,..,31: thread-local
constexpr int QTAB_WINDOWS = (GLV_M_BITS + QTAB_W - 1) / QTAB_W;
static_assert(GLV_M_BITS - QTAB_W * (QTAB_WINDOWS - 1) <= QTAB_W - 1, "top digit 2m+1 must stay below 2^W");
static_assert(QTAB_W * QTAB_WINDOWS <= 5 * 32, "m1 and m2 are stored as 5 words each");
#if EB_K256_FQ
constexpr int QTAB_WORDS = QTABQ_WORDS;        // per item: (x, y, beta*x) x 8, 9 limbs padded to 12 words each
#else
constexpr int QTAB_WORDS = QTAB_ENTRIES * 24;  // per item: (x, y, beta*x) x 8
#endif
#ifndef EB_GW
#define EB_GW 20                         // fixed-base window width in bits (wider windows measured faster up to 20; 20 = 13 windows, 436 MB)
#endif
constexpr int GTAB_W = EB_GW;
constexpr int GTAB_WINDOWS = (255 + GTAB_W - 1) / GTAB_W;     // digits of m = (u1'-1)/2 (255 bits)
constexpr int GTAB_ENTRIES = 1 << (GTAB_W - 1);               // (2i+1) * 2^(W*j) * G, i < 2^(W-1)
static_assert(255 - GTAB_W * (GTAB_WINDOWS - 1) <= GTAB_W - 1, "top digit 2m+1 must stay below 2^W");

// W-bit digit chunk at bit `pos` of the nwords-word number stored SoA from word `base` of ws
EB_HD u32 ks_chunk(const u32* ws, size_t N, size_t i, int base, int nwords, int pos, int W) {
  int wi = pos >> 5;
  u32 lo = ws[(size_t)(base + wi) * N + i];
  u32 hi = (wi + 1 < nwords) ? ws[(size_t)(base + wi + 1) * N + i] : 0u;
  u64 both = ((u64)hi << 32) | lo;
  return (u32)(both >> (pos & 31)) & ((1u << W) - 1);
}
// regular signed-odd recoding: chunk c of window w stands for the digit 2c + 1 - 2^W (top window: 2c + 1);
// returns the table index of |digit| and whether the digit is negative
EB_HD u32 ks_digit(u32 chunk, bool top, int W, bool* dneg) {
  const u32 half = 1u << (W - 1);
  *dneg = !top && chunk < half;
  return top ? (chunk & (half - 1)) : (*dneg ? half - 1 - chunk : chunk - half);
}

struct madd_out { ge_jac r; fe h; };

#if defined(__CUDACC__)
#define EB_FN __host__ __device__ __noinline__
#else
#define EB_FN
#endif

EB_FN ge_jac jac_dbl(ge_jac p) { return jac_dbl_inl(p); }
EB_FN ge_jac jac_madd(ge_jac a, ge_aff p) { return jac_madd_inl(a, p); }

// madd that also returns h with Z3 = Z1*h (table build; inputs never exceptional).
EB_HD madd_out jac_madd_h(const ge_jac& a, const ge_aff& p) {
  madd_out o;
  fe z2 = fe_sqr(a.z);
  fe u2 = fe_mul(p.x, z2);
  fe s2 = fe_mul(fe_mul(p.y, z2), a.z);
  fe h = fe_sub(a.x, u2);
  fe rr = fe_sub(a.y, s2);
  fe h2 = fe_sqr(h);
  fe h3 = fe_mul(h2, h);
  fe v = fe_mul(a.x, h2);
  o.r.x = fe_sub(fe_sub(fe_add(fe_sqr(rr), h3), v), v);
  o.r.y = fe_sub(fe_mul(rr, fe_sub(v, o.r.x)), fe_mul(a.y, h3));
  o.r.z = fe_mul(a.z, h);
  o.h = h;
  return o;
}

EB_HD fe fe_beta() {
  fe b;
  const u32 v[8] = {0x719501eeu, 0xc1396c28u, 0x12f58995u, 0x9cf04975u, 0xac3434e9u, 0x6e64479eu, 0x657c0710u, 0x7ae96a2bu};
  for (int i = 0; i < 8; i++) b.v[i] = v[i];
  return b;
}

EB_HD ge_aff k256_G() {
  ge_aff g;
  const u32 x[8] = {0x16f81798u, 0x59f2815bu, 0x2dce28d9u, 0x029bfcdbu, 0xce870b07u, 0x55a06295u, 0xf9dcbbacu, 0x79be667eu};
  const u32 y[8] = {0xfb10d4b8u, 0x9c47d08fu, 0xa6855419u, 0xfd17b448u, 0x0e1108a8u, 0x5da4fbfcu, 0x26a3c465u, 0x483ada77u};
  for (int i = 0; i < 8; i++) { g.x.v[i] = x[i]; g.y.v[i] = y[i]; }
  return g;
}

// ---------------------------------------------------------------------------
// G table entry (j, idx) = (2*idx+1) * 2^(W*j) * G, affine, normalized.
EB_HD void gtab_entry(int j, int idx, u32* out16) {
  ge_jac b = jac_from_aff(k256_G());
  for (int k = 0; k < GTAB_W * j; k++) b = jac_dbl(b);
  ge_aff base = jac_to_aff(b);
  u32 s = 2 * idx + 1;  // W-bit odd scalar
  ge_jac acc = jac_infinity();
  for (int k = GTAB_W - 1; k >= 0; k--) {
    acc = jac_dbl(acc);
    if ((s >> k) & 1) acc = jac_madd(acc, base);
  }
  ge_aff r = jac_to_aff(acc);
  r.x = fe_normalize(r.x);
  r.y = fe_normalize(r.y);
  for (int i = 0; i < 8; i++) { out16[i] = r.x.v[i]; out16[8 + i] = r.y.v[i]; }
}

// Recode (u1, u2) for k256_dsm and store them SoA: u1 odd-ified for the fixed-base windows, u2 GLV-split
// into odd halves.
EB_HD void prep_store(size_t i, size_t N, u32* u1, const u32* u2, u32 flags, u32* ws) {
  u32 nn[8];
  K256N::n(nn);
  // u1 odd-ify: u1' = n - u1 when u1 is even (then the G part is negated)
  if ((u1[0] & 1) == 0) {
    sub_n<8>(u1, nn, u1);
    flags |= FL_NEGG;
  }
  u32 m1[5], m2[5];
  bool n1, n2;
  glv_split_odd(u2, m1, &n1, m2, &n2);
  if (n1) flags |= FL_NEG1;
  if (n2) flags |= FL_NEG2;
  for (int w = 0; w < 8; w++) {
    u32 hi = (w < 7) ? u1[w + 1] : 0;
    ws[(size_t)w * N + i] = (u1[w] >> 1) | (hi << 31);
  }
  for (int w = 0; w < 5; w++) {
    ws[(size_t)(8 + w) * N + i] = m1[w];
    ws[(size_t)(13 + w) * N + i] = m2[w];
  }
  ws[(size_t)18 * N + i] = flags;
}

// ---------------------------------------------------------------------------
// prep: thread `tid` of `T` handles items tid, tid+T, ... (up to `batch` <= 64; T * batch >= N).
// e, r, s: N x 32 bytes big-endian.  ws: PREP_WORDS x N words.
// scratch: 8 x N words (prefix products).
// mode 0 (verify, ec/index.js:199-207): invert s; u1 = e/s, u2 = r/s; r, s outside [1, n-1] -> FALSE.
// mode 1 (recoverPubKey, ec/index.js:250-258): invert r; u1 = -e/r, u2 = s/r; no range checks
//         (r = 0 mod n gives rInv = 0 exactly like BN.invm, i.e. the point at infinity).
// mode 2 (getKeyRecoveryParam, recovery_param_item): invert s mod n; u1 = e/s, u2 = (r mod n)/s; no range checks;
//         s = 0 (mod n) -> FL_INVALID (recovery_param_cold_item decides those items).
EB_HD void prep_thread(size_t tid, size_t T, size_t N, const uint8_t* e, const uint8_t* r,
                       const uint8_t* s, u32* ws, u32* scratch, int mode = 0, int batch = PREP_BATCH) {
  u32 R2[8], one[8], nn[8];
  K256N::r2(R2); K256N::r1(one); K256N::n(nn);
  u32 prod[8];
  copy_n<8>(prod, one);
  u64 invalid_mask = 0;
  int cnt = 0;
  for (int j = 0; j < batch; j++) {
    size_t i = tid + (size_t)j * T;
    if (i >= N) break;
    cnt = j + 1;
    u32 sv[8], rv[8];
    load_be<8>(sv, s + 32 * i);
    load_be<8>(rv, r + 32 * i);
    bool ok = sc_in_range(sv) && sc_in_range(rv);   // ec/index.js:199-202
    u32 sm[8];
    if (mode == 1) {
      sc_mont_mul(sm, rv, R2);                      // r mod n, Montgomery form
      ok = !is_zero_n<8>(sm);
    } else {
      sc_mont_mul(sm, sv, R2);
      if (mode == 2) ok = !is_zero_n<8>(sm);        // s mod n
    }
    if (!ok) invalid_mask |= (u64)1 << j;
    cmov_n<8>(sm, one, !ok);
    // scratch[i] = prefix product BEFORE this item
    for (int w = 0; w < 8; w++) scratch[(size_t)w * N + i] = prod[w];
    u32 t[8];
    sc_mont_mul(t, prod, sm);
    copy_n<8>(prod, t);
  }
  if (cnt == 0) return;
  u32 inv[8];
  sc_mont_inv(inv, prod);
  for (int j = cnt - 1; j >= 0; j--) {
    size_t i = tid + (size_t)j * T;
    bool ok = !((invalid_mask >> j) & 1);
    u32 sv[8], rv[8], ev[8], sm[8], pre[8], sinv[8], t[8];
    load_be<8>(sv, s + 32 * i);
    load_be<8>(rv, r + 32 * i);
    sc_mont_mul(sm, mode == 1 ? rv : sv, R2);
    cmov_n<8>(sm, one, !ok);
    for (int w = 0; w < 8; w++) pre[w] = scratch[(size_t)w * N + i];
    sc_mont_mul(sinv, inv, pre);      // s_i^-1 (Montgomery form)
    sc_mont_mul(t, inv, sm);          // drop s_i from the running inverse
    copy_n<8>(inv, t);
    u32 flags = (ok || mode == 1) ? 0 : FL_INVALID;
    load_be<8>(ev, e + 32 * i);
    u32 u1[8], u2[8];
    if (mode == 1) {
      u32 zero8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      cmov_n<8>(sinv, zero8, !ok);    // invm(0) = 0
      sc_mont_mul(u1, ev, sinv);      // e / r
      if (!is_zero_n<8>(u1)) sub_n<8>(u1, nn, u1);   // s1 = (n - e) * rInv mod n   (ec/index.js:251)
      sc_mont_mul(u2, sv, sinv);      // s2 = s * rInv mod n         (ec/index.js:252)
    } else {
      sc_mont_mul(u1, ev, sinv);      // e * s^-1 mod n   (ec/index.js:206)
      sc_mont_mul(u2, rv, sinv);      // r * s^-1 mod n   (ec/index.js:207)
    }
    prep_store(i, N, u1, u2, flags, ws);
  }
}

// Generic scalars for BasePoint.mul / mulAdd callers (short.js:422-441): k1, k2 are any 256-bit
// integers (big-endian), reduced mod n here (the group law only sees the residue for on-curve
// points).  k1 == nullptr: no base-point term.
EB_HD void prep_scalars_item(size_t i, size_t N, const uint8_t* k1, const uint8_t* k2, u32* ws) {
  u32 nn[8], u1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, u2[8];
  K256N::n(nn);
  u32 flags = 0;
  if (k1) {
    load_be<8>(u1, k1 + 32 * i);
    if (geq_n<8>(u1, nn)) sub_n<8>(u1, u1, nn);
  } else {
    flags |= FL_NOG;
  }
  load_be<8>(u2, k2 + 32 * i);
  if (geq_n<8>(u2, nn)) sub_n<8>(u2, u2, nn);
  prep_store(i, N, u1, u2, flags, ws);
}

// ---------------------------------------------------------------------------
// main: one signature.  pub: N x 64 bytes (x || y big-endian).  r: N x 32.
// gtab: GTAB_WINDOWS x GTAB_ENTRIES x 16 words.  qtab: N x QTAB_WORDS words.
EB_HD void store_fe(u32* dst, const fe& a) { for (int i = 0; i < 8; i++) dst[i] = a.v[i]; }
EB_HD fe load_fe(const u32* src) { fe a; for (int i = 0; i < 8; i++) a.v[i] = src[i]; return a; }

#if EB_K256_FQ
// u1*G + u2*Q for an ON-CURVE Q, scalars as prepared by prep_thread in ws.  Jacobian result.
// Carry-free field version: the whole double/add schedule runs on 9 x 29-bit lazy limbs (gq_k256.cuh);
// the packed 8 x 32 form only appears at the two ends (Q in, the fixed-base table entries, R out).
EB_HD ge_jac k256_dsm(size_t i, size_t N, const ge_aff& Q, u32 flags, const u32* ws, const u32* gtab, u32* qtab) {
  // ---- per-item table: (2k+1)*Q, k < 16, as affine points on an isomorphic
  // curve y^2 = x^3 + 7*Zg^6 (the a = 0 formulas never use b), Zg = zglobal.
  u32* tab = qtab + (size_t)i * QTAB_WORDS;
  alignas(16) u32 hi[QTAB_HI_ENTRIES * QTABQ_ENTRY_WORDS];
  auto ent = [&](u32 k) { return k < QTAB_ENTRIES ? tab + QTABQ_ENTRY_WORDS * k : hi + QTABQ_ENTRY_WORDS * (k - QTAB_ENTRIES); };
  constexpr int NE = QTAB_ENTRIES + QTAB_HI_ENTRIES;
  fqk<1> zglobal;
  {
    gq_jac Qj; Qj.x = fqk_from_fe(Q.x); Qj.y = fqk_from_fe(Q.y); Qj.z = fqk_one();
    gq_jac D = gq_dbl(Qj);                   // 2Q, finite for an on-curve Q
    fqk<1> C2 = fq_sqr(D.z);
    fqk<1> C3 = fq_mul(C2, D.z);
    gq_jac P;                                // 2Q is affine on the curve scaled by C = D.z
    P.x = fq_mul(Qj.x, C2);
    P.y = fq_mul(Qj.y, C3);
    P.z = fqk_one();
    fq_store12(tab + 0, P.x); fq_store12(tab + FQ_PAD, P.y);
    for (int k = 1; k < NE; k++) {
      gq_madd_out o = gq_madd_h(P, D.x, D.y);
      P = o.r;
      u32* e = ent(k);
      fq_store12(e, P.x); fq_store12(e + FQ_PAD, P.y);
      fq_store12(e + 2 * FQ_PAD, o.h);       // Z_k / Z_{k-1}, consumed below
    }
    zglobal = fq_mul(P.z, D.z);
    // rescale every entry to the last entry's Z and append beta*x
    const fqk<1> beta = fqk_from_fe(fe_beta());
    fqk<1> zs = fqk_one();
    for (int k = NE - 1; k >= 0; k--) {
      u32* e = ent(k);
      fqk<1> X = fq_load12(e), Y = fq_load12(e + FQ_PAD);
      fqk<1> hk = fqk_one();
      if (k > 0) hk = fq_load12(e + 2 * FQ_PAD);
      if (k < NE - 1) {
        fqk<1> zs2 = fq_sqr(zs);
        fqk<1> zs3 = fq_mul(zs2, zs);
        X = fq_mul(X, zs2);
        Y = fq_mul(Y, zs3);
        fq_store12(e, X); fq_store12(e + FQ_PAD, Y);
      }
      fq_store12(e + 2 * FQ_PAD, fq_mul(X, beta));
      zs = fq_mul(zs, hk);
    }
  }

  // ---- u2*Q = k1*Q + k2*(lambda*Q): QTAB_WINDOWS windows of QTAB_W bits, regular signed-odd digits
  gq_jac acc;
  acc.x = fqk_one(); acc.y = fqk_one(); acc.z = fqk_zero();
  for (int w = QTAB_WINDOWS - 1; w >= 0; w--) {
    const bool top = w == QTAB_WINDOWS - 1;
    if (!top)
      for (int d = 0; d < QTAB_W; d++) acc = gq_dbl(acc);    // (the top window starts from its first table entry)
    for (int h = 0; h < 2; h++) {
      bool dneg;
      u32 idx = ks_digit(ks_chunk(ws, N, i, h ? 13 : 8, 5, QTAB_W * w, QTAB_W), top, QTAB_W, &dneg);
      bool neg = dneg != (((flags & (h ? FL_NEG2 : FL_NEG1)) != 0));
      const u32* e = ent(idx);
      gq_aff P;
      P.x = fq_load12(e + (h ? 2 * FQ_PAD : 0));
      P.y = fq_cneg(fq_load12(e + FQ_PAD), neg);
      if (top && h == 0) acc = gq_from_aff(P);
      else acc = gq_madd(acc, P);
    }
  }
  // back to the real curve: Z *= Zg
  acc.z = fq_mul(acc.z, zglobal);

  // ---- u1*G from the fixed table: GTAB_WINDOWS windows of GTAB_W bits, regular signed-odd digits
  if (!(flags & FL_NOG)) {                    // Point.mul: no base-point term (uniform across a batch)
    for (int j = 0; j < GTAB_WINDOWS; j++) {
      bool dneg;
      u32 idx = ks_digit(ks_chunk(ws, N, i, 0, 8, GTAB_W * j, GTAB_W), j == GTAB_WINDOWS - 1, GTAB_W, &dneg);
      bool neg = dneg != ((flags & FL_NEGG) != 0);
      const u32* ent = gtab + ((size_t)j * GTAB_ENTRIES + idx) * 16;
      gq_aff P;
      P.x = fqk_from_fe(load_fe(ent));
      P.y = fq_cneg(fqk_from_fe(load_fe(ent + 8)), neg);
      acc = gq_madd(acc, P);
    }
  }
  return gq_to_jac(acc);
}
#else
// Per-item table (2k+1)*Q, k < QTAB_ENTRIES + NHI, for an ON-CURVE Q: entry k = (x, y, beta*x) at tab + 24k for
// k < QTAB_ENTRIES (the item's workspace table), at hi + 24(k - QTAB_ENTRIES) after that, as affine points on the
// isomorphic curve y^2 = x^3 + 7*Zg^6 (the a = 0 formulas never use b); returns Zg.  Built with co-Z additions
// (Meloni): all points of one step share a Z, so no addition needs it.  NHI = 0 is the table of 4-bit windows.
template <int NHI = 0>
EB_HD fe qtab_build(const ge_aff& Q, u32* tab, u32* hi = nullptr) {
  constexpr int NE = QTAB_ENTRIES + NHI;
  auto ent = [&](int k) { return k < QTAB_ENTRIES ? tab + 24 * k : hi + 24 * (k - QTAB_ENTRIES); };
  // co-Z doubling of the affine Q (dbl-2009-l at Z = 1): D = 2Q and P = Q, both on Z = 2*y(Q), i.e. affine on
  // the curve scaled by 2*y(Q).  y(Q) != 0: the group has odd order.
  fe B = fe_sqr(Q.x);
  fe E = fe_sqr(Q.y);
  fe L = fe_sqr(E);
  fe S = fe_dbl(fe_sub(fe_sub(fe_sqr(fe_add(Q.x, E)), B), L));   // 4 x y^2 = x * (2y)^2
  fe M = fe_add(B, fe_dbl(B));
  fe L8 = fe_dbl(fe_dbl(fe_dbl(L)));                               // 8 y^4 = y * (2y)^3
  fe Dx = fe_sub(fe_sqr(M), fe_dbl(S));
  fe Dy = fe_sub(fe_mul(M, fe_sub(S, Dx)), L8);
  fe Px = S, Py = L8;
  store_fe(tab + 0, Px); store_fe(tab + 8, Py);
  for (int k = 1; k < NE; k++) {
    // ZADDU: P += D with D moved to the new Z; Z_k = Z_{k-1} * h.  (2k-1)Q = +-2Q is impossible in a group of
    // large prime order, so h != 0.
    fe h = fe_sub(Px, Dx);
    fe C = fe_sqr(h);
    fe W1 = fe_mul(Px, C), W2 = fe_mul(Dx, C);
    fe A2 = fe_mul(Dy, fe_sub(W1, W2));                            // y_D * h^3
    fe dy = fe_sub(Py, Dy);
    Px = fe_sub(fe_sub(fe_sqr(dy), W1), W2);
    Py = fe_sub(fe_mul(dy, fe_sub(W2, Px)), A2);
    Dx = W2; Dy = A2;
    u32* e = ent(k);
    store_fe(e, Px); store_fe(e + 8, Py);
    store_fe(e + 16, h);                                           // Z_k / Z_{k-1}, consumed below
  }
  // rescale every entry to the last entry's Z and append beta*x
  fe beta = fe_beta();
  fe zs = fe_one();
  for (int k = NE - 1; k >= 0; k--) {
    u32* e = ent(k);
    fe X = load_fe(e), Y = load_fe(e + 8);
    if (k < NE - 1) {
      fe zs2 = fe_sqr(zs);
      fe zs3 = fe_mul(zs2, zs);
      X = fe_mul(X, zs2);
      Y = fe_mul(Y, zs3);
      store_fe(e, X); store_fe(e + 8, Y);
    }
    if (k > 0) zs = fe_mul(zs, load_fe(e + 16));
    store_fe(e + 16, fe_mul(X, beta));
  }
  return fe_mul(zs, fe_dbl(Q.y));                                  // Z_last * 2y(Q)
}

// u1*G + u2*Q for an ON-CURVE Q, scalars as prepared by prep_thread in ws.  Jacobian result.
EB_HD ge_jac k256_dsm(size_t i, size_t N, const ge_aff& Q, u32 flags, const u32* ws, const u32* gtab, u32* qtab) {
  u32* tab = qtab + (size_t)i * QTAB_WORDS;
  alignas(16) u32 hi[QTAB_HI_ENTRIES * 24];
  fe zglobal = qtab_build<QTAB_HI_ENTRIES>(Q, tab, hi);

  // ---- u2*Q = k1*Q + k2*(lambda*Q): QTAB_WINDOWS windows of QTAB_W bits, regular signed-odd digits
  ge_jac acc = jac_infinity();
  for (int w = QTAB_WINDOWS - 1; w >= 0; w--) {
    const bool top = w == QTAB_WINDOWS - 1;
    if (!top)
      for (int d = 0; d < QTAB_W; d++) acc = jac_dbl(acc);   // (the top window starts from its first table entry)
    for (int h = 0; h < 2; h++) {
      bool dneg;
      u32 idx = ks_digit(ks_chunk(ws, N, i, h ? 13 : 8, 5, QTAB_W * w, QTAB_W), top, QTAB_W, &dneg);
      bool neg = dneg != (((flags & (h ? FL_NEG2 : FL_NEG1)) != 0));
      const u32* e = idx < QTAB_ENTRIES ? tab + 24 * idx : hi + 24 * (idx - QTAB_ENTRIES);
      ge_aff P;
      P.x = load_fe(e + (h ? 16 : 0));
      P.y = load_fe(e + 8);
      P = aff_neg_if(P, neg);
      if (top && h == 0) acc = jac_from_aff(P);
      else acc = jac_madd(acc, P);
    }
  }
  // back to the real curve: Z *= Zg
  acc.z = fe_mul(acc.z, zglobal);

  // ---- u1*G from the fixed table: GTAB_WINDOWS windows of GTAB_W bits, regular signed-odd digits
  if (flags & FL_NOG) return acc;             // Point.mul: no base-point term (uniform across a batch)
  for (int j = 0; j < GTAB_WINDOWS; j++) {
    bool dneg;
    u32 idx = ks_digit(ks_chunk(ws, N, i, 0, 8, GTAB_W * j, GTAB_W), j == GTAB_WINDOWS - 1, GTAB_W, &dneg);
    bool neg = dneg != ((flags & FL_NEGG) != 0);
    const u32* ent = gtab + ((size_t)j * GTAB_ENTRIES + idx) * 16;
    ge_aff P;
    P.x = load_fe(ent);
    P.y = load_fe(ent + 8);
    acc = jac_madd(acc, aff_neg_if(P, neg));
  }
  return acc;
}

#endif  // EB_K256_FQ

EB_HD uint8_t verify_item(size_t i, size_t N, const uint8_t* pub, const uint8_t* r,
                          const u32* ws, const u32* gtab, u32* qtab) {
  u32 flags = ws[(size_t)18 * N + i];
  if (flags & FL_INVALID) return ST_FALSE;
  ge_aff Q;
  Q.x = fe_from_be(pub + 64 * i);
  Q.y = fe_from_be(pub + 64 * i + 32);
  if (!aff_on_curve(Q)) return ST_NEEDS_HOST;
  ge_jac acc = k256_dsm(i, N, Q, flags, ws, gtab, qtab);

  // ---- accept iff R != O and x(R) == r (mod n)   (ec/index.js:222-228, short.js:908-925)
  if (fe_is_zero(acc.z)) return ST_FALSE;
  fe z2 = fe_sqr(acc.z);
  fe rf = fe_from_be(r + 32 * i);
  if (fe_eq(acc.x, fe_mul(rf, z2))) return ST_TRUE;
  const u32 pmn[8] = {0x2fc9baeeu, 0x402da172u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0, 0, 0};  // p - n
  if (!geq_n<8>(rf.v, pmn)) {      // r + n < p: second candidate
    u32 nn[8]; K256N::n(nn);
    fe rn;
    add_n<8>(rn.v, rf.v, nn);
    if (fe_eq(acc.x, fe_mul(rn, z2))) return ST_TRUE;
  }
  return ST_FALSE;
}

// EC.prototype.recoverPubKey (ec/index.js:231-259): Q = r^-1 (s*R - e*G), R = pointFromX(r or r+n, odd).
// recid: 1 byte per item (0..3).  out: 64 bytes x||y big-endian.  Status: ST_TRUE = point returned,
// ST_INFINITY = the reference returns the point at infinity, ST_THROW_INVALID_POINT (short.js:195),
// ST_THROW_SECOND_KEY ('Unable to find sencond key candinate', ec/index.js:243-244).
EB_HD uint8_t recover_item(size_t i, size_t N, const uint8_t* r, const uint8_t* recid,
                           const u32* ws, const u32* gtab, u32* qtab, uint8_t* out) {
  for (int b = 0; b < 64; b++) out[64 * i + b] = 0;
  u32 j = recid[i];
  bool odd = j & 1, second = (j >> 1) & 1;
  u32 rv[8];
  load_be<8>(rv, r + 32 * i);
  const u32 pmn[8] = {0x2fc9baeeu, 0x402da172u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0, 0, 0};  // p mod n = p - n
  if (second && geq_n<8>(rv, pmn)) return ST_THROW_SECOND_KEY;
  fe x; copy_n<8>(x.v, rv);
  if (second) { u32 nn[8]; K256N::n(nn); add_n<8>(x.v, rv, nn); }      // r + n < p here
  fe seven = fe_zero(); seven.v[0] = 7;
  fe y2 = fe_add(fe_mul(fe_sqr(x), x), seven);
  fe y = fe_sqrt_candidate(y2);
  if (!fe_eq(fe_sqr(y), y2)) return ST_THROW_INVALID_POINT;
  if (fe_is_odd(y) != odd) y = fe_neg(y);
  ge_aff R; R.x = x; R.y = y;
  u32 flags = ws[(size_t)18 * N + i];
  ge_jac acc = k256_dsm(i, N, R, flags, ws, gtab, qtab);
  if (fe_is_zero(acc.z)) return ST_INFINITY;
  ge_aff q = jac_to_aff(acc);
  fe qx = fe_normalize(q.x), qy = fe_normalize(q.y);
  store_be<8>(out + 64 * i, qx.v);
  store_be<8>(out + 64 * i + 32, qy.v);
  return ST_TRUE;
}

// EC.prototype.getKeyRecoveryParam (ec/index.js:261-278) with one double-scalar multiplication instead of its loop over
// recoverPubKey.  The group has prime order, so for r, s != 0 (mod n): r^-1 (s R - e G) = Q  <=>  R = s^-1 (e G + r Q) = P.
// prep_thread mode 2 leaves u1 = e/s, u2 = r/s, and the answer is read off P: x(P) = r mod p gives j = parity(y(P)),
// x(P) = r + n (r < p - n) gives j = 2 + parity(y(P)), anything else (or P = O) no j.  P itself proves that pointFromX
// finds that candidate.  recid: 1 byte per item, 0 unless ST_TRUE.  Status ST_TRUE, ST_THROW_NO_RECOVERY, or
// ST_NEEDS_HOST for s = 0 (mod n), which recovery_param_cold_item (ecdsa_k256_sign.cuh) decides.
EB_HD uint8_t recovery_param_item(size_t i, size_t N, const uint8_t* q, const uint8_t* r, const u32* ws, const u32* gtab,
                                  u32* qtab, uint8_t* recid) {
  recid[i] = 0;
  ge_aff Q;
  Q.x = fe_from_be(q + 64 * i);
  Q.y = fe_from_be(q + 64 * i + 32);
  if (!aff_on_curve(Q)) return ST_THROW_NO_RECOVERY;       // a recovered point is always on the curve
  u32 rv[8], nn[8];
  load_be<8>(rv, r + 32 * i);
  K256N::n(nn);
  if (is_zero_n<8>(rv) || eq_n<8>(rv, nn)) return ST_THROW_NO_RECOVERY;   // r = 0 (mod n): rInv = 0, every Q' is O
  u32 flags = ws[(size_t)18 * N + i];
  if (flags & FL_INVALID) return ST_NEEDS_HOST;             // s = 0 (mod n)
  ge_jac acc = k256_dsm(i, N, Q, flags, ws, gtab, qtab);
  if (fe_is_zero(acc.z)) return ST_THROW_NO_RECOVERY;
  fe z2 = fe_sqr(acc.z);
  u32 j = 0;
  if (!fe_eq(acc.x, fe_mul(fe_from_be(r + 32 * i), z2))) {
    const u32 pmn[8] = {0x2fc9baeeu, 0x402da172u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0, 0, 0};  // p mod n = p - n
    if (geq_n<8>(rv, pmn)) return ST_THROW_NO_RECOVERY;    // no second candidate (ec/index.js:243)
    fe rn;
    add_n<8>(rn.v, rv, nn);
    if (!fe_eq(acc.x, fe_mul(rn, z2))) return ST_THROW_NO_RECOVERY;
    j = 2;
  }
  fe zi = fe_inv(acc.z);
  if (fe_is_odd(fe_mul(fe_mul(acc.y, fe_sqr(zi)), zi))) j |= 1;
  recid[i] = (uint8_t)j;
  return ST_TRUE;
}

// BasePoint.mul / Point.mulAdd (short.js:422-441) for an on-curve point: k1*G + k2*P (or k2*P alone), affine
// result as Point.toP / JPoint.toP (short.js:516-526).  ST_TRUE = point written, ST_INFINITY = the point at
// infinity (out zeroed), ST_NEEDS_HOST = P is off the curve (the replay kernel re-runs it).
EB_HD uint8_t mul_add_item(size_t i, size_t N, const uint8_t* pts, const u32* ws, const u32* gtab, u32* qtab,
                           uint8_t* out) {
  for (int b = 0; b < 64; b++) out[64 * i + b] = 0;
  ge_aff P;
  P.x = fe_from_be(pts + 64 * i);
  P.y = fe_from_be(pts + 64 * i + 32);
  if (!aff_on_curve(P)) return ST_NEEDS_HOST;
  u32 flags = ws[(size_t)18 * N + i];
  ge_jac acc = k256_dsm(i, N, P, flags, ws, gtab, qtab);
  if (fe_is_zero(acc.z)) return ST_INFINITY;
  ge_aff q = jac_to_aff(acc);
  fe qx = fe_normalize(q.x), qy = fe_normalize(q.y);
  store_be<8>(out + 64 * i, qx.v);
  store_be<8>(out + 64 * i + 32, qy.v);
  return ST_TRUE;
}

}  // namespace eb
