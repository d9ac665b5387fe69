// ecdsa_sw_body.cuh -- batch ECDSA verify on short Weierstrass curves with a = -3 and no
// endomorphism (p256, p384), generic over a curve-parameter struct C (sw_params_gen.inc).
//
// Reference path (lib/elliptic): ec/index.js:188-229 EC.verify -> short.js:443-450
// jmulAdd -> base.js:128-253 _wnafMulAdd(1, [G, Q], [u1, u2], 2, true) with G's wnd-8 table
// (ec/index.js:36, base.js:321) and JPoint._threeDbl (short.js:739-800); field = BN.mont(p)
// (curves.js:75,90).  Same outputs, GPU schedule: one thread per signature; u2*Q by regular
// signed-odd 4-bit windows over a per-item Jacobian table {1,3,..,15}Q, u1*G by GW-bit windows
// over a fixed affine table; CIOS Montgomery field; exceptional cases in cold paths.
#pragma once
#include "fp_mont.cuh"
#include "sw_params.cuh"

namespace eb {

template <class C>
struct SW {
  typedef typename C::F F;
  typedef typename C::S S;
  typedef typename F::fe fe;
  static constexpr int N = C::N;
  struct jac { fe x, y, z; };
  struct aff { fe x, y; };

  static constexpr int MBITS = C::BITS - 1;                  // bits of m = (u'-1)/2
  static constexpr int QWINDOWS = MBITS / 4 + 1;              // the top digit then has at most 3 bits
  static_assert(MBITS - 4 * (QWINDOWS - 1) <= 3, "top 4-bit digit must stay positive");
  static constexpr int GW = C::GW;
  static constexpr int GWINDOWS = MBITS / GW + 1;
  static constexpr int GENTRIES = 1 << (GW - 1);
  static_assert(MBITS - GW * (GWINDOWS - 1) <= GW - 1, "top fixed-base digit must stay positive");
  static constexpr int PREP_WORDS = 2 * N + 1;               // mG[N], m2[N], flags
  static constexpr int QTAB_WORDS = 8 * 3 * N;               // 8 Jacobian entries
  static constexpr int BATCH = 16;
  static constexpr u32 FL_INVALID = 1, FL_NEGG = 2, FL_NEG2 = 4, FL_NOG = 8;

  // field-sized big-endian strings: 4N bytes, except p521 (66 bytes in 18 limbs)
  static EB_HD void ldb(u32* r, const uint8_t* p) {
    if (C::LEN == 4 * N) load_be<N>(r, p); else load_be_len<N>(r, p, C::LEN);
  }
  static EB_HD void stb(uint8_t* p, const u32* a) {
    if (C::LEN == 4 * N) store_be<N>(p, a); else store_be_len<N>(p, a, C::LEN);
  }

  static EB_HD jac infinity() { jac r; r.x = F::one(); r.y = F::one(); r.z = F::zero(); return r; }
  static EB_HD jac from_aff(const aff& p) { jac r; r.x = p.x; r.y = p.y; r.z = F::one(); return r; }

  // dbl-2001-b (a = -3): 3M + 5S   (short.js:766-796)
  static EB_HD jac dbl_inl(const jac& p) {
    fe delta = F::sqr(p.z);
    fe gamma = F::sqr(p.y);
    fe beta4 = F::template mul_k<4>(p.x, gamma);                                    // 4 x y^2
    fe alpha = F::template mul_k<3>(F::sub(p.x, delta), F::add(p.x, delta));        // 3 (x - z^2)(x + z^2)
    jac r;
    r.x = F::sub(F::sqr(alpha), F::dbl(beta4));
    r.z = F::sub(F::sub(F::sqr(F::add(p.y, p.z)), gamma), delta);
    fe g8 = F::template sqr_k<8>(gamma);                                            // 8 y^4
    r.y = F::sub(F::mul(alpha, F::sub(beta4, r.x)), g8);
    return r;
  }

  // Jacobian + affine, all cases exact (short.js:569-603)
  static EB_HD jac madd_inl(const jac& a, const aff& p) {
    fe z2 = F::sqr(a.z);
    fe u2 = F::mul(p.x, z2);
    fe s2 = F::mul(F::mul(p.y, z2), a.z);
    fe h = F::sub(a.x, u2);
    fe rr = F::sub(a.y, s2);
    fe h2 = F::sqr(h);
    fe h3 = F::mul(h2, h);
    fe v = F::mul(a.x, h2);
    jac r;
    r.x = F::sub(F::sub(F::add(F::sqr(rr), h3), v), v);
    r.y = F::sub(F::mul(rr, F::sub(v, r.x)), F::mul(a.y, h3));
    r.z = F::mul(a.z, h);
    if (F::is_zero(r.z)) {
      if (F::is_zero(a.z)) return from_aff(p);
      if (F::is_zero(rr)) return dbl(a);          // cold: through the out-of-line copy, not another inlined doubling
      return infinity();
    }
    return r;
  }

  // Jacobian + Jacobian, all cases exact (short.js:532-567)
  static EB_HD jac add_inl(const jac& a, const jac& b) {
    fe bz2 = F::sqr(b.z);
    fe az2 = F::sqr(a.z);
    fe u1 = F::mul(a.x, bz2);
    fe u2 = F::mul(b.x, az2);
    fe s1 = F::mul(a.y, F::mul(bz2, b.z));
    fe s2 = F::mul(b.y, F::mul(az2, a.z));
    fe h = F::sub(u1, u2);
    fe rr = F::sub(s1, s2);
    fe h2 = F::sqr(h);
    fe h3 = F::mul(h2, h);
    fe v = F::mul(u1, h2);
    jac r;
    r.x = F::sub(F::sub(F::add(F::sqr(rr), h3), v), v);
    r.y = F::sub(F::mul(rr, F::sub(v, r.x)), F::mul(s1, h3));
    r.z = F::mul(F::mul(a.z, b.z), h);
    if (F::is_zero(r.z)) {
      if (F::is_zero(a.z)) return b;
      if (F::is_zero(b.z)) return a;
      if (F::is_zero(rr)) return dbl(a);
      return infinity();
    }
    return r;
  }

#if defined(__CUDACC__)
#define EB_SWFN static __host__ __device__ __noinline__
#else
#define EB_SWFN static
#endif
  EB_SWFN jac dbl(jac p) { return dbl_inl(p); }
  EB_SWFN jac madd(jac a, aff p) { return madd_inl(a, p); }
  EB_SWFN jac add(jac a, jac b) { return add_inl(a, b); }

  static EB_HD aff to_aff(const jac& a) {
    fe zi = F::inv(a.z);
    fe zi2 = F::sqr(zi);
    aff r;
    r.x = F::mul(a.x, zi2);
    r.y = F::mul(F::mul(a.y, zi2), zi);
    return r;
  }

  // Red.prototype.sqrt (bn.js, dist/elliptic.js:7177-7232) on a Montgomery-form operand.  p = 3 mod 4: a^((p+1)/4).
  // p = 1 mod 4 (p224): Tonelli-Shanks with the reference's own non-residue; for a non-residue its
  // `assert(i < m)` fires (status 5, 'Assertion failed') before the caller's own y^2 check can.
  // Returns 0 with a candidate root (the caller still squares it), or 5.
  static EB_HD uint8_t sqrt_ref(const fe& a, fe* out) {
    u32 pm[N];
    F::Params::mod(pm);
    if ((pm[0] & 3) == 3) {
      u32 one[N];
      for (int w = 0; w < N; w++) one[w] = w == 0;
      add_n<N>(pm, pm, one);
      for (int k = 0; k < N; k++) pm[k] = (pm[k] >> 2) | ((k + 1 < N ? pm[k + 1] : 0u) << 30);
      *out = F::pow(a, pm);
      return 0;
    }
    if (F::is_zero(a)) { *out = F::zero(); return 0; }
    u32 q[N], q1h[N];
    C::ts_q(q); C::ts_q1h(q1h);
    fe c = C::ts_c();
    fe r = F::pow(a, q1h), t = F::pow(a, q);
    const fe one = F::one();
    int mm = C::TS_S;
    while (!F::eq(t, one)) {
      fe tmp = t;
      int i = 0;
      while (!F::eq(tmp, one)) {
        tmp = F::sqr(tmp);
        if (++i >= mm) return 5;
      }
      fe b = c;
      for (int k = 0; k < mm - i - 1; k++) b = F::sqr(b);
      r = F::mul(r, b);
      c = F::sqr(b);
      t = F::mul(t, c);
      mm = i;
    }
    *out = r;
    return 0;
  }

  // y^2 == x^3 - 3x + b  (ShortCurve.validate, short.js:206-216)
  static EB_HD bool on_curve(const aff& p) {
    fe x3 = F::mul(F::sqr(p.x), p.x);
    fe t = F::sub(x3, F::add(F::dbl(p.x), p.x));
    return F::eq(F::sqr(p.y), F::add(t, C::b()));
  }

  // ---- fixed-base table entry (j, idx) = (2 idx + 1) 2^(GW j) G, affine, Montgomery form
  static EB_HD void gtab_entry(int j, int idx, u32* out) {
    aff g; g.x = C::gx(); g.y = C::gy();
    jac b = from_aff(g);
    for (int k = 0; k < GW * j; k++) b = dbl(b);
    aff base = to_aff(b);
    u32 s = 2 * idx + 1;
    jac acc = infinity();
    for (int k = GW - 1; k >= 0; k--) {
      acc = dbl(acc);
      if ((s >> k) & 1) acc = madd(acc, base);
    }
    aff r = to_aff(acc);
    store_fe_n<N>(out, F::canon(r.x));       // table entries are stored canonical (and compared as such by the tests)
    store_fe_n<N>(out + N, F::canon(r.y));
  }

  // ---- prep: batched s^-1 (Montgomery trick, BATCH items/thread), u1, u2, odd-ification
  static EB_HD void prep_thread(size_t tid, size_t T, size_t cnt_items, const uint8_t* e, const uint8_t* r,
                                const uint8_t* s, u32* ws, u32* scratch) {
    typedef typename S::fe sc;
    const size_t LEN = C::LEN;
    u32 nmod[N];
    n_limbs(nmod);
    sc prod = S::one();
    u32 invalid_mask = 0;
    int cnt = 0;
    for (int j = 0; j < BATCH; j++) {
      size_t i = tid + (size_t)j * T;
      if (i >= cnt_items) break;
      cnt = j + 1;
      sc sv, rv;
      ldb(sv.v, s + LEN * i);
      ldb(rv.v, r + LEN * i);
      bool ok = !is_zero_n<N>(sv.v) && !geq_n<N>(sv.v, nmod) && !is_zero_n<N>(rv.v) && !geq_n<N>(rv.v, nmod);
      if (!ok) invalid_mask |= 1u << j;
      sc sm = S::cmov(S::to_mont(sv), S::one(), !ok);
      for (int w = 0; w < N; w++) scratch[(size_t)w * cnt_items + i] = prod.v[w];
      prod = S::mul(prod, sm);
    }
    if (cnt == 0) return;
    sc inv = S::inv(prod);
    for (int j = cnt - 1; j >= 0; j--) {
      size_t i = tid + (size_t)j * T;
      bool ok = !((invalid_mask >> j) & 1);
      sc sv, rv, ev, pre;
      ldb(sv.v, s + LEN * i);
      sc sm = S::cmov(S::to_mont(sv), S::one(), !ok);
      for (int w = 0; w < N; w++) pre.v[w] = scratch[(size_t)w * cnt_items + i];
      sc sinv = S::mul(inv, pre);
      inv = S::mul(inv, sm);
      u32 flags = ok ? 0 : FL_INVALID;
      ldb(rv.v, r + LEN * i);
      ldb(ev.v, e + LEN * i);
      sc u1 = S::mul(ev, sinv);     // plain e * Montgomery s^-1 -> plain   (ec/index.js:206)
      sc u2 = S::mul(rv, sinv);     //                                        (ec/index.js:207)
      prep_store(i, cnt_items, u1.v, u2.v, flags, ws);
    }
  }

  // odd-ify and store (u1, u2) SoA for dsm()
  static EB_HD void prep_store(size_t i, size_t cnt_items, u32* u1, u32* u2, u32 flags, u32* ws) {
    u32 nmod[N];
    n_limbs(nmod);
    if ((u1[0] & 1) == 0) { sub_n<N>(u1, nmod, u1); flags |= FL_NEGG; }
    if ((u2[0] & 1) == 0) { sub_n<N>(u2, nmod, u2); flags |= FL_NEG2; }
    for (int w = 0; w < N; w++) {
      u32 h1 = (w < N - 1) ? u1[w + 1] : 0, h2 = (w < N - 1) ? u2[w + 1] : 0;
      ws[(size_t)w * cnt_items + i] = (u1[w] >> 1) | (h1 << 31);
      ws[(size_t)(N + w) * cnt_items + i] = (u2[w] >> 1) | (h2 << 31);
    }
    ws[(size_t)(2 * N) * cnt_items + i] = flags;
  }

  // recoverPubKey scalars (ec/index.js:250-258): s1 = (n - e) r^-1, s2 = s r^-1 (mod n), with BN.invm's
  // convention that a multiple of n inverts to 0 (the result is then the point at infinity).  One inversion per
  // item: recovery is not on the headline path and stays simple.
  static EB_HD void prep_recover_item(size_t i, size_t cnt_items, const uint8_t* e, const uint8_t* r, const uint8_t* s,
                                      u32* ws) {
    typedef typename S::fe sc;
    const size_t LEN = C::LEN;
    u32 nmod[N];
    n_limbs(nmod);
    sc rv, sv, ev;
    ldb(rv.v, r + LEN * i); ldb(sv.v, s + LEN * i); ldb(ev.v, e + LEN * i);
    sc rm = S::to_mont(rv);                              // r mod n, Montgomery form (r < R)
    sc rinv = S::zero();
    if (!S::is_zero(rm)) rinv = S::inv(rm);
    sc u1 = S::mul(ev, rinv);                            // e / r (plain; e < R)
    if (!is_zero_n<N>(u1.v)) sub_n<N>(u1.v, nmod, u1.v); // (n - e) / r
    sc u2 = S::mul(sv, rinv);
    prep_store(i, cnt_items, u1.v, u2.v, 0, ws);
  }

  // k < 2^(8 LEN) -> k mod n.  One conditional subtraction when 2^(8 LEN) <= 2n; p521 (528-bit strings,
  // 521-bit n) goes through the Montgomery round trip x -> xR -> x.
  static EB_HD void reduce_scalar(u32* k) {
    if (8 * C::LEN <= C::BITS) {
      u32 nmod[N];
      n_limbs(nmod);
      if (geq_n<N>(k, nmod)) sub_n<N>(k, k, nmod);
    } else {
      typename S::fe t;
      for (int w = 0; w < N; w++) t.v[w] = k[w];
      t = S::from_mont(S::to_mont(t));
      for (int w = 0; w < N; w++) k[w] = t.v[w];
    }
  }

  // Point.mul / mulAdd callers (short.js:422-441): k1, k2 any integers below 2^(8 LEN), reduced mod n here
  // (for an on-curve point only the residue matters).  k1 == nullptr: no base-point term.
  static EB_HD void prep_scalars_item(size_t i, size_t cnt_items, const uint8_t* k1, const uint8_t* k2, u32* ws) {
    const size_t LEN = C::LEN;
    u32 nmod[N], u1[N], u2[N];
    n_limbs(nmod);
    u32 flags = 0;
    for (int w = 0; w < N; w++) u1[w] = 0;
    if (k1) { ldb(u1, k1 + LEN * i); reduce_scalar(u1); }
    else flags |= FL_NOG;
    ldb(u2, k2 + LEN * i);
    reduce_scalar(u2);
    prep_store(i, cnt_items, u1, u2, flags, ws);
  }

  static EB_HD void n_limbs(u32* r) { S::Params::mod(r); }

  static EB_HD u32 extract(const u32* ws, size_t cnt_items, size_t i, int base_word, int pos, int width) {
    int wi = pos >> 5;
    u32 lo = ws[(size_t)(base_word + wi) * cnt_items + i];
    u32 hi = (wi + 1 < N) ? ws[(size_t)(base_word + wi + 1) * cnt_items + i] : 0u;
    u64 both = ((u64)hi << 32) | lo;
    return (u32)(both >> (pos & 31)) & ((1u << width) - 1);
  }

  // ---- u1*G + u2*Q for an on-curve Q, scalars as stored by prep_store.  Jacobian result.
  static EB_HD jac dsm(size_t i, size_t cnt_items, const aff& Q, u32 flags, const u32* ws, const u32* gtab, u32* qtab) {
    u32* tab = qtab + (size_t)i * QTAB_WORDS;
    {
      jac P = from_aff(Q);
      jac D = dbl(P);
      for (int k = 0; k < 8; k++) {
        store_fe_n<N>(tab + 3 * N * k, P.x);
        store_fe_n<N>(tab + 3 * N * k + N, P.y);
        store_fe_n<N>(tab + 3 * N * k + 2 * N, P.z);
        if (k < 7) P = add(P, D);
      }
    }
    jac acc = infinity();
    for (int w = QWINDOWS - 1; w >= 0; w--) {
      if (w != QWINDOWS - 1)
        for (int d = 0; d < 4; d++) acc = dbl(acc);
      u32 nib = extract(ws, cnt_items, i, N, 4 * w, 4);
      bool dneg = (w != QWINDOWS - 1) && (nib < 8);
      u32 idx = (w == QWINDOWS - 1) ? (nib & 7) : (dneg ? 7 - nib : nib - 8);
      bool neg = dneg != ((flags & FL_NEG2) != 0);
      jac P;
      P.x = load_fe_n<N>(tab + 3 * N * idx);
      P.y = load_fe_n<N>(tab + 3 * N * idx + N);
      P.z = load_fe_n<N>(tab + 3 * N * idx + 2 * N);
      P.y = F::cmov(P.y, F::neg(P.y), neg);
      if (w == QWINDOWS - 1) acc = P;
      else acc = add(acc, P);
    }
    if (flags & FL_NOG) return acc;      // Point.mul: no base-point term
    for (int j = 0; j < GWINDOWS; j++) {
      u32 chunk = extract(ws, cnt_items, i, 0, GW * j, GW);
      const u32 half = 1u << (GW - 1);
      bool dneg = (j != GWINDOWS - 1) && (chunk < half);
      u32 idx = (j == GWINDOWS - 1) ? (chunk & (half - 1)) : (dneg ? half - 1 - chunk : chunk - half);
      bool neg = dneg != ((flags & FL_NEGG) != 0);
      const u32* ent = gtab + ((size_t)j * GENTRIES + idx) * 2 * N;
      aff P;
      P.x = load_fe_n<N>(ent);
      P.y = load_fe_n<N>(ent + N);
      P.y = F::cmov(P.y, F::neg(P.y), neg);
      acc = madd(acc, P);
    }
    return acc;
  }

  static EB_HD aff load_point(const uint8_t* pts, size_t i) {
    const size_t LEN = C::LEN;
    aff Q;
    fe t;
    ldb(t.v, pts + 2 * LEN * i);       Q.x = F::to_mont(t);
    ldb(t.v, pts + 2 * LEN * i + LEN); Q.y = F::to_mont(t);
    return Q;
  }
  static EB_HD void store_point(uint8_t* out, size_t i, const aff& a) {
    const size_t LEN = C::LEN;
    fe x = F::from_mont(a.x), y = F::from_mont(a.y);
    stb(out + 2 * LEN * i, x.v);
    stb(out + 2 * LEN * i + LEN, y.v);
  }

  // ---- main: one signature
  static EB_HD uint8_t verify_item(size_t i, size_t cnt_items, const uint8_t* pub, const uint8_t* r,
                                   const u32* ws, const u32* gtab, u32* qtab) {
    const size_t LEN = C::LEN;
    u32 flags = ws[(size_t)(2 * N) * cnt_items + i];
    if (flags & FL_INVALID) return 0;   // ST_FALSE
    aff Q = load_point(pub, i);
    if (!on_curve(Q)) return 4;          // ST_NEEDS_HOST (un-validated off-curve key, SURVEY 8a Q1)
    jac acc = dsm(i, cnt_items, Q, flags, ws, gtab, qtab);
    // accept iff R != O and x(R) == r (mod n)  (ec/index.js:222-228, eqXToP short.js:908-925)
    if (F::is_zero(acc.z)) return 0;
    fe z2 = F::sqr(acc.z);
    fe rp;
    ldb(rp.v, r + LEN * i);
    if (F::eq(acc.x, F::mul(F::to_mont(rp), z2))) return 1;
    u32 pmn[N]; C::p_minus_n(pmn);
    if (!geq_n<N>(rp.v, pmn)) {
      u32 nmod[N]; n_limbs(nmod);
      fe rn;
      add_n<N>(rn.v, rp.v, nmod);
      if (F::eq(acc.x, F::mul(F::to_mont(rn), z2))) return 1;
    }
    return 0;
  }

  // BasePoint.mul / Point.mulAdd (short.js:422-441) for an on-curve point, affine result (JPoint.toP,
  // short.js:516-526).  1 = point written, 7 = infinity, 4 = off-curve (replayed by SWReplay).
  static EB_HD uint8_t mul_add_item(size_t i, size_t cnt_items, const uint8_t* pts, const u32* ws, const u32* gtab,
                                    u32* qtab, uint8_t* out) {
    const size_t LEN = C::LEN;
    for (size_t b = 0; b < 2 * LEN; b++) out[2 * LEN * i + b] = 0;
    aff P = load_point(pts, i);
    if (!on_curve(P)) return 4;
    u32 flags = ws[(size_t)(2 * N) * cnt_items + i];
    jac acc = dsm(i, cnt_items, P, flags, ws, gtab, qtab);
    if (F::is_zero(acc.z)) return 7;
    store_point(out, i, to_aff(acc));
    return 1;
  }

  // EC.prototype.recoverPubKey (ec/index.js:231-259): R = pointFromX(r or r + n, odd) (short.js:187-204, p = 3 mod 4),
  // Q = s1*G + s2*R.  1 = point written, 7 = infinity, 2 = 'invalid point', 8 = 'Unable to find sencond key candinate'.
  static EB_HD uint8_t recover_item(size_t i, size_t cnt_items, const uint8_t* r, const uint8_t* recid, const u32* ws,
                                    const u32* gtab, u32* qtab, uint8_t* out) {
    const size_t LEN = C::LEN;
    for (size_t b = 0; b < 2 * LEN; b++) out[2 * LEN * i + b] = 0;
    u32 j = recid[i];
    bool odd = j & 1, second = (j >> 1) & 1;
    fe xr;
    ldb(xr.v, r + LEN * i);
    u32 pmn[N];
    C::p_minus_n(pmn);                                   // p mod n
    if (second && geq_n<N>(xr.v, pmn)) return 8;
    if (second) { u32 nmod[N]; n_limbs(nmod); add_n<N>(xr.v, xr.v, nmod); }   // r + n < p < 2^(32N)
    fe x = F::to_mont(xr);
    fe y2 = F::add(F::sub(F::mul(F::sqr(x), x), F::add(F::dbl(x), x)), C::b());
    fe y;
    if (uint8_t ss = sqrt_ref(y2, &y)) return ss;
    if (!F::eq(F::sqr(y), y2)) return 2;
    fe yp = F::from_mont(y);
    if (((yp.v[0] & 1) != 0) != odd) y = F::neg(y);
    aff R; R.x = x; R.y = y;
    u32 flags = ws[(size_t)(2 * N) * cnt_items + i];
    jac acc = dsm(i, cnt_items, R, flags, ws, gtab, qtab);
    if (F::is_zero(acc.z)) return 7;
    store_point(out, i, to_aff(acc));
    return 1;
  }

  // getKeyRecoveryParam scalars (recovery_param_item): u1 = e / s, u2 = (r mod n) / s for r, s any values below
  // 2^(8 LEN); s = 0 (mod n) is flagged FL_INVALID for the cold path.  One inversion per item, as prep_recover_item.
  static EB_HD void prep_recovery_param_item(size_t i, size_t cnt_items, const uint8_t* e, const uint8_t* r,
                                             const uint8_t* s, u32* ws) {
    typedef typename S::fe sc;
    const size_t LEN = C::LEN;
    sc rv, sv, ev;
    ldb(rv.v, r + LEN * i); ldb(sv.v, s + LEN * i); ldb(ev.v, e + LEN * i);
    sc sm = S::to_mont(sv);                              // s mod n, Montgomery form
    sc sinv = S::zero();
    u32 flags = FL_INVALID;
    if (!S::is_zero(sm)) { sinv = S::inv(sm); flags = 0; }
    sc u1 = S::mul(ev, sinv);                            // e / s (plain; e < n)
    sc u2 = S::mul(rv, sinv);                            // r / s (plain; r < R)
    prep_store(i, cnt_items, u1.v, u2.v, flags, ws);
  }

  // EC.prototype.getKeyRecoveryParam (ec/index.js:261-278) with one double-scalar multiplication: the group has prime
  // order, so for r, s != 0 (mod n), recoverPubKey(e, sig, j) = Q exactly when its candidate R_j equals
  // P = s^-1 (e G + r Q) = u1 G + u2 Q.  x(P) = r mod p gives j = parity(y(P)); x(P) = r + n (r < p mod n) gives
  // j = 2 + parity(y(P)); anything else (or P = O) no j.  P proves that pointFromX finds that candidate, Tonelli-Shanks
  // included (it succeeds on every square).  recid 0 unless 1; 1 = found, 11 = 'Unable to find valid recovery factor',
  // 4 = s = 0 (mod n), decided by recovery_param_cold_item.
  static EB_HD uint8_t recovery_param_item(size_t i, size_t cnt_items, const uint8_t* q, const uint8_t* r, const u32* ws,
                                           const u32* gtab, u32* qtab, uint8_t* recid) {
    const size_t LEN = C::LEN;
    recid[i] = 0;
    aff Q = load_point(q, i);
    if (!on_curve(Q)) return 11;                         // a recovered point is always on the curve
    u32 rn[N];
    ldb(rn, r + LEN * i);
    reduce_scalar(rn);
    if (is_zero_n<N>(rn)) return 11;                     // r = 0 (mod n): rInv = 0, every Q' is the point at infinity
    u32 flags = ws[(size_t)(2 * N) * cnt_items + i];
    if (flags & FL_INVALID) return 4;
    jac acc = dsm(i, cnt_items, Q, flags, ws, gtab, qtab);
    if (F::is_zero(acc.z)) return 11;
    fe z2 = F::sqr(acc.z);
    fe rp;
    ldb(rp.v, r + LEN * i);
    u32 j = 0;
    if (!F::eq(acc.x, F::mul(F::to_mont(rp), z2))) {
      u32 pmn[N]; C::p_minus_n(pmn);
      if (geq_n<N>(rp.v, pmn)) return 11;                // no second candidate (ec/index.js:243)
      u32 nmod[N]; n_limbs(nmod);
      add_n<N>(rp.v, rp.v, nmod);                        // r + n < p
      if (!F::eq(acc.x, F::mul(F::to_mont(rp), z2))) return 11;
      j = 2;
    }
    fe y = F::from_mont(to_aff(acc).y);
    recid[i] = (uint8_t)(j | (y.v[0] & 1));
    return 1;
  }

  // pointFromX(x) does not throw (recover_item's test); x plain, reduced mod p here as toRed does
  static EB_HD bool has_point_at(const fe& xr) {
    fe x = F::to_mont(xr);
    fe y2 = F::add(F::sub(F::mul(F::sqr(x), x), F::add(F::dbl(x), x)), C::b());
    fe y;
    if (sqrt_ref(y2, &y)) return false;
    return F::eq(F::sqr(y), y2);
  }

  // The items recovery_param_item leaves as 4: s = 0, r != 0 (mod n).  recoverPubKey then returns s1 G = ((n - e) / r) G
  // for every j whose candidate exists, so the answer is the first such j when Q is that point: j = 0 when r is an x
  // coordinate, else j = 2 when r + n < p is one.
  static EB_HD uint8_t recovery_param_cold_item(size_t i, const uint8_t* e, const uint8_t* r, const uint8_t* q,
                                                const u32* gtab, uint8_t* recid) {
    typedef typename S::fe sc;
    const size_t LEN = C::LEN;
    u32 nmod[N];
    n_limbs(nmod);
    sc rv, ev;
    ldb(rv.v, r + LEN * i); ldb(ev.v, e + LEN * i);
    sc k = S::mul(ev, S::inv(S::to_mont(rv)));          // e / r
    if (S::is_zero(k)) return 11;                        // s1 = 0: every Q' is the point at infinity
    sub_n<N>(k.v, nmod, k.v);                            // (n - e) / r
    uint8_t kb[C::LEN], t[2 * C::LEN], qb[2 * C::LEN];
    stb(kb, k.v);
    mul_g_item(0, kb, gtab, t);
    store_point(qb, 0, load_point(q, i));                // Q reduced mod p, as curve.point holds it
    for (size_t b = 0; b < 2 * LEN; b++)
      if (t[b] != qb[b]) return 11;
    fe x;
    ldb(x.v, r + LEN * i);
    if (has_point_at(x)) { recid[i] = 0; return 1; }
    u32 pmn[N];
    C::p_minus_n(pmn);
    if (geq_n<N>(x.v, pmn)) return 11;                   // 'Unable to find sencond key candinate'
    add_n<N>(x.v, x.v, nmod);
    if (has_point_at(x)) { recid[i] = 2; return 1; }
    return 11;
  }

  // G.mul(k) (short.js:422-427 -> _fixedNafMul, base.js:52-84): fixed table only
  static EB_HD uint8_t mul_g_item(size_t i, const uint8_t* k, const u32* gtab, uint8_t* out) {
    const size_t LEN = C::LEN;
    u32 nmod[N], kv[N];
    n_limbs(nmod);
    ldb(kv, k + LEN * i);
    reduce_scalar(kv);
    for (size_t b = 0; b < 2 * LEN; b++) out[2 * LEN * i + b] = 0;
    if (is_zero_n<N>(kv)) return 7;
    bool negg = (kv[0] & 1) == 0;
    if (negg) sub_n<N>(kv, nmod, kv);
    u32 m[N];
    for (int w = 0; w < N; w++) m[w] = (kv[w] >> 1) | ((w < N - 1 ? kv[w + 1] : 0u) << 31);
    jac acc = infinity();
    for (int j = 0; j < GWINDOWS; j++) {
      u32 chunk = extract(m, 1, 0, 0, GW * j, GW);
      const u32 half = 1u << (GW - 1);
      bool dneg = (j != GWINDOWS - 1) && (chunk < half);
      u32 idx = (j == GWINDOWS - 1) ? (chunk & (half - 1)) : (dneg ? half - 1 - chunk : chunk - half);
      const u32* ent = gtab + ((size_t)j * GENTRIES + idx) * 2 * N;
      aff P;
      P.x = load_fe_n<N>(ent);
      P.y = load_fe_n<N>(ent + N);
      P.y = F::cmov(P.y, F::neg(P.y), dneg != negg);
      acc = madd(acc, P);
    }
    store_point(out, i, to_aff(acc));
    return 1;
  }
};

}  // namespace eb
