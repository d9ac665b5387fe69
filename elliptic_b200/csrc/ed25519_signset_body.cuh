// ed25519_signset_body.cuh -- per-thread bodies of the EdDSA signing-set kernels (eddsa_signset.cu): the batch form of
// `key = eddsa.keyFromSecret(secret)` once and `key.sign(msg)` many times (lib/elliptic/eddsa/key.js:40-75,
// eddsa/index.js:34-44).  Host+device like the other bodies, so that the host emulation runs them.
//
// Create, once per key: hash = SHA512(secret), a = clamp(hash[0..31]), prefix = hash[32..63], A = encode(a G) -- the
// first half of ed25519_sign_item.  The set keeps a (Montgomery form of the scalar field, as the signing arithmetic
// uses it), the prefix and the 32 bytes of A; not the secret.
// Sign, per item, in three kernels:
//   nonce      r = SHA512(prefix || M) mod n, R = r G (extended coordinates) into the workspace;
//   normalise  one thread per ED_SS_BATCH items: Montgomery's trick over their Zs, one inversion, Renc into the signature;
//   challenge  h = SHA512(Renc || A || M) mod n, S = (r + h a) mod n.
// Every step is the unkeyed body's own arithmetic on the same values, so the signatures are byte-identical to
// ed25519_sign_item's.
#pragma once
#include "ed25519_body.cuh"

namespace eb {

constexpr int ED_SS_BATCH = 16;         // items per normalisation thread (DESIGN §6: B = 8 / 16 / 32 measured)
// normalisation block: 1024 items at any B, so a 2^18-item chunk launches 256 blocks (132 SMs)
constexpr int ED_SS_NORM_THREADS = 1024 / ED_SS_BATCH;
constexpr int ED_SS_KEY_WORDS = 16;     // per key: a (Montgomery form mod n), then the 32 prefix bytes
// Workspace, word-major (word w of item i at ws[w * ld + i]: a warp's accesses to one word are coalesced), per item:
// R's X, Y, Z, the running product of the batch's Zs, r (Montgomery form mod n).
constexpr int ED_SS_WS_X = 0, ED_SS_WS_Y = 8, ED_SS_WS_Z = 16, ED_SS_WS_PROD = 24, ED_SS_WS_R = 32, ED_SS_WS_WORDS = 40;

EB_HD f25 ed_ss_ws_load(const u32* ws, int w, size_t ld, size_t i) {
  f25 a;
  for (int q = 0; q < 8; q++) a.v[q] = ws[(size_t)(w + q) * ld + i];
  return a;
}
EB_HD void ed_ss_ws_store(u32* ws, int w, size_t ld, size_t i, const f25& a) {
  for (int q = 0; q < 8; q++) ws[(size_t)(w + q) * ld + i] = a.v[q];
}

// KeyPair.fromSecret for key k (eddsa/key.js:52-75): key words out, pub[32 k ..] = pubBytes
EB_HD void ed_ss_create_item(size_t k, const uint8_t* secrets, const u32* gtab, u32* keys, uint8_t* pub) {
  typedef Fp<ED25519_FN> S;
  uint8_t hash[64];
  sha512_ctx c;
  sha512_init(&c);
  sha512_update(&c, secrets + 32 * k, 32);
  sha512_final(&c, hash);
  hash[0] &= 248; hash[31] &= 127; hash[31] |= 64;                  // eddsa/key.js:58-62
  S::fe am;
  load_le<8>(am.v, hash);
  ed_encode(ed_mul_base(am.v, gtab), pub + 32 * k);                 // create is one-off: a per-item inversion
  const S::fe a = S::to_mont(am);
  u32* o = keys + ED_SS_KEY_WORDS * k;
  for (int q = 0; q < 8; q++) o[q] = a.v[q];
  uint8_t* prefix = reinterpret_cast<uint8_t*>(o + 8);             // messagePrefix
  for (int b = 0; b < 32; b++) prefix[b] = hash[32 + b];
  // the clamped key must not stay in local memory beyond this call
  for (int b = 0; b < 64; b++) hash[b] = 0;
}

// r = SHA512(prefix || M) mod n and R = r G for item i, signed by key key_idx[i]; ld: the workspace's item stride
EB_HD void ed_ss_nonce_item(size_t i, size_t ld, const uint8_t* msgs, const u64* msg_off, const u32* key_idx, const u32* keys,
                            const u32* gtab, u32* ws) {
  typedef Fp<ED25519_FN> S;
  const uint8_t* prefix = reinterpret_cast<const uint8_t*>(keys + ED_SS_KEY_WORDS * (size_t)key_idx[i] + 8);
  uint8_t dg[64];
  sha512_ctx c;
  sha512_init(&c);
  sha512_update(&c, prefix, 32);
  sha512_update(&c, msgs + msg_off[i], (size_t)(msg_off[i + 1] - msg_off[i]));
  sha512_final(&c, dg);
  const S::fe r = ed_digest_mod_n(dg);
  const S::fe rp = S::from_mont(r);                                 // r < n, plain
  const ed_ext R = ed_mul_base(rp.v, gtab);
  ed_ss_ws_store(ws, ED_SS_WS_X, ld, i, R.x);
  ed_ss_ws_store(ws, ED_SS_WS_Y, ld, i, R.y);
  ed_ss_ws_store(ws, ED_SS_WS_Z, ld, i, R.z);
  for (int q = 0; q < 8; q++) ws[(size_t)(ED_SS_WS_R + q) * ld + i] = r.v[q];
}

// Thread t of ceil(n / ED_SS_BATCH) encodes R for items t, t + T, t + 2 T, ... below n (T: the thread count; a strided
// batch, so that a warp's workspace loads are coalesced), with one inversion for the batch.  No Z is 0: R comes from
// ed_mul_base, which starts at the identity (0 : 1 : 1) and adds points of the fixed table, all on the curve, with
// complete formulas, and those never give Z = 0 for points on the curve.  So the product of the batch's Zs is
// invertible and each 1 / Z_u is exact.
EB_HD void ed_ss_normalise_item(size_t t, size_t n, size_t ld, u32* ws, uint8_t* sig) {
  const size_t T = (n + ED_SS_BATCH - 1) / ED_SS_BATCH;
  int cnt = 0;
  f25 prod = f25_one();
  for (int u = 0; u < ED_SS_BATCH; u++) {
    const size_t i = t + (size_t)u * T;
    if (i >= n) break;
    prod = f25_mul(prod, ed_ss_ws_load(ws, ED_SS_WS_Z, ld, i));
    ed_ss_ws_store(ws, ED_SS_WS_PROD, ld, i, prod);                // Z_0 .. Z_u
    cnt++;
  }
  f25 inv = f25_inv(prod);
  for (int u = cnt - 1; u >= 0; u--) {
    const size_t i = t + (size_t)u * T;
    const f25 zi = u ? f25_mul(inv, ed_ss_ws_load(ws, ED_SS_WS_PROD, ld, i - T)) : inv;
    inv = f25_mul(inv, ed_ss_ws_load(ws, ED_SS_WS_Z, ld, i));
    const f25 x = f25_normalize(f25_mul(ed_ss_ws_load(ws, ED_SS_WS_X, ld, i), zi));
    const f25 y = f25_normalize(f25_mul(ed_ss_ws_load(ws, ED_SS_WS_Y, ld, i), zi));
    ed_encode_affine(x, y, sig + 64 * i);
  }
}

// h = SHA512(Renc || A || M) mod n and S = (r + h a) mod n into sig[64 i + 32 ..]; Renc is sig[64 i ..], A the key's bytes
EB_HD void ed_ss_challenge_item(size_t i, size_t ld, const uint8_t* msgs, const u64* msg_off, const u32* key_idx,
                                const u32* keys, const uint8_t* A, const u32* ws, uint8_t* sig) {
  typedef Fp<ED25519_FN> S;
  const size_t k = key_idx[i];
  uint8_t dg[64];
  sha512_ctx c;
  sha512_init(&c);
  sha512_update(&c, sig + 64 * i, 32);
  sha512_update(&c, A + 32 * k, 32);
  sha512_update(&c, msgs + msg_off[i], (size_t)(msg_off[i + 1] - msg_off[i]));
  sha512_final(&c, dg);
  const S::fe h = ed_digest_mod_n(dg);
  S::fe r, a;
  for (int q = 0; q < 8; q++) { r.v[q] = ws[(size_t)(ED_SS_WS_R + q) * ld + i]; a.v[q] = keys[ED_SS_KEY_WORDS * k + q]; }
  const S::fe sv = S::from_mont(S::add(r, S::mul(h, a)));          // (r + h a) mod n
  for (int q = 0; q < 8; q++) {
    sig[64 * i + 32 + 4 * q] = (uint8_t)sv.v[q]; sig[64 * i + 32 + 4 * q + 1] = (uint8_t)(sv.v[q] >> 8);
    sig[64 * i + 32 + 4 * q + 2] = (uint8_t)(sv.v[q] >> 16); sig[64 * i + 32 + 4 * q + 3] = (uint8_t)(sv.v[q] >> 24);
  }
}

}  // namespace eb
