// keyset_forms_body.cuh -- item bodies of the kernels that frame the unchanged keyed ECDSA verify (keyset.cu) for its DER
// and device-pointer forms (keyset_forms.cu): a DER decode that also takes the key's verdict, an index screen, and the
// verdict merge behind the keyed replay; and, for the device-pointer forms of the other keyed calls, the scalar and
// message-range screens, a merge that also zeroes outputs, and screened wrappers of the bodies that read messages.
//
// A verdict byte per item carries what must override the keyed main kernel's answer: 0 = nothing (the keyed verify
// decides), else the status the item gets.  The precedence is the reference's order of evaluation in key.verify with a
// DER signature (ec/index.js:194-202): keyFromPublic's throw, then new Signature's, then the range test and the verify
// itself, which the keyed kernels already answer.  An index >= m has no key at all, so its verdict overrides everything.
#pragma once
#include "../../include/elliptic_b200.h"
#include "der_sig.cuh"
#include "ed25519_signset_body.cuh"

namespace eb {

// Item i of a DER block: decodes der[off[i] .. off[i+1]) to fixed-width r, s (len bytes each, zero when _importDER
// rejects the encoding, so the prep kernel never reads stale bytes) and returns the item's verdict: the throw of key
// key_idx[i] if it threw at import, else ST_THROW_SIG_FORMAT for a rejected encoding, else 0.
EB_HD uint8_t ks_der_verdict_item(size_t i, u32 len, const uint8_t* der, const unsigned long long* off, const u32* key_idx,
                                  const uint8_t* kst, uint8_t* r, uint8_t* s) {
  uint8_t* ri = r + (size_t)len * i;
  uint8_t* si = s + (size_t)len * i;
  const bool ok = der_import(der + off[i], (size_t)(off[i + 1] - off[i]), len, ri, si);
  if (!ok)
    for (u32 k = 0; k < len; k++) ri[k] = si[k] = 0;
  const uint8_t ks = kst[key_idx[i]];
  if (ks > EB200_ST_TRUE) return ks;
  return ok ? 0 : (uint8_t)EB200_ST_THROW_SIG_FORMAT;
}

// Item i of a device-pointer block: copies key_idx[i] to idx_out[i], or 0 when it is not below m, and returns the item's
// verdict (EB200_ST_BAD_KEY_INDEX or 0).  Only idx_out addresses the set afterwards.
EB_HD uint8_t ks_index_screen_item(size_t i, const u32* key_idx, size_t m, u32* idx_out) {
  const u32 k = key_idx[i];
  const bool bad = (size_t)k >= m;
  idx_out[i] = bad ? 0u : k;
  return bad ? (uint8_t)EB200_ST_BAD_KEY_INDEX : 0;
}

// ks_der_verdict_item behind the index-and-range screen (ks_index_range_screen_item), for the keyed DER verify on
// device pointers: pre[i] is the screen's verdict and idx the screened indices.  A screened item reads no byte of its
// range, gets r = s = 0 and keeps its verdict; any other is decoded with its key's verdict exactly as there.  So the
// precedence is BAD_KEY_INDEX, BAD_ITEM, the key's import throw, THROW_SIG_FORMAT.
EB_HD uint8_t ks_der_screened_item(size_t i, u32 len, const uint8_t* pre, const uint8_t* der, const unsigned long long* off,
                                   const u32* idx, const uint8_t* kst, uint8_t* r, uint8_t* s) {
  const uint8_t v = pre[i];
  if (!v) return ks_der_verdict_item(i, len, der, off, idx, kst, r, s);
  for (u32 k = 0; k < len; k++) r[(size_t)len * i + k] = s[(size_t)len * i + k] = 0;
  return v;
}

// Item i after the keyed replay: a non-zero verdict replaces the keyed status.
EB_HD void ks_verdict_merge_item(size_t i, const uint8_t* verdict, uint8_t* status) {
  const uint8_t v = verdict[i];
  if (v) status[i] = v;
}

// ---- the device-pointer forms of the other keyed calls -----------------------------------------------------------------
// A host form refuses a bad argument with EB200_ERR_ARG before launch; a device-pointer call cannot read its arguments
// without synchronising the caller's stream, so a screen gives each such item a verdict instead, and only screened
// copies (index 0, scalar 0) or skipped bodies ever see it.  The keyed ed25519 and curve25519 tables cover 253 bits and
// their top digit is bounded only for scalars below n, so a scalar >= n must never reach them, as an index >= m must
// never address the set and a range past msgs_len must never be read.  BAD_KEY_INDEX takes precedence over BAD_ITEM.

// w < n of ed25519 / curve25519 (2^252 + 27742317777372353535851937790883648493) for w as 8 little-endian words
EB_HD bool ks_below_n25519(const u32* w) {
  const u32 n[8] = {0x5cf5d3edu, 0x5812631au, 0xa2f79cd6u, 0x14def9deu, 0u, 0u, 0u, 0x10000000u};
  for (int q = 7; q >= 0; q--)
    if (w[q] != n[q]) return w[q] < n[q];
  return false;
}

// A 16-byte-aligned group of four words, so that an aligned 32-byte scalar moves in two 16-byte loads and stores
struct alignas(16) ks_w4 { u32 v[4]; };

// Item i of a block with a 32-byte scalar per item (k: little-endian EdDSA h, or big_endian curve25519 priv): copies
// key_idx[i] to idx_out[i] and the scalar to k_out[32 i ..], or 0 and 32 zero bytes for a screened item, and returns
// the item's verdict: BAD_KEY_INDEX for key_idx[i] >= m, else BAD_ITEM for a scalar >= n, else 0.  When k and k_out
// are 16-byte aligned (the caller's tensors, and the workspace always) the scalar moves as words, else byte by byte.
EB_HD uint8_t ks_index_scalar_screen_item(size_t i, const u32* key_idx, size_t m, const uint8_t* k, bool big_endian,
                                          u32* idx_out, uint8_t* k_out) {
  const uint8_t* ki = k + 32 * i;
  uint8_t* ko = k_out + 32 * i;
  const bool aligned = (((uintptr_t)k | (uintptr_t)k_out) & 15) == 0;
  u32 le[8];                                       // the 32 bytes as little-endian words, in memory order
  if (aligned) {
    const ks_w4 a = reinterpret_cast<const ks_w4*>(ki)[0], b = reinterpret_cast<const ks_w4*>(ki)[1];
    for (int q = 0; q < 4; q++) { le[q] = a.v[q]; le[4 + q] = b.v[q]; }
  } else {
    for (int q = 0; q < 8; q++)
      le[q] = (u32)ki[4 * q] | (u32)ki[4 * q + 1] << 8 | (u32)ki[4 * q + 2] << 16 | (u32)ki[4 * q + 3] << 24;
  }
  u32 w[8];                                        // the scalar's value, least significant word first
  for (int q = 0; q < 8; q++) {
    const u32 x = le[big_endian ? 7 - q : q];
    w[q] = big_endian ? (x >> 24) | (x >> 8 & 0xff00u) | (x << 8 & 0xff0000u) | (x << 24) : x;
  }
  const u32 ix = key_idx[i];
  const uint8_t v = (size_t)ix >= m ? (uint8_t)EB200_ST_BAD_KEY_INDEX : !ks_below_n25519(w) ? (uint8_t)EB200_ST_BAD_ITEM : 0;
  idx_out[i] = v ? 0u : ix;
  if (aligned) {
    ks_w4 a, b;
    for (int q = 0; q < 4; q++) { a.v[q] = v ? 0u : le[q]; b.v[q] = v ? 0u : le[4 + q]; }
    reinterpret_cast<ks_w4*>(ko)[0] = a;
    reinterpret_cast<ks_w4*>(ko)[1] = b;
  } else {
    for (int b = 0; b < 32; b++) ko[b] = v ? 0 : ki[b];
  }
  return v;
}

// Item i of a block of messages (off: n + 1 absolute offsets into a buffer of msgs_len bytes): the index screen, then
// BAD_ITEM for a range that decreases or ends past msgs_len.  Only items with verdict 0 may read their range.
EB_HD uint8_t ks_index_range_screen_item(size_t i, const u32* key_idx, size_t m, const u64* off, u64 msgs_len, u32* idx_out) {
  const u32 ix = key_idx[i];
  const u64 a = off[i], b = off[i + 1];
  const uint8_t v = (size_t)ix >= m ? (uint8_t)EB200_ST_BAD_KEY_INDEX : (b < a || b > msgs_len) ? (uint8_t)EB200_ST_BAD_ITEM : 0;
  idx_out[i] = v ? 0u : ix;
  return v;
}

// Item i after the keyed kernels of a call with outputs: a non-zero verdict replaces the status and zeroes the item's
// ol-byte output row (ol = 1 for the recovery parameter).
EB_HD void ks_verdict_merge_out_item(size_t i, const uint8_t* verdict, uint8_t* status, uint8_t* out, u32 ol) {
  const uint8_t v = verdict[i];
  if (!v) return;
  status[i] = v;
  for (u32 b = 0; b < ol; b++) out[(size_t)ol * i + b] = 0;
}

// ed25519_hash_item for a screened item i: h = 0 and no message byte read.
EB_HD void ks_ed_hash_screened_item(size_t i, const uint8_t* verdict, const uint8_t* R, const uint8_t* A, const uint8_t* msgs,
                                    const u64* msg_off, uint8_t* h) {
  if (verdict[i]) {
    for (int b = 0; b < 32; b++) h[32 * i + b] = 0;
    return;
  }
  ed25519_hash_item(i, R, A, msgs, msg_off, h);
}

// ed_ss_nonce_item for a screened item i: no message byte read, and R = the identity (0 : 1 : 1) with r = 0 in the
// workspace, so that the batched normalisation, which multiplies the Zs of ED_SS_BATCH items together, still sees an
// invertible Z in this slot and encodes the other items' R exactly.
EB_HD void ks_ss_nonce_screened_item(size_t i, size_t ld, const uint8_t* verdict, const uint8_t* msgs, const u64* msg_off,
                                     const u32* key_idx, const u32* keys, const u32* gtab, u32* ws) {
  if (verdict[i]) {
    const ed_ext I = ed_identity();
    ed_ss_ws_store(ws, ED_SS_WS_X, ld, i, I.x);
    ed_ss_ws_store(ws, ED_SS_WS_Y, ld, i, I.y);
    ed_ss_ws_store(ws, ED_SS_WS_Z, ld, i, I.z);
    for (int q = 0; q < 8; q++) ws[(size_t)(ED_SS_WS_R + q) * ld + i] = 0;
    return;
  }
  ed_ss_nonce_item(i, ld, msgs, msg_off, key_idx, keys, gtab, ws);
}

// ed_ss_challenge_item, skipped for a screened item (the merge zeroes its signature).
EB_HD void ks_ss_challenge_screened_item(size_t i, size_t ld, const uint8_t* verdict, const uint8_t* msgs, const u64* msg_off,
                                         const u32* key_idx, const u32* keys, const uint8_t* A, const u32* ws, uint8_t* sig) {
  if (!verdict[i]) ed_ss_challenge_item(i, ld, msgs, msg_off, key_idx, keys, A, ws, sig);
}

}  // namespace eb
