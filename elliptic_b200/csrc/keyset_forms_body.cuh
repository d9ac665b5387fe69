// keyset_forms_body.cuh -- item bodies of the kernels that frame the unchanged keyed ECDSA verify (keyset.cu) for its DER
// and device-pointer forms (keyset_forms.cu): a DER decode that also takes the key's verdict, an index screen, and the
// verdict merge behind the keyed replay.
//
// A verdict byte per item carries what must override the keyed main kernel's answer: 0 = nothing (the keyed verify
// decides), else the status the item gets.  The precedence is the reference's order of evaluation in key.verify with a
// DER signature (ec/index.js:194-202): keyFromPublic's throw, then new Signature's, then the range test and the verify
// itself, which the keyed kernels already answer.  An index >= m has no key at all, so its verdict overrides everything.
#pragma once
#include "../../include/elliptic_b200.h"
#include "der_sig.cuh"

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

// Item i after the keyed replay: a non-zero verdict replaces the keyed status.
EB_HD void ks_verdict_merge_item(size_t i, const uint8_t* verdict, uint8_t* status) {
  const uint8_t v = verdict[i];
  if (v) status[i] = v;
}

}  // namespace eb
