// unkeyed_forms_body.cuh -- item bodies of the kernels that frame the unchanged unkeyed kernels for the device-pointer
// forms of the calls that take variable-length ranges (unkeyed_forms.cu): eb200_ecdsa_verify_batch_der_dev,
// eb200_eddsa_verify_batch_msgs_dev and eb200_eddsa_sign_batch_dev.
//
// Their host forms refuse a decreasing offset with EB200_ERR_ARG before launch.  A device-pointer call cannot read its
// offsets without synchronising the caller's stream, so a range screen gives each item a verdict instead (0, or
// EB200_ST_BAD_ITEM for a range that decreases or ends past the buffer), the bodies below skip a screened item without
// reading a byte of its range, and the merge of keyset_forms_body.cuh writes the verdict over the item's status and
// zeroes its outputs.
//
// A screened item cannot simply be handed an empty range in a sanitised copy of the n + 1 offsets: item i's end is item
// i + 1's start, so a decreasing range between two good ones has no empty replacement that leaves both neighbours
// intact.  The DER decode is therefore screened itself, as the EdDSA hash (ks_ed_hash_screened_item) already is.
#pragma once
#include "keyset_forms_body.cuh"

namespace eb {

// Item i of a block of ranges without key indices (off: n + 1 absolute offsets into a buffer of len bytes): BAD_ITEM
// for a range that decreases or ends past len, else 0.  The keyed range screen's own body decides, on a one-item view
// (offsets off[i], off[i + 1]) with the one key index 0 of a one-key set, so both screens share one predicate.
EB_HD uint8_t ud_range_screen_item(size_t i, const u64* off, u64 len) {
  const u32 key0 = 0;
  u32 idx_sink;
  return ks_index_range_screen_item(0, &key0, 1, off + i, len, &idx_sink);
}

// der_decode_kernel's item behind a range screen.  An item with verdict 0 is decoded exactly as there, except that a
// rejected encoding leaves r = s = 0 instead of what the buffers held (its status is the throw either way); a screened
// item reads nothing, gets r = s = 0 and the status of a rejected encoding, which the merge then replaces.  pre: the
// key decoder's statuses when pre_valid, overwritten with the item's pre-status as der_decode_kernel does.
EB_HD void ud_der_decode_screened_item(size_t i, u32 len, const uint8_t* verdict, const uint8_t* der,
                                       const unsigned long long* off, uint8_t* r, uint8_t* s, uint8_t* pre, int pre_valid) {
  uint8_t* ri = r + (size_t)len * i;
  uint8_t* si = s + (size_t)len * i;
  const bool ok = !verdict[i] && der_import(der + off[i], (size_t)(off[i + 1] - off[i]), len, ri, si);
  if (!ok)
    for (u32 k = 0; k < len; k++) ri[k] = si[k] = 0;
  uint8_t st = pre_valid ? pre[i] : 0;
  if (!st && !ok) st = (uint8_t)EB200_ST_THROW_SIG_FORMAT;
  pre[i] = st;
}

// ed25519_sign_item behind a range screen: a screened item reads neither its message nor its secret, zeroes its public
// key row (pub may be NULL) and returns 0; the merge writes its status and zeroes its signature.
EB_HD uint8_t ud_ed25519_sign_screened_item(size_t i, const uint8_t* verdict, const uint8_t* secrets, const uint8_t* msgs,
                                            const u64* msg_off, const u32* gtab, uint8_t* sig, uint8_t* pub) {
  if (verdict[i]) {
    if (pub)
      for (int b = 0; b < 32; b++) pub[32 * i + b] = 0;
    return 0;
  }
  return ed25519_sign_item(i, secrets, msgs, msg_off, gtab, sig, pub);
}

}  // namespace eb
