"""Host-side mirror of the reference's ECDSA object for the accelerated path.

`EC(name)` corresponds to `new elliptic.ec(name)` (lib/elliptic/ec/index.js:13-40);
`verify(msg, sig, key)` keeps the reference's argument forms and error
behaviour (ec/index.js:188-229) and `verify_batch` is the new batch entry
point (SURVEY 8b: `EC#verifyBatch(msgs, sigs, pubs) -> Uint8Array`).  Parsing
(hex / byte arrays / DER / SEC1) is done here exactly as the reference's JS
does it; all curve arithmetic happens in libelliptic_b200.so on the GPU.
"""
import re

import ctypes

import numpy as np

from . import _native as nat

_CURVES = {
    # name -> C-ABI id, byte length of a field element, group order n, field prime p (curves.js:43-206)
    "secp256k1": dict(id=nat.CURVE_SECP256K1, len=32,
                      n=0xfffffffffffffffffffffffffffffffebaaedce6af48a03bbfd25e8cd0364141,
                      p=2**256 - 2**32 - 977),
    "p256": dict(id=nat.CURVE_P256, len=32,
                 n=0xffffffff00000000ffffffffffffffffbce6faada7179e84f3b9cac2fc632551,
                 p=2**256 - 2**224 + 2**192 + 2**96 - 1),
    "curve25519": dict(id=nat.CURVE_CURVE25519, len=32,
                       n=0x1000000000000000000000000000000014def9dea2f79cd65812631a5cf5d3ed, p=2**255 - 19),
    "p384": dict(id=nat.CURVE_P384, len=48,
                 n=0xffffffffffffffffffffffffffffffffffffffffffffffffc7634d81f4372ddf581a0db248b0a77aecec196accc52973,
                 p=2**384 - 2**128 - 2**96 + 2**32 - 1),
    "p521": dict(id=nat.CURVE_P521, len=66,
                 n=0x1fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d03bb5c9b8899c47aebb6fb71e91386409,
                 p=2**521 - 1),
    "ed25519": dict(id=nat.CURVE_ED25519, len=32,
                    n=0x1000000000000000000000000000000014def9dea2f79cd65812631a5cf5d3ed, p=2**255 - 19),
    "p192": dict(id=nat.CURVE_P192, len=24, n=0xffffffffffffffffffffffff99def836146bc9b1b4d22831, p=0xfffffffffffffffffffffffffffffffeffffffffffffffff),
    "p224": dict(id=nat.CURVE_P224, len=28, n=0xffffffffffffffffffffffffffff16a2e0b8f03e13dd29455c5c2a3d, p=0xffffffffffffffffffffffffffffffff000000000000000000000001),
}


_SHORT = ("secp256k1", "p256", "p384", "p521", "p192", "p224")
# presets whose points are (x, y) pairs with batch sign / keygen / mul / mulAdd / ECDH entry points: the six short
# curves and the twisted Edwards preset (new elliptic.ec('ed25519'), test/ecdsa-test.js:130, test/ecdh-test.js:26)
_XY = _SHORT + ("ed25519",)


class EllipticError(Exception):
    """An `Error` the reference would have thrown (message = the JS message)."""


class NeedsReferencePath(EllipticError):
    """The reference's result for this item is not a group-law function of the
    inputs (un-validated off-curve public key, SURVEY 8a Q1); the engine does
    not guess -- run the reference's single-item path for it."""


_THROW_MSG = {
    nat.ST_THROW_INVALID_POINT: "invalid point",
    nat.ST_THROW_NOT_VALIDATED: "public point not validated",
    nat.ST_THROW_ASSERT: "Assertion failed",
    nat.ST_THROW_POINT_FORMAT: "Unknown point format",
    nat.ST_THROW_SECOND_KEY: "Unable to find sencond key candinate",
    nat.ST_THROW_SIG_FORMAT: "Signature without r or s",
    nat.ST_THROW_NO_RECOVERY: "Unable to find valid recovery factor",
}


def _to_array(msg, enc=None):
    """minimalistic-crypto-utils.toArray (reference dist/elliptic.js:8847-8876)."""
    if isinstance(msg, (bytes, bytearray)):
        return bytes(msg)
    if isinstance(msg, (list, tuple, np.ndarray)):
        return bytes(int(b) & 0xFF for b in msg)
    if not msg:
        return b""
    if isinstance(msg, str):
        if enc == "hex":
            msg = re.sub(r"[^a-zA-Z0-9]+", "", msg)
            if len(msg) % 2:
                msg = "0" + msg
            out = bytearray()
            for i in range(0, len(msg), 2):
                try:
                    out.append(int(msg[i:i + 2], 16))
                except ValueError:
                    out.append(0)
            return bytes(out)
        out = bytearray()
        for ch in msg:
            c = ord(ch)
            if c >> 8:
                out.append(c >> 8)
            out.append(c & 0xFF)
        return bytes(out)
    raise TypeError("unsupported input form")


def _parse_hex(s):
    """bn.js 4.11.9 `new BN(str, 16)` (dist/elliptic.js:4135-4157 parseHex, :4003-4017): whitespace is dropped, a
    leading '-' negates, and a character outside [0-9a-fA-F] contributes (charCode - 48) & 0xf instead of throwing."""
    s = "".join(s.split())
    neg = s.startswith("-")
    if neg:
        s = s[1:]
    v = 0
    for ch in s:
        c = ord(ch) - 48
        if 49 <= c <= 54:
            d = c - 49 + 10
        elif 17 <= c <= 22:
            d = c - 17 + 10
        else:
            d = c & 0xF
        v = (v << 4) | d
    return -v if neg else v


def _bn(v):
    """`new BN(v, 16)` for int / hex string / byte array."""
    if isinstance(v, int):
        return v
    if isinstance(v, str):
        return _parse_hex(v)
    return int.from_bytes(bytes(v), "big")


def _msg_int(msg):
    """`new BN(msg)` as recoverPubKey / getKeyRecoveryParam take the message: byte arrays big-endian, else as _bn."""
    if isinstance(msg, (bytes, bytearray, list, tuple)):
        return int.from_bytes(_to_array(msg), "big")
    return _bn(msg)


def _signature(sig, enc):
    """new Signature(sig, enc) (ec/signature.js:8-22) -> (r, s)."""
    if isinstance(sig, dict):
        if not (sig.get("r") and sig.get("s")):
            raise EllipticError("Signature without r or s")
        return _bn(sig["r"]), _bn(sig["s"])
    if hasattr(sig, "r") and hasattr(sig, "s"):
        return int(sig.r), int(sig.s)
    rs = parse_der(_to_array(sig, enc))
    if rs is None:
        raise EllipticError("Signature without r or s")
    return rs


def _pers(pers, pers_enc):
    """The `pers` option after `persEnc` decoding (utf8 by default, ec/index.js:150) as a NUL-terminated uint8 array,
    and its length; (None, 0) without one."""
    if pers is None:
        return None, 0
    b = bytes(_to_array(pers, pers_enc or "utf8"))
    return np.frombuffer(b + b"\x00", np.uint8), len(b)


def _pack(vals, width, order="big"):
    """Ints as an (n, width) uint8 array, one `width`-byte row each: the C ABI's item-major layout.  Each value is
    encoded as `vals` yields it, so a generator that parses items stops at the first one that does not fit."""
    return np.frombuffer(b"".join(v.to_bytes(width, order) for v in vals), np.uint8).reshape(-1, width)


def _pack_points(pts, p, ln):
    """curve.point(x, y) for (x, y) pairs or {x, y} dicts (short.js:251-271): an (n, 2 ln) array of x || y,
    coordinates reduced mod p, not validated."""
    xy = ((pt["x"], pt["y"]) if isinstance(pt, dict) else pt for pt in pts)
    return _pack((_bn(c) % p for x, y in xy for c in (x, y)), ln).reshape(-1, 2 * ln)


def _unpack(out, ln, st=None, needs_host=False):
    """The rows of an (n, ln) output as ints, of an (n, 2 ln) one as (x, y) pairs; None where `st` is not TRUE.
    needs_host: refuse the batch if the engine flagged an input point as off the curve (ST_NEEDS_HOST)."""
    if needs_host and bool((st == nat.ST_NEEDS_HOST).any()):
        raise NeedsReferencePath("point %d is not on the curve; the reference does not validate it" % int(np.flatnonzero(st == nat.ST_NEEDS_HOST)[0]))
    b = out.tobytes()
    vals = [int.from_bytes(b[i:i + ln], "big") for i in range(0, len(b), ln)]
    if out.shape[1] != ln:
        vals = list(zip(vals[::2], vals[1::2]))
    return [v if st is None or st[i] == nat.ST_TRUE else None for i, v in enumerate(vals)]


def _blob(items):
    """Byte strings back to back as a uint8 array, and the n + 1 uint64 offsets of the items in it."""
    off = np.zeros(len(items) + 1, np.uint64)
    off[1:] = np.cumsum([len(b) for b in items])
    return np.frombuffer(b"".join(items), np.uint8), off


def _answer(value, st, answers):
    """One item's result: `value` where its status is one of `answers`, else the exception the reference throws."""
    st = int(st)
    if st not in answers:
        raise EllipticError(_THROW_MSG.get(st, "status %d" % st))
    return value


def parse_der(data):
    """Signature._importDER (ec/signature.js:73-134).  Returns (r, s) or None."""
    n = len(data)
    pos = 0

    def byte(i):
        return data[i] if 0 <= i < n else None

    def get_length():
        nonlocal pos
        initial = byte(pos)
        pos += 1
        if initial is None:
            return 0
        if not (initial & 0x80):
            return initial
        octets = initial & 0xF
        if octets == 0 or octets > 4:
            return None
        if byte(pos) == 0:
            return None
        val = 0
        off = pos
        for _ in range(octets):
            val = ((val << 8) | (byte(off) or 0)) & 0xFFFFFFFF
            off += 1
        if val <= 0x7F:
            return None
        pos = off
        return val

    if byte(pos) != 0x30:
        return None
    pos += 1
    ln = get_length()
    if ln is None or ln + pos != n:
        return None
    if byte(pos) != 0x02:
        return None
    pos += 1
    rlen = get_length()
    if rlen is None or ((byte(pos) or 0) & 0x80):
        return None
    r = data[pos:pos + rlen]
    pos += rlen
    if byte(pos) != 0x02:
        return None
    pos += 1
    slen = get_length()
    if slen is None or n != slen + pos or ((byte(pos) or 0) & 0x80):
        return None
    s = data[pos:pos + slen]
    for v in (r, s):
        if len(v) and v[0] == 0 and not (len(v) > 1 and v[1] & 0x80):
            return None
    return int.from_bytes(r, "big"), int.from_bytes(s, "big")


class _KeyObjects:
    """The key-object side of the `ec` API (ec/key.js), in batch form; EC inherits it."""

    def key_set(self, keys, enc=None, table_bits=0):
        """The batch form of `key = ec.keyFromPublic(pub, enc)` + `key.getPublic().precompute()`: a KeySet on the GPU
        (an X25519KeySet on curve25519)."""
        if self.name == "curve25519":
            return X25519KeySet(self, keys, table_bits)
        return KeySet(self, keys, enc, table_bits)


class _TensorForms:
    """The device-buffer calls on CUDA tensors, on the caller's stream (conventions: _tensors); EC inherits them."""

    def _tensor_call(self, name, fn, specs, head, outs, zeroed=False, ws=True):
        """Checks specs, then fn(*head(n), *outs, status[, workspace], stream) with outs new (n, ...) uint8 tensors (zeroed:
        filled with zeros first).  Returns the outputs and the status."""
        from . import _tensors as T
        if self.name == "curve25519" and name not in ("derive_batch_tensors", "x_mul_batch_tensors"):
            raise EllipticError("%s: not available on curve25519" % name)
        n, dev = T.check(name, specs)
        res = [(T.zeros if zeroed else T.empty)(dev, n, *shape) for shape in outs] + [T.empty(dev, n)]
        T.launch(fn, dev, head(n) + res, T.ws_unkeyed(self._c["id"], n) if ws else None)
        return res

    def _rows(self, *named, width=None):
        from . import _tensors as T
        return [(a, t, T.ROWS, width or self._len) for a, t in named]

    def verify_batch_tensors(self, e, r, s, pub, pub_fmt=nat.PUB_XY):
        """verify_batch_packed on CUDA tensors (eb200_ecdsa_verify_batch_dev): e, r, s (n, len), pub (n, k) in pub_fmt.
        Returns the (n,) statuses."""
        if pub_fmt not in (nat.PUB_XY, nat.PUB_SEC1_65, nat.PUB_SEC1_33):
            raise ValueError("verify_batch_tensors: unknown pub_fmt %r" % (pub_fmt,))
        specs = self._rows(("e", e), ("r", r), ("s", s)) + self._rows(("pub", pub), width=self._pub_bytes(pub_fmt))
        (st,) = self._tensor_call("verify_batch_tensors", "eb200_ecdsa_verify_batch_dev", specs,
                                  lambda n: [self._c["id"], n, e, r, s, pub, pub_fmt], [])
        return st

    def verify_batch_der_tensors(self, e, sigs, sig_off, pub, pub_fmt=nat.PUB_XY):
        """verify_batch_der_packed on CUDA tensors (eb200_ecdsa_verify_batch_der_dev): e (n, len), the DER encodings back
        to back in sigs (1-D uint8) with (n + 1,) int64 offsets, pub (n, k) in pub_fmt.  Returns the (n,) statuses; an
        item whose range decreases or ends past sigs gets ST_BAD_ITEM."""
        from . import _tensors as T
        if pub_fmt not in (nat.PUB_XY, nat.PUB_SEC1_65, nat.PUB_SEC1_33):
            raise ValueError("verify_batch_der_tensors: unknown pub_fmt %r" % (pub_fmt,))
        specs = self._rows(("e", e)) + [("sigs", sigs, T.BYTES, 0), ("sig_off", sig_off, T.OFF, 0)] + \
            self._rows(("pub", pub), width=self._pub_bytes(pub_fmt))
        (st,) = self._tensor_call("verify_batch_der_tensors", "eb200_ecdsa_verify_batch_der_dev", specs,
                                  lambda n: [self._c["id"], n, e, sigs, sigs.numel(), sig_off, pub, pub_fmt], [])
        return st

    def sign_batch_tensors(self, e, priv, canonical=False, k=None, pers=None):
        """One batch of EC.sign on CUDA tensors: e (n, len) truncated hashes (< n), priv (n, len) reduced mod n, as
        eb200_ecdsa_sign_batch takes them.  k: (n, len) nonces for one attempt (eb200_ecdsa_sign_batch_k_dev; a RETRY
        item's r, s and recid stay zero), or pers: the personalisation bytes as a 1-D uint8 tensor
        (eb200_ecdsa_sign_batch_pers_dev); neither: RFC 6979 nonces.  Returns (r, s, recid, status)."""
        from . import _tensors as T
        if self.name not in _XY:
            raise EllipticError("sign_batch_tensors: not available on " + self.name)
        if k is not None and pers is not None:
            raise ValueError("sign_batch_tensors: k and pers exclude each other")
        cid, flags = self._c["id"], 1 if canonical else 0
        specs = self._rows(("e", e), ("priv", priv), ("k", k)) + [("pers", pers, T.BYTES, 0)]
        outs = [(self._len,), (self._len,), ()]
        if k is not None:
            return self._tensor_call("sign_batch_tensors", "eb200_ecdsa_sign_batch_k_dev", specs,
                                     lambda n: [cid, n, e, priv, k, flags], outs, zeroed=True)
        if pers is not None:
            return self._tensor_call("sign_batch_tensors", "eb200_ecdsa_sign_batch_pers_dev", specs,
                                     lambda n: [cid, n, e, priv, pers, pers.numel(), flags], outs)
        return self._tensor_call("sign_batch_tensors", "eb200_ecdsa_sign_batch_dev", specs,
                                 lambda n: [cid, n, e, priv, flags], outs)

    def gen_key_pair_batch_tensors(self, entropy, pers=None):
        """gen_key_pair_batch on CUDA tensors (eb200_ec_keygen_batch_dev): entropy (n, k) uint8, k >= 24, one row per key;
        pers: the personalisation bytes as a 1-D uint8 tensor, or None.  Returns (priv (n, len), pub (n, 2 len), status)."""
        from . import _tensors as T
        if self.name not in _XY:
            raise EllipticError("gen_key_pair_batch_tensors: not available on " + self.name)
        specs = [("entropy", entropy, T.ROWS, None), ("pers", pers, T.BYTES, 0)]
        return self._tensor_call("gen_key_pair_batch_tensors", "eb200_ec_keygen_batch_dev", specs,
                                 lambda n: [self._c["id"], n, entropy, entropy.shape[1], pers,
                                            0 if pers is None else pers.numel()], [(self._len,), (2 * self._len,)])

    def recover_pub_key_batch_tensors(self, e, r, s, recid):
        """recoverPubKey on CUDA tensors (eb200_ecdsa_recover_batch_dev): e, r, s (n, len) as recover_pub_key_batch's call
        takes them, recid (n,) uint8.  Returns (points (n, 2 len), status)."""
        from . import _tensors as T
        specs = self._rows(("e", e), ("r", r), ("s", s)) + [("recid", recid, T.VEC, 0)]
        return self._tensor_call("recover_pub_key_batch_tensors", "eb200_ecdsa_recover_batch_dev", specs,
                                 lambda n: [self._c["id"], n, e, r, s, recid], [(2 * self._len,)])

    def get_key_recovery_param_batch_tensors(self, e, r, s, q):
        """getKeyRecoveryParam on CUDA tensors (eb200_ecdsa_recovery_param_batch_dev): e, r, s (n, len) as
        get_key_recovery_param_batch's call takes them, q (n, 2 len) the points.  Returns (recid (n,), status)."""
        specs = self._rows(("e", e), ("r", r), ("s", s)) + self._rows(("q", q), width=2 * self._len)
        return self._tensor_call("get_key_recovery_param_batch_tensors", "eb200_ecdsa_recovery_param_batch_dev",
                                 specs, lambda n: [self._c["id"], n, e, r, s, q], [()])

    def mul_batch_tensors(self, k, points=None):
        """Point.mul on CUDA tensors (eb200_scalar_mul_batch_dev): k (n, len) scalars, points (n, 2 len) x || y, or None
        for the base point.  Returns (out (n, 2 len), status)."""
        specs = self._rows(("k", k)) + self._rows(("points", points), width=2 * self._len)
        return self._tensor_call("mul_batch_tensors", "eb200_scalar_mul_batch_dev", specs,
                                 lambda n: [self._c["id"], n, k, points], [(2 * self._len,)])

    def mul_add_batch_tensors(self, k1, k2, points):
        """G.mulAdd(k1, P, k2) on CUDA tensors (eb200_mul_add_batch_dev): k1, k2 (n, len), points (n, 2 len).  Returns
        (out (n, 2 len), status)."""
        specs = self._rows(("k1", k1), ("k2", k2)) + self._rows(("points", points), width=2 * self._len)
        return self._tensor_call("mul_add_batch_tensors", "eb200_mul_add_batch_dev", specs,
                                 lambda n: [self._c["id"], n, k1, k2, points], [(2 * self._len,)])

    def derive_batch_tensors(self, priv, pub):
        """ECDH on CUDA tensors: priv (n, len) reduced mod n; pub (n, 2 len) peer points (eb200_ecdh_derive_batch_dev), or
        on curve25519 (n, 32) peer x (eb200_x25519_derive_batch_dev), as derive_batch_packed.  Returns (x (n, len),
        status)."""
        if self.name == "curve25519":
            return self._tensor_call("derive_batch_tensors", "eb200_x25519_derive_batch_dev",
                                     self._rows(("priv", priv), ("pub", pub)), lambda n: [n, priv, pub], [(32,)], ws=False)
        specs = self._rows(("priv", priv)) + self._rows(("pub", pub), width=2 * self._len)
        return self._tensor_call("derive_batch_tensors", "eb200_ecdh_derive_batch_dev", specs,
                                 lambda n: [self._c["id"], n, priv, pub], [(self._len,)])

    def x_mul_batch_tensors(self, k, px):
        """curve25519 x_mul_batch on CUDA tensors (eb200_x25519_mul_batch_dev): k, px (n, 32) big-endian.  Returns (x (n,
        32), status)."""
        if self.name != "curve25519":
            raise EllipticError("x_mul_batch_tensors: curve25519 only")
        return self._tensor_call("x_mul_batch_tensors", "eb200_x25519_mul_batch_dev",
                                 self._rows(("k", k), ("px", px)), lambda n: [n, k, px], [(32,)], ws=False)


class EC(_KeyObjects, _TensorForms):
    def __init__(self, curve="secp256k1", device=0):
        if curve not in _CURVES:
            raise EllipticError("Unknown curve " + str(curve))   # ec/index.js:19-20
        self.name = curve
        self._c = _CURVES[curve]
        self.n = self._c["n"]
        self._len = self._c["len"]
        self._device = device

    # ---- reference-compatible scalar preparation (host side, cheap) -------------
    def _truncate_to_n(self, msg, msg_bit_length=None):
        """EC._truncateToN (ec/index.js:81-108), including its single conditional `- n`."""
        if isinstance(msg, int):
            v = msg
            byte_length = (v.bit_length() + 7) // 8
        elif isinstance(msg, str):
            byte_length = (len(msg) + 1) >> 1
            v = _parse_hex(msg)
        else:
            b = _to_array(msg)
            byte_length = len(b)
            v = int.from_bytes(b, "big")
        bit_length = byte_length * 8 if msg_bit_length is None else msg_bit_length
        delta = bit_length - self.n.bit_length()
        if delta > 0:
            v >>= delta
        if v >= self.n:
            v -= self.n
        return v

    def _public(self, key, enc=None):
        """KeyPair._importPublic (ec/key.js:84-99) -> (fmt, bytes)."""
        ln = self._len
        if isinstance(key, dict) and (key.get("x") or key.get("y")):
            if not (key.get("x") and key.get("y")):
                raise EllipticError("Need both x and y coordinate")
            x, y = _bn(key["x"]), _bn(key["y"])
            if x < 0 or y < 0:
                raise EllipticError("red works only with positives")
            # toRed reduces oversize coordinates mod p (short.js:258-268); the engine
            # does that for anything that fits the wire width, wider values here.
            if x >> (8 * ln) or y >> (8 * ln):
                x %= self._c["p"]
                y %= self._c["p"]
            return nat.PUB_XY, _pack([x, y], ln).tobytes()
        b = _to_array(key, enc)
        if len(b) and b[0] in (4, 6, 7) and len(b) - 1 == 2 * ln:
            if (b[0] == 6 and b[-1] % 2 != 0) or (b[0] == 7 and b[-1] % 2 != 1):
                raise EllipticError("Assertion failed")            # base.js:278-281
            return nat.PUB_XY, b[1:]
        if len(b) and b[0] in (2, 3) and len(b) - 1 == ln:
            return nat.PUB_SEC1_33, b
        raise EllipticError("Unknown point format")                # base.js:291

    def _pub_bytes(self, pub_fmt):
        """Bytes per public key in `pub_fmt` (include/elliptic_b200.h: EB200_PUB_*)."""
        return {nat.PUB_XY: 2 * self._len, nat.PUB_SEC1_65: 1 + 2 * self._len, nat.PUB_SEC1_33: 1 + self._len}[pub_fmt]

    # ---- batch entry points ---------------------------------------------------
    def verify_batch_packed(self, e, r, s, pub, pub_fmt=nat.PUB_XY):
        """Packed form: e, r, s are (n, len) uint8 arrays (big-endian), pub is
        (n, 2*len).  Returns the per-item status bytes (see _native.ST_*)."""
        lib = nat.init(self._device)
        e, r, s, pub = (np.ascontiguousarray(a, dtype=np.uint8) for a in (e, r, s, pub))
        n = e.shape[0]
        if not (e.shape == (n, self._len) and r.shape == e.shape and s.shape == e.shape):      # raw pointers go down
            raise ValueError("e, r, s must be (n, %d) uint8 arrays" % self._len)
        pb = self._pub_bytes(pub_fmt)
        if pub.shape != (n, pb):
            raise ValueError("pub must be (n, %d) for this format, got %r" % (pb, pub.shape))
        status = np.empty(n, dtype=np.uint8)
        nat.call(lib.eb200_ecdsa_verify_batch, self._c["id"], n, e, r, s, pub, pub_fmt, status)
        return status

    def verify_batch_der_packed(self, e, ders, pub, pub_fmt=nat.PUB_XY):
        """e: (n, len) uint8 truncated hashes; ders: list of DER byte strings (parsed on the GPU exactly as
        Signature._importDER, ec/signature.js:73-134); pub: (n, k) uint8 in `pub_fmt`.  Returns statuses."""
        lib = nat.init(self._device)
        n = len(ders)
        blob, off = _blob([bytes(d) for d in ders])
        e = np.ascontiguousarray(e, np.uint8); pub = np.ascontiguousarray(pub, np.uint8)
        pb = self._pub_bytes(pub_fmt)
        if e.shape != (n, self._len) or pub.shape != (n, pb):
            raise EllipticError("verify_batch_der_packed: e must be (n, %d) and pub (n, %d)" % (self._len, pb))
        status = np.zeros(n, np.uint8)
        nat.call(lib.eb200_ecdsa_verify_batch_der, self._c["id"], n, e, blob, off, pub, pub_fmt, status)
        return status

    def verify_batch(self, msgs, sigs, keys, enc=None, msg_bit_length=None):
        """EC#verifyBatch: lists of the reference's own argument forms.
        Returns a uint8 array of statuses; items whose *parsing* throws in the
        reference raise here, like a loop over `verify` would at that item."""
        n = len(msgs)
        groups = {}          # pub format -> (item indices, key bytes)
        early = {}

        def items():         # parsed one item at a time, as _pack encodes them: an e that does not fit raises at its item
            for i in range(n):
                ev = self._truncate_to_n(msgs[i], msg_bit_length)
                fmt, pb = self._public(keys[i], enc)
                rv, sv = _signature(sigs[i], "hex")
                if rv < 1 or rv >= self.n or sv < 1 or sv >= self.n:
                    early[i] = nat.ST_FALSE       # ec/index.js:199-202 (after the key import, which may throw)
                    rv = sv = 0
                g = groups.setdefault(fmt, ([], []))
                g[0].append(i)
                g[1].append(pb)
                yield from (ev, rv, sv)
        ers = _pack(items(), self._len).reshape(n, 3, self._len)
        st = np.zeros(n, np.uint8)
        for fmt, (idx, pbs) in groups.items():
            idx = np.asarray(idx)
            pub = np.frombuffer(b"".join(pbs), np.uint8).reshape(len(pbs), -1)
            st[idx] = self.verify_batch_packed(ers[idx, 0], ers[idx, 1], ers[idx, 2], pub, fmt)
        for i, v in early.items():
            if st[i] in (nat.ST_TRUE, nat.ST_FALSE, nat.ST_NEEDS_HOST):
                st[i] = v
        return st

    # ---- signing ---------------------------------------------------------------------------------------------
    def sign_batch(self, msgs, privs, canonical=False, msg_bit_length=None, pers=None, pers_enc=None, k=None):
        """Batch of EC.prototype.sign (ec/index.js:110-186) with the curve's default hash.
        pers / pers_enc: the `pers` / `persEnc` options (one personalisation string for the batch; persEnc defaults
        to 'utf8' as in ec/index.js:150).  k: the `k` option as a callable k(item, iter) -> nonce (int / hex / bytes);
        without it the nonces are RFC 6979 (HMAC-DRBG on the GPU).  Returns (r list, s list, recoveryParam array)."""
        if self.name not in _XY:
            raise EllipticError("sign_batch: not available on " + self.name)
        lib = nat.init(self._device)
        n, ln = len(msgs), self._len
        es, ds = [], []
        for i in range(n):
            ev = self._truncate_to_n(msgs[i], msg_bit_length)                  # includes the single `- n` (ec/index.js:105-106)
            if ev >> (8 * ln):
                raise EllipticError("byte array longer than desired length")   # msg.toArray('be', bytes), dist bn.js toArrayLike
            es.append(ev)
            ds.append(_bn(privs[i]) % self.n)                                  # _importPrivate
        e, d = _pack(es, ln), _pack(ds, ln)
        r = np.zeros((n, ln), np.uint8); s = np.zeros((n, ln), np.uint8)
        rec = np.zeros(n, np.uint8); st = np.zeros(n, np.uint8)
        flags = 1 if canonical else 0
        if k is not None:
            def nonce(i, it):
                kv = _bn(k(int(i), it))
                # _truncateToN(k, true) on a BN wider than the field: shift by its own byte length (ec/index.js:96-103)
                delta = ((kv.bit_length() + 7) // 8) * 8 - self.n.bit_length()
                return kv >> delta if kv.bit_length() > 8 * ln and delta > 0 else kv
            todo = np.arange(n)
            for it in range(1 << 16):
                kb = _pack((nonce(i, it) for i in todo), ln)     # k(i, it) is encoded before the next item's is asked for
                rr = np.zeros((len(todo), ln), np.uint8); ss = np.zeros((len(todo), ln), np.uint8)
                cc = np.zeros(len(todo), np.uint8); tt = np.zeros(len(todo), np.uint8)
                nat.call(lib.eb200_ecdsa_sign_batch_k, self._c["id"], len(todo), e[todo], d[todo], kb, flags,
                         rr, ss, cc, tt)
                ok = tt == nat.ST_TRUE
                r[todo[ok]], s[todo[ok]], rec[todo[ok]], st[todo[ok]] = rr[ok], ss[ok], cc[ok], tt[ok]
                if not bool(((tt == nat.ST_TRUE) | (tt == nat.ST_RETRY)).all()):
                    raise nat.NativeError("sign_batch: unexpected status")
                todo = todo[~ok]
                if not len(todo):
                    break
        elif pers is not None:
            pb, pb_len = _pers(pers, pers_enc)
            nat.call(lib.eb200_ecdsa_sign_batch_pers, self._c["id"], n, e, d, pb, pb_len, flags, r, s, rec, st)
        else:
            nat.call(lib.eb200_ecdsa_sign_batch, self._c["id"], n, e, d, flags, r, s, rec, st)
        if not bool((st == nat.ST_TRUE).all()):
            bad = int(np.flatnonzero(st != nat.ST_TRUE)[0])
            raise nat.NativeError("sign_batch: item %d returned status %d" % (bad, int(st[bad])))
        return _unpack(r, ln), _unpack(s, ln), rec

    def gen_key_pair_batch(self, entropies, entropy_enc=None, pers=None, pers_enc=None):
        """Batch of EC.prototype.genKeyPair({entropy, entropyEnc, pers, persEnc}) (ec/index.js:55-79): every item's key
        comes from its own HMAC-DRBG(hash, entropy, nonce = n, pers).  All entropies must have the same byte length
        (>= 24, the reference's 'Not enough entropy' assertion).  Returns (private keys, public points (x, y))."""
        if self.name not in _XY:
            raise EllipticError("gen_key_pair_batch: not available on " + self.name)
        lib = nat.init(self._device)
        ents = [bytes(_to_array(x, entropy_enc or "utf8")) for x in entropies]
        n, ln = len(ents), self._len
        if not n:
            return [], []
        ne = len(ents[0])
        if any(len(x) < 24 for x in ents):
            raise EllipticError("Not enough entropy. Minimum is: 192 bits")     # hmac-drbg ctor, dist:8708-8710
        if any(len(x) != ne for x in ents):
            raise EllipticError("gen_key_pair_batch: entropies of one batch must have the same length")
        pb, pb_len = _pers(pers, pers_enc)
        priv = np.zeros((n, ln), np.uint8); pub = np.zeros((n, 2 * ln), np.uint8); st = np.zeros(n, np.uint8)
        nat.call(lib.eb200_ec_keygen_batch, self._c["id"], n, _blob(ents)[0], ne, pb, pb_len, priv, pub, st)
        if not bool((st == nat.ST_TRUE).all()):
            raise nat.NativeError("gen_key_pair_batch: unexpected status")
        return _unpack(priv, ln), _unpack(pub, ln)

    def sign(self, msg, priv, canonical=False, pers=None, pers_enc=None, k=None):
        """EC.prototype.sign (ec/index.js:110-186); k: the reference's options.k(iter)."""
        r, s, rec = self.sign_batch([msg], [priv], canonical, None, pers, pers_enc, (lambda i, it: k(it)) if k else None)
        return {"r": r[0], "s": s[0], "recoveryParam": int(rec[0])}

    # ---- public-key recovery -----------------------------------------------------------------------------
    def _recover_args(self, es, rss):
        """e mod n, r, s mod n as (n, len) arrays, as the recover and recovery-parameter entry points take them."""
        ln = self._len
        return _pack([e % self.n for e in es], ln), _pack([r for r, _ in rss], ln), _pack([s % self.n for _, s in rss], ln)

    def recover_pub_key_batch(self, msgs, sigs, js, enc=None):
        """Batch of EC.prototype.recoverPubKey (ec/index.js:231-259).  msgs as `new BN(msg)` takes them
        (int / hex / bytes, NOT truncated), sigs as Signature takes them, js the recovery params.
        Returns (points, statuses): points[i] = (x, y), None for the point at infinity / a throw."""
        if self.name not in _SHORT:
            raise EllipticError("recover_pub_key_batch: short curves only")
        lib = nat.init(self._device)
        n, ln = len(msgs), self._len
        es, rss, rid = [], [], []
        for i in range(n):
            if (3 & js[i]) != js[i]:
                raise EllipticError("The recovery param is more than two bits")      # ec/index.js:232
            rv, sv = _signature(sigs[i], enc)
            es.append(_msg_int(msgs[i]))
            if rv >> (8 * ln):
                raise NeedsReferencePath("r does not fit the curve's field width")
            rss.append((rv, sv))
            rid.append(js[i])
        out = np.zeros((n, 2 * ln), np.uint8)
        st = np.zeros(n, np.uint8)
        nat.call(lib.eb200_ecdsa_recover_batch, self._c["id"], n, *self._recover_args(es, rss), np.array(rid, np.uint8), out, st)
        return _unpack(out, ln, st), st

    def recover_pub_key(self, msg, signature, j, enc=None):
        pts, st = self.recover_pub_key_batch([msg], [signature], [j], enc)
        return _answer(pts[0], st[0], (nat.ST_TRUE, nat.ST_INFINITY))

    def get_key_recovery_param_batch(self, msgs, sigs, qs, enc=None):
        """Batch of EC.prototype.getKeyRecoveryParam (ec/index.js:261-278): per item the first j in 0..3 whose
        recoverPubKey(msg, sig, j) equals Q.  msgs and sigs as recover_pub_key_batch takes them, qs the public points
        as (x, y) pairs or {x, y} dicts (reduced mod p like curve.point).  A signature that carries a recoveryParam is
        answered with it without any computation, as the reference does (ec/index.js:263-264).
        Returns (js, statuses): js[i] is the parameter, or None where the reference throws
        'Unable to find valid recovery factor' (status ST_THROW_NO_RECOVERY)."""
        if self.name not in _SHORT:
            raise EllipticError("get_key_recovery_param_batch: short curves only")
        js, st, todo, rss = self._recovery_param_split(msgs, sigs, qs, enc)
        if not todo:
            return js, st
        lib = nat.init(self._device)
        m = len(todo)
        ers = self._recover_args([_msg_int(msgs[i]) for i in todo], rss)
        q = self._points([qs[i] for i in todo])
        rid = np.zeros(m, np.uint8); sub = np.zeros(m, np.uint8)
        nat.call(lib.eb200_ecdsa_recovery_param_batch, self._c["id"], m, *ers, q, rid, sub)
        for k, i in enumerate(todo):
            st[i] = sub[k]
            js[i] = int(rid[k]) if sub[k] == nat.ST_TRUE else None
        return js, st

    def _recovery_param_split(self, msgs, sigs, qs, enc):
        """getKeyRecoveryParam's host side before the engine: (js, statuses) with the items whose signature carries a
        recoveryParam answered (ec/index.js:263-264), and the indices and (r, s) of the others.  qs: the points, or None
        when a key set supplies them."""
        n, ln = len(msgs), self._len
        js = [None] * n
        st = np.zeros(n, np.uint8)
        todo = []
        rss = []
        for i in range(n):
            rv, sv = _signature(sigs[i], enc)                  # new Signature(signature, enc) may throw first
            rp = sigs[i].get("recoveryParam") if isinstance(sigs[i], dict) else \
                getattr(sigs[i], "recoveryParam", getattr(sigs[i], "recovery_param", None))
            if rp is not None:
                js[i], st[i] = rp, nat.ST_TRUE
                continue
            if qs is not None and qs[i] is None:
                raise NeedsReferencePath("Q is the point at infinity")
            if rv >> (8 * ln):
                raise NeedsReferencePath("r does not fit the curve's field width")
            todo.append(i)
            rss.append((rv, sv))
        return js, st, todo, rss

    def get_key_recovery_param(self, e, signature, Q, enc=None):
        """EC.prototype.getKeyRecoveryParam (ec/index.js:261-278): the parameter, or raises like the reference."""
        js, st = self.get_key_recovery_param_batch([e], [signature], [Q], enc)
        return _answer(js[0], st[0], (nat.ST_TRUE,))

    # ---- curve.point(...).mul / mulAdd batches (short.js:422-441) ---------------------------------------------
    def _scalars(self, ks):
        # k P == (k mod order) P for every on-curve P: the group has order n on the short curves, 8n on ed25519 (cofactor 8)
        order = 8 * self.n if self.name == "ed25519" else self.n
        vals = []
        for k in ks:
            k = _bn(k)
            if k < 0:
                raise EllipticError("negative scalars are not supported by the batch path")
            vals.append(k % order if k >> (8 * self._len) else k)
        return _pack(vals, self._len)

    def _points(self, pts):
        """curve.point(x, y) (short.js:251-271): coordinates reduced mod p, not validated."""
        return _pack_points(pts, self._c["p"], self._len)

    def _mul_common(self, k1, k2, pts):
        if self.name == "curve25519":
            raise EllipticError("Not supported on Montgomery curve")      # mont.js: mulAdd / jumlAdd throw; mul: x_mul_batch
        if self.name not in _XY:
            raise EllipticError("mul/mulAdd batches: not available on " + self.name)
        lib = nat.init(self._device)
        n, ln = len(k2), self._len
        out = np.zeros((n, 2 * ln), np.uint8)
        st = np.zeros(n, np.uint8)
        if k1 is None:
            nat.call(lib.eb200_scalar_mul_batch, self._c["id"], n, k2, pts, out, st)
        else:
            nat.call(lib.eb200_mul_add_batch, self._c["id"], n, k1, k2, pts, out, st)
        return _unpack(out, ln, st, needs_host=True)      # (only the Edwards preset reports it; the short curves replay)

    def x_mul_batch(self, xs, ks):
        """curve25519: [curve.point(x).mul(k).getX()] (mont.js:130-153, 173-178) -- x-only points, no validation."""
        if self.name != "curve25519":
            raise EllipticError("x_mul_batch: curve25519 only")
        lib = nat.init(self._device)
        n = len(ks)
        kvs, xvs = [], []
        for i in range(n):
            kv, xv = _bn(ks[i]), _bn(xs[i])
            if kv >> 256:
                raise NeedsReferencePath("scalar wider than 256 bits")
            kvs.append(kv)
            xvs.append(xv % self._c["p"] if xv >> 256 else xv)
        out = np.zeros((n, 32), np.uint8); st = np.zeros(n, np.uint8)
        nat.call(lib.eb200_x25519_mul_batch, n, _pack(kvs, 32), _pack(xvs, 32), out, st)
        return _unpack(out, 32)

    def g_mul_batch(self, ks):
        """[G.mul(k) for k in ks] (short.js:422-427, the keygen product ec/key.js:55-60): (x, y) or None = infinity."""
        return self._mul_common(None, self._scalars(ks), None)

    def mul_batch(self, points, ks):
        """[curve.point(x, y).mul(k)] (short.js:422-432): (x, y) or None = infinity."""
        return self._mul_common(None, self._scalars(ks), self._points(points))

    def mul_add_batch(self, k1s, p2s, k2s):
        """[G.mulAdd(k1, P2, k2)] (short.js:434-441): (x, y) or None = infinity."""
        return self._mul_common(self._scalars(k1s), self._scalars(k2s), self._points(p2s))

    # ---- ECDH --------------------------------------------------------------------------------------------
    def derive_batch(self, privs, pubs):
        """Batch of `ec.keyFromPrivate(priv).derive(ec.keyFromPublic(pub).getPublic())`
        (ec/key.js:76-82, 102-107) on curve25519.  privs: ints / hex / bytes; pubs: the peer's x as
        int / hex / big-endian bytes (mont.js:46-48).  Returns (list of int-or-None, statuses)."""
        if self.name != "curve25519":
            return self._derive_short(privs, pubs)
        lib = nat.init(self._device)
        n = len(privs)
        kvs, xvs = [], []
        for i in range(n):
            kvs.append(_bn(privs[i]) % self.n)                      # _importPrivate: umod n
            xv = _bn(pubs[i])
            xvs.append(xv % self._c["p"] if xv >> 256 else xv)
        out = np.zeros((n, 32), np.uint8)
        st = np.zeros(n, np.uint8)
        nat.call(lib.eb200_x25519_derive_batch, n, _pack(kvs, 32), _pack(xvs, 32), out, st)
        return _unpack(out, 32, st), st

    def derive_batch_packed(self, priv, pubx, out=None, status=None):
        """Packed curve25519 ECDH: priv, pubx are (n, 32) uint8 arrays (big-endian; priv already reduced mod n as
        _importPrivate does, ec/key.js:76-82).  Returns ((n, 32) shared x big-endian, statuses); `out` / `status`
        let the caller supply (and reuse) the result buffers, e.g. pinned ones."""
        if self.name != "curve25519":
            raise EllipticError("derive_batch_packed: curve25519 only (short curves: derive_batch)")
        lib = nat.init(self._device)
        priv = np.ascontiguousarray(priv, dtype=np.uint8)
        pubx = np.ascontiguousarray(pubx, dtype=np.uint8)
        n = priv.shape[0]
        if priv.shape != (n, 32) or pubx.shape != (n, 32):
            raise EllipticError("derive_batch_packed: (n, 32) arrays expected")
        out = np.empty((n, 32), np.uint8) if out is None else out
        st = np.empty(n, np.uint8) if status is None else status
        if out.shape != (n, 32) or out.dtype != np.uint8 or not out.flags.c_contiguous or st.shape != (n,) or st.dtype != np.uint8:
            raise EllipticError("derive_batch_packed: out must be a contiguous (n, 32) uint8 array, status (n,) uint8")
        nat.call(lib.eb200_x25519_derive_batch, n, priv, pubx, out, st)
        return out, st

    def _derive_short(self, privs, pubs):
        """Short curves: pubs are the peer's points as {x, y} / (x, y) (keyFromPublic(...).getPublic())."""
        lib = nat.init(self._device)
        n, ln = len(privs), self._len
        k = self._scalars([_bn(p) % self.n for p in privs])
        pts = self._points(pubs)
        out = np.zeros((n, ln), np.uint8)
        st = np.zeros(n, np.uint8)
        nat.call(lib.eb200_ecdh_derive_batch, self._c["id"], n, k, pts, out, st)
        return _unpack(out, ln, st), st

    def derive(self, priv, pub):
        """KeyPair.prototype.derive: the shared x as an int, or raises like the reference."""
        vals, st = self.derive_batch([priv], [pub])
        return _answer(vals[0], st[0], (nat.ST_TRUE,))

    def verify(self, msg, signature, key, enc=None, options=None):
        """EC.prototype.verify (ec/index.js:188-229): bool, or raises."""
        mbl = (options or {}).get("msgBitLength")
        st = int(self.verify_batch([msg], [signature], [key], enc, mbl)[0])
        if st == nat.ST_NEEDS_HOST:
            raise NeedsReferencePath("public key is not on the curve; the reference does not validate it")
        return _answer(st == nat.ST_TRUE, st, (nat.ST_TRUE, nat.ST_FALSE))


class _NativeSets:
    """The lifecycle of key-set handles (eb200_keyset) shared by KeySet and eddsa.EdKeySet: `_sets` holds the live
    handles; close() destroys them (the object is then closed), the object is a context manager and closes on
    collection."""
    _sets = ()

    def close(self):
        lib = nat.load()
        for h in self._sets:
            nat.check(lib.eb200_keyset_destroy(h))
        self._sets = []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class KeySet(_NativeSets):
    """Public keys imported once and kept on the GPU with their precomputed tables (eb200_keyset_create); item i of a
    verify call is checked against key key_idx[i], with the status EC.verify_batch gives for that key.  Keys come in the
    reference's argument forms through EC._public; a set that mixes {x, y} / uncompressed keys with compressed ones holds
    one native set per wire format, so no key is converted (or validated) on the host and every throw stays the engine's.
    `status`: per key, a throw status, ST_TRUE (on the curve) or ST_FALSE (imported, off the curve).  close() frees the
    device memory; the object is a context manager."""

    def __init__(self, ec, keys, enc=None, table_bits=0):
        if ec.name not in _SHORT:
            raise EllipticError("key_set: short curves only")
        self._ec = ec
        lib = nat.init(ec._device)
        groups = {}                                   # pub format -> (key indices, key bytes)
        for j, key in enumerate(keys):
            fmt, pb = ec._public(key, enc)
            g = groups.setdefault(fmt, ([], []))
            g[0].append(j)
            g[1].append(pb)
        m = len(keys)
        self.status = np.zeros(m, np.uint8)
        self._where = np.zeros((m, 2), np.uint32)     # key -> (sub-set, index in it)
        self._sets = []
        self.table_bits, self.device_bytes = [], 0
        try:
            for fmt, (idx, pbs) in groups.items():
                pub = np.frombuffer(b"".join(pbs), np.uint8).reshape(len(pbs), -1).copy()
                st = np.zeros(len(idx), np.uint8)
                h = ctypes.c_void_p()
                nat.check(lib.eb200_keyset_create(ec._c["id"], len(idx), pub.ctypes.data, fmt, table_bits, st.ctypes.data,
                                                  ctypes.byref(h)))
                self._sets.append(h)
                self.status[idx] = st
                self._where[idx, 0] = len(self._sets) - 1
                self._where[idx, 1] = np.arange(len(idx))
                w, db = ctypes.c_uint32(), ctypes.c_size_t()
                nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), ctypes.byref(db)))
                self.table_bits.append(w.value)
                self.device_bytes += db.value
        except Exception:
            self.close()
            raise
        self.table_bits = self.table_bits[0] if len(set(self.table_bits)) == 1 else tuple(self.table_bits)

    def _keyed(self, fn, ins, key_idx, outs):
        """fn(set, n, *ins, key_idx, *outs) for the items of each native set: ins and outs are arrays with one row per
        item (None passes NULL); a set that holds one native set per wire format gets its items split by `_where`."""
        key_idx = np.asarray(key_idx)
        n = len(key_idx)
        if n and (key_idx.min() < 0 or key_idx.max() >= len(self.status)):
            raise ValueError("key_idx out of range")
        if not self._sets and n:
            raise EllipticError("key set is closed")
        if len(self._sets) == 1:
            nat.call(fn, self._sets[0], n, *ins, np.ascontiguousarray(key_idx, np.uint32), *outs)
            return
        where = self._where[key_idx]
        for k, h in enumerate(self._sets):
            sel = np.nonzero(where[:, 0] == k)[0]
            if len(sel):
                part = [np.empty((len(sel),) + o.shape[1:], o.dtype) for o in outs]
                nat.call(fn, h, len(sel), *(None if a is None else np.ascontiguousarray(a[sel]) for a in ins),
                         np.ascontiguousarray(where[sel, 1]), *part)
                for o, p in zip(outs, part):
                    o[sel] = p

    def _packed_scalars(self, name, ks, n):
        ks = [np.ascontiguousarray(a, dtype=np.uint8) for a in ks]
        if any(a.shape != (n, self._ec._len) for a in ks):
            raise ValueError("%s: scalars must be (n, %d) uint8 arrays, n = len(key_idx)" % (name, self._ec._len))
        return ks

    def verify_batch_packed(self, e, r, s, key_idx):
        """e, r, s: (n, len) uint8 arrays (big-endian); key_idx: n indices into the set.  Returns the status bytes."""
        lib = nat.load()
        ln = self._ec._len
        e, r, s = (np.ascontiguousarray(a, dtype=np.uint8) for a in (e, r, s))
        key_idx = np.asarray(key_idx)
        n = e.shape[0]
        if not (e.shape == (n, ln) and r.shape == e.shape and s.shape == e.shape and key_idx.shape == (n,)):
            raise ValueError("e, r, s must be (n, %d) uint8 arrays and key_idx (n,)" % ln)
        status = np.empty(n, np.uint8)
        self._keyed(lib.eb200_ecdsa_verify_batch_keyed, (e, r, s), key_idx, (status,))
        return status

    def verify_batch_der_packed(self, e, ders, key_idx):
        """e: (n, len) uint8 truncated hashes; ders: n DER byte strings, parsed on the GPU exactly as
        EC.verify_batch_der_packed parses them; key_idx: n indices into the set.  Returns the status bytes
        EC.verify_batch_der_packed gives with pub[i] = key key_idx[i] (eb200_ecdsa_verify_batch_keyed_der)."""
        lib = nat.load()
        ln = self._ec._len
        ders = [bytes(d) for d in ders]
        e = np.ascontiguousarray(e, dtype=np.uint8)
        key_idx = np.asarray(key_idx)
        n = len(ders)
        if not (e.shape == (n, ln) and key_idx.shape == (n,)):
            raise ValueError("e must be (n, %d) uint8, ders n byte strings and key_idx (n,)" % ln)
        if n and (key_idx.min() < 0 or key_idx.max() >= len(self.status)):
            raise ValueError("key_idx out of range")
        if not self._sets and n:
            raise EllipticError("key set is closed")
        status = np.empty(n, np.uint8)
        # one native set per wire format: each gets its own items' DER blob and offsets
        where = self._where[key_idx] if len(self._sets) > 1 else None
        for k, h in enumerate(self._sets):
            sel = np.arange(n) if where is None else np.nonzero(where[:, 0] == k)[0]
            if not len(sel):
                continue
            blob, off = _blob([ders[i] for i in sel])
            idx = key_idx if where is None else where[sel, 1]
            part = np.empty(len(sel), np.uint8)
            nat.call(lib.eb200_ecdsa_verify_batch_keyed_der, h, len(sel), np.ascontiguousarray(e[sel]), blob, off,
                     np.ascontiguousarray(idx, np.uint32), part)
            status[sel] = part
        return status

    def mul_batch_packed(self, k, key_idx):
        """pub.mul(k) for key key_idx[i] of the set (eb200_scalar_mul_batch_keyed): k is an (n, len) uint8 array, any
        value below 2^(8 len).  Returns ((n, 2 len) x || y big-endian, statuses) as EC.mul_batch's call leaves them."""
        key_idx = np.asarray(key_idx)
        n = len(key_idx)
        (k,) = self._packed_scalars("mul_batch_packed", (k,), n)
        out, st = np.empty((n, 2 * self._ec._len), np.uint8), np.empty(n, np.uint8)
        self._keyed(nat.load().eb200_scalar_mul_batch_keyed, (k,), key_idx, (out, st))
        return out, st

    def mul_add_batch_packed(self, k1, k2, key_idx):
        """G.mulAdd(k1, pub, k2) for key key_idx[i] (eb200_mul_add_batch_keyed); as mul_batch_packed."""
        key_idx = np.asarray(key_idx)
        n = len(key_idx)
        k1, k2 = self._packed_scalars("mul_add_batch_packed", (k1, k2), n)
        out, st = np.empty((n, 2 * self._ec._len), np.uint8), np.empty(n, np.uint8)
        self._keyed(nat.load().eb200_mul_add_batch_keyed, (k1, k2), key_idx, (out, st))
        return out, st

    def derive_batch_packed(self, priv, key_idx):
        """keyPair.derive(pub) for key key_idx[i] (eb200_ecdh_derive_batch_keyed): priv is an (n, len) uint8 array.
        Returns ((n, len) shared x big-endian, statuses)."""
        key_idx = np.asarray(key_idx)
        n = len(key_idx)
        (priv,) = self._packed_scalars("derive_batch_packed", (priv,), n)
        out, st = np.empty((n, self._ec._len), np.uint8), np.empty(n, np.uint8)
        self._keyed(nat.load().eb200_ecdh_derive_batch_keyed, (priv,), key_idx, (out, st))
        return out, st

    def recovery_param_batch_packed(self, e, r, s, key_idx):
        """getKeyRecoveryParam(e, sig, pub) for pub = key key_idx[i] (eb200_ecdsa_recovery_param_batch_keyed): e, r, s are
        (n, len) uint8 arrays as EC.get_key_recovery_param_batch's call takes them (e, s reduced mod n; r any value below
        2^(8 len)).  Returns (recid, statuses): recid[i] is the parameter where the status is ST_TRUE, else 0."""
        key_idx = np.asarray(key_idx)
        n = len(key_idx)
        e, r, s = self._packed_scalars("recovery_param_batch_packed", (e, r, s), n)
        recid, st = np.empty(n, np.uint8), np.empty(n, np.uint8)
        self._keyed(nat.load().eb200_ecdsa_recovery_param_batch_keyed, (e, r, s), key_idx, (recid, st))
        return recid, st

    def _check_imported(self, key_idx):
        """Raise the reference's error for the first item whose key threw at import, as keyFromPublic would."""
        key_idx = np.asarray(key_idx, np.int64)
        if len(key_idx) and (key_idx.min() < 0 or key_idx.max() >= len(self.status)):
            raise ValueError("key_idx out of range")
        ks = self.status[key_idx]
        bad = np.flatnonzero(ks > nat.ST_TRUE)
        if len(bad):
            raise EllipticError(_THROW_MSG.get(int(ks[bad[0]]), "status %d" % int(ks[bad[0]])))

    def mul_batch(self, key_idx, ks):
        """[pub.mul(k)] for pub = key key_idx[i]: what EC.mul_batch returns for those points, (x, y) or None = infinity."""
        self._check_imported(key_idx)
        out, st = self.mul_batch_packed(self._ec._scalars(ks), key_idx)
        return _unpack(out, self._ec._len, st)

    def mul_add_batch(self, k1s, key_idx, k2s):
        """[G.mulAdd(k1, pub, k2)] for pub = key key_idx[i]: what EC.mul_add_batch returns."""
        self._check_imported(key_idx)
        out, st = self.mul_add_batch_packed(self._ec._scalars(k1s), self._ec._scalars(k2s), key_idx)
        return _unpack(out, self._ec._len, st)

    def derive_batch(self, privs, key_idx):
        """[keyPair(priv).derive(pub)] for pub = key key_idx[i]: what EC.derive_batch returns, (values, statuses)."""
        self._check_imported(key_idx)
        ec = self._ec
        out, st = self.derive_batch_packed(ec._scalars([_bn(p) % ec.n for p in privs]), key_idx)
        return _unpack(out, ec._len, st), st

    def get_key_recovery_param_batch(self, msgs, sigs, key_idx, enc=None):
        """[ec.getKeyRecoveryParam(msg, sig, pub)] for pub = key key_idx[i]: what EC.get_key_recovery_param_batch returns
        for those keys' points, (js, statuses), js[i] None where the reference throws 'Unable to find valid recovery
        factor'.  A signature that carries a recoveryParam is answered with it; a key whose import threw raises its error."""
        self._check_imported(key_idx)
        ec = self._ec
        js, st, todo, rss = ec._recovery_param_split(msgs, sigs, None, enc)
        if not todo:
            return js, st
        recid, sub = self.recovery_param_batch_packed(*ec._recover_args([_msg_int(msgs[i]) for i in todo], rss),
                                                      np.asarray(key_idx)[todo])
        for k, i in enumerate(todo):
            st[i] = sub[k]
            js[i] = int(recid[k]) if sub[k] == nat.ST_TRUE else None
        return js, st

    def verify_batch(self, msgs, sigs, key_idx, enc=None, msg_bit_length=None):
        """Lists of the reference's message and signature forms, as EC.verify_batch takes them; `enc` is accepted for
        symmetry (signatures are read as the reference reads them, 'hex')."""
        ec, n = self._ec, len(msgs)
        early = {}

        def items():
            for i in range(n):
                ev = ec._truncate_to_n(msgs[i], msg_bit_length)
                rv, sv = _signature(sigs[i], "hex")
                if rv < 1 or rv >= ec.n or sv < 1 or sv >= ec.n:
                    early[i] = nat.ST_FALSE
                    rv = sv = 0
                yield from (ev, rv, sv)
        ers = _pack(items(), ec._len).reshape(n, 3, ec._len)
        st = self.verify_batch_packed(ers[:, 0], ers[:, 1], ers[:, 2], key_idx)
        for i, v in early.items():
            if st[i] in (nat.ST_TRUE, nat.ST_FALSE, nat.ST_NEEDS_HOST):
                st[i] = v
        return st

    # ---- tensor forms: the keyed device-buffer calls on CUDA tensors (conventions: _tensors) -------------------------
    def _where_on(self, dev):
        """_where on `dev` as (native set of each key, its index there, the native sets' sizes), built once per device."""
        cache = self.__dict__.setdefault("_where_dev", {})
        if dev not in cache:
            import torch
            w = torch.from_numpy(self._where.astype(np.int64)).to(dev)
            cache[dev] = (w[:, 0].contiguous(), w[:, 1].contiguous(),
                          np.bincount(self._where[:, 0], minlength=len(self._sets)).tolist())
        return cache[dev]

    def _keyed_tensors(self, name, fn, specs, ins, key_idx, outs):
        from . import _tensors as T
        n, dev = T.check(name, specs + [("key_idx", key_idx, T.IDX, 0)], self._sets)
        return T.keyed(name, self._sets, len(self.status), self._where_on if len(self._sets) > 1 else None, fn, n, dev,
                       ins, key_idx, [(n,) + o for o in outs])

    def _rows(self, *named, width=None):
        from . import _tensors as T
        return [(a, t, T.ROWS, width or self._ec._len) for a, t in named]

    def verify_batch_tensors(self, e, r, s, key_idx):
        """verify_batch_packed on CUDA tensors (eb200_ecdsa_verify_batch_keyed_dev).  Returns the (n,) statuses."""
        (st,) = self._keyed_tensors("verify_batch_tensors", "eb200_ecdsa_verify_batch_keyed_dev",
                                    self._rows(("e", e), ("r", r), ("s", s)), [e, r, s], key_idx, [])
        return st

    def verify_batch_der_tensors(self, e, sigs, sig_off, key_idx):
        """verify_batch_der_packed on CUDA tensors (eb200_ecdsa_verify_batch_keyed_der_dev): e (n, len), the DER encodings
        back to back in sigs (1-D uint8) with (n + 1,) int64 offsets.  Returns the (n,) statuses; a range that decreases
        or ends past sigs gets ST_BAD_ITEM."""
        from . import _tensors as T
        specs = self._rows(("e", e)) + [("sigs", sigs, T.BYTES, 0), ("sig_off", sig_off, T.OFF, 0)]
        (st,) = self._keyed_tensors("verify_batch_der_tensors", "eb200_ecdsa_verify_batch_keyed_der_dev", specs,
                                    [e, sigs, sigs.numel(), sig_off], key_idx, [])
        return st

    def mul_batch_tensors(self, k, key_idx):
        """mul_batch_packed on CUDA tensors (eb200_scalar_mul_batch_keyed_dev).  Returns (out (n, 2 len), status)."""
        return self._keyed_tensors("mul_batch_tensors", "eb200_scalar_mul_batch_keyed_dev", self._rows(("k", k)),
                                   [k], key_idx, [(2 * self._ec._len,)])

    def mul_add_batch_tensors(self, k1, k2, key_idx):
        """mul_add_batch_packed on CUDA tensors (eb200_mul_add_batch_keyed_dev).  Returns (out (n, 2 len), status)."""
        return self._keyed_tensors("mul_add_batch_tensors", "eb200_mul_add_batch_keyed_dev",
                                   self._rows(("k1", k1), ("k2", k2)), [k1, k2], key_idx, [(2 * self._ec._len,)])

    def derive_batch_tensors(self, priv, key_idx):
        """derive_batch_packed on CUDA tensors (eb200_ecdh_derive_batch_keyed_dev).  Returns (x (n, len), status)."""
        return self._keyed_tensors("derive_batch_tensors", "eb200_ecdh_derive_batch_keyed_dev",
                                   self._rows(("priv", priv)), [priv], key_idx, [(self._ec._len,)])

    def recovery_param_batch_tensors(self, e, r, s, key_idx):
        """recovery_param_batch_packed on CUDA tensors (eb200_ecdsa_recovery_param_batch_keyed_dev).  Returns (recid (n,),
        status)."""
        return self._keyed_tensors("recovery_param_batch_tensors", "eb200_ecdsa_recovery_param_batch_keyed_dev",
                                   self._rows(("e", e), ("r", r), ("s", s)), [e, r, s], key_idx, [()])


class X25519KeySet(_NativeSets):
    """curve25519 peer keys imported once (eb200_x25519_keyset_create) and kept on the GPU as their edwards25519 images
    with per-key tables; item i of a derive call uses key key_idx[i].  Keys come in the forms EC.derive_batch takes on
    curve25519 (int, hex or big-endian bytes, reduced mod p when wider than 256 bits).  `status`: per key, ST_TRUE, or
    ST_THROW_ASSERT for a point on the twist (whose derives then give that status, as in EC.derive_batch).  close()
    frees the device memory; the object is a context manager."""

    def __init__(self, ec, keys, table_bits=0):
        self._ec = ec
        p = ec._c["p"]
        pubx = _pack((x % p if x >> 256 else x for x in (_bn(k) for k in keys)), 32)
        lib = nat.init(ec._device)
        self.status = np.zeros(len(pubx), np.uint8)
        h = ctypes.c_void_p()
        nat.check(lib.eb200_x25519_keyset_create(len(pubx), pubx.ctypes.data, table_bits, self.status.ctypes.data,
                                                 ctypes.byref(h)))
        self._sets = [h]
        w, db = ctypes.c_uint32(), ctypes.c_size_t()
        nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), ctypes.byref(db)))
        self.table_bits, self.device_bytes = w.value, db.value

    def derive_batch_packed(self, priv, key_idx, out=None, status=None):
        """keyPair.derive(pub) for pub = key key_idx[i] (eb200_x25519_derive_batch_keyed): priv is an (n, 32) uint8 array,
        big-endian, each below n (reduced mod n as _importPrivate does, ec/key.js:76-82).  Returns ((n, 32) shared x
        big-endian, statuses), as EC.derive_batch_packed for those keys; `out` / `status` let the caller supply (and
        reuse) the result buffers, e.g. pinned ones."""
        priv = np.ascontiguousarray(priv, dtype=np.uint8)
        key_idx = np.asarray(key_idx)
        n = len(key_idx)
        if priv.shape != (n, 32) or key_idx.shape != (n,):
            raise ValueError("derive_batch_packed: priv must be an (n, 32) uint8 array, n = len(key_idx)")
        if n and (key_idx.min() < 0 or key_idx.max() >= len(self.status)):
            raise ValueError("key_idx out of range")
        out = np.empty((n, 32), np.uint8) if out is None else out
        st = np.empty(n, np.uint8) if status is None else status
        if out.shape != (n, 32) or out.dtype != np.uint8 or not out.flags.c_contiguous or st.shape != (n,) or st.dtype != np.uint8:
            raise ValueError("derive_batch_packed: out must be a contiguous (n, 32) uint8 array, status (n,) uint8")
        if not self._sets:
            if n:
                raise EllipticError("key set is closed")
            return out, st
        nat.call(nat.load().eb200_x25519_derive_batch_keyed, self._sets[0], n, priv, np.ascontiguousarray(key_idx, np.uint32),
                 out, st)
        return out, st

    def derive_batch(self, privs, key_idx):
        """[keyPair(priv).derive(pub)] for pub = key key_idx[i]: what EC.derive_batch returns for those keys, (values,
        statuses); a twist key's items are None with ST_THROW_ASSERT."""
        if len(privs) != len(key_idx):
            raise ValueError("derive_batch: one key index per private key")
        out, st = self.derive_batch_packed(_pack((_bn(k) % self._ec.n for k in privs), 32), key_idx)
        return _unpack(out, 32, st), st

    def derive_batch_tensors(self, priv, key_idx):
        """derive_batch_packed on CUDA tensors (eb200_x25519_derive_batch_keyed_dev): priv (n, 32) big-endian; a priv >= n
        gets ST_BAD_ITEM.  Returns (x (n, 32), status)."""
        from . import _tensors as T
        n, dev = T.check("derive_batch_tensors", [("priv", priv, T.ROWS, 32), ("key_idx", key_idx, T.IDX, 0)], self._sets)
        return T.keyed("derive_batch_tensors", self._sets, len(self.status), None,
                       "eb200_x25519_derive_batch_keyed_dev", n, dev, [priv], key_idx, [(n, 32)])
