"""DER signatures for the keyed DER verify tests: the canonical encoding and the malformed forms a wire parser meets
(long-form lengths, padded integers, truncation, trailing bytes, bit flips), with the oracle's status for each item."""
import numpy as np

ST_FALSE, ST_TRUE, ST_SIG_FORMAT = 0, 1, 9


def _int_der(v):
    b = v.to_bytes(max(1, (v.bit_length() + 7) // 8), "big")
    return b"\x00" + b if b[0] & 0x80 else b


def canonical(r, s):
    ri, si = _int_der(r), _int_der(s)
    body = b"\x02" + bytes([len(ri)]) + ri + b"\x02" + bytes([len(si)]) + si
    return b"\x30" + bytes([len(body)]) + body


def variants(r, s, rnd):
    """Encodings of (r, s) that a parser must accept or reject exactly as Signature._importDER does."""
    der = canonical(r, s)
    ri, si = _int_der(r), _int_der(s)
    body = b"\x02" + bytes([len(ri)]) + ri + b"\x02" + bytes([len(si)]) + si
    flip = bytearray(der)
    flip[rnd.randrange(len(flip))] ^= 1 << rnd.randrange(8)
    return [
        der,
        b"\x30\x81" + bytes([len(body)]) + body,                              # long-form length under 0x80
        b"\x30" + bytes([len(body) + 1]) + b"\x02" + bytes([len(ri) + 1]) + b"\x00" + ri + body[2 + len(ri):],  # padded r
        der[:-rnd.randrange(1, 4)],                                          # truncated
        der + b"\x00",                                                       # trailing byte
        bytes(flip),                                                         # one bit flipped
        b"",
    ]


def parse(der):
    """(r, s) as the oracle's Signature._importDER reads `der`, or None where it rejects it."""
    from oracle.ref_py.signature import Signature
    chk = Signature.__new__(Signature)
    if not chk._import_der(bytes(der), None):
        return None
    return int(chk.r), int(chk.s)


def status(ec, e, der, xy, key_throw=0):
    """key.verify(e, der) for key xy: the key's throw, THROW_SIG_FORMAT, FALSE out of range, then the verify."""
    if key_throw:
        return key_throw
    rs = parse(der)
    if rs is None:
        return ST_SIG_FORMAT
    r, s = rs
    if not (1 <= r < ec.n and 1 <= s < ec.n):
        return ST_FALSE
    return int(ec.verify(e, {"r": r, "s": s}, {"x": xy[0], "y": xy[1]}))


def blob(ders):
    """The DER encodings back to back and their n + 1 offsets, as the C ABI takes them."""
    off = np.zeros(len(ders) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d in ders])
    return np.frombuffer(b"".join(ders) + b"\x00", np.uint8).copy(), off
