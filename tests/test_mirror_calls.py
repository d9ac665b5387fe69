"""Every call the Python mirror (elliptic_b200/ec.py, eddsa.py, curve.py) makes into the C ABI, against a recorded log.

The mirror runs here over a fake library: one Python method per eb200_* entry point, which reads every input buffer
at the size include/elliptic_b200.h gives it, fills the outputs deterministically (SHAKE-256 of the call's inputs)
and answers with the statuses and return codes each case plans.  Each case records the ordered library calls (values,
input bytes, NULLs), the init(device) calls and the result or exception, once with the fake and once with an
init() that fails as it does without a device.  tests/golden/mirror_calls.json.gz holds that record;
`python tests/test_mirror_calls.py --regen` rewrites it.
"""
import ctypes
import gzip
import hashlib
import importlib
import inspect
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from elliptic_b200 import _native as nat  # noqa: E402

ecm = importlib.import_module("elliptic_b200.ec")
edm = importlib.import_module("elliptic_b200.eddsa")
cvm = importlib.import_module("elliptic_b200.curve")
EC, EDDSA, ShortCurve = ecm.EC, edm.EDDSA, cvm.ShortCurve

GOLDEN = os.path.join(ROOT, "tests", "golden", "mirror_calls.json.gz")

# ---- the fake library -----------------------------------------------------------------------------------------------
CURVE_LEN = {1: 32, 2: 32, 3: 48, 4: 32, 5: 32, 6: 66, 7: 24, 8: 28}     # EB200_CURVE_* -> field bytes


def _L(c, k=1):
    return lambda a: a["n"] * k * c.len


def _pub(c):
    return lambda a: a["n"] * {0: 2 * c.len, 1: 1 + 2 * c.len, 2: 1 + c.len}[a["pub_fmt"]]


# Argument layouts of the header: (name, kind, bytes) with kind "v" (a value), "in", "out", "st" (the status
# output), "desc" (eb200_short_curve*), "off" (n + 1 uint64 offsets) or "blob" (bytes up to the last offset of
# the "off" argument named in the third field).  `c` carries the call's field length.
def _layouts(c):
    n = lambda a: a["n"]
    n32, n64 = (lambda a: 32 * a["n"]), (lambda a: 64 * a["n"])
    k = lambda a: a["n"] * a["klen"]
    L, L2, P = _L(c), _L(c, 2), _pub(c)
    st, cur, nn = ("status", "st", n), ("curve", "v", None), ("n", "v", None)
    sign_out = [("out_r", "out", L), ("out_s", "out", L), ("out_recid", "out", n), st]
    return {
        "eb200_ecdsa_verify_batch": [cur, nn, ("e", "in", L), ("r", "in", L), ("s", "in", L), ("pub", "in", P),
                                     ("pub_fmt", "v", None), st],
        "eb200_ecdsa_verify_batch_der": [cur, nn, ("e", "in", L), ("sigs", "blob", "sig_off"), ("sig_off", "off", None),
                                         ("pub", "in", P), ("pub_fmt", "v", None), st],
        "eb200_ecdsa_sign_batch": [cur, nn, ("e", "in", L), ("priv", "in", L), ("flags", "v", None)] + sign_out,
        "eb200_ecdsa_sign_batch_k": [cur, nn, ("e", "in", L), ("priv", "in", L), ("k", "in", L),
                                     ("flags", "v", None)] + sign_out,
        "eb200_ecdsa_sign_batch_pers": [cur, nn, ("e", "in", L), ("priv", "in", L), ("pers", "in", lambda a: a["pers_len"]),
                                        ("pers_len", "v", None), ("flags", "v", None)] + sign_out,
        "eb200_ec_keygen_batch": [cur, nn, ("entropy", "in", lambda a: a["n"] * a["entropy_len"]), ("entropy_len", "v", None),
                                  ("pers", "in", lambda a: a["pers_len"]), ("pers_len", "v", None),
                                  ("out_priv", "out", L), ("out_pub_xy", "out", L2), st],
        "eb200_ecdsa_recover_batch": [cur, nn, ("e", "in", L), ("r", "in", L), ("s", "in", L), ("recid", "in", n),
                                      ("out_xy", "out", L2), st],
        "eb200_ecdsa_recovery_param_batch": [cur, nn, ("e", "in", L), ("r", "in", L), ("s", "in", L), ("q_xy", "in", L2),
                                             ("out_recid", "out", n), st],
        "eb200_scalar_mul_batch": [cur, nn, ("k", "in", L), ("points_xy", "in", L2), ("out_xy", "out", L2), st],
        "eb200_mul_add_batch": [cur, nn, ("k1", "in", L), ("k2", "in", L), ("p2_xy", "in", L2), ("out_xy", "out", L2), st],
        "eb200_ecdh_derive_batch": [cur, nn, ("priv", "in", L), ("pub_xy", "in", L2), ("out_x", "out", L), st],
        "eb200_eddsa_verify_batch": [nn, ("R", "in", n32), ("S", "in", n32), ("A", "in", n32), ("h", "in", n32), st],
        "eb200_eddsa_verify_batch_msgs": [nn, ("R", "in", n32), ("S", "in", n32), ("A", "in", n32),
                                          ("msgs", "blob", "msg_off"), ("msg_off", "off", None), st],
        "eb200_eddsa_sign_batch": [nn, ("secrets", "in", n32), ("msgs", "blob", "msg_off"), ("msg_off", "off", None),
                                   ("out_sig", "out", n64), ("out_pub", "out", n32), st],
        "eb200_x25519_derive_batch": [nn, ("priv", "in", n32), ("pubx", "in", n32), ("out", "out", n32), st],
        "eb200_x25519_mul_batch": [nn, ("k", "in", n32), ("px", "in", n32), ("out_x", "out", n32), st],
        "eb200_curve_mul_batch": [("curve", "desc", None), nn, ("k", "in", k), ("klen", "v", None), ("points_xy", "in", L2),
                                  ("out_xy", "out", L2), st],
        "eb200_curve_mul_add_batch": [("curve", "desc", None), nn, ("k1", "in", k), ("p1_xy", "in", L2), ("k2", "in", k),
                                      ("p2_xy", "in", L2), ("klen", "v", None), ("out_xy", "out", L2), st],
        "eb200_curve_add_batch": [("curve", "desc", None), nn, ("p1_xy", "in", L2), ("p2_xy", "in", L2),
                                  ("out_xy", "out", L2), st],
        "eb200_curve_dbl_batch": [("curve", "desc", None), nn, ("p_xy", "in", L2), ("out_xy", "out", L2), st],
        "eb200_curve_validate_batch": [("curve", "desc", None), nn, ("p_xy", "in", L2), st],
    }


FUNCS = sorted(_layouts(types.SimpleNamespace(len=0)))


def _addr(p):
    """What a c_void_p argument accepts: an int, None, or an object with _as_parameter_ -> address or None (NULL)."""
    while hasattr(p, "_as_parameter_"):
        p = p._as_parameter_
    if isinstance(p, ctypes.c_void_p):
        p = p.value
    assert p is None or isinstance(p, int), "not a pointer argument: %r" % (p,)
    return p or None


def _desc(d):
    d = getattr(d, "_obj", d)                      # ctypes.byref(desc)
    if isinstance(d, ctypes._Pointer):
        d = d.contents
    assert isinstance(d, nat.ShortCurveDesc), d
    return d


class FakeLib:
    """Stands in for libelliptic_b200.so.  plan[k]: the statuses of the k-th call (item i gets plan[k][i % len]; the
    last list repeats); rcs[k]: its return code (the last one repeats)."""

    def __init__(self, plan, rcs):
        self.plan, self.rcs = plan, rcs
        self.calls, self.addrs = [], []
        for name in FUNCS:
            setattr(self, name, self._entry(name))

    def eb200_strerror(self, rc):
        return b"fake error %d" % rc

    def eb200_last_error(self):
        return b"fake last error"

    def _entry(self, name):
        def fn(*args):
            c = types.SimpleNamespace(len=None)
            lay = _layouts(c)[name]
            assert len(args) == len(lay), (name, len(args))
            vals, rec, ins, outs, addrs = {}, [], [], [], {}
            for (an, kind, _), a in zip(lay, args):
                if kind == "v":
                    assert isinstance(a, int) and not isinstance(a, bool), (name, an, a)
                    vals[an] = a
                    if an == "curve":
                        c.len = CURVE_LEN.get(a, 0)
                elif kind == "desc":
                    d = _desc(a)
                    c.len = d.len
                    vals[an] = {"len": d.len, **{f: ctypes.string_at(getattr(d, f), d.len).hex() for f in ("p", "a", "b")}}
                else:
                    addrs[an] = _addr(a)
            for an, kind, size in lay:
                if kind in ("v", "desc"):
                    rec.append(vals[an])
                    continue
                p = addrs[an]
                if kind in ("out", "st"):
                    rec.append(None if p is None else "out")
                    if p is not None:
                        outs.append((an, kind, p, size(vals)))
                    continue
                if kind == "off":
                    nb = 8 * (vals["n"] + 1)
                elif kind == "blob":
                    po = addrs[size]
                    nb = 0 if po is None else int(np.frombuffer(ctypes.string_at(po, 8 * (vals["n"] + 1)), "<u8")[-1])
                else:
                    nb = size(vals)
                b = None if p is None else ctypes.string_at(p, nb)
                rec.append(None if b is None else b.hex())
                ins.append(b or b"")
            k = len(self.calls)
            self.calls.append({"fn": name, "args": rec})
            self.addrs.append(addrs)
            seed = hashlib.sha256(name.encode() + b"".join(ins)).digest()
            sts = self.plan[min(k, len(self.plan) - 1)]
            for an, kind, p, nb in outs:
                if kind == "st":
                    data = bytes(sts[i % len(sts)] for i in range(nb))
                else:
                    data = hashlib.shake_256(seed + an.encode()).digest(nb)
                ctypes.memmove(p, data, nb)
            return self.rcs[min(k, len(self.rcs) - 1)]
        fn.__name__ = name
        return fn


def _norm(v):
    """A result as JSON, its shape kept: list / tuple / ndarray (dtype, shape, bytes) / numpy scalar / int / bool."""
    if v is None or isinstance(v, str):
        return v
    if isinstance(v, bool):
        return {"bool": v}
    if isinstance(v, np.ndarray):
        return {"ndarray": v.dtype.str, "shape": list(v.shape), "hex": v.tobytes().hex()}
    if isinstance(v, np.generic):
        return {"np": v.dtype.str, "v": v.item()}
    if isinstance(v, int):
        return {"int": hex(v)}
    if isinstance(v, (bytes, bytearray)):
        return {type(v).__name__: bytes(v).hex()}
    if isinstance(v, list):
        return [_norm(x) for x in v]
    if isinstance(v, tuple):
        return {"tuple": [_norm(x) for x in v]}
    if isinstance(v, dict):
        return {"dict": [[_norm(k), _norm(x)] for k, x in v.items()]}
    raise TypeError("unrecorded result type %r" % type(v))


def run_case(fn, plan=((1,),), rcs=(0,), device_ok=True):
    """fn() over a fake library -> (record, fake)."""
    fake = FakeLib([list(p) for p in plan], list(rcs))
    inits = []

    def init(device=0, flags=0):
        inits.append([device, flags])
        if not device_ok:
            raise nat.NativeError("no CUDA device [fake]")
        return fake

    def init_devices(devices=None, flags=0):
        inits.append(["devices", devices, flags])
        if not device_ok:
            raise nat.NativeError("no CUDA device [fake]")
        return fake

    saved = nat.init, nat.init_devices, nat.load
    nat.init, nat.init_devices, nat.load = init, init_devices, (lambda: fake)
    try:
        try:
            out = {"result": _norm(fn())}
        except Exception as e:      # noqa: BLE001 -- the exception is the recorded outcome
            out = {"raise": [type(e).__name__, str(e)]}
    finally:
        nat.init, nat.init_devices, nat.load = saved
    return dict(init=inits, calls=fake.calls, **out), fake


# ---- the corpus ---------------------------------------------------------------------------------------------------
SHORT = ("secp256k1", "p256", "p384", "p521", "p192", "p224")
XY = SHORT + ("ed25519",)
ALL = XY + ("curve25519",)
N = {c: ecm._CURVES[c]["n"] for c in ALL}
P = {c: ecm._CURVES[c]["p"] for c in ALL}
LN = {c: ecm._CURVES[c]["len"] for c in ALL}
STATUSES = range(12)


def arr(n, w, seed, dtype=np.uint8):
    return np.frombuffer(hashlib.shake_256(seed.encode()).digest(n * w), np.uint8).reshape(n, w).astype(dtype)


def B(b):
    return np.frombuffer(b, np.uint8)


def num(seed, bits=256):
    return int.from_bytes(hashlib.shake_256(seed.encode()).digest((bits + 7) // 8), "big") >> (-bits % 8)


def der(r, s):
    def i(v):
        b = v.to_bytes(max(1, (v.bit_length() + 7) // 8), "big")
        return b"\x02" + bytes([len(b) + (b[0] >> 7)]) + (b"\x00" if b[0] & 0x80 else b"") + b
    body = i(r) + i(s)
    return b"\x30" + (bytes([len(body)]) if len(body) < 0x80 else b"\x81" + bytes([len(body)])) + body


def _no_more_k():
    raise RuntimeError("k called after a nonce that does not fit")


def RS(r, s, **kw):
    return types.SimpleNamespace(r=r, s=s, **kw)


def corpus():
    cs = []

    def case(name, fn, plan=((1,),), rcs=(0,)):
        cs.append((name, fn, plan, rcs))

    msg_forms = [12345, "abcdef0123", b"\x01\x02\x03" * 11, list(range(40)), "xyz", 2**300 + 7, "", bytearray(b"\xff" * 33)]

    # -- constructors
    case("EC('bogus')", lambda: EC("bogus"))
    case("EDDSA('p256')", lambda: EDDSA("p256"))
    case("ShortCurve p even", lambda: ShortCurve(100, 1, 1))
    case("ShortCurve p=3", lambda: ShortCurve(3, 1, 1))
    case("ShortCurve p too wide", lambda: ShortCurve(2**577 + 1, 1, 1))

    # -- EC.verify_batch_packed / verify_batch_der_packed
    for c in ALL:
        ln = LN[c]
        for fmt, pb in ((0, 2 * ln), (1, 1 + 2 * ln), (2, 1 + ln)):
            case("%s verify_batch_packed fmt %d" % (c, fmt),
                 lambda c=c, ln=ln, fmt=fmt, pb=pb: EC(c).verify_batch_packed(
                     arr(3, ln, c + "e"), arr(3, ln, c + "r"), arr(3, ln, c + "s"), arr(3, pb, c + "q"), fmt),
                 plan=((1, 0, 2),))
        ders = [der(num(c + "r1", 8 * ln), num(c + "s1", 8 * ln)), b"", b"\x30\x00", der(1, 2), bytearray(der(3, 4))]
        case("%s verify_batch_der_packed" % c,
             lambda c=c, ln=ln, ders=ders: EC(c).verify_batch_der_packed(arr(5, ln, c + "e"), ders, arr(5, 2 * ln, c + "q")),
             plan=((1, 9, 0, 3),))
        case("%s verify_batch_der_packed sec1_33" % c,
             lambda c=c, ln=ln, ders=ders: EC(c).verify_batch_der_packed(arr(5, ln, c + "e"), ders, arr(5, 1 + ln, c + "q"), 2))
    k1 = LN["secp256k1"]
    case("verify_batch_packed n=0", lambda: EC().verify_batch_packed(*(np.zeros((0, 32), np.uint8),) * 3, np.zeros((0, 64), np.uint8)))
    case("verify_batch_packed int64 input", lambda: EC().verify_batch_packed(
        arr(2, 32, "e", np.int64), arr(2, 32, "r"), arr(2, 32, "s"), arr(2, 64, "q")))
    case("verify_batch_packed strided input", lambda: EC().verify_batch_packed(
        arr(4, 32, "e")[::2], arr(2, 32, "r"), np.asfortranarray(arr(2, 32, "s")), arr(2, 64, "q")))
    case("verify_batch_packed list input", lambda: EC().verify_batch_packed(
        arr(2, 32, "e").tolist(), arr(2, 32, "r"), arr(2, 32, "s"), arr(2, 64, "q")))
    case("verify_batch_packed bad e", lambda: EC().verify_batch_packed(arr(2, 31, "e"), arr(2, 32, "r"), arr(2, 32, "s"), arr(2, 64, "q")))
    case("verify_batch_packed bad s", lambda: EC().verify_batch_packed(arr(2, 32, "e"), arr(2, 32, "r"), arr(3, 32, "s"), arr(2, 64, "q")))
    case("verify_batch_packed bad pub", lambda: EC().verify_batch_packed(arr(2, 32, "e"), arr(2, 32, "r"), arr(2, 32, "s"), arr(2, 65, "q")))
    case("verify_batch_packed bad fmt", lambda: EC().verify_batch_packed(arr(2, 32, "e"), arr(2, 32, "r"), arr(2, 32, "s"), arr(2, 64, "q"), 7))
    case("verify_batch_packed rc", lambda: EC().verify_batch_packed(arr(2, 32, "e"), arr(2, 32, "r"), arr(2, 32, "s"), arr(2, 64, "q")),
         rcs=(nat.ERR_ARG,))
    case("verify_batch_packed device 3", lambda: EC("p256", device=3).verify_batch_packed(
        arr(1, 32, "e"), arr(1, 32, "r"), arr(1, 32, "s"), arr(1, 33, "q"), nat.PUB_SEC1_33))
    case("verify_batch_der_packed n=0", lambda: EC().verify_batch_der_packed(np.zeros((0, 32), np.uint8), [], np.zeros((0, 64), np.uint8)))
    case("verify_batch_der_packed bad e", lambda: EC().verify_batch_der_packed(arr(2, 32, "e"), [b"", b""], arr(1, 64, "q")))
    case("verify_batch_der_packed bad pub", lambda: EC().verify_batch_der_packed(arr(2, 32, "e"), [b"", b""], arr(2, 65, "q"), 1))
    case("verify_batch_der_packed bad fmt", lambda: EC().verify_batch_der_packed(arr(2, 32, "e"), [b"", b""], arr(2, 64, "q"), 9))

    # -- EC.verify_batch / verify
    for c in XY + ("curve25519",):
        ln, n = LN[c], N[c]
        r, s = num(c + "r") % n, num(c + "s") % n
        x, y = num(c + "x", 8 * ln), num(c + "y", 8 * ln)
        keys = [{"x": x, "y": y}, b"\x04" + x.to_bytes(ln, "big") + y.to_bytes(ln, "big"),
                [3] + list(x.to_bytes(ln, "big")), {"x": hex(x)[2:], "y": hex(y)[2:]}]
        sigs = [{"r": r, "s": s}, RS(r, s), der(r, s), {"r": hex(r)[2:], "s": hex(s)[2:]}]
        case("%s verify_batch forms" % c, lambda c=c, keys=keys, sigs=sigs: EC(c).verify_batch(msg_forms[:4], sigs, keys),
             plan=((1, 0, 4, 2, 1),))
        case("%s verify_batch hex keys" % c,
             lambda c=c, ln=ln, x=x, y=y, sigs=sigs: EC(c).verify_batch(
                 ["00ff", "abc"], [der(r, s).hex(), sigs[0]],
                 ["04" + x.to_bytes(ln, "big").hex() + y.to_bytes(ln, "big").hex(), "02" + x.to_bytes(ln, "big").hex()], "hex"))
    n, ln = N["secp256k1"], 32
    x, y = num("x"), num("y")
    xy = {"x": x, "y": y}
    b65 = lambda h: bytes([h]) + x.to_bytes(32, "big") + (y | 1).to_bytes(32, "big")
    case("verify_batch early FALSE", lambda: EC().verify_batch([1] * 6, [{"r": 0, "s": 5}, {"r": n, "s": 5}, {"r": 5, "s": n}, RS(5, 0),
                                                                          {"r": 5, "s": n - 1}, {"r": -1, "s": 5}], [xy] * 6),
         plan=((1, 0, 4, 2, 7, 11),))
    case("verify_batch msg_bit_length", lambda: EC().verify_batch(msg_forms, [{"r": 1, "s": 2}] * 8, [xy] * 8, None, 100))
    case("verify_batch msg_bit_length 400", lambda: EC().verify_batch(msg_forms, [{"r": 1, "s": 2}] * 8, [xy] * 8, None, 400))
    case("verify_batch msg_bit_length 8", lambda: EC().verify_batch([12345, "abcdef0123", "", 0], [RS(1, 2)] * 4, [xy] * 4, None, 8))
    case("verify_batch wide key", lambda: EC().verify_batch([1, 2], [RS(1, 2)] * 2, [{"x": 2**300 + 5, "y": 7}, {"x": 7, "y": P["secp256k1"] + 1}]))
    case("verify_batch hybrid keys", lambda: EC().verify_batch([1, 2], [RS(1, 2)] * 2, [b65(6)[:-1] + b"\x00", b65(7)]))
    case("verify_batch hybrid 06 odd", lambda: EC().verify_batch([1], [RS(1, 2)], [b65(6)]))
    case("verify_batch hybrid 07 even", lambda: EC().verify_batch([1], [RS(1, 2)], [b65(7)[:-1] + b"\x02"]))
    case("verify_batch only x", lambda: EC().verify_batch([1], [RS(1, 2)], [{"x": 5}]))
    case("verify_batch negative x", lambda: EC().verify_batch([1], [RS(1, 2)], [{"x": -5, "y": 3}]))
    case("verify_batch unknown format", lambda: EC().verify_batch([1], [RS(1, 2)], [b"\x05" + bytes(32)]))
    case("verify_batch empty key", lambda: EC().verify_batch([1], [RS(1, 2)], [b""]))
    case("verify_batch sig without s", lambda: EC().verify_batch([1], [{"r": 1}], [xy]))
    case("verify_batch sig s=0 dict", lambda: EC().verify_batch([1], [{"r": 1, "s": 0}], [xy]))
    case("verify_batch bad DER", lambda: EC().verify_batch([1], [b"\x30\x01\x02"], [xy]))
    case("verify_batch key before sig", lambda: EC().verify_batch([1], [b"\x30"], [{"x": 5}]))
    case("verify_batch bad msg before key", lambda: EC().verify_batch([{"a": 1}], [b"\x30"], [{"x": 5}]))
    case("verify_batch second item throws", lambda: EC().verify_batch([1, 2], [RS(1, 2), {"r": 1}], [xy, xy]))
    case("verify_batch n=0", lambda: EC().verify_batch([], [], []))
    case("verify_batch negative e before later key", lambda: EC().verify_batch(["-ab", 1], [RS(1, 2)] * 2, [xy, b"\x05" + bytes(32)]))
    case("verify_batch wide e before later sig", lambda: EC().verify_batch([2**300, 1], [RS(1, 2), {"r": 1}], [xy, xy], None, 100))
    case("verify_batch negative int e before later msg", lambda: EC().verify_batch([-5, {"a": 1}], [RS(1, 2)] * 2, [xy, xy]))
    for st in STATUSES:
        case("verify status %d" % st, lambda: EC().verify(b"\x01" * 32, {"r": 1, "s": 2}, xy), plan=((st,),))
        case("verify early FALSE status %d" % st, lambda: EC("p384").verify(b"\x01" * 32, {"r": 0, "s": 2}, {"x": 1, "y": 2}), plan=((st,),))
    case("verify msgBitLength", lambda: EC().verify(2**256 - 1, der(3, 4).hex(), b65(4).hex(), "hex", {"msgBitLength": 64}))
    case("verify options without msgBitLength", lambda: EC().verify(2**256 - 1, der(3, 4), b65(4), None, {}))

    # -- EC.sign_batch / sign
    privs = [5, "abcdef", b"\x01" * 20, N["secp256k1"] + 9, [1, 2, 3]]
    for c in XY + ("curve25519",):
        ln = LN[c]
        privs_c = [5, "abcdef", b"\x01" * 20, N[c] + 9, [1, 2, 3]]
        case("%s sign_batch" % c, lambda c=c, privs_c=privs_c: EC(c).sign_batch(msg_forms[:5], privs_c))
        case("%s sign_batch canonical pers" % c,
             lambda c=c, privs_c=privs_c: EC(c).sign_batch(msg_forms[:5], privs_c, canonical=True, pers="hello"))
        case("%s sign_batch k" % c, lambda c=c, privs_c=privs_c: EC(c).sign_batch(
            msg_forms[:5], privs_c, msg_bit_length=200, k=lambda i, it: [i + 1, "abcd", b"\x07" * 9, 2**600 + i, 7][i]),
             plan=((10, 1, 10, 1, 1), (1,)))
    case("sign_batch pers hex", lambda: EC().sign_batch([1, 2], [3, 4], pers="00ff10", pers_enc="hex"))
    case("sign_batch pers empty", lambda: EC().sign_batch([1, 2], [3, 4], pers=""))
    case("sign_batch pers bytes", lambda: EC("p521").sign_batch([1, 2], [3, 4], pers=b"\x00\x01"))
    case("sign_batch k over pers", lambda: EC().sign_batch([1, 2], [3, 4], pers="x", k=lambda i, it: 1000 * it + i + 1),
         plan=((10, 1), (10,), (1,)))
    case("sign_batch k wide", lambda: EC("p384").sign_batch([1, 2, 3], [3, 4, 5],
                                                            k=lambda i, it: [2**384 + 5, 2**390 + 2**389, (2**384 - 1).to_bytes(48, "big") + b"\x05"][i]))
    case("sign_batch k p521 wide", lambda: EC("p521").sign_batch([1, 2], [3, 4], k=lambda i, it: [2**528 + 5, 2**521 + 3][i]))
    case("sign_batch k unexpected", lambda: EC().sign_batch([1, 2, 3], [3, 4, 5], k=lambda i, it: i + 1), plan=((1, 10, 0),))
    case("sign_batch k retry twice", lambda: EC().sign_batch([1, 2, 3], [3, 4, 5], k=lambda i, it: i + it + 1),
         plan=((10, 1, 10), (10, 1), (1,)))
    case("sign_batch unexpected", lambda: EC().sign_batch([1, 2, 3], privs[:3]), plan=((1, 1, 0),))
    case("sign_batch pers unexpected", lambda: EC().sign_batch([1, 2], [1, 2], pers="p"), plan=((10, 1),))
    case("sign_batch rc", lambda: EC().sign_batch([1, 2], [1, 2]), rcs=(nat.ERR_CUDA,))
    case("sign_batch k rc", lambda: EC().sign_batch([1, 2], [1, 2], k=lambda i, it: 5), rcs=(nat.ERR_ARG,))
    case("sign_batch too long", lambda: EC().sign_batch([1, 2**300], [1, 2], msg_bit_length=0))
    case("sign_batch bad priv", lambda: EC().sign_batch([1, 2], [1, None]))
    case("sign_batch msg_bit_length 0", lambda: EC("p192").sign_batch([5, 2**200], [1, 2], msg_bit_length=0))
    case("sign_batch n=0", lambda: EC().sign_batch([], []))
    case("sign_batch k negative before next k", lambda: EC().sign_batch([1, 2], [3, 4], k=lambda i, it: "-5" if i == 0 else _no_more_k()))
    case("sign_batch k retry negative before next k",
         lambda: EC().sign_batch([1, 2, 3], [3, 4, 5], k=lambda i, it: 7 if it == 0 else ("-5" if i == 0 else _no_more_k())),
         plan=((10, 1, 10),))
    case("sign_batch pers n=0", lambda: EC().sign_batch([], [], pers="x"))
    case("sign_batch k n=0", lambda: EC().sign_batch([], [], k=lambda i, it: 1))
    case("sign", lambda: EC("p256").sign("abcdef", 77, canonical=True))
    case("sign pers", lambda: EC("p256").sign([1, 2, 3], "77", pers="0102", pers_enc="hex"))
    case("sign k", lambda: EC().sign(b"\x01" * 32, 77, k=lambda it: it + 3), plan=((10,), (10,), (1,)))
    case("sign curve25519", lambda: EC("curve25519").sign(1, 2))

    # -- EC.gen_key_pair_batch
    for c in XY + ("curve25519",):
        case("%s gen_key_pair_batch" % c, lambda c=c: EC(c).gen_key_pair_batch(["a" * 24, "b" * 24, "ā" * 12]))
        case("%s gen_key_pair_batch pers" % c,
             lambda c=c: EC(c).gen_key_pair_batch(["00" * 30, "ff" * 30], entropy_enc="hex", pers="0a0b", pers_enc="hex"))
    case("gen_key_pair_batch bytes", lambda: EC().gen_key_pair_batch([b"\x01" * 32, list(range(32))], pers="pp"))
    case("gen_key_pair_batch short", lambda: EC().gen_key_pair_batch(["a" * 24, "b" * 23]))
    case("gen_key_pair_batch lengths", lambda: EC().gen_key_pair_batch(["a" * 24, "b" * 25]))
    case("gen_key_pair_batch short before lengths", lambda: EC().gen_key_pair_batch(["a" * 30, "b" * 23]))
    case("gen_key_pair_batch unexpected", lambda: EC().gen_key_pair_batch(["a" * 24] * 3), plan=((1, 0, 1),))
    case("gen_key_pair_batch rc", lambda: EC().gen_key_pair_batch(["a" * 24]), rcs=(nat.ERR_NOT_INIT,))
    case("gen_key_pair_batch n=0", lambda: EC().gen_key_pair_batch([]))
    case("gen_key_pair_batch n=0 curve25519", lambda: EC("curve25519").gen_key_pair_batch([]))

    # -- EC.recover_pub_key_batch / recover_pub_key
    for c in XY + ("curve25519",):
        ln, n = LN[c], N[c]
        r, s = num(c + "r", 8 * ln), num(c + "s", 8 * ln + 8)
        sigs = [{"r": r, "s": s}, RS(r, s), der(r % 2**(8 * ln - 1), s % n), {"r": hex(r), "s": hex(s)}, der(r % n, 5)]
        case("%s recover_pub_key_batch" % c,
             lambda c=c, sigs=sigs: EC(c).recover_pub_key_batch([12345, "abcdef", b"\x01" * 70, list(range(40)), (1, 2)],
                                                                sigs, [0, 1, 2, 3, 1]),
             plan=((1, 7, 2, 8, 1),))
        case("%s recover_pub_key_batch hex" % c,
             lambda c=c, r=r, s=s, n=n: EC(c).recover_pub_key_batch(["ab"], [der(r % n, s % n).hex()], [2], "hex"))
    case("recover_pub_key_batch j=4", lambda: EC().recover_pub_key_batch([1], [RS(1, 2)], [4]))
    case("recover_pub_key_batch j before sig", lambda: EC().recover_pub_key_batch([1], [b"\x30"], [5]))
    case("recover_pub_key_batch j=-1", lambda: EC().recover_pub_key_batch([1], [RS(1, 2)], [-1]))
    case("recover_pub_key_batch sig before r width", lambda: EC().recover_pub_key_batch([1, 2], [RS(2**256, 2), {"r": 1}], [0, 0]))
    case("recover_pub_key_batch wide r", lambda: EC().recover_pub_key_batch([1], [RS(2**256, 2)], [0]))
    case("recover_pub_key_batch bad msg", lambda: EC().recover_pub_key_batch([None], [RS(1, 2)], [0]))
    case("recover_pub_key_batch n=0", lambda: EC().recover_pub_key_batch([], [], []))
    case("recover_pub_key_batch rc", lambda: EC().recover_pub_key_batch([1], [RS(1, 2)], [0]), rcs=(nat.ERR_UNSUPPORTED,))
    for st in STATUSES:
        case("recover_pub_key status %d" % st, lambda: EC("p256").recover_pub_key(b"\x05" * 32, {"r": 3, "s": 4}, 1), plan=((st,),))
    case("recover_pub_key hex", lambda: EC().recover_pub_key("05", der(3, 4).hex(), 0, "hex"))

    # -- EC.get_key_recovery_param_batch / get_key_recovery_param
    for c in XY + ("curve25519",):
        ln, n, p = LN[c], N[c], P[c]
        r, s = num(c + "r", 8 * ln), num(c + "s", 8 * ln + 8)
        qx, qy = num(c + "qx", 8 * ln + 8), num(c + "qy", 8 * ln)
        case("%s get_key_recovery_param_batch" % c,
             lambda c=c, r=r, s=s, qx=qx, qy=qy, n=n: EC(c).get_key_recovery_param_batch(
                 [12345, "abcdef", b"\x01" * 70, list(range(40)), 9, 10],
                 [{"r": r, "s": s}, RS(r, s), der(r % n, s % n), {"r": r, "s": s, "recoveryParam": 2}, RS(r, s, recoveryParam=1),
                  RS(r, s, recovery_param=3)],
                 [(qx, qy), {"x": hex(qx), "y": qy}, (qx + 1, qy), None, None, (1, 2)]),
             plan=((1, 11, 1),))
    case("get_key_recovery_param_batch hex", lambda: EC().get_key_recovery_param_batch(["ab"], [der(3, 4).hex()], [(1, 2)], "hex"))
    case("get_key_recovery_param_batch all carried",
         lambda: EC().get_key_recovery_param_batch([1, 2], [{"r": 1, "s": 2, "recoveryParam": 0}, RS(1, 2, recoveryParam=3)], [None, 5]))
    case("get_key_recovery_param_batch rp zero", lambda: EC().get_key_recovery_param_batch([1], [RS(1, 2, recoveryParam=0)], [None]))
    case("get_key_recovery_param_batch rp None attr", lambda: EC().get_key_recovery_param_batch([1], [RS(1, 2, recoveryParam=None)], [None]))
    case("get_key_recovery_param_batch Q None", lambda: EC().get_key_recovery_param_batch([1], [RS(1, 2)], [None]))
    case("get_key_recovery_param_batch rp before Q", lambda: EC().get_key_recovery_param_batch([1, 1], [RS(1, 2, recoveryParam=1), RS(1, 2)], [None, None]))
    case("get_key_recovery_param_batch Q before r width", lambda: EC().get_key_recovery_param_batch([1], [RS(2**256, 2)], [None]))
    case("get_key_recovery_param_batch wide r", lambda: EC().get_key_recovery_param_batch([1], [RS(2**256, 2)], [(1, 2)]))
    case("get_key_recovery_param_batch wide r carried", lambda: EC().get_key_recovery_param_batch([1], [RS(2**256, 2, recoveryParam=2)], [(1, 2)]))
    case("get_key_recovery_param_batch bad sig carried", lambda: EC().get_key_recovery_param_batch([1], [{"r": 0, "s": 1, "recoveryParam": 1}], [None]))
    case("get_key_recovery_param_batch bad msg", lambda: EC().get_key_recovery_param_batch([None, 1], [RS(1, 2), RS(1, 2)], [(1, 2), (1, 2)]))
    case("get_key_recovery_param_batch bad msg carried", lambda: EC().get_key_recovery_param_batch([None], [RS(1, 2, recoveryParam=1)], [(1, 2)]))
    case("get_key_recovery_param_batch bad Q", lambda: EC().get_key_recovery_param_batch([1], [RS(1, 2)], [(1, 2, 3)]))
    case("get_key_recovery_param_batch n=0", lambda: EC().get_key_recovery_param_batch([], [], []))
    case("get_key_recovery_param_batch rc", lambda: EC().get_key_recovery_param_batch([1], [RS(1, 2)], [(1, 2)]), rcs=(nat.ERR_CUDA,))
    for st in STATUSES:
        case("get_key_recovery_param status %d" % st,
             lambda: EC("p224").get_key_recovery_param(b"\x05" * 28, {"r": 3, "s": 4}, {"x": 5, "y": 6}), plan=((st,),))
    case("get_key_recovery_param carried", lambda: EC().get_key_recovery_param(1, {"r": 3, "s": 4, "recoveryParam": 2}, None))

    # -- EC.g_mul_batch / mul_batch / mul_add_batch / x_mul_batch
    for c in ALL:
        ln, n, p = LN[c], N[c], P[c]
        ks = [0, 1, "abcdef", b"\x02" * ln, n - 1, 2**(8 * ln) + 5, [1, 2]]
        pts = [(1, 2), {"x": p + 3, "y": "ff"}, (2**(8 * ln + 3), p - 1), ("aa", b"\x01\x02"), {"x": 0, "y": 0}, (p, 2 * p), (5, 6)]
        case("%s g_mul_batch" % c, lambda c=c, ks=ks: EC(c).g_mul_batch(ks), plan=((1, 7, 1),))
        case("%s mul_batch" % c, lambda c=c, ks=ks, pts=pts: EC(c).mul_batch(pts, ks), plan=((7, 1),))
        case("%s mul_add_batch" % c, lambda c=c, ks=ks, pts=pts: EC(c).mul_add_batch(ks, pts, ks[::-1]), plan=((1, 1, 7),))
        case("%s x_mul_batch" % c, lambda c=c, ks=ks: EC(c).x_mul_batch([9, 2**256 + 3, "ff", b"\x01" * 40, 0, 1, 2], ks[:1] + ks[2:5] + [2**256 - 1, 3, 4]),
             plan=((1, 0, 5),))
        case("%s g_mul_batch n=0" % c, lambda c=c: EC(c).g_mul_batch([]))
        case("%s mul_batch n=0" % c, lambda c=c: EC(c).mul_batch([], []))
        case("%s mul_add_batch n=0" % c, lambda c=c: EC(c).mul_add_batch([], [], []))
        case("%s x_mul_batch n=0" % c, lambda c=c: EC(c).x_mul_batch([], []))
    case("g_mul_batch negative", lambda: EC().g_mul_batch([1, -1]))
    case("g_mul_batch negative curve25519", lambda: EC("curve25519").g_mul_batch([-1]))
    case("mul_batch negative before point", lambda: EC().mul_batch([(1,)], [-1]))
    case("mul_batch bad point", lambda: EC().mul_batch([(1, 2, 3)], [1]))
    case("mul_batch None point", lambda: EC().mul_batch([None], [1]))
    case("mul_add_batch k2 negative", lambda: EC().mul_add_batch([1], [(1, 2)], [-2]))
    case("x_mul_batch wide k", lambda: EC("curve25519").x_mul_batch([1, 2], [1, 2**256]))
    case("x_mul_batch bad x", lambda: EC("curve25519").x_mul_batch([None], [1]))
    for st in (4,):
        case("mul_batch NEEDS_HOST", lambda: EC("ed25519").mul_batch([(1, 2), (3, 4)], [1, 2]), plan=((1, st),))
        case("g_mul_batch NEEDS_HOST", lambda: EC().g_mul_batch([1, 2]), plan=((st,),))
        case("mul_add_batch NEEDS_HOST", lambda: EC("p521").mul_add_batch([1, 2], [(1, 2), (3, 4)], [1, 2]), plan=((7, st),))
    case("mul_batch statuses", lambda: EC().mul_batch([(1, 2)] * 12, list(range(12))), plan=(tuple(range(12)),))
    case("mul_batch rc", lambda: EC().mul_batch([(1, 2)], [1]), rcs=(nat.ERR_ARG,))
    case("x_mul_batch rc", lambda: EC("curve25519").x_mul_batch([1], [1]), rcs=(nat.ERR_ARG,))

    # -- EC.derive_batch / derive / derive_batch_packed
    for c in ALL:
        ln, n, p = LN[c], N[c], P[c]
        privs_c = [5, "abcdef", b"\x01" * (ln + 3), n + 9, [1, 2, 3]]
        pubs = ([9, 2**256 + 3, "ff", b"\x01" * 40, 2**255 - 19] if c == "curve25519"
                else [(1, 2), {"x": p + 3, "y": "ff"}, (2**(8 * ln + 3), p - 1), ("aa", b"\x01\x02"), {"x": 0, "y": 0}])
        case("%s derive_batch" % c, lambda c=c, privs_c=privs_c, pubs=pubs: EC(c).derive_batch(privs_c, pubs), plan=((1, 5, 3, 7),))
        case("%s derive_batch n=0" % c, lambda c=c: EC(c).derive_batch([], []))
        for st in STATUSES:
            case("%s derive status %d" % (c, st), lambda c=c, pubs=pubs: EC(c).derive(7, pubs[0]), plan=((st,),))
        case("%s derive_batch_packed" % c, lambda c=c: EC(c).derive_batch_packed(arr(3, 32, "k"), arr(3, 32, "x")), plan=((1, 5),))
    case("derive_batch bad pub", lambda: EC("curve25519").derive_batch([1], [None]))
    case("derive_batch short bad pub", lambda: EC("p256").derive_batch([1], [(1,)]))
    case("derive_batch short negative priv", lambda: EC("p256").derive_batch([-3], [(1, 2)]))
    case("derive_batch rc", lambda: EC("curve25519").derive_batch([1], [2]), rcs=(nat.ERR_CUDA,))
    c25 = lambda: EC("curve25519")
    case("derive_batch_packed out", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x"), out=np.zeros((2, 32), np.uint8),
                                                                      status=np.full(2, 9, np.uint8)), plan=((1, 3),))
    case("derive_batch_packed out only", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x"), out=np.zeros((2, 32), np.uint8)))
    case("derive_batch_packed status only", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x"), status=np.zeros(2, np.uint8)))
    case("derive_batch_packed n=0", lambda: c25().derive_batch_packed(np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8)))
    case("derive_batch_packed bad shape", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(3, 32, "x")))
    case("derive_batch_packed bad out dtype", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x"), out=np.zeros((2, 32), np.int8)))
    case("derive_batch_packed strided out", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x"), out=np.zeros((2, 64), np.uint8)[:, ::2]))
    case("derive_batch_packed bad status", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x"), status=np.zeros(3, np.uint8)))
    case("derive_batch_packed bad status dtype", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x"), status=np.zeros(2, np.int32)))
    case("derive_batch_packed strided in", lambda: c25().derive_batch_packed(arr(4, 32, "k")[::2], arr(2, 32, "x", np.int16)))
    case("derive_batch_packed rc", lambda: c25().derive_batch_packed(arr(2, 32, "k"), arr(2, 32, "x")), rcs=(nat.ERR_CUDA,))

    # -- EDDSA
    ed = EDDSA
    sig64, pub32 = bytes(range(64)), bytes(range(100, 132))
    case("hash_int", lambda: ed().hash_int(b"\x01" * 32, [1, 2, 3], bytearray(b"xyz")))
    case("eddsa verify_batch_packed", lambda: ed().verify_batch_packed(*(arr(3, 32, s) for s in "RSAh")), plan=((1, 0, 2, 5),))
    case("eddsa verify_batch_packed n=0", lambda: ed().verify_batch_packed(*(np.zeros((0, 32), np.uint8),) * 4))
    case("eddsa verify_batch_packed bad", lambda: ed().verify_batch_packed(arr(3, 32, "R"), arr(3, 32, "S"), arr(3, 32, "A"), arr(3, 31, "h")))
    case("eddsa verify_batch_packed strided", lambda: ed().verify_batch_packed(arr(6, 32, "R")[::2], arr(3, 32, "S", np.int32),
                                                                               arr(3, 32, "A").tolist(), arr(3, 32, "h")))
    case("eddsa verify_batch_packed rc", lambda: ed().verify_batch_packed(*(arr(1, 32, s) for s in "RSAh")), rcs=(nat.ERR_NO_DEVICE,))
    off3 = np.array([0, 3, 3, 10], np.uint64)
    case("eddsa verify_batch_msgs_packed", lambda: ed().verify_batch_msgs_packed(*(arr(3, 32, s) for s in "RSA"), arr(1, 10, "m")[0], off3),
         plan=((1, 0, 5),))
    case("eddsa verify_batch_msgs_packed int offsets", lambda: ed().verify_batch_msgs_packed(*(arr(3, 32, s) for s in "RSA"), list(range(10)), [0, 3, 3, 10]))
    case("eddsa verify_batch_msgs_packed empty msgs", lambda: ed().verify_batch_msgs_packed(*(arr(2, 32, s) for s in "RSA"), B(b""), np.zeros(3, np.uint64)))
    case("eddsa verify_batch_msgs_packed n=0", lambda: ed().verify_batch_msgs_packed(*(np.zeros((0, 32), np.uint8),) * 3, np.zeros(0, np.uint8), np.zeros(1, np.uint64)))
    case("eddsa verify_batch_msgs_packed bad shape", lambda: ed().verify_batch_msgs_packed(arr(2, 32, "R"), arr(3, 32, "S"), arr(2, 32, "A"), B(b""), np.zeros(3, np.uint64)))
    case("eddsa verify_batch_msgs_packed bad offsets", lambda: ed().verify_batch_msgs_packed(*(arr(2, 32, s) for s in "RSA"), arr(1, 4, "m")[0], np.array([0, 1, 3], np.uint64)))
    case("eddsa verify_batch_msgs_packed bad offsets n", lambda: ed().verify_batch_msgs_packed(*(arr(2, 32, s) for s in "RSA"), B(b""), np.zeros(2, np.uint64)))
    case("eddsa verify_batch_msgs_packed rc", lambda: ed().verify_batch_msgs_packed(*(arr(1, 32, s) for s in "RSA"), B(b"ab"), [0, 2]), rcs=(nat.ERR_ARG,))
    for gh in (True, False):
        forms = dict(messages=["abcd", b"\x01\x02", list(range(5)), "", bytearray(b"q"), [], "zz"],
                     sigs=[sig64.hex(), sig64, list(sig64), bytearray(sig64), sig64[::-1], sig64, sig64.hex().upper()],
                     pubs=[pub32.hex(), pub32, list(pub32), bytearray(pub32), pub32[::-1], pub32, pub32.hex()])
        case("eddsa verify_batch gpu_hash=%s" % gh, lambda gh=gh, f=forms: ed().verify_batch(f["messages"], f["sigs"], f["pubs"], gpu_hash=gh),
             plan=((1, 0, 2, 5),))
        case("eddsa verify_batch empty msgs gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch(["", b""], [sig64] * 2, [pub32] * 2, gh))
        case("eddsa verify_batch n=0 gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch([], [], [], gh))
        case("eddsa verify_batch sig size gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch(["ab", "cd"], [sig64, sig64[:63]], [pub32] * 2, gh))
        case("eddsa verify_batch pub size gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch(["ab"], [sig64], [pub32 + b"\x00"], gh))
        case("eddsa verify_batch sig before pub gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch(["ab"], [b"\x01"], [b"\x02"], gh))
        case("eddsa verify_batch bad msg gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch([5], [sig64], [pub32], gh))
        case("eddsa verify_batch bad msg bad sig gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch([5], [b"\x01"], [pub32], gh))
        case("eddsa verify_batch bad msg bad pub gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch([5], [sig64], [b"\x01"], gh))
        case("eddsa verify_batch rc gpu_hash=%s" % gh, lambda gh=gh: ed().verify_batch(["ab"], [sig64], [pub32], gh), rcs=(nat.ERR_CUDA,))
    for st in STATUSES:
        case("eddsa verify status %d" % st, lambda: ed().verify("abcd", sig64.hex(), pub32), plan=((st,),))
    case("eddsa sign_batch_packed", lambda: ed().sign_batch_packed(arr(3, 32, "k"), arr(1, 10, "m")[0], off3))
    case("eddsa sign_batch_packed want_pub", lambda: ed().sign_batch_packed(arr(3, 32, "k"), arr(1, 10, "m")[0], off3, want_pub=True))
    case("eddsa sign_batch_packed empty msgs", lambda: ed().sign_batch_packed(arr(2, 32, "k"), [], [0, 0, 0]))
    case("eddsa sign_batch_packed n=0", lambda: ed().sign_batch_packed(np.zeros((0, 32), np.uint8), B(b""), [0]))
    case("eddsa sign_batch_packed n=0 want_pub", lambda: ed().sign_batch_packed(np.zeros((0, 32), np.uint8), B(b""), [0], True))
    case("eddsa sign_batch_packed bad secrets", lambda: ed().sign_batch_packed(arr(2, 31, "k"), B(b""), [0, 0, 0]))
    case("eddsa sign_batch_packed bad offsets", lambda: ed().sign_batch_packed(arr(2, 32, "k"), B(b"abc"), [0, 1, 2]))
    case("eddsa sign_batch_packed unexpected", lambda: ed().sign_batch_packed(arr(2, 32, "k"), B(b"abc"), [0, 1, 3]), plan=((1, 0),))
    case("eddsa sign_batch_packed unexpected want_pub", lambda: ed().sign_batch_packed(arr(2, 32, "k"), B(b"abc"), [0, 1, 3], True), plan=((5,),))
    case("eddsa sign_batch_packed rc", lambda: ed().sign_batch_packed(arr(2, 32, "k"), B(b"abc"), [0, 1, 3]), rcs=(nat.ERR_ARG,))
    case("eddsa sign_batch", lambda: ed().sign_batch(["abcd", b"\x01\x02", list(range(5)), "", "zz"],
                                                     [pub32.hex(), pub32, list(pub32), bytearray(pub32), pub32[::-1]]))
    case("eddsa sign_batch empty msgs", lambda: ed().sign_batch(["", b""], [pub32] * 2))
    case("eddsa sign_batch n=0", lambda: ed().sign_batch([], []))
    case("eddsa sign_batch bad secret", lambda: ed().sign_batch(["ab", "cd"], [pub32, pub32[:31]]))
    case("eddsa sign_batch bad msg", lambda: ed().sign_batch([5], [pub32]))
    case("eddsa sign_batch bad msg bad secret", lambda: ed().sign_batch([5], [pub32[:3]]))
    case("eddsa sign_batch unexpected", lambda: ed().sign_batch(["ab"], [pub32]), plan=((0,),))
    case("eddsa sign", lambda: ed().sign("abcd", pub32.hex()))
    case("eddsa public_from_secret_batch", lambda: ed().public_from_secret_batch(arr(3, 32, "k")))
    case("eddsa public_from_secret_batch list", lambda: ed().public_from_secret_batch(arr(2, 32, "k").tolist()))
    case("eddsa public_from_secret_batch n=0", lambda: ed().public_from_secret_batch(np.zeros((0, 32), np.uint8)))
    case("eddsa public_from_secret_batch unexpected", lambda: ed().public_from_secret_batch(arr(1, 32, "k")), plan=((4,),))

    # -- ShortCurve
    curves = {"toy": (97, 2, 3), "k256": ("fffffffffffffffffffffffffffffffffffffffffffffffffffffffefffffc2f", 0, 7),
              "p521": (P["p521"], P["p521"] - 3, 2**520 + 5), "w576": (2**576 - 2**32 + 1, -1, [1, 2, 3])}
    for name, (p, a, b) in curves.items():
        cv = lambda p=p, a=a, b=b: ShortCurve(p, a, b)
        pp = ecm._bn(p)
        pts = [(1, 2), {"x": pp + 3, "y": "ff"}, (2**600, pp - 1), ("aa", b"\x01\x02"), (0, 0)]
        ks = [0, 1, "abcdef", b"\x02" * 70, 2**1000 + 1]
        case("ShortCurve %s mul_batch" % name, lambda cv=cv, pts=pts, ks=ks: cv().mul_batch(pts, ks), plan=((1, 7),))
        case("ShortCurve %s mul_batch small k" % name, lambda cv=cv, pts=pts: cv().mul_batch(pts, [0, 1, 2, 3, 4]))
        case("ShortCurve %s mul_add_batch" % name, lambda cv=cv, pts=pts, ks=ks: cv().mul_add_batch(pts, [1, 2, 3, 4, 5], pts[::-1], ks),
             plan=((7, 1, 1),))
        case("ShortCurve %s add_batch" % name, lambda cv=cv, pts=pts: cv().add_batch(pts, pts[::-1]), plan=((1, 1, 7),))
        case("ShortCurve %s dbl_batch" % name, lambda cv=cv, pts=pts: cv().dbl_batch(pts), plan=((1, 7),))
        case("ShortCurve %s validate_batch" % name, lambda cv=cv, pts=pts: cv().validate_batch(pts), plan=((1, 0, 0),))
        for m in ("mul_batch", "dbl_batch", "validate_batch"):
            case("ShortCurve %s %s n=0" % (name, m), lambda cv=cv, m=m: getattr(cv(), m)(*([[], []] if m == "mul_batch" else [[]])))
        for m in ("mul_add_batch", "add_batch"):
            case("ShortCurve %s %s n=0" % (name, m), lambda cv=cv, m=m: getattr(cv(), m)(*([[]] * (4 if m == "mul_add_batch" else 2))))
    toy = lambda: ShortCurve(97, 2, 3)
    case("ShortCurve None point", lambda: toy().mul_batch([(1, 2), None], [1, 2]))
    case("ShortCurve bad point before None", lambda: toy().add_batch([(1, 2, 3), None], [(1, 2), (1, 2)]))
    case("ShortCurve None before bad point", lambda: toy().add_batch([None, (1, 2, 3)], [(1, 2), (1, 2)]))
    case("ShortCurve None in p2", lambda: toy().mul_add_batch([(1, 2)], [1], [None], [2]))
    case("ShortCurve None in dbl", lambda: toy().dbl_batch([None]))
    case("ShortCurve None in validate", lambda: toy().validate_batch([(5, 5), None]))
    case("ShortCurve negative k", lambda: toy().mul_batch([(1, 2)], [-1]))
    case("ShortCurve negative k2", lambda: toy().mul_add_batch([(1, 2)], [1], [(1, 2)], [-1]))
    case("ShortCurve wide k", lambda: toy().mul_batch([(1, 2), (1, 2)], [1, 2**1024]))
    case("ShortCurve widest k", lambda: toy().mul_batch([(1, 2)], [2**1024 - 1]))
    case("ShortCurve wide k1", lambda: toy().mul_add_batch([(1, 2)], [2**1024], [(1, 2)], [1]))
    case("ShortCurve point before k", lambda: toy().mul_batch([None], [-1]))
    case("ShortCurve mul_add k lengths", lambda: toy().mul_add_batch([(1, 2), (3, 4)], [1, 2, 3], [(1, 2), (3, 4)], [4]))
    case("ShortCurve NEEDS_HOST mul", lambda: toy().mul_batch([(1, 2), (3, 4)], [1, 2]), plan=((1, 4),))
    case("ShortCurve NEEDS_HOST add", lambda: toy().add_batch([(1, 2)], [(3, 4)]), plan=((4,),))
    case("ShortCurve NEEDS_HOST dbl", lambda: toy().dbl_batch([(1, 2)]), plan=((4,),))
    case("ShortCurve NEEDS_HOST mul_add", lambda: toy().mul_add_batch([(1, 2)], [1], [(3, 4)], [2]), plan=((4,),))
    case("ShortCurve validate statuses", lambda: toy().validate_batch([(1, 2)] * 12), plan=(tuple(range(12)),))
    case("ShortCurve mul statuses", lambda: toy().mul_batch([(1, 2)] * 12, list(range(12))), plan=(tuple(range(12)),))
    case("ShortCurve rc", lambda: toy().dbl_batch([(1, 2)]), rcs=(nat.ERR_ARG,))
    case("ShortCurve device 2", lambda: ShortCurve(97, 2, 3, device=2).validate_batch([(1, 2)]))
    return cs


def api():
    """The public surface: inspect.signature of every public method, and each module's public names (plus the
    private names other modules import from ec.py)."""
    sigs = {}
    for cls in (EC, EDDSA, ShortCurve):
        for name, fn in sorted(vars(cls).items()):
            if callable(fn) and (not name.startswith("_") or name == "__init__"):
                sigs["%s.%s" % (cls.__name__, name)] = str(inspect.signature(fn))
    names = {}
    for mod in (ecm, edm, cvm):
        pub = [k for k, v in vars(mod).items() if not k.startswith("_") and not inspect.ismodule(v)
               and not ((inspect.isclass(v) or inspect.isfunction(v)) and v.__module__ != mod.__name__)]
        names[mod.__name__] = sorted(pub + (["_CURVES", "_THROW_MSG", "_bn", "_to_array"] if mod is ecm else []))
    return {"signatures": sigs, "names": names}


def record():
    out = []
    for name, fn, plan, rcs in corpus():
        for device_ok in (True, False):
            rec, _ = run_case(fn, plan, rcs, device_ok)
            out.append(dict(case=name, device=device_ok, **rec))
    return {"api": api(), "cases": out}


def _dump(rec):
    return gzip.compress(json.dumps(rec, sort_keys=True, separators=(",", ":")).encode(), 9, mtime=0)


def _golden():
    with gzip.open(GOLDEN) as f:
        return json.load(f)


# ---- tests ----------------------------------------------------------------------------------------------------------
def test_mirror_calls_match_the_recording():
    want = _golden()["cases"]
    got = json.loads(json.dumps(record()["cases"]))
    assert [(c["case"], c["device"]) for c in got] == [(c["case"], c["device"]) for c in want]
    for g, w in zip(got, want):
        assert g == w, "case %r (device %s) differs" % (g["case"], g["device"])


def test_mirror_public_surface_is_kept():
    want, got = _golden()["api"], api()
    assert got["signatures"] == want["signatures"]
    for mod, names in want["names"].items():
        assert set(names) <= set(got["names"][mod]), (mod, set(names) - set(got["names"][mod]))


def _pinned_inputs(rec_fake, names, arrays):
    seen = rec_fake.addrs[-1]
    return {k: seen[k] for k in names} == {k: a.ctypes.data for k, a in zip(names, arrays)}


def test_packed_entry_points_pass_the_callers_buffers_through():
    """bench.py hands these calls pinned host buffers; a copy would send the library down its pageable staging path."""
    e, r, s, q = arr(4, 32, "e"), arr(4, 32, "r"), arr(4, 32, "s"), arr(4, 33, "q")
    rec, fake = run_case(lambda: EC().verify_batch_packed(e, r, s, q, nat.PUB_SEC1_33))
    assert "raise" not in rec and _pinned_inputs(fake, ("e", "r", "s", "pub"), (e, r, s, q))

    R, S, A, m = arr(3, 32, "R"), arr(3, 32, "S"), arr(3, 32, "A"), arr(1, 10, "m")[0]
    off = np.array([0, 3, 3, 10], np.uint64)
    rec, fake = run_case(lambda: EDDSA().verify_batch_msgs_packed(R, S, A, m, off))
    assert "raise" not in rec and _pinned_inputs(fake, ("R", "S", "A", "msgs", "msg_off"), (R, S, A, m, off))

    k, x = arr(3, 32, "k"), arr(3, 32, "x")
    out, st = np.empty((3, 32), np.uint8), np.empty(3, np.uint8)
    res = []
    rec, fake = run_case(lambda: res.append(EC("curve25519").derive_batch_packed(k, x, out=out, status=st)))
    assert "raise" not in rec and _pinned_inputs(fake, ("priv", "pubx", "out", "status"), (k, x, out, st))
    assert res[0][0] is out and res[0][1] is st
    assert st.tolist() == [1, 1, 1] and out.any()


if __name__ == "__main__":
    if sys.argv[1:] != ["--regen"]:
        sys.exit("usage: python tests/test_mirror_calls.py --regen")
    with open(GOLDEN, "wb") as f:
        f.write(_dump(record()))
    print("wrote", GOLDEN)
