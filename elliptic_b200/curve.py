"""Host-side mirror of `elliptic.curve.short` for the batch path (SURVEY 8f-4).

`ShortCurve(p, a, b)` corresponds to `new elliptic.curve.short({p, a, b})` (lib/elliptic/curve/short.js:10-24) with
parameters chosen at run time -- any odd prime p > 3 of up to 576 bits, e.g. the toy curve of the reference's own
test (test/curve-test.js:9-22).  Points are (x, y) pairs (ints / hex / byte arrays, as `curve.point(x, y)` takes
them); `None` stands for the point at infinity in results.  Every method takes and returns whole batches and runs
on the GPU (include/elliptic_b200.h: eb200_curve_*_batch); the named presets have their own tuned entry points in
elliptic_b200.ec.EC (mul_batch, mul_add_batch, g_mul_batch)."""
import numpy as np

from . import _native as nat
from .ec import EllipticError, NeedsReferencePath, _bn, _pack, _pack_points, _unpack


class ShortCurve:
    def __init__(self, p, a, b, device=0):
        self.p, self.a, self.b = _bn(p), _bn(a), _bn(b)
        if self.p <= 3 or self.p % 2 == 0:
            raise EllipticError("ShortCurve: p must be an odd prime > 3")
        if self.p.bit_length() > 576:
            raise EllipticError("ShortCurve: p wider than 576 bits is not supported")
        self.len = max(1, (self.p.bit_length() + 7) // 8)
        self._device = device
        self._pab = _pack([self.p, self.a % self.p, self.b % self.p], self.len)
        self._desc = nat.short_curve(self._pab)

    # ---- packing --------------------------------------------------------------------------------------------
    def _pts(self, pts):
        def finite(pt):
            if pt is None:
                raise EllipticError("the point at infinity is not accepted as a batch input")
            return pt
        return _pack_points(map(finite, pts), self.p, self.len)

    def _scalars(self, ks):
        vals = [_bn(k) for k in ks]
        if any(v < 0 for v in vals):
            raise EllipticError("negative scalars are not supported by the batch path")
        klen = max(1, max((v.bit_length() + 7) // 8 for v in vals)) if vals else 1
        if klen > 128:
            raise NeedsReferencePath("scalar wider than 1024 bits")
        return _pack(vals, klen), klen

    def _run(self, fn, n, *args):
        """fn(desc, n, *args, out_xy, status) -> the n result points (None = infinity)."""
        out = np.zeros((n, 2 * self.len), np.uint8); st = np.zeros(n, np.uint8)
        nat.call(fn, self._desc, n, *args, out, st)
        return _unpack(out, self.len, st, needs_host=True)

    # ---- batch entry points ---------------------------------------------------------------------------------
    def mul_batch(self, points, ks):
        """[curve.point(x, y).mul(k)] (short.js:422-432)."""
        lib = nat.init(self._device)
        pts = self._pts(points)
        k, klen = self._scalars(ks)
        return self._run(lib.eb200_curve_mul_batch, len(pts), k, klen, pts)

    def mul_add_batch(self, p1s, k1s, p2s, k2s):
        """[p1.mulAdd(k1, p2, k2)] = k1*p1 + k2*p2 (short.js:434-441)."""
        lib = nat.init(self._device)
        a, b = self._pts(p1s), self._pts(p2s)
        kk, klen = self._scalars(list(k1s) + list(k2s))
        n = len(a)
        return self._run(lib.eb200_curve_mul_add_batch, n, kk[:n], a, kk[n:], b, klen)

    def add_batch(self, p1s, p2s):
        """[p1.add(p2)] (short.js:365-392)."""
        lib = nat.init(self._device)
        a, b = self._pts(p1s), self._pts(p2s)
        return self._run(lib.eb200_curve_add_batch, len(a), a, b)

    def dbl_batch(self, points):
        """[p.dbl()] (short.js:394-412)."""
        lib = nat.init(self._device)
        a = self._pts(points)
        return self._run(lib.eb200_curve_dbl_batch, len(a), a)

    def validate_batch(self, points):
        """[curve.validate(p)] (short.js:206-216): booleans."""
        lib = nat.init(self._device)
        a = self._pts(points)
        st = np.zeros(len(a), np.uint8)
        nat.call(lib.eb200_curve_validate_batch, self._desc, len(a), a, st)
        return [bool(v) for v in st]
