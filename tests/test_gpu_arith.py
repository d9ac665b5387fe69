"""Device field arithmetic against Python integers on the operands of tests/arith_cases.py: word patterns, boundary
values, CIOS extremes and products aimed at every rare reduction branch, plus a uniform baseline, through the
self-test hook eb200_selftest_fe (ops in include/elliptic_b200.h).  These run the inline-PTX carry chains the kernels
execute, which the host-emulation tests do not."""
import random

import numpy as np
import pytest

import arith_cases as ac

pytestmark = pytest.mark.gpu

UNIFORM = 100000          # uniform pairs per field for the products
UNIFORM_OTHER = 1 << 14   # and for the other ops
N_INV = 256


def to_limbs(vals, nl):
    return np.frombuffer(b"".join(v.to_bytes(4 * nl, "little") for v in vals), "<u4").reshape(len(vals), nl).copy()


def from_limbs(arr):
    return [int.from_bytes(r.tobytes(), "little") for r in arr]


def hook(native, name, op, a, b):
    from elliptic_b200 import _native as nat
    nl = ac.LIMBS[name]
    A, B = to_limbs(a, nl), to_limbs(b, nl)
    out = np.zeros_like(A)
    nat.check(native.eb200_selftest_fe(ac.CURVE_ID[name], op, len(a), A.ctypes.data, B.ctypes.data, out.ctypes.data))
    return from_limbs(out)


def _pairs(name, scalar, seed):
    rnd = random.Random(seed)
    return ac.operand_pairs(name, scalar, rnd), rnd


@pytest.mark.parametrize("name", ["secp256k1", "25519"])
def test_weakly_reduced_fields(native, name):
    """secp256k1 and 25519 hold values weakly reduced: every result is < 2^256 and right mod p, and a product is
    exactly the value the reduction's integer model gives (so the rare wraps and the >= p outputs are checked)."""
    ac._init_models()
    p = ac.PRIMES[name]
    pairs, rnd = _pairs(name, False, 21)
    top = 1 << 256
    a = [x for x, _ in pairs] + [rnd.randrange(top) for _ in range(UNIFORM)]
    b = [y for _, y in pairs] + [rnd.randrange(top) for _ in range(UNIFORM)]
    got = hook(native, name, 0, a, b)
    for x, y, g in zip(a, b, got):
        assert g == ac.classify(name, x, y)[1], (name, hex(x), hex(y), hex(g))
    k = len(pairs) + UNIFORM_OTHER
    for op, fn in ((1, lambda x, y: x * x), (2, lambda x, y: x + y), (3, lambda x, y: x - y), (4, lambda x, y: -x)):
        for x, y, g in zip(a[:k], b[:k], hook(native, name, op, a[:k], b[:k])):
            assert g < top and g % p == fn(x, y) % p, (name, op, hex(x), hex(y), hex(g))
    for x, g in zip(a[:k], hook(native, name, 6, a[:k], b[:k])):
        assert g == x % p, (name, hex(x))
    for x, g in zip(a[:N_INV], hook(native, name, 7, a[:N_INV], b[:N_INV])):
        assert g < top and g % p == pow(x % p, p - 2, p), (name, hex(x))


@pytest.mark.parametrize("name", ["p256", "p384", "p521", "p192", "p224"])
def test_short_curve_coordinate_fields(native, name):
    """Canonical results for the products, the doubling's scaled products (3ab, 4ab, 8a^2, 2a as SW::dbl_inl calls
    them), add, sub, neg and inv; the cases include products that take the second fold of the p256 / p384
    reductions (both directions on p256), the final subtraction taken and screened, and the p521 lo == p screen."""
    p = ac.PRIMES[name]
    nl = ac.LIMBS[name]
    pairs, rnd = _pairs(name, False, 22)
    top = 1 << (32 * nl)
    a = [x for x, _ in pairs] + [rnd.randrange(top) for _ in range(UNIFORM)]
    b = [y for _, y in pairs] + [rnd.randrange(p) for _ in range(UNIFORM)]
    k = len(pairs) + UNIFORM_OTHER
    ops = ((0, lambda x, y: x * y), (1, lambda x, y: x * x), (2, lambda x, y: x + y), (3, lambda x, y: x - y),
           (4, lambda x, y: -x), (8, lambda x, y: 3 * x * y), (9, lambda x, y: 4 * x * y), (10, lambda x, y: 8 * x * x),
           (11, lambda x, y: 2 * x))
    for op, fn in ops:
        n = len(a) if op in (0, 1) else k
        for x, y, g in zip(a[:n], b[:n], hook(native, name, op, a[:n], b[:n])):
            assert g == fn(x, y) % p, (name, op, hex(x), hex(y), hex(g))
    for x, g in zip(a[:N_INV], hook(native, name, 7, a[:N_INV], b[:N_INV])):
        assert g == pow(x % p, p - 2, p), (name, hex(x))


@pytest.mark.parametrize("name", list(ac.ORDERS))
def test_scalar_fields(native, name):
    """The scalar field mod n (mod l for ed25519) on the Montgomery multiplier every verify, sign and recover uses:
    the raw product a b R^-1 with a up to R - 1 (exact and < n), Montgomery conversions, add, sub and the inverse.
    On secp256k1 these go through sc_mont_mul / sc_mont_inv, including the prep's extreme e = 2^256 - 1 times
    s^-1 for s near n."""
    n = ac.ORDERS[name]
    nl = ac.LIMBS[name]
    R = 1 << (32 * nl)
    Ri = pow(R, -1, n)
    pairs, rnd = _pairs(name, True, 23)
    pairs = [(x, y) for x, y in pairs if y < n]
    # e * s^-1 in the prep: e raw (any 256-bit value), s^-1 in Montgomery form
    pairs += [(e, pow(s, -1, n) * R % n) for e in (R - 1, R - 2, n, n - 1) for s in (n - 1, n - 2, 1, 2, (n + 1) // 2)]
    a = [x for x, _ in pairs] + [rnd.randrange(R) for _ in range(UNIFORM)]
    b = [y for _, y in pairs] + [rnd.randrange(n) for _ in range(UNIFORM)]
    for x, y, g in zip(a, b, hook(native, name, 16, a, b)):
        assert g == x * y * Ri % n, (name, hex(x), hex(y), hex(g))
    k = len(pairs) + UNIFORM_OTHER
    for x, g in zip(a[:k], hook(native, name, 17, a[:k], b[:k])):
        assert g == x * R % n, (name, "to_mont", hex(x))
    for x, g in zip(a[:k], hook(native, name, 18, a[:k], b[:k])):
        assert g == x * Ri % n, (name, "from_mont", hex(x))
    ca = [x % n for x in a[:k]]
    for op, fn in ((19, lambda x, y: x + y), (20, lambda x, y: x - y)):
        for x, y, g in zip(ca, b[:k], hook(native, name, op, ca, b[:k])):
            assert g == fn(x, y) % n, (name, op, hex(x), hex(y))
    inv_in = [0, 1, n - 1, n - 2, R % n, (n - 1) * R % n] + ca[:N_INV]
    for x, g in zip(inv_in, hook(native, name, 21, inv_in, inv_in)):
        assert g == pow(x * Ri % n, n - 2, n) * R % n, (name, "inv", hex(x))


def test_glv_split_on_the_device(native):
    """glv_split_odd on the device equals its Python restatement (arith_cases.glv_split_odd) on small and special
    scalars, on both sides of the rounding boundaries of c1 and c2, and on the scalars with the largest halves; the
    halves are odd, k1 + k2 lambda = k (mod n), and m = (|k| - 1) / 2 fits what its consumers budget: 131 bits in
    the keyed tables (keyset_plan.h) and the 33 four-bit windows of k256_dsm, whose top digit holds 3 bits.
    Observed maximum over these cases: |k1|, |k2| < 2^129, m < 2^128."""
    n = ac.ORDERS["secp256k1"]
    ks = ac.glv_cases(random.Random(31))
    out1 = hook(native, "secp256k1", 24, ks, ks)
    out2 = hook(native, "secp256k1", 25, ks, ks)
    mask = (1 << 160) - 1
    widest = 0
    for k, o1, o2 in zip(ks, out1, out2):
        m1, m2 = o1 & mask, o2 & mask
        n1, n2 = (o1 >> 160) & 0xFFFFFFFF, (o1 >> 192) & 0xFFFFFFFF
        assert ((o2 >> 160) & 0xFFFFFFFF, (o2 >> 192) & 0xFFFFFFFF) == (n1, n2) and o1 >> 224 == 0
        k1 = (2 * m1 + 1) * (-1 if n1 else 1)
        k2 = (2 * m2 + 1) * (-1 if n2 else 1)
        assert (k1, k2) == ac.glv_split_odd(k), hex(k)
        assert (k1 + k2 * ac.LAMBDA - k) % n == 0
        widest = max(widest, m1.bit_length(), m2.bit_length())
    assert widest <= 131 and widest <= 4 * 32 + 3, widest
