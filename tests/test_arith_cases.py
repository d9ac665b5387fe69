"""The operand generator of tests/arith_cases.py on the CPU: every rare reduction branch gets its quota of products of
canonical operands (checked with the reduction's integer model), the branches no product can reach are shown
unreachable on every case, and the host-emulation builds of the field products agree with Python integers on the
same cases.  The device runs the same cases in tests/test_gpu_arith.py."""
import ctypes
import random

import pytest

import arith_cases as ac
from test_hostemu_k256 import he  # noqa: F401  (the host-emulation library fixture)

QUOTA = 50


def L(x, k):
    return (ctypes.c_uint32 * k)(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(k)])


def I(a, k):
    return sum(int(a[i]) << (32 * i) for i in range(k))


def test_moduli_match_the_oracle():
    from oracle.ref_py import curves
    for name in ("secp256k1", "p256", "p384", "p521", "p192", "p224"):
        c = curves.get(name)
        assert (c.curve.p, c.n) == (ac.PRIMES[name], ac.ORDERS[name]), name
    ed = curves.get("ed25519")
    assert (ed.curve.p, ed.n) == (ac.PRIMES["25519"], ac.ORDERS["ed25519"])


@pytest.mark.parametrize("name,scalar", ac.fields(), ids=lambda v: str(v))
def test_every_rare_branch_gets_its_quota(name, scalar):
    m = ac.modulus(name, scalar)
    got = ac.aimed_products(name, scalar, QUOTA, random.Random(hash((name, scalar)) & 0xFFFF))
    for br in ac.quota_branches(name, scalar):
        assert len(got[br]) >= QUOTA, (name, scalar, br, len(got[br]))
        for a, b in got[br]:
            assert b < m and (scalar or a < m)
            taken, out = ac.classify(name, a, b, scalar)
            assert br in taken
            R = ac.radix(name)
            assert out % m == (a * b * pow(R, -1, m) if scalar else a * b) % m
    # the branches no product of canonical operands can take: never taken by any case of this field
    rnd = random.Random(5)
    pairs = ac.operand_pairs(name, scalar, rnd, n_patterns=64, quota=8)
    pairs += [(rnd.randrange(m), rnd.randrange(m)) for _ in range(2000)]
    for (field, br), why in ac.UNREACHABLE.items():
        if field != name or scalar:
            continue
        for a, b in pairs:
            if a < m and b < m:
                assert br not in ac.classify(name, a, b)[0], (why, hex(a), hex(b))


def test_p521_screen_zero_is_reached_by_a_raw_input():
    """The lo == p zeroing of RedP521 is unreachable from canonical products, and to_mont(p) is what reaches it."""
    p = ac.PRIMES["p521"]
    assert ac._p521_model(p) == ({"screen", "screen_zero"}, 0)


@pytest.mark.parametrize("name,scalar", [(n, s) for n, s in ac.fields() if not s or n == "secp256k1"],
                         ids=lambda v: str(v))
def test_host_emulation_matches_integers_on_the_cases(he, name, scalar):  # noqa: F811
    """The portable C++ products (tests/hostemu) on the same cases: the reduction's output itself where it is weakly
    reduced (secp256k1, 25519), the canonical residue otherwise."""
    ac._init_models()
    nl = ac.LIMBS[name]
    m = ac.modulus(name, scalar)
    pairs = [(a, b) for a, b in ac.operand_pairs(name, scalar, random.Random(9), n_patterns=64, quota=QUOTA)
             if (a < m or scalar) and b < m]
    assert len(pairs) > 100
    for a, b in pairs:
        out = (ctypes.c_uint32 * nl)()
        if scalar:
            he.he_sc_mont_mul(L(a, 8), L(b, 8), out)
        elif name == "secp256k1":
            he.he_fe_op(0, L(a, 8), L(b, 8), out)
        elif name == "25519":
            he.he_f25_op(0, L(a, 8), L(b, 8), out)
        else:
            he.he_sw_fe_op(ac.CURVE_ID[name], 0, L(a, nl), L(b, nl), out)
        got = I(out, nl)
        assert got == ac.classify(name, a, b, scalar)[1], (name, hex(a), hex(b), hex(got))
