"""Operands that drive the device field arithmetic into the paths uniform random inputs almost never reach.

Pure Python, shared by the host-emulation branch-quota test (tests/test_arith_cases.py) and the device tests
(tests/test_gpu_arith.py).  Every modulus the kernels reduce by is here: the seven coordinate primes, the six group
orders and the ed25519 group order l.  For each there are

- word patterns: every 32-bit limb drawn from WORDS;
- boundary values: 0, 1, 2, m-2, m-1, m, m+1, R-1, R-m, (m-1)/2, (m+1)/2, 2^(bits-1);
- CIOS extremes for the Montgomery products: a = R-1 against b in {m-1, m-2, word patterns below m};
- products aimed at the reductions' rare branches: pick a target residue t in a band, a random a, b = t a^-1 mod m,
  and keep the pair when the reduction's own integer model (classify) says it takes a branch whose quota is not met.

R is 2^(32 L) for the L limbs the device holds an element in.
"""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PRIMES = {
    "secp256k1": 2**256 - 2**32 - 977,
    "p256": 2**256 - 2**224 + 2**192 + 2**96 - 1,
    "p384": 2**384 - 2**128 - 2**96 + 2**32 - 1,
    "p521": 2**521 - 1,
    "p192": 2**192 - 2**64 - 1,
    "p224": 2**224 - 2**96 + 1,
    "25519": 2**255 - 19,
}
ORDERS = {
    "secp256k1": 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141,
    "p256": 0xFFFFFFFF00000000FFFFFFFFFFFFFFFFBCE6FAADA7179E84F3B9CAC2FC632551,
    "p384": int("FFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFC7634D81F4372DDF581A0DB248B0A77AECEC196ACCC52973", 16),
    "p521": int("1fffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffffa51868783bf2f966b7fcc0148f709a5d0"
                "3bb5c9b8899c47aebb6fb71e91386409", 16),
    "p192": 0xFFFFFFFFFFFFFFFFFFFFFFFF99DEF836146BC9B1B4D22831,
    "p224": 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFF16A2E0B8F03E13DD29455C5C2A3D,
    "ed25519": 2**252 + 27742317777372353535851937790883648493,
}
LIMBS = {"secp256k1": 8, "p256": 8, "p384": 12, "p521": 18, "p192": 6, "p224": 8, "25519": 8, "ed25519": 8}
# the curve id whose self-test hook serves the field (include/elliptic_b200.h)
CURVE_ID = {"secp256k1": 1, "p256": 2, "p384": 3, "25519": 4, "ed25519": 4, "p521": 6, "p192": 7, "p224": 8}
WORDS = (0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF)

# secp256k1 GLV constants of glv_split_odd (sc_k256.cuh): the reference's basis (curves.js) and the 2^384-scaled
# rounding constants
LAMBDA = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
G1 = 0x3086D221A7D46BCDE86C90E49284EB153DAA8A1471E8CA7FE893209A45DBB031
G2 = 0xE4437ED6010E88286F547FA90ABFE4C4221208AC9DF506C61571B4AE8AC47F71
A1 = 0x3086D221A7D46BCDE86C90E49284EB15
B1 = -0xE4437ED6010E88286F547FA90ABFE4C3
A2 = 0x114CA50F7A8E2F3F657C1108D9D44CFD8
B2 = A1


def radix(name):
    return 1 << (32 * LIMBS[name])


def modulus(name, scalar):
    return ORDERS[name] if scalar else PRIMES[name]


def word_patterns(nl, count, rnd, below=None):
    """`count` values whose limbs are all drawn from WORDS (below `below`, when given: the top limbs that `below`
    leaves empty stay zero, and values >= below are redrawn)."""
    bits = below.bit_length() if below else 32 * nl
    used = (bits + 31) // 32
    out = []
    while len(out) < count:
        v = sum(rnd.choice(WORDS) << (32 * i) for i in range(used)) & ((1 << bits) - 1)
        if below is None or v < below:
            out.append(v)
    return out


def boundary(m, nl):
    R = 1 << (32 * nl)
    vals = [0, 1, 2, m - 2, m - 1, m, m + 1, R - 1, R - m, (m - 1) // 2, (m + 1) // 2, 1 << (m.bit_length() - 1)]
    return sorted({v for v in vals if 0 <= v < R})


def cios_extremes(m, nl, rnd, count=64):
    """(a, b) pairs for a b R^-1 with a = R - 1, the largest multiplicand the product accepts."""
    R = 1 << (32 * nl)
    bs = [m - 1, m - 2] + word_patterns(nl, count, rnd, below=m)
    return [(R - 1, b) for b in bs]


# ---- integer models of the reductions: which branch does the product a * b take? ------------------------------
def _solinas_model(name):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_solinas as g
    cfg = g.P256 if name == "p256" else g.P384
    nl = cfg["N"]
    cols = g.columns(cfg)
    K = sum(d << (32 * j) for j, d in cfg["K"].items())
    R = 1 << (32 * nl)
    p = PRIMES[name]

    def model(v):
        """The generated column reduction followed by sp_final_rare (fp_special.cuh), step by step."""
        c = [(v >> (32 * i)) & 0xFFFFFFFF for i in range(2 * nl)]
        tot = sum(coef * c[i] << (32 * j) for j, col in enumerate(cols) for i, coef in col.items())
        top, w = tot >> (32 * nl), tot & (R - 1)
        v2 = w + top * K
        top2 = v2 >> (32 * nl)
        v3 = (v2 & (R - 1)) + top2 * K
        taken = set()
        if top2 == 1:
            taken.add("fold_up")
        if top2 == -1:
            taken.add("fold_down")
        if v3 >> (32 * (nl - 1)) == 0xFFFFFFFF:
            taken.add("final_taken" if v3 >= p else "final_screened")
        return taken, v3 - p if v3 >= p else v3
    return model


def _p521_model(v):
    """RedP521::reduce: two folds of 2^521 = 1, then the word-15 screen for lo == p."""
    M = (1 << 521) - 1
    lo = (v & M) + (v >> 521)
    lo = (lo & M) + (lo >> 521)
    taken = set()
    if (lo >> 480) & 0xFFFFFFFF == 0xFFFFFFFF:
        taken.add("screen")
        if lo == M:
            taken.add("screen_zero")
    return taken, 0 if lo == M else lo


def _fold_model(c0, wrap_label):
    """fe_reduce512 (secp256k1, C = 2^32 + 977) and f25_reduce512 (25519, C = 38): lo + C hi, the top folded again,
    then one more fold of a wrap out of 2^256.  The result is weakly reduced, in [0, 2^256)."""
    R = 1 << 256

    def model(v):
        A = (v & (R - 1)) + c0 * (v >> 256)
        r1 = (A & (R - 1)) + c0 * (A >> 256)
        taken = set()
        if A >> 288:
            taken.add("a9")                  # fe_reduce512_ptx's A[9] branch (secp256k1 only)
        if r1 >> 256:
            taken.add(wrap_label)
        r = (r1 & (R - 1)) + c0 * (r1 >> 256)
        return taken, r
    return model


def _cios_model(m, nl):
    """Montgomery product T = (x y + q m) / R, q = -x y m^-1 mod R; the final subtraction fires when T >= m."""
    R = 1 << (32 * nl)
    minv = pow(-m, -1, R)

    def model(x, y):
        q = x * y * minv % R
        T = (x * y + q * m) // R
        return ({"final_taken"} if T >= m else set()), T - m if T >= m else T
    return model


def classify(name, a, b, scalar=False):
    """(set of rare branches taken, the reduction's output) for the device product of a and b as the self-test hook
    computes it: op 0 on the coordinate field (the hook converts plain a, b to the field's form first), op 16 on
    the scalar field (a b R^-1, operands as given)."""
    nl = LIMBS[name]
    if scalar:
        return _cios_model(ORDERS[name], nl)(a, b)
    p = PRIMES[name]
    if name in ("p256", "p384"):
        taken, out = _MODELS[name](a * b)
    elif name == "p521":
        taken, out = _p521_model(a * b)
    elif name == "secp256k1":
        taken, out = _MODELS[name](a * b)
        weak = "weak_ge_p" if out >= p else None
        taken = taken | ({weak} if weak else set())
    elif name == "25519":
        taken, out = _MODELS[name](a * b)
        if out >= 2 * p:
            taken.add("weak_ge_2p")
        elif out >= p:
            taken.add("weak_ge_p")
    else:                                    # p192, p224: CIOS on the Montgomery forms, then from_mont
        R = 1 << (32 * nl)
        taken, _ = _cios_model(p, nl)(a * R % p, b * R % p)
        out = a * b % p
    return taken, out


_MODELS = {}


def _init_models():
    if not _MODELS:
        _MODELS["p256"] = _solinas_model("p256")
        _MODELS["p384"] = _solinas_model("p384")
        _MODELS["secp256k1"] = _fold_model(2**32 + 977, "wrap")
        _MODELS["25519"] = _fold_model(38, "wrap")


# Branches a product of canonical operands can take, and the residue bands that lead there.  A branch missing from
# a field's list is unreachable for such products (see UNREACHABLE).
def _bands(name, scalar):
    m = modulus(name, scalar)
    nl = LIMBS[name]
    R = 1 << (32 * nl)
    if scalar:
        # T = a b R^-1 + m needs a b / R > t: small targets, large a (aimed_products draws a from [R/2, R))
        return {"final_taken": [(0, m // 4)]}
    if name == "p256":
        K = 2**224 - 2**192 - 2**96 + 1
        return {"fold_up": [(R - m, R - m + 4 * K)], "fold_down": [(m - 4 * K, m)],
                "final_taken": [(0, R - m)], "final_screened": [(R - 2**224, m)]}
    if name == "p384":
        K = 2**128 + 2**96 - 2**32 + 1
        return {"fold_up": [(R - m, R - m + 3 * K)], "final_taken": [(0, R - m)],
                "final_screened": [(R - 2**352, m)]}
    if name == "p521":
        return {"screen": [(2**512 - 2**480 + i * 2**512, 2**512 + i * 2**512) for i in range(2**9 - 1)]}
    if name == "secp256k1":
        # a wrap out of 2^256 leaves r1 - p in [C, C (top + 1)), top = A >> 256 < 2^34
        return {"weak_ge_p": [(1, R - m)], "wrap": [(R - m, 2**66)]}
    if name == "25519":
        return {"weak_ge_p": [(0, m)], "weak_ge_2p": [(0, R - 2 * m)]}
    if name == "p192":
        return {"final_taken": [(0, m)]}
    # p224 (see MONT_TARGET): T = c + p when the Montgomery result c is below x y / R, which reaches 2^192
    return {"final_taken": [(1, 2**180)]}


# Coordinate fields held in Montgomery form: their bands are for the multiplier's result c = x y R^-1, so the plain
# residue to aim at is c R^-1.  On p224, p < R 2^-32 makes T = (x y + q p) / R < p (1 + 2^-32): T >= p needs x y >= R
# with a small result, which uniform residues hit with probability 2^-32 and this band hits about half the time.
MONT_TARGET = {"p224"}


def quota_branches(name, scalar):
    """The branches aimed_products fills a quota for."""
    return sorted(_bands(name, scalar))


# Why the remaining branches cannot be reached by a product of canonical operands (tests assert it on every case):
UNREACHABLE = {
    # p384's column sums put top in [-1, 3], and a negative top cannot meet a low part below K: no downward wrap
    ("p384", "fold_down"): "top >= -1 and w + top K >= 0 for every product",
    # lo == p needs a b = 0 (mod p) with a nonzero double-width value; a, b < p makes a b = 0 only when one is 0, and
    # then every word is 0.  The screen's zeroing is reached by to_mont(p) instead (a raw input equal to p).
    ("p521", "screen_zero"): "a b = 0 mod p only for a = 0 or b = 0, whose product folds to 0, not p",
}

def aimed_products(name, scalar, quota, rnd, max_tries=200000):
    """{branch: [(a, b), ...]} with `quota` canonical pairs per reachable branch, each verified by classify()."""
    _init_models()
    m = modulus(name, scalar)
    R = radix(name)
    bands = _bands(name, scalar)
    got = {br: [] for br in bands}
    for _ in range(max_tries):
        open_ = [br for br in bands if len(got[br]) < quota]
        if not open_:
            break
        lo, hi = rnd.choice(bands[rnd.choice(open_)])
        t = rnd.randrange(lo, hi)
        a = rnd.randrange(R // 2, R) if scalar else rnd.randrange(1, m)
        if scalar and a % m == 0:
            continue
        # raw Montgomery product: a b R^-1 = t  ->  b = t R a^-1
        if name in MONT_TARGET and not scalar:
            t = t * pow(R, -1, m) % m          # plain a b whose Montgomery product (a R)(b R) R^-1 is t
        b = t * (R if scalar else 1) * pow(a, -1, m) % m
        taken, _ = classify(name, a, b, scalar)
        for br in taken:
            if br in got and len(got[br]) < quota:
                got[br].append((a, b))
    return got


def fields():
    """(name, scalar) of every field the hooks serve: 7 coordinate fields and 7 scalar fields."""
    return [(n, False) for n in PRIMES] + [(n, True) for n in ORDERS]


def operand_pairs(name, scalar, rnd, n_patterns=200, quota=64):
    """The structured (a, b) pairs of one field: boundary x boundary, patterns x patterns, CIOS extremes (scalar
    fields) and aimed products.  a may reach R - 1 where the op allows it; b < m except in the boundary cross."""
    m = modulus(name, scalar)
    nl = LIMBS[name]
    edge = boundary(m, nl)
    pats = word_patterns(nl, n_patterns // 2, rnd) + word_patterns(nl, n_patterns - n_patterns // 2, rnd, below=m)
    pairs = [(x, y) for x in edge for y in edge]
    pairs += [(pats[i], pats[(7 * i + 3) % len(pats)]) for i in range(len(pats))]
    pairs += [(x, y) for x in pats[:16] for y in edge]
    if scalar:
        pairs += cios_extremes(m, nl, rnd)
    for br, ps in aimed_products(name, scalar, quota, rnd).items():
        pairs += ps
    return pairs


# ---- secp256k1 GLV split, restated ----------------------------------------------------------------------------
def glv_split_odd(k):
    """glv_split_odd (sc_k256.cuh) on Python ints: (k1, k2), both odd, k1 + k2 lambda = k (mod n)."""
    c1 = (k * G1 + (1 << 383)) >> 384
    c2 = (k * G2 + (1 << 383)) >> 384
    k1 = k - c1 * A1 - c2 * A2
    k2 = -c1 * B1 - c2 * B2
    if k1 % 2 == 0:
        if k1 >= 0:
            k1, k2 = k1 - A1, k2 - B1
        else:
            k1, k2 = k1 + A1, k2 + B1
    if k2 % 2 == 0:
        if k1 >= 0:
            k1, k2 = k1 - A2, k2 - B2
        else:
            k1, k2 = k1 + A2, k2 + B2
    return k1, k2


def glv_cases(rnd, n_random=20000, keep=64):
    """Scalars for the split: small and special values, the k on each side of the rounding boundaries of c1 and c2
    (k g mod 2^384 straddling 2^383), and the k with the largest |k1| and |k2| among all of these and n_random
    random scalars."""
    n = ORDERS["secp256k1"]
    ks = [0, 1, 2, 3, n - 1, n - 2, LAMBDA, LAMBDA - 1, LAMBDA + 1, (n - 1) // 2, (n + 1) // 2]
    # (j + 1/2) 2^384 / g: the smallest k with k g / 2^384 past j + 1/2, and the one before it, so the rounding of c
    # flips between the two.  k g then lies within g < 2^256 of the boundary; a lattice solve over all k < n could
    # bring it to about 2^384 / n = 2^128, but the straddle is what the rounding sees
    for g in (G1, G2):
        top = n * g >> 384
        for _ in range(200):
            j = rnd.randrange(top)
            k = (((2 * j + 1) << 383) + g - 1) // g
            ks += [k, k - 1]
    cand = ks + [rnd.randrange(n) for _ in range(n_random)]
    split = [(k, glv_split_odd(k)) for k in cand]
    big1 = sorted(split, key=lambda s: -abs(s[1][0]))[:keep]
    big2 = sorted(split, key=lambda s: -abs(s[1][1]))[:keep]
    return sorted({k for k in ks} | {s[0] for s in big1 + big2})
