"""new elliptic.ec('ed25519') on the GPU -- the generic `describe('curve ed25519')` block of the reference's
test/ecdsa-test.js:17-130 and test/ecdh-test.js:26, through the reference-shaped host API, checked against the
oracle; plus the .curve batch entry points Point.mul / mulAdd on the Edwards preset and Point.mul on curve25519."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ENTROPY = list(range(1, 26))          # test/ecdsa-test.js:11-14


def test_reference_generic_block(native):
    from elliptic_b200.ec import EC as GpuEC
    from oracle.ref_py.ec import EC
    ec, gec = EC("ed25519"), GpuEC("ed25519")
    privs, pubs = gec.gen_key_pair_batch([ENTROPY])
    kp = ec.gen_key_pair(bytes(ENTROPY))
    q = ec.g.mul(kp.priv)
    assert privs[0] == kp.priv and pubs[0] == (q.get_x(), q.get_y())
    assert len("%064x" % privs[0]) == 64                                           # 'should generate proper key pair'
    msg = "deadbeef"
    sig = gec.sign(msg, privs[0])
    ref = ec.sign(msg, kp.priv)
    assert (sig["r"], sig["s"], sig["recoveryParam"]) == (ref.r, ref.s, ref.recovery_param)
    key = {"x": pubs[0][0], "y": pubs[0][1]}
    assert gec.verify(msg, sig, key) is True                                       # 'should sign and verify'
    can = gec.sign("hello", privs[0], canonical=True)
    assert can["s"] <= ec.n >> 1                                                   # 'signature.s <= keys.ec.nh'
    ksig = gec.sign(msg, privs[0], k=lambda it: 1358)                              # 'should support options.k'
    assert gec.verify(msg, ksig, key) is True
    rk = ec.sign(msg, kp.priv, k_fn=lambda it: 1358)
    assert (ksig["r"], ksig["s"]) == (rk.r, rk.s)
    s2 = gec.sign(msg, privs[0], pers="1234", pers_enc="hex")                      # 'another signature with pers'
    rp = ec.sign(msg, kp.priv, pers=bytes.fromhex("1234"))
    assert (s2["r"], s2["s"]) == (rp.r, rp.s) and (s2["r"], s2["s"]) != (sig["r"], sig["s"])
    # compact and full hex keys (decodePoint / pointFromX), DER signatures
    x, y = pubs[0]
    compact = ("03" if y & 1 else "02") + "%064x" % x
    full = "04" + "%064x%064x" % (x, y)
    from oracle.ref_py.signature import Signature
    der = Signature({"r": sig["r"], "s": sig["s"]}).to_der()
    for k in (compact, full):
        assert gec.verify(msg, sig, k, "hex") is True
        assert gec.verify(msg, bytes(der).hex(), k, "hex") is True
    wp, wq = gec.gen_key_pair_batch([bytes(range(40, 72))])                         # 'wrong public key'
    assert gec.verify(msg, sig, {"x": wq[0][0], "y": wq[0][1]}) is False


def test_verify_sign_batches_against_the_oracle(native):
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC as GpuEC, NeedsReferencePath
    from oracle.ref_py.ec import EC
    ec, gec = EC("ed25519"), GpuEC("ed25519")
    rnd = random.Random(77)
    n = 192
    privs = [rnd.randrange(1, ec.n) for _ in range(n)]
    msgs = [rnd.randrange(1 << 248) for _ in range(n)]
    r, s, rec = gec.sign_batch(msgs, privs)
    pubs = gec.g_mul_batch(privs)
    for i in range(0, n, 3):
        sg = ec.sign(msgs[i], privs[i])
        q = ec.g.mul(privs[i])
        assert (r[i], s[i], int(rec[i])) == (sg.r, sg.s, sg.recovery_param) and pubs[i] == (q.get_x(), q.get_y())
    sigs = [{"r": a, "s": b} for a, b in zip(r, s)]
    keys = [{"x": p[0], "y": p[1]} for p in pubs]
    assert (gec.verify_batch(msgs, sigs, keys) == 1).all()
    assert sum(1 for v in rec if v & 2) > n // 2                 # x(R) >= n for most items: eqXToP's candidate loop
    bad = [m ^ (1 << (i % 200)) for i, m in enumerate(msgs)]
    st = gec.verify_batch(bad, sigs, keys)
    assert [int(v) for v in st] == [int(ec.verify(bad[i], sigs[i], keys[i])) for i in range(n)] and not st.any()
    with pytest.raises(NeedsReferencePath):
        gec.verify(msgs[0], sigs[0], {"x": pubs[0][0], "y": (pubs[0][1] + 1) % (2**255 - 19)})
    # 2^16 sign -> verify round trip through the packed ABI
    lib = nat.init(0)
    m = 1 << 16
    rng = np.random.default_rng(5)
    e = rng.integers(0, 256, size=(m, 32), dtype=np.uint8); e[:, 0] = 0
    d = rng.integers(0, 256, size=(m, 32), dtype=np.uint8); d[:, 0] &= 0x0F; d[:, 31] |= 1
    rr = np.zeros((m, 32), np.uint8); ss = np.zeros((m, 32), np.uint8); rc = np.zeros(m, np.uint8); st = np.zeros(m, np.uint8)
    pub = np.zeros((m, 64), np.uint8)
    nat.check(lib.eb200_scalar_mul_batch(nat.CURVE_ED25519, m, d.ctypes.data, None, pub.ctypes.data, st.ctypes.data))
    assert (st == 1).all()
    nat.check(lib.eb200_ecdsa_sign_batch(nat.CURVE_ED25519, m, e.ctypes.data, d.ctypes.data, 0, rr.ctypes.data, ss.ctypes.data, rc.ctypes.data, st.ctypes.data))
    assert (st == 1).all()
    assert (gec.verify_batch_packed(e, rr, ss, pub) == 1).all()
    e[:, 9] ^= 4
    assert (gec.verify_batch_packed(e, rr, ss, pub) == 0).all()


def test_curve_api_mul_mul_add_and_ecdh(native):
    from elliptic_b200.ec import EC as GpuEC, EllipticError
    from oracle.ref_py.ec import EC, KeyPair
    from oracle.ref_py import curves
    ec, gec = EC("ed25519"), GpuEC("ed25519")
    rnd = random.Random(79)
    n = 96
    ds = [rnd.randrange(1, ec.n) for _ in range(n)]
    pts = gec.g_mul_batch(ds)
    k1 = [rnd.randrange(2**256) for _ in range(n)]
    k2 = [rnd.randrange(2**256) for _ in range(n)]
    k2[0], k2[1] = 0, ec.n
    got = gec.mul_add_batch(k1, pts, k2)
    mul = gec.mul_batch(pts, k2)
    for i in range(0, n, 2):
        P = ec.curve.point(pts[i][0], pts[i][1])
        w = ec.g.mul_add(k1[i], P, k2[i])
        assert got[i] == (w.get_x(), w.get_y())
        w = P.mul(k2[i])
        assert mul[i] == (w.get_x(), w.get_y())
    assert mul[0] == (0, 1) and mul[1] == (0, 1)                     # the neutral element is an ordinary point
    # ECDH (test/ecdh-test.js:26): both sides agree, and equal the oracle
    a, b = ds[:n // 2], ds[n // 2:]
    A, B = pts[:n // 2], pts[n // 2:]
    sa, st1 = gec.derive_batch(a, [{"x": q[0], "y": q[1]} for q in B])
    sb, st2 = gec.derive_batch(b, [{"x": q[0], "y": q[1]} for q in A])
    assert sa == sb and (st1 == 1).all() and (st2 == 1).all()
    assert sa[3] == KeyPair(ec, priv=a[3]).derive(ec.curve.point(B[3][0], B[3][1]))
    with pytest.raises(EllipticError, match="public point not validated"):
        gec.derive(a[0], {"x": B[0][0], "y": (B[0][1] + 1) % (2**255 - 19)})
    # curve25519: Point.mul on x-only points (test/curve-test.js:348-356: g.mul(6) KAT)
    c25 = curves.get("curve25519").curve
    g25 = GpuEC("curve25519")
    xs = [9, 9] + [rnd.randrange(2**255 - 19) for _ in range(30)]
    ks = [6, 0] + [rnd.randrange(2**256) for _ in range(30)]
    out = g25.x_mul_batch(xs, ks)
    assert out == [c25.point(xs[i], 1).mul(ks[i]).get_x() for i in range(32)]
    assert "%x" % out[0] == "26954ccdc99ebf34f8f1dde5e6bb080685fec73640494c28f9fe0bfa8c794531"
    with pytest.raises(EllipticError, match="Not supported on Montgomery curve"):
        g25.mul_add_batch([1], [(9, 0)], [2])
