"""Time EC.getKeyRecoveryParam on one GPU and print one JSON line.

Per curve (secp256k1 and p256 at N = 2^20, p384 at 2^18) the items are valid signatures made by
eb200_ecdsa_sign_batch, with their keys from eb200_scalar_mul_batch, so j is mixed as signing leaves it.  Three calls
are timed, alternated in one process after a warm-up, and the median of --reps rounds is reported:
  recovery_param : eb200_ecdsa_recovery_param_batch
  composed       : the same answer from eb200_ecdsa_recover_batch at j = 0, then at j = 1 on the items still
                   unmatched, with a numpy comparison against Q (what a caller without the new call does)
  verify         : eb200_ecdsa_verify_batch on the same items, as the yardstick
main_kernel_ms comes from eb200_last_timing() (summed over the composition's two calls); wall_ms includes the copies.
Every round's answers are checked against the signer's recovery parameters.

    python tools/bench_recovery_param.py [--reps 10] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = [("secp256k1", 1, 32, 1 << 20), ("p256", 2, 32, 1 << 20), ("p384", 3, 48, 1 << 18)]


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def items(lib, nat, cid, ln, n, seed):
    rng = np.random.default_rng(seed)
    e = rng.integers(0, 256, size=(n, ln), dtype=np.uint8)
    d = rng.integers(0, 256, size=(n, ln), dtype=np.uint8)
    e[:, 0] &= 0x7F                                       # below n on these three curves
    d[:, 0] &= 0x7F
    d[:, -1] |= 1
    r, s = np.zeros((n, ln), np.uint8), np.zeros((n, ln), np.uint8)
    rec, st = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    nat.check(lib.eb200_ecdsa_sign_batch(cid, n, e.ctypes.data, d.ctypes.data, 0, r.ctypes.data, s.ctypes.data,
                                         rec.ctypes.data, st.ctypes.data))
    q = np.zeros((n, 2 * ln), np.uint8)
    nat.check(lib.eb200_scalar_mul_batch(cid, n, d.ctypes.data, None, q.ctypes.data, st.ctypes.data))
    assert (st == nat.ST_TRUE).all()
    return e, r, s, q, rec


def timed(fn):
    t = time.perf_counter()
    out = fn()
    wall = (time.perf_counter() - t) * 1e3
    return out, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from elliptic_b200 import _native as nat
    if not torch.cuda.is_available():
        sys.exit("bench_recovery_param: no CUDA device")
    lib = nat.init(0)
    res = {"metric": "EC.getKeyRecoveryParam batch: new call vs composed recover calls vs verify",
           "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "reps": a.reps, "warmup": a.warmup,
           "statistic": "median", "curves": {}}
    for name, cid, ln, n in SIZES:
        e, r, s, q, rec = items(lib, nat, cid, ln, n, seed=cid)
        rid, st = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        out, sj = np.zeros((n, 2 * ln), np.uint8), np.zeros(n, np.uint8)
        vst = np.zeros(n, np.uint8)
        zeros, ones = np.zeros(n, np.uint8), np.ones(n, np.uint8)

        def new():
            nat.check(lib.eb200_ecdsa_recovery_param_batch(cid, n, e.ctypes.data, r.ctypes.data, s.ctypes.data, q.ctypes.data,
                                                           rid.ctypes.data, st.ctypes.data))
            return [nat.last_timing()["main_kernel_ms"]], np.where(st == nat.ST_TRUE, rid, 255)

        def composed():
            ks = []
            nat.check(lib.eb200_ecdsa_recover_batch(cid, n, e.ctypes.data, r.ctypes.data, s.ctypes.data, zeros.ctypes.data,
                                                    out.ctypes.data, sj.ctypes.data))
            ks.append(nat.last_timing()["main_kernel_ms"])
            ans = np.full(n, 255, np.uint8)
            hit = (sj == nat.ST_TRUE) & (out == q).all(axis=1)
            ans[hit] = 0
            left = np.flatnonzero(~hit)
            if len(left):
                e1, r1, s1 = e[left], r[left], s[left]
                o1, t1 = np.zeros((len(left), 2 * ln), np.uint8), np.zeros(len(left), np.uint8)
                nat.check(lib.eb200_ecdsa_recover_batch(cid, len(left), e1.ctypes.data, r1.ctypes.data, s1.ctypes.data,
                                                        ones[:len(left)].ctypes.data, o1.ctypes.data, t1.ctypes.data))
                ks.append(nat.last_timing()["main_kernel_ms"])
                ans[left[(t1 == nat.ST_TRUE) & (o1 == q[left]).all(axis=1)]] = 1
            return ks, ans

        def verify():
            nat.check(lib.eb200_ecdsa_verify_batch(cid, n, e.ctypes.data, r.ctypes.data, s.ctypes.data, q.ctypes.data,
                                                   nat.PUB_XY, vst.ctypes.data))
            return [nat.last_timing()["main_kernel_ms"]], vst.copy()

        rows = {"recovery_param": [], "composed_recover": [], "verify": []}
        for it in range(a.warmup + a.reps):
            for key, fn, want in (("recovery_param", new, rec), ("composed_recover", composed, rec),
                                  ("verify", verify, np.ones(n, np.uint8))):
                (ks, ans), wall = timed(fn)
                if not np.array_equal(ans, want):
                    sys.exit("bench_recovery_param: %s on %s disagrees with the signer" % (key, name))
                if it >= a.warmup:
                    rows[key].append((ks, wall))
        med = lambda xs: float(np.median(xs))
        cur = {"n": n, "recids": {str(j): int((rec == j).sum()) for j in range(4)}}
        for key, v in rows.items():
            cur[key] = {"main_kernel_ms": med([sum(k) for k, _ in v]), "wall_ms": med([w for _, w in v]),
                        "main_kernel_ms_min": float(min(sum(k) for k, _ in v)), "wall_ms_min": float(min(w for _, w in v))}
        one_recover = med([k[0] for k, _ in rows["composed_recover"]])        # one recover call over all N items
        cur["composed_recover"]["first_call_main_kernel_ms"] = one_recover
        cur["main_kernel_vs_one_recover"] = cur["recovery_param"]["main_kernel_ms"] / one_recover
        cur["main_kernel_vs_verify"] = cur["recovery_param"]["main_kernel_ms"] / cur["verify"]["main_kernel_ms"]
        cur["wall_vs_composed"] = cur["recovery_param"]["wall_ms"] / cur["composed_recover"]["wall_ms"]
        res["curves"][name] = cur
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
