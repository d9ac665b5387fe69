"""Time keyed against unkeyed getKeyRecoveryParam on one GPU and print one JSON line.

Per shape, m keys are made on the GPU and n items are GPU signatures by keys picked at random (the workload of a signer
that does not report the recovery bit: every item recovers).  The set is created at the given table width, and the keyed
call (eb200_ecdsa_recovery_param_batch_keyed) and its unkeyed twin (eb200_ecdsa_recovery_param_batch, keys gathered)
are called alternately on the same inputs after a warm-up; medians of --reps rounds are reported.  recid and statuses of
the two calls are asserted equal, and equal to the signer's recid, in every round.  wall_ms includes the copies.
Kernel times come from a separate torch.profiler pass over --reps calls of each, summed per call over its chunks:
main_kernel_ms is the keyed main kernel against the unkeyed main kernel (each call's prep and cold kernels are
listed apart), norm_kernel_ms the recid normalisation.  create_ms is the median wall time of three eb200_keyset_create
calls after a warm-up one; break_even_per_key: the items per key at which create + keyed calls beat the unkeyed calls by
wall time (null when keyed is not faster).

    python tools/bench_keyset_recovery_param.py [--reps 10] [--warmup 2] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (curve, id, len, items, keys, width)
SHAPES = ([("secp256k1", 1, 32, 1 << 20, 4096, W) for W in (4, 6, 8)] + [("p256", 2, 32, 1 << 20, 4096, W) for W in (4, 6, 8)] +
          [("p384", 3, 48, 1 << 18, 4096, 6), ("p521", 6, 66, 1 << 18, 4096, 6)])


def gpu_query():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        return out[0].strip(), float(out[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None, None


def kernel_kind(name):
    if "recid_norm_kernel" in name:
        return "norm"
    if "recovery_param_keyed_kernel" in name:
        return "keyed_main"
    if "prep_recovery_param_kernel" in name:
        return "prep"
    if "recovery_param_cold" in name:
        return "cold"
    if "recovery_param_kernel" in name:
        return "unkeyed_main"
    return None


def kernel_ms(fn, reps):
    """Median over `reps` calls of fn() of each kernel kind's device time per call (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        k = kernel_kind(e.name)
        if k:
            per.setdefault(k, []).append(e.time_range.elapsed_us())
    return {k: float(np.sum(v) / reps / 1e3) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    from elliptic_b200 import _native as nat
    from oracle.ref_py.ec import EC
    lib = nat.init(0)
    name, watts = gpu_query()
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps, "shapes": []}
    for curve, cid, ln, n, m, W in SHAPES:
        order = EC(curve).n
        rng = np.random.default_rng(cid * 1000 + W)
        d = np.frombuffer(b"".join((int.from_bytes(rng.bytes(ln + 8), "big") % (order - 1) + 1).to_bytes(ln, "big")
                                   for _ in range(m)), np.uint8).reshape(m, ln)
        xy, kst = np.zeros((m, 2 * ln), np.uint8), np.zeros(m, np.uint8)
        nat.call(lib.eb200_scalar_mul_batch, cid, m, d, None, xy, kst)
        idx = rng.integers(0, m, size=n).astype(np.uint32)
        e = rng.integers(0, 256, size=(n, ln), dtype=np.uint8)
        e[:, 0] = 0                                   # e < n
        r, s, rec, st = np.zeros((n, ln), np.uint8), np.zeros((n, ln), np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        nat.call(lib.eb200_ecdsa_sign_batch, cid, n, e, np.ascontiguousarray(d[idx]), 0, r, s, rec, st)
        q = np.ascontiguousarray(xy[idx])
        h = ctypes.c_void_p()
        creates = []
        for rep in range(4):                          # the first create of a shape is a warm-up
            if h.value:
                nat.check(lib.eb200_keyset_destroy(h))
            t = time.perf_counter()
            nat.check(lib.eb200_keyset_create(cid, m, xy.ctypes.data, 0, W, kst.ctypes.data, ctypes.byref(h)))
            creates.append((time.perf_counter() - t) * 1e3)
        create_ms = float(np.median(creates[1:]))
        assert (kst == 1).all()
        db = ctypes.c_size_t()
        nat.check(lib.eb200_keyset_info(h, None, None, None, ctypes.byref(db)))
        rk, ru = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        sk, su = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        keyed = lambda: nat.call(lib.eb200_ecdsa_recovery_param_batch_keyed, h, n, e, r, s, idx, rk, sk)
        unkeyed = lambda: nat.call(lib.eb200_ecdsa_recovery_param_batch, cid, n, e, r, s, q, ru, su)
        walls = {True: [], False: []}
        for rep in range(a.warmup + a.reps):
            for is_keyed in (True, False):
                t = time.perf_counter()
                (keyed if is_keyed else unkeyed)()
                if rep >= a.warmup:
                    walls[is_keyed].append((time.perf_counter() - t) * 1e3)
            assert (sk == su).all() and (rk == ru).all() and (sk == nat.ST_TRUE).all() and (rk == rec).all()
        kk, ku = kernel_ms(keyed, a.reps), kernel_ms(unkeyed, a.reps)
        wk, wu = float(np.median(walls[True])), float(np.median(walls[False]))
        gain = (wu - wk) / n                          # wall ms saved per item
        row = {"curve": curve, "items": n, "keys": m, "table_bits": W, "device_bytes": db.value, "create_ms": create_ms,
               "keyed_main_kernel_ms": kk.get("keyed_main"), "unkeyed_main_kernel_ms": ku.get("unkeyed_main"),
               "main_kernel_speedup": ku.get("unkeyed_main") / kk.get("keyed_main"),
               "norm_kernel_ms": kk.get("norm"), "keyed_prep_ms": kk.get("prep"), "keyed_cold_ms": kk.get("cold"),
               "unkeyed_prep_ms": ku.get("prep"), "unkeyed_cold_ms": ku.get("cold"),
               "keyed_wall_ms": wk, "unkeyed_wall_ms": wu, "wall_speedup": wu / wk,
               "break_even_per_key": (create_ms / m / gain) if gain > 0 else None}
        nat.check(lib.eb200_keyset_destroy(h))
        res["shapes"].append(row)
        print(json.dumps(row), file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
