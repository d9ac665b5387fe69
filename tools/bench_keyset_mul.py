"""Time keyed against unkeyed Point.mul, G.mulAdd and ECDH derive on one GPU and print one JSON line.

Per shape, m keys are made on the GPU and n items get a random key index and random full-width scalars; the set is
created at the given table width, and each keyed call (eb200_scalar_mul_batch_keyed, eb200_mul_add_batch_keyed,
eb200_ecdh_derive_batch_keyed) and its unkeyed twin (keys gathered) are called alternately on the same inputs after a
warm-up; medians of --reps rounds are reported.  main_kernel_ms comes from eb200_last_timing() (the span of the chunks'
main kernels, which takes in the scalar prep and normalisation of every chunk but the last), wall_ms includes the
copies, create_ms is the median wall time of three eb200_keyset_create calls after a warm-up one.  Outputs and statuses
of the two calls are asserted equal in every round.  norm_kernel_ms (the batched normalisation, summed over a call's
chunks) comes from a separate torch.profiler pass over --reps keyed calls.  break_even_per_key: the scalars per key at
which create + keyed calls beat the unkeyed calls by wall time (null when keyed is not faster).

    python tools/bench_keyset_mul.py [--reps 10] [--warmup 2] [--out FILE]
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
SHAPES = [("secp256k1", 1, 32, 1 << 20, 4096, W) for W in (4, 6, 8)] + [("p256", 2, 32, 1 << 20, 4096, W) for W in (4, 6, 8)] + [
    ("p384", 3, 48, 1 << 18, 1024, 6)]
OPS = ("mul", "mul_add", "derive")


def gpu_query():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        return out[0].strip(), float(out[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None, None


def call(lib, nat, op, keyed, h_or_cid, n, k1, k2, idx, pts, out, st):
    if keyed:
        fn = {"mul": lib.eb200_scalar_mul_batch_keyed, "mul_add": lib.eb200_mul_add_batch_keyed,
              "derive": lib.eb200_ecdh_derive_batch_keyed}[op]
        args = (k1, k2, idx) if op == "mul_add" else (k2, idx)
    else:
        fn = {"mul": lib.eb200_scalar_mul_batch, "mul_add": lib.eb200_mul_add_batch, "derive": lib.eb200_ecdh_derive_batch}[op]
        args = (k1, k2, pts) if op == "mul_add" else (k2, pts)
    nat.call(fn, h_or_cid, n, *args, out, st)


def norm_ms(lib, nat, op, h, n, k1, k2, idx, out, st, reps):
    """Median over `reps` keyed calls of the normalisation kernels' device time per call (torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call(lib, nat, op, True, h, n, k1, k2, idx, None, out, st)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if "keyed_norm_kernel" in e.name), key=lambda e: e.time_range.start)
    if not ev or len(ev) % reps:
        return None
    per = len(ev) // reps
    return float(np.median([sum(e.time_range.elapsed_us() for e in ev[r * per:(r + 1) * per]) for r in range(reps)]) / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    name, watts = gpu_query()
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps, "shapes": []}
    for curve, cid, ln, n, m, W in SHAPES:
        rng = np.random.default_rng(cid * 1000 + W)
        d = rng.integers(0, 256, size=(m, ln), dtype=np.uint8)
        xy, kst = np.zeros((m, 2 * ln), np.uint8), np.zeros(m, np.uint8)
        nat.call(lib.eb200_scalar_mul_batch, cid, m, d, None, xy, kst)
        idx = rng.integers(0, m, size=n).astype(np.uint32)
        pts = np.ascontiguousarray(xy[idx])
        k1, k2 = (rng.integers(0, 256, size=(n, ln), dtype=np.uint8) for _ in range(2))
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
        row = {"curve": curve, "items": n, "keys": m, "table_bits": W, "device_bytes": db.value, "create_ms": create_ms}
        for op in OPS:
            ol = ln if op == "derive" else 2 * ln
            ok, ou = np.zeros((n, ol), np.uint8), np.zeros((n, ol), np.uint8)
            sk, su = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
            rows = {True: [], False: []}
            for rep in range(a.warmup + a.reps):
                for keyed in (True, False):
                    t = time.perf_counter()
                    call(lib, nat, op, keyed, h if keyed else cid, n, k1, k2, idx, pts, ok if keyed else ou, sk if keyed else su)
                    wall = (time.perf_counter() - t) * 1e3
                    if rep >= a.warmup:
                        rows[keyed].append((nat.last_timing()["main_kernel_ms"], wall))
                assert (sk == su).all() and (ok == ou).all() and (sk == nat.ST_TRUE).all()
            med = lambda keyed, j: float(np.median([x[j] for x in rows[keyed]]))
            gain = (med(False, 1) - med(True, 1)) / n          # wall ms saved per item
            row[op] = {"keyed_main_kernel_ms": med(True, 0), "unkeyed_main_kernel_ms": med(False, 0),
                       "keyed_wall_ms": med(True, 1), "unkeyed_wall_ms": med(False, 1),
                       "main_kernel_speedup": med(False, 0) / med(True, 0),
                       "norm_kernel_ms": norm_ms(lib, nat, op, h, n, k1, k2, idx, ok, sk, a.reps),
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
