"""Time keyed against unkeyed ECDSA verify on one GPU and print one JSON line.

Per shape the items are valid signatures made by eb200_ecdsa_sign_batch over m keys (one in 64 damaged), the set is
created at the given table width, and eb200_ecdsa_verify_batch_keyed and eb200_ecdsa_verify_batch (keys gathered) are
called alternately on the same items after a warm-up; the median of --reps rounds is reported.  main_kernel_ms comes
from eb200_last_timing(); wall_ms includes the copies; create_ms is the wall time of eb200_keyset_create.  The statuses of
the two calls are asserted equal in every round.  break_even_sigs_per_key: the signatures per key at which create +
keyed verify beats unkeyed verify by wall time (null when keyed is not faster).

    python tools/bench_keyset.py [--reps 10] [--warmup 2] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (curve, id, len, items, keys, width)
SHAPES = [("secp256k1", 1, 32, 1 << 20, 4096, W) for W in (4, 6, 8)] + [("p256", 2, 32, 1 << 20, 4096, W) for W in (4, 6, 8)] + [
    ("p384", 3, 48, 1 << 18, 1024, 6), ("secp256k1", 1, 32, 1 << 20, 16, 8), ("secp256k1", 1, 32, 1 << 20, 1 << 16, 4),
    ("secp256k1", 1, 32, 1 << 20, 1 << 16, 8)]


def gpu_query():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        return out[0].strip(), float(out[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    from elliptic_b200 import _native as nat
    from gpu_keyset_items import gpu_items
    lib = nat.init(0)
    name, watts = gpu_query()
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps, "shapes": []}
    cache = {}
    for curve, cid, ln, n, m, W in SHAPES:
        if (cid, n, m) not in cache:
            cache.clear()
            cache[(cid, n, m)] = gpu_items(lib, nat, cid, ln, m, n, seed=cid * 1000 + m % 997)
        xy, e, r, s, idx = cache[(cid, n, m)]
        pub = np.ascontiguousarray(xy[idx])
        kst, h = np.zeros(m, np.uint8), ctypes.c_void_p()
        t = time.perf_counter()
        nat.check(lib.eb200_keyset_create(cid, m, xy.ctypes.data, 0, W, kst.ctypes.data, ctypes.byref(h)))
        create_ms = (time.perf_counter() - t) * 1e3
        build_kernel_ms = nat.last_timing()["kernel_ms"]
        db = ctypes.c_size_t()
        nat.check(lib.eb200_keyset_info(h, None, None, None, ctypes.byref(db)))
        sk, su = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        rows = {"keyed": [], "unkeyed": []}
        for rep in range(a.warmup + a.reps):
            for kind in ("keyed", "unkeyed"):
                t = time.perf_counter()
                if kind == "keyed":
                    nat.call(lib.eb200_ecdsa_verify_batch_keyed, h, n, e, r, s, idx, sk)
                else:
                    nat.call(lib.eb200_ecdsa_verify_batch, cid, n, e, r, s, pub, 0, su)
                wall = (time.perf_counter() - t) * 1e3
                if rep >= a.warmup:
                    rows[kind].append((nat.last_timing()["main_kernel_ms"], wall))
            assert (sk == su).all() and sk.sum() == n - (n + 63) // 64
        nat.check(lib.eb200_keyset_destroy(h))
        med = lambda kind, j: float(np.median([x[j] for x in rows[kind]]))
        gain = (med("unkeyed", 1) - med("keyed", 1)) / n            # wall ms saved per signature
        res["shapes"].append({
            "curve": curve, "items": n, "keys": m, "table_bits": W, "device_bytes": db.value, "create_ms": create_ms,
            "build_kernel_ms": build_kernel_ms,
            "keyed_main_kernel_ms": med("keyed", 0), "unkeyed_main_kernel_ms": med("unkeyed", 0),
            "keyed_wall_ms": med("keyed", 1), "unkeyed_wall_ms": med("unkeyed", 1),
            "main_kernel_speedup": med("unkeyed", 0) / med("keyed", 0),
            "break_even_sigs_per_key": (create_ms / m / gain) if gain > 0 else None})
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
