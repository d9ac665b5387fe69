"""Time keyed against unkeyed curve25519 ECDH derive on one GPU and print one JSON line.

Per shape the items are benchdata.gen_x25519_derive's (priv below n, item i against peer key i mod m, one in 256 a
twist point instead).  The set is built from the distinct peer keys the items use, the 16 twist x values included, so
the twist items go through the set too.  It is created at the given table width (0: the automatic choice), and
eb200_x25519_derive_batch_keyed and eb200_x25519_derive_batch on the same items are called alternately after a
warm-up; the median of --reps rounds is reported.  main_kernel_ms comes from eb200_last_timing() (the keyed main
kernel, or the ladder); wall_ms includes the copies and, for the keyed call, the normalisation.  create_ms is the wall
time of eb200_x25519_keyset_create.  Both calls' outputs and statuses are asserted equal, and the statuses equal to
the generator's, in every round.  break_even_derives_per_key: the derives per key at which create + keyed derive beats
unkeyed derive by wall time (null when keyed is not faster).

--profile makes a separate run under torch.profiler at the first automatic-width shape instead, and reports the mean
time per call of each kernel (keyed main, normalisation; the unkeyed ladder).

    python tools/bench_x25519_keyset.py [--reps 10] [--warmup 2] [--profile] [--out FILE]
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

# (items, peer keys, width)
SHAPES = [(1 << 20, 4096, W) for W in (4, 6, 0, 8)] + [(1 << 20, 16, 8), (1 << 20, 1 << 16, 4)]
KERNELS = {"x25519_derive_keyed_kernel": "keyed_main", "x25519_keyed_norm_kernel": "keyed_norm",
           "x25519_derive_kernel": "unkeyed_ladder"}


def gpu_query():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        return out[0].strip(), float(out[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None, None


def shape_items(n, m):
    """The generator's items, the set's keys (the distinct pubx rows) and each item's key index."""
    import benchdata
    ds = benchdata.gen_x25519_derive(n, n_pubs=m, cache_dir=benchdata.cache_dir())
    keys, idx = np.unique(ds["pubx"].view("V32").reshape(-1), return_inverse=True)
    keys = np.ascontiguousarray(keys.view(np.uint8).reshape(-1, 32))
    idx = idx.reshape(-1).astype(np.uint32)
    assert (keys[idx] == ds["pubx"]).all()
    return ds, keys, idx


def create(lib, nat, keys, W):
    kst, h = np.zeros(len(keys), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_x25519_keyset_create(len(keys), keys.ctypes.data, W, kst.ctypes.data, ctypes.byref(h)))
    return h, kst


def profile(lib, nat, reps):
    import torch
    from torch.profiler import ProfilerActivity
    n, m, W = next(s for s in SHAPES if s[2] == 0)
    ds, keys, idx = shape_items(n, m)
    h, _ = create(lib, nat, keys, W)
    ko = (np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8))
    uo = (np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8))
    fns = {"keyed": lambda: nat.call(lib.eb200_x25519_derive_batch_keyed, h, n, ds["priv"], idx, *ko),
           "unkeyed": lambda: nat.call(lib.eb200_x25519_derive_batch, n, ds["priv"], ds["pubx"], *uo)}
    for f in fns.values():
        f()
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fns["keyed"](); fns["unkeyed"]()
        torch.cuda.synchronize()
    assert (ko[0] == uo[0]).all() and (ko[1] == uo[1]).all() and (ko[1] == ds["expected"]).all()
    nat.check(lib.eb200_keyset_destroy(h))
    per = {}
    for e in prof.events():
        k = next((v for name, v in KERNELS.items() if e.name.startswith(name)), None)
        if k:
            per.setdefault(k, []).append(e.time_range.elapsed_us())
    return {"items": n, "keys": m, "table_bits_requested": W, "reps": reps,
            "kernel_ms_per_call": {k: float(np.sum(v) / reps / 1e3) for k, v in per.items()},
            "launches_per_call": {k: len(v) // reps for k, v in per.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    name, watts = gpu_query()
    res = {"gpu": name, "power_limit_w": watts}
    if a.profile:
        res["profile"] = profile(lib, nat, a.reps)
    else:
        res.update(reps=a.reps, warmup=a.warmup, shapes=[])
        for n, m, W in SHAPES:
            ds, keys, idx = shape_items(n, m)
            t = time.perf_counter()
            h, kst = create(lib, nat, keys, W)
            create_ms = (time.perf_counter() - t) * 1e3
            build_kernel_ms = nat.last_timing()["kernel_ms"]
            w, db = ctypes.c_uint32(), ctypes.c_size_t()
            nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), ctypes.byref(db)))
            ok, sk = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
            ou, su = np.zeros((n, 32), np.uint8), np.zeros(n, np.uint8)
            rows = {"keyed": [], "unkeyed": []}
            for rep in range(a.warmup + a.reps):
                for kind in ("keyed", "unkeyed"):
                    t = time.perf_counter()
                    if kind == "keyed":
                        nat.call(lib.eb200_x25519_derive_batch_keyed, h, n, ds["priv"], idx, ok, sk)
                    else:
                        nat.call(lib.eb200_x25519_derive_batch, n, ds["priv"], ds["pubx"], ou, su)
                    wall = (time.perf_counter() - t) * 1e3
                    if rep >= a.warmup:
                        rows[kind].append((nat.last_timing()["main_kernel_ms"], wall))
                assert (ok == ou).all() and (sk == su).all() and (sk == ds["expected"]).all()
            nat.check(lib.eb200_keyset_destroy(h))
            med = lambda kind, j: float(np.median([x[j] for x in rows[kind]]))
            gain = (med("unkeyed", 1) - med("keyed", 1)) / n             # wall ms saved per derive
            res["shapes"].append({
                "items": n, "keys": len(keys), "twist_keys": int((kst != 1).sum()), "table_bits": w.value,
                "device_bytes": db.value, "create_ms": create_ms, "build_kernel_ms": build_kernel_ms,
                "keyed_main_kernel_ms": med("keyed", 0), "unkeyed_main_kernel_ms": med("unkeyed", 0),
                "keyed_wall_ms": med("keyed", 1), "unkeyed_wall_ms": med("unkeyed", 1),
                "main_kernel_speedup": med("unkeyed", 0) / med("keyed", 0),
                "break_even_derives_per_key": (create_ms / len(keys) / gain) if gain > 0 else None})
            print(json.dumps(res["shapes"][-1]), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
