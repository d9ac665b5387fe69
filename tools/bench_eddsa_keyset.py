"""Time keyed against unkeyed EdDSA verify on one GPU and print one JSON line.

Per shape the items are benchdata.gen_ed25519_verify's (ed25519 signatures over m keys, item i by key i mod m, one in 64
forged).  The set is created at the given table width (0: the automatic choice), and the keyed call and the unkeyed
call on the same items are made alternately after a warm-up, through the `h` or the raw-message (`msgs`) entry points;
the median of --reps rounds is reported.  main_kernel_ms comes from eb200_last_timing(); wall_ms includes the copies (and,
for msgs, the hash kernel); create_ms is the wall time of eb200_eddsa_keyset_create.  Both calls' statuses are asserted
equal to each other and to the generator's expected bytes in every round.  break_even_sigs_per_key: the signatures per
key at which create + keyed verify beats unkeyed verify by wall time (null when keyed is not faster).

    python tools/bench_eddsa_keyset.py [--reps 10] [--warmup 2] [--out FILE]
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

# (items, keys, width, call)
SHAPES = [(1 << 20, 4096, W, call) for W in (4, 6, 0, 8) for call in ("h", "msgs")] + [
    (1 << 20, 16, 8, "h"), (1 << 20, 1 << 16, 4, "h")]


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
    import benchdata
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    name, watts = gpu_query()
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps, "shapes": []}
    cache = {}
    for n, m, W, call in SHAPES:
        if (n, m) not in cache:
            cache.clear()
            ds = benchdata.gen_ed25519_verify(n, n_keys=m, cache_dir=benchdata.cache_dir(), with_msgs=True)
            keys, idx = np.ascontiguousarray(ds["A"][:m]), np.arange(n, dtype=np.uint32) % m
            assert (ds["A"] == keys[idx]).all()
            msgs, off = np.ascontiguousarray(ds["msgs"].reshape(-1)), np.arange(n + 1, dtype=np.uint64) * 32
            cache[(n, m)] = ds, keys, idx, msgs, off
        ds, keys, idx, msgs, off = cache[(n, m)]
        kst, h = np.zeros(m, np.uint8), ctypes.c_void_p()
        t = time.perf_counter()
        nat.check(lib.eb200_eddsa_keyset_create(m, keys.ctypes.data, W, kst.ctypes.data, ctypes.byref(h)))
        create_ms = (time.perf_counter() - t) * 1e3
        build_kernel_ms = nat.last_timing()["kernel_ms"]
        w, db = ctypes.c_uint32(), ctypes.c_size_t()
        nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), ctypes.byref(db)))
        sk, su = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        rows = {"keyed": [], "unkeyed": []}
        for rep in range(a.warmup + a.reps):
            for kind in ("keyed", "unkeyed"):
                t = time.perf_counter()
                if kind == "keyed" and call == "h":
                    nat.call(lib.eb200_eddsa_verify_batch_keyed, h, n, ds["R"], ds["S"], ds["h"], idx, sk)
                elif kind == "keyed":
                    nat.call(lib.eb200_eddsa_verify_batch_keyed_msgs, h, n, ds["R"], ds["S"], msgs, off, idx, sk)
                elif call == "h":
                    nat.call(lib.eb200_eddsa_verify_batch, n, ds["R"], ds["S"], ds["A"], ds["h"], su)
                else:
                    nat.call(lib.eb200_eddsa_verify_batch_msgs, n, ds["R"], ds["S"], ds["A"], msgs, off, su)
                wall = (time.perf_counter() - t) * 1e3
                if rep >= a.warmup:
                    rows[kind].append((nat.last_timing()["main_kernel_ms"], wall))
            assert (sk == su).all() and (sk == ds["expected"]).all()
        nat.check(lib.eb200_keyset_destroy(h))
        med = lambda kind, j: float(np.median([x[j] for x in rows[kind]]))
        gain = (med("unkeyed", 1) - med("keyed", 1)) / n            # wall ms saved per signature
        res["shapes"].append({
            "call": call, "items": n, "keys": m, "table_bits": w.value, "device_bytes": db.value, "create_ms": create_ms,
            "build_kernel_ms": build_kernel_ms,
            "keyed_main_kernel_ms": med("keyed", 0), "unkeyed_main_kernel_ms": med("unkeyed", 0),
            "keyed_wall_ms": med("keyed", 1), "unkeyed_wall_ms": med("unkeyed", 1),
            "main_kernel_speedup": med("unkeyed", 0) / med("keyed", 0),
            "break_even_sigs_per_key": (create_ms / m / gain) if gain > 0 else None})
        print(json.dumps(res["shapes"][-1]), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
