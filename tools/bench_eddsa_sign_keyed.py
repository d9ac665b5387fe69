"""Time keyed against unkeyed EdDSA sign on one GPU and print one JSON line.

Per shape: m random 32-byte secrets, n random messages of a fixed length, item i signed by a random key.  The signing
set is created once after a warm-up create (create_ms: wall time of eb200_eddsa_signing_set_create), then
eb200_eddsa_sign_batch_keyed and eb200_eddsa_sign_batch (with each item's secret) are called alternately on the same
items after a warm-up; the median of --reps rounds is reported.  From eb200_last_timing(): main_kernel_ms (keyed: the
span of the chunks' nonce kernels, which includes waits for later chunks' inputs; unkeyed: the sign kernel, after all
inputs are resident) and call_gpu_ms (the whole call on the GPU timeline, copies included); wall_ms is the host clock
around the call.  In every round the two calls' signatures are asserted equal, and a sample of them equal to PyNaCl's.
break_even_sigs_per_key: the signatures per key at which create + keyed sign beats unkeyed sign by wall time (null when
keyed is not faster).

--profile makes a separate run under torch.profiler at the first shape instead, and reports the mean time per call of
each kernel (nonce, normalise, challenge; and the unkeyed sign kernel).

    python tools/bench_eddsa_sign_keyed.py [--reps 5] [--warmup 2] [--profile] [--out FILE]
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

# (items, keys, message bytes)
SHAPES = [(1 << 20, 4096, 32), (1 << 20, 4096, 256), (1 << 20, 16, 32), (1 << 20, 1 << 16, 32)]


def gpu_query():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        return out[0].strip(), float(out[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None, None


def shape_items(n, m, mlen, seed=2024):
    rng = np.random.default_rng(seed + m + mlen)
    sec = rng.integers(0, 256, (m, 32), dtype=np.uint8)
    idx = rng.integers(0, m, n).astype(np.uint32)
    msgs = rng.integers(0, 256, n * mlen, dtype=np.uint8)
    off = np.arange(n + 1, dtype=np.uint64) * mlen
    return sec, idx, msgs, off, np.ascontiguousarray(sec[idx])


def calls(lib, nat, n, h, msgs, off, idx, sec_i):
    sk, su = np.empty((n, 64), np.uint8), np.empty((n, 64), np.uint8)
    st = np.empty(n, np.uint8)
    keyed = lambda: nat.call(lib.eb200_eddsa_sign_batch_keyed, h, n, msgs, off, idx, sk, st)
    unkeyed = lambda: nat.call(lib.eb200_eddsa_sign_batch, n, sec_i, msgs, off, su, None, st)
    return {"keyed": keyed, "unkeyed": unkeyed}, sk, su


def check_nacl(sk, sec_i, msgs, off, count=16):
    import nacl.signing
    n = len(sk)
    for i in range(0, n, max(1, n // count)):
        s = nacl.signing.SigningKey(sec_i[i].tobytes()).sign(msgs[int(off[i]):int(off[i + 1])].tobytes()).signature
        assert s == sk[i].tobytes(), i


def profile(lib, nat, out_dir):
    import torch
    from torch.profiler import ProfilerActivity
    n, m, mlen = SHAPES[0]
    sec, idx, msgs, off, sec_i = shape_items(n, m, mlen)
    h = ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_signing_set_create(m, sec.ctypes.data, None, ctypes.byref(h)))
    fns, sk, su = calls(lib, nat, n, h, msgs, off, idx, sec_i)
    for _ in range(2):
        fns["keyed"](); fns["unkeyed"]()
    reps = 5
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fns["keyed"](); fns["unkeyed"]()
    assert (sk == su).all()
    nat.check(lib.eb200_keyset_destroy(h))
    kern = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if "kernel" in e.key and t:
            kern[e.key.split("(")[0]] = {"ms_per_call": t / 1e3 / reps, "launches_per_call": e.count / reps}
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "eddsa_sign_keyed.pt.trace.json"))
    return {"items": n, "keys": m, "msg_bytes": mlen, "reps": reps, "kernels": kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--trace-dir")
    ap.add_argument("--out")
    a = ap.parse_args()
    from elliptic_b200 import _native as nat
    lib = nat.init(0)
    name, watts = gpu_query()
    res = {"gpu": name, "power_limit_w": watts, "lib": os.path.basename(nat.LIB_PATH)}
    if a.profile:
        res["profile"] = profile(lib, nat, a.trace_dir)
    else:
        res.update(reps=a.reps, warmup=a.warmup, shapes=[])
        for n, m, mlen in SHAPES:
            sec, idx, msgs, off, sec_i = shape_items(n, m, mlen)
            h = ctypes.c_void_p()
            nat.check(lib.eb200_eddsa_signing_set_create(m, sec.ctypes.data, None, ctypes.byref(h)))   # warm-up
            nat.check(lib.eb200_keyset_destroy(h))
            t = time.perf_counter()
            nat.check(lib.eb200_eddsa_signing_set_create(m, sec.ctypes.data, None, ctypes.byref(h)))
            create_ms = (time.perf_counter() - t) * 1e3
            create_kernel_ms = nat.last_timing()["kernel_ms"]
            fns, sk, su = calls(lib, nat, n, h, msgs, off, idx, sec_i)
            rows = {"keyed": [], "unkeyed": []}
            launches = None
            for rep in range(a.warmup + a.reps):
                for kind in ("keyed", "unkeyed"):
                    t = time.perf_counter()
                    fns[kind]()
                    wall = (time.perf_counter() - t) * 1e3
                    tm = nat.last_timing()
                    if kind == "keyed":
                        launches = tm["launches"]
                    # the whole call on the GPU timeline: the chunked keyed call reports it as kernel_ms, the
                    # single-stream unkeyed call splits it into copies up, kernels and copies home
                    gpu = tm["kernel_ms"] if kind == "keyed" else tm["h2d_ms"] + tm["kernel_ms"] + tm["d2h_ms"]
                    if rep >= a.warmup:
                        rows[kind].append((tm["main_kernel_ms"], gpu, wall))
                assert (sk == su).all()
                check_nacl(sk, sec_i, msgs, off)
            nat.check(lib.eb200_keyset_destroy(h))
            med = lambda kind, j: float(np.median([x[j] for x in rows[kind]]))
            gain = (med("unkeyed", 2) - med("keyed", 2)) / n            # wall ms saved per signature
            res["shapes"].append({
                "items": n, "keys": m, "msg_bytes": mlen, "create_ms": create_ms, "create_kernel_ms": create_kernel_ms,
                "keyed_launches": launches,
                "keyed_main_kernel_ms": med("keyed", 0), "unkeyed_main_kernel_ms": med("unkeyed", 0),
                "keyed_call_gpu_ms": med("keyed", 1), "unkeyed_call_gpu_ms": med("unkeyed", 1),
                "keyed_wall_ms": med("keyed", 2), "unkeyed_wall_ms": med("unkeyed", 2),
                "call_gpu_speedup": med("unkeyed", 1) / med("keyed", 1),
                "break_even_sigs_per_key": (create_ms / m / gain) if gain > 0 else None})
            print(json.dumps(res["shapes"][-1]), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
