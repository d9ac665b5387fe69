"""A/B timing of two builds of the library on bench.py's headline workload, and one JSON line.

Both builds are loaded into one process: the baseline from --base, the candidate from $EB200_LIB (default: the
in-tree build).  Each round runs the 2^20-item secp256k1 verify of bench.py (same generator and seed) through
eb200_ecdsa_verify_batch_dev, --steps calls per build, the builds alternating every round so that clock and
neighbour drift fall on both alike.  Every call's statuses must equal the generator's expectation.  Per build:
median and min-max over rounds of the main kernel ms (eb200_last_timing), the other kernels' ms (the prep kernel;
kernel_ms - main_kernel_ms) and the step ms (CUDA events around one call).  The card's name, power limit and SM
clock are read in the same run.

    EB200_LIB=<candidate .so> python tools/bench_k256_ab.py --base <baseline .so> [--rounds 12] [--steps 5] [--out F]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_query():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1]), "sm_clock_mhz": float(out[2]), "max_sm_clock_mhz": float(out[3])}
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return {"gpu": None}


class Build:
    def __init__(self, path, nat, n, d, stream):
        c = ctypes
        self.path, self.nat, self.n, self.d, self.stream = path, nat, n, d, stream
        lib = self.lib = c.CDLL(path)
        lib.eb200_init.argtypes = [c.POINTER(c.c_int), c.c_int, c.c_uint32]
        lib.eb200_last_timing.argtypes = [c.POINTER(nat.Timing)]
        lib.eb200_ecdsa_verify_workspace_bytes.restype = c.c_size_t
        lib.eb200_ecdsa_verify_workspace_bytes.argtypes = [c.c_int, c.c_size_t]
        lib.eb200_ecdsa_verify_batch_dev.argtypes = [c.c_int, c.c_size_t] + [c.c_void_p] * 4 + [c.c_uint32] + [c.c_void_p] * 3
        lib.eb200_strerror.restype = c.c_char_p
        dev = (c.c_int * 1)(0)
        self.check(lib.eb200_init(dev, 1, 0))
        import torch
        self.ws = torch.empty(lib.eb200_ecdsa_verify_workspace_bytes(nat.CURVE_SECP256K1, n), dtype=torch.uint8, device="cuda")
        self.status = torch.empty(n, dtype=torch.uint8, device="cuda")
        self.rows = []

    def check(self, rc):
        if rc != self.nat.OK:
            raise RuntimeError("%s: %s" % (self.path, self.lib.eb200_strerror(rc).decode()))

    def call(self):
        d = self.d
        self.check(self.lib.eb200_ecdsa_verify_batch_dev(self.nat.CURVE_SECP256K1, self.n, d["e"].data_ptr(), d["r"].data_ptr(),
                                                         d["s"].data_ptr(), d["pub"].data_ptr(), self.nat.PUB_XY,
                                                         self.status.data_ptr(), self.ws.data_ptr(), self.stream))

    def timing(self):
        t = self.nat.Timing()
        self.check(self.lib.eb200_last_timing(ctypes.byref(t)))
        return t


def summary(vals):
    return {"median": float(np.median(vals)), "min": float(np.min(vals)), "max": float(np.max(vals))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="baseline libelliptic_b200.so")
    ap.add_argument("--rounds", type=int, default=12)
    ap.add_argument("--steps", type=int, default=5, help="calls per build per round")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--label", default="")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import benchdata
    from elliptic_b200 import _native as nat
    n = 1 << 20
    ds = benchdata.gen_secp256k1_verify(n, seed=0xE1110002, cache_dir=benchdata.cache_dir())
    torch.cuda.set_device(0)
    d = {k: torch.from_numpy(ds[k]).cuda() for k in ("e", "r", "s", "pub")}
    expected = torch.from_numpy(ds["expected"]).cuda()
    stream = torch.cuda.current_stream().cuda_stream
    builds = [Build(os.path.abspath(a.base), nat, n, d, stream), Build(os.path.abspath(nat.LIB_PATH), nat, n, d, stream)]
    for b in builds:
        for _ in range(a.warmup):
            b.call()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rnd in range(a.rounds):
        for b in (builds if rnd % 2 == 0 else builds[::-1]):
            for _ in range(a.steps):
                ev0.record()
                b.call()
                ev1.record()
                ev1.synchronize()
                t = b.timing()
                b.rows.append((t.main_kernel_ms, t.kernel_ms - t.main_kernel_ms, ev0.elapsed_time(ev1)))
                assert bool((b.status == expected).all()), "%s: statuses differ from the generator's expectation" % b.path
    res = dict(gpu_query(), label=a.label, items=n, rounds=a.rounds, steps_per_round=a.steps)
    for key, b in zip(("base", "cand"), builds):
        res[key] = {"lib": os.path.relpath(b.path, ROOT), "main_kernel_ms": summary([r[0] for r in b.rows]),
                    "other_kernels_ms": summary([r[1] for r in b.rows]), "step_ms": summary([r[2] for r in b.rows])}
    res["step_speedup"] = res["base"]["step_ms"]["median"] / res["cand"]["step_ms"]["median"]
    res["main_kernel_speedup"] = res["base"]["main_kernel_ms"]["median"] / res["cand"]["main_kernel_ms"]["median"]
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
