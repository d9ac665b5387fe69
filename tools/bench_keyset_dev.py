"""Time the device-pointer forms of the keyed calls against their host forms on one GPU and print one JSON line.

Shape: 2^20 items over 4096 keys at the default table width, on secp256k1 and p256 (keyed mul, mulAdd, ECDH derive,
getKeyRecoveryParam), ed25519 (keyed verify from h and from raw messages, keyed sign) and curve25519 (keyed derive).
In each of --reps alternated rounds (after --warmup), on the same items:
  host   the host-pointer keyed call from pinned buffers; wall_ms is the host clock around it (it returns synchronised)
  dev    the `_dev` call on torch tensors, timed with CUDA events around it on the caller's stream
Outputs and statuses of both forms are asserted equal in every round; medians are reported, with main_kernel_ms and
launches from eb200_last_timing().  A separate torch.profiler run per call (after the timed rounds) gives the share of
the `_dev` call's kernel time spent in the screen and merge kernels; that run is a second process of this script
(--profile-only), so that tracing never overlaps the timed rounds.

    python tools/bench_keyset_dev.py [--reps 5] [--warmup 1] [--out FILE]
"""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

N, M = 1 << 20, 4096
FRAME_KERNELS = ("keyset_index", "keyset_verdict_merge")      # the screens and merges this form adds


def pinned(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    return t.numpy()


class Call:
    """One keyed call in both forms: host(*hargs, *outs) and dev(*dargs, *douts, ws, stream)."""

    def __init__(self, label, h, host_fn, dev_fn, hargs, dargs, out_bytes):
        import torch
        self.label, self.h, self.host_fn, self.dev_fn = label, h, host_fn, dev_fn
        self.hargs = [pinned(a) if isinstance(a, np.ndarray) else a for a in hargs]
        self.dt = [torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
                   if isinstance(a, np.ndarray) else a for a in dargs]
        self.houts = [pinned(np.zeros(b, np.uint8)) for b in out_bytes]
        self.douts = [torch.empty(b, dtype=torch.uint8, device="cuda") for b in out_bytes]
        self.ws = torch.empty(lib_.eb200_keyset_dev_workspace_bytes(h, N), dtype=torch.uint8, device="cuda")

    def run_host(self):
        from elliptic_b200 import _native as nat
        t = time.perf_counter()
        nat.call(self.host_fn, self.h, N, *self.hargs, *self.houts)
        return (time.perf_counter() - t) * 1e3

    def launch_dev(self, stream):
        from elliptic_b200 import _native as nat
        cargs = [ctypes.c_void_p(x.data_ptr()) if hasattr(x, "data_ptr") else None if x is None else ctypes.c_uint64(x)
                 for x in self.dt + self.douts]
        nat.check(self.dev_fn(self.h, N, *cargs, ctypes.c_void_p(self.ws.data_ptr()), ctypes.c_void_p(stream.cuda_stream)))

    def run_dev(self, stream):
        import torch
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        self.launch_dev(stream)
        ev1.record(stream)
        stream.synchronize()
        return ev0.elapsed_time(ev1)

    def equal(self):
        return all((d.cpu().numpy() == h).all() for d, h in zip(self.douts, self.houts))


def build_calls(lib, nat):
    from gpu_keyset_items import gpu_items
    import benchdata
    calls, handles = [], []
    rng = np.random.default_rng(1)
    for curve, cid, ln in (("secp256k1", 1, 32), ("p256", 2, 32)):
        xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, M, N, seed=cid * 1000 + M % 997)
        kst, h = np.zeros(M, np.uint8), ctypes.c_void_p()
        nat.check(lib.eb200_keyset_create(cid, M, xy.ctypes.data, 0, 0, kst.ctypes.data, ctypes.byref(h)))
        handles.append(h)
        k1, k2 = (rng.integers(0, 256, (N, ln), dtype=np.uint8) for _ in range(2))
        calls += [
            Call(curve + " mul", h, lib.eb200_scalar_mul_batch_keyed, lib.eb200_scalar_mul_batch_keyed_dev, [k2, idx],
                 [k2, idx], [2 * ln * N, N]),
            Call(curve + " mul_add", h, lib.eb200_mul_add_batch_keyed, lib.eb200_mul_add_batch_keyed_dev, [k1, k2, idx],
                 [k1, k2, idx], [2 * ln * N, N]),
            Call(curve + " derive", h, lib.eb200_ecdh_derive_batch_keyed, lib.eb200_ecdh_derive_batch_keyed_dev, [k2, idx],
                 [k2, idx], [ln * N, N]),
            Call(curve + " recovery_param", h, lib.eb200_ecdsa_recovery_param_batch_keyed,
                 lib.eb200_ecdsa_recovery_param_batch_keyed_dev, [e, r, s, idx], [e, r, s, idx], [N, N])]
    # ed25519: keys and signatures from a signing set, so that the verifies are TRUE
    sec = rng.integers(0, 256, (M, 32), dtype=np.uint8)
    pub, hs = np.zeros((M, 32), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_signing_set_create(M, sec.ctypes.data, pub.ctypes.data, ctypes.byref(hs)))
    handles.append(hs)
    lens = rng.integers(0, 129, N)
    off = np.zeros(N + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    L = int(off[N])
    msgs = rng.integers(0, 256, L, dtype=np.uint8)
    idx = rng.integers(0, M, N).astype(np.uint32)
    sig = np.zeros((N, 64), np.uint8)
    nat.call(lib.eb200_eddsa_sign_batch_keyed, hs, N, msgs, off, idx, sig, np.zeros(N, np.uint8))
    kst, hv = np.zeros(M, np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_eddsa_keyset_create(M, pub.ctypes.data, 0, kst.ctypes.data, ctypes.byref(hv)))
    handles.append(hv)
    R, S = np.ascontiguousarray(sig[:, :32]), np.ascontiguousarray(sig[:, 32:])
    n25519 = 2**252 + 27742317777372353535851937790883648493
    mb, pb, rb = msgs.tobytes(), pub.tobytes(), R.tobytes()
    hh = np.frombuffer(b"".join(
        (int.from_bytes(hashlib.sha512(rb[32 * i:32 * i + 32] + pb[32 * int(idx[i]):32 * int(idx[i]) + 32] +
                                       mb[int(off[i]):int(off[i + 1])]).digest(), "little") % n25519).to_bytes(32, "little")
        for i in range(N)), np.uint8).reshape(N, 32)
    calls += [
        Call("ed25519 verify", hv, lib.eb200_eddsa_verify_batch_keyed, lib.eb200_eddsa_verify_batch_keyed_dev,
             [R, S, hh, idx], [R, S, hh, idx], [N]),
        Call("ed25519 verify_msgs", hv, lib.eb200_eddsa_verify_batch_keyed_msgs, lib.eb200_eddsa_verify_batch_keyed_msgs_dev,
             [R, S, msgs, off, idx], [R, S, msgs, L, off, idx], [N]),
        Call("ed25519 sign", hs, lib.eb200_eddsa_sign_batch_keyed, lib.eb200_eddsa_sign_batch_keyed_dev,
             [msgs, off, idx], [msgs, L, off, idx], [64 * N, N])]
    ds = benchdata.gen_x25519_derive(N, n_pubs=M, cache_dir=benchdata.cache_dir())
    keys, xidx = np.unique(ds["pubx"].view("V32").reshape(-1), return_inverse=True)
    keys = np.ascontiguousarray(keys.view(np.uint8).reshape(-1, 32))
    xidx = xidx.reshape(-1).astype(np.uint32)
    priv = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    priv[:, 0] &= 0x0F
    kst, hx = np.zeros(len(keys), np.uint8), ctypes.c_void_p()
    nat.check(lib.eb200_x25519_keyset_create(len(keys), keys.ctypes.data, 0, kst.ctypes.data, ctypes.byref(hx)))
    handles.append(hx)
    calls.append(Call("curve25519 derive", hx, lib.eb200_x25519_derive_batch_keyed, lib.eb200_x25519_derive_batch_keyed_dev,
                      [priv, xidx], [priv, xidx], [32 * N, N]))
    return calls, handles


def frame_share(call, stream):
    """Share of the `_dev` call's kernel time spent in the screen and merge kernels, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call.launch_dev(stream)
        stream.synchronize()
    total = frame = 0.0
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.name.startswith("Memset"):
            us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            total += us
            if any(k in ev.name for k in FRAME_KERNELS):
                frame += us
    return {"frame_kernels_us": frame, "all_kernels_us": total, "frame_share": frame / total if total else None}


lib_ = None


def main():
    global lib_
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out")
    ap.add_argument("--profile-only", action="store_true")
    a = ap.parse_args()
    import torch
    from bench_keyset import gpu_query
    from elliptic_b200 import _native as nat
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyset_dev: no CUDA device (there is no CPU path to measure)")
    lib_ = lib = nat.init(0)
    name, watts = gpu_query()
    calls, handles = build_calls(lib, nat)
    stream = torch.cuda.Stream()
    if a.profile_only:
        for c in calls:
            c.run_dev(stream)                                  # warm-up
        print(json.dumps({c.label: frame_share(c, stream) for c in calls}))
        return
    res = {"gpu": name, "power_limit_w": watts, "items": N, "keys": M, "table_bits": "default", "reps": a.reps,
           "calls": []}
    for c in calls:
        rows = {"host": [], "dev": []}
        for rep in range(a.warmup + a.reps):
            for kind in ("host", "dev"):
                t = c.run_host() if kind == "host" else c.run_dev(stream)
                tm = nat.last_timing()
                if rep >= a.warmup:
                    rows[kind].append((t, tm["main_kernel_ms"], tm["launches"]))
            assert c.equal(), c.label
        med = lambda kind, j: float(np.median([x[j] for x in rows[kind]]))
        res["calls"].append({"call": c.label,
                             "host": {"wall_ms": med("host", 0), "main_kernel_ms": med("host", 1),
                                      "launches": int(rows["host"][0][2])},
                             "dev": {"dev_ms": med("dev", 0), "main_kernel_ms": med("dev", 1),
                                     "launches": int(rows["dev"][0][2])},
                             "host_wall_vs_dev": med("host", 0) / med("dev", 0)})
    for h in handles:
        nat.check(lib.eb200_keyset_destroy(h))
    del calls
    torch.cuda.empty_cache()
    prof = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile-only"], check=True, capture_output=True,
                          text=True).stdout.strip().splitlines()[-1]
    for row, share in zip(res["calls"], json.loads(prof).values()):
        row["profile"] = share
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
