"""Time the device-pointer forms of the unkeyed calls against their host forms on one GPU and write one JSON document.

Shape: 2^20 items (sign and keygen: 2^18) on secp256k1 and p256 (sign, sign with k, sign with pers, keygen, recover,
getKeyRecoveryParam, mul, G.mul, mulAdd, derive, verify from DER), ed25519 (EdDSA sign, EdDSA verify from raw messages)
and curve25519 (Point.mul).  In each of --reps alternated rounds (after --warmup), on the same items:
  host   the host-pointer call from pinned buffers; wall_ms is the host clock around it (it returns synchronised)
  dev    the `_dev` call on torch tensors, timed with CUDA events around it on the caller's stream
Outputs and statuses of both forms are asserted equal in every round; medians are reported, with main_kernel_ms and
launches from eb200_last_timing(), and the GPU's name and power limit read in the same run.

    python tools/bench_unkeyed_dev.py [--reps 5] [--warmup 1] [--out profiles/h100_unkeyed_dev.json]
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

N, N_SIGN = 1 << 20, 1 << 18


def pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()


class Call:
    """One call in both forms: host(*lead, *hargs, *outs) and dev(*lead, *dargs, *douts, [ws,] stream)."""

    def __init__(self, lib, label, lead, host_fn, dev_fn, hargs, dargs, out_bytes, ws_curve):
        import torch
        self.label, self.lead, self.host_fn, self.dev_fn = label, lead, host_fn, dev_fn
        self.hargs = [pinned(a) if isinstance(a, np.ndarray) else a for a in hargs]
        self.dt = [torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
                   if isinstance(a, np.ndarray) else a for a in dargs]
        self.houts = [pinned(np.zeros(b, np.uint8)) for b in out_bytes]
        self.douts = [torch.empty(b, dtype=torch.uint8, device="cuda") for b in out_bytes]
        n = lead[-1]
        self.ws = None if ws_curve is None else \
            torch.empty(lib.eb200_dev_workspace_bytes(ws_curve, n), dtype=torch.uint8, device="cuda")

    def run_host(self):
        from elliptic_b200 import _native as nat
        t = time.perf_counter()
        nat.call(self.host_fn, *self.lead, *self.hargs, *self.houts)
        return (time.perf_counter() - t) * 1e3

    def launch_dev(self, stream):
        from elliptic_b200 import _native as nat
        cargs = [ctypes.c_void_p(x.data_ptr()) if hasattr(x, "data_ptr") else None if x is None else x
                 for x in self.dt + self.douts]
        tail = [] if self.ws is None else [ctypes.c_void_p(self.ws.data_ptr())]
        nat.check(self.dev_fn(*self.lead, *cargs, *tail, ctypes.c_void_p(stream.cuda_stream)))

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


def der(r, s):
    def integer(b):
        b = b.lstrip(b"\0") or b"\0"
        return b"\x02" + bytes([len(b) + (b[0] >> 7)]) + (b"\0" if b[0] & 0x80 else b"") + b
    parts = []
    for ri, si in zip(r, s):
        body = integer(ri.tobytes()) + integer(si.tobytes())
        parts.append(b"\x30" + bytes([len(body)]) + body)
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in parts])
    return np.frombuffer(b"".join(parts), np.uint8).copy(), off


def build_calls(lib, nat):
    rng = np.random.default_rng(1)
    calls = []
    for curve, cid, ln in (("secp256k1", 1, 32), ("p256", 2, 32)):
        e, d, k = (rng.integers(0, 256, (N, ln), dtype=np.uint8) for _ in range(3))
        for a in (e, d, k):
            a[:, 0] &= 0x7F
        r, s, rec, st = np.zeros((N, ln), np.uint8), np.zeros((N, ln), np.uint8), np.zeros(N, np.uint8), np.zeros(N, np.uint8)
        nat.call(lib.eb200_ecdsa_sign_batch, cid, N, e, d, 0, r, s, rec, st)
        q = np.zeros((N, 2 * ln), np.uint8)
        nat.call(lib.eb200_scalar_mul_batch, cid, N, d, None, q, st)
        sigs, off = der(r, s)
        pers = rng.integers(0, 256, 32, dtype=np.uint8)
        ent = rng.integers(0, 256, (N_SIGN, 32), dtype=np.uint8)
        es, ds, ks = e[:N_SIGN], d[:N_SIGN], k[:N_SIGN]
        so = [ln * N_SIGN, ln * N_SIGN, N_SIGN, N_SIGN]
        calls += [
            Call(lib, curve + " sign", (cid, N_SIGN), lib.eb200_ecdsa_sign_batch, lib.eb200_ecdsa_sign_batch_dev,
                 [es, ds, 0], [es, ds, 0], so, cid),
            Call(lib, curve + " sign_k", (cid, N_SIGN), lib.eb200_ecdsa_sign_batch_k, lib.eb200_ecdsa_sign_batch_k_dev,
                 [es, ds, ks, 0], [es, ds, ks, 0], so, cid),
            Call(lib, curve + " sign_pers", (cid, N_SIGN), lib.eb200_ecdsa_sign_batch_pers, lib.eb200_ecdsa_sign_batch_pers_dev,
                 [es, ds, pers, 32, 0], [es, ds, pers, 32, 0], so, cid),
            Call(lib, curve + " keygen", (cid, N_SIGN), lib.eb200_ec_keygen_batch, lib.eb200_ec_keygen_batch_dev,
                 [ent, 32, None, 0], [ent, 32, None, 0], [ln * N_SIGN, 2 * ln * N_SIGN, N_SIGN], cid),
            Call(lib, curve + " recover", (cid, N), lib.eb200_ecdsa_recover_batch, lib.eb200_ecdsa_recover_batch_dev,
                 [e, r, s, rec], [e, r, s, rec], [2 * ln * N, N], cid),
            Call(lib, curve + " recovery_param", (cid, N), lib.eb200_ecdsa_recovery_param_batch,
                 lib.eb200_ecdsa_recovery_param_batch_dev, [e, r, s, q], [e, r, s, q], [N, N], cid),
            Call(lib, curve + " mul", (cid, N), lib.eb200_scalar_mul_batch, lib.eb200_scalar_mul_batch_dev,
                 [k, q], [k, q], [2 * ln * N, N], cid),
            Call(lib, curve + " mul_g", (cid, N), lib.eb200_scalar_mul_batch, lib.eb200_scalar_mul_batch_dev,
                 [k, None], [k, None], [2 * ln * N, N], cid),
            Call(lib, curve + " mul_add", (cid, N), lib.eb200_mul_add_batch, lib.eb200_mul_add_batch_dev,
                 [e, k, q], [e, k, q], [2 * ln * N, N], cid),
            Call(lib, curve + " derive", (cid, N), lib.eb200_ecdh_derive_batch, lib.eb200_ecdh_derive_batch_dev,
                 [k, q], [k, q], [ln * N, N], cid),
            Call(lib, curve + " verify_der", (cid, N), lib.eb200_ecdsa_verify_batch_der, lib.eb200_ecdsa_verify_batch_der_dev,
                 [e, sigs, off, q, nat.PUB_XY], [e, sigs, ctypes.c_uint64(len(sigs)), off, q, ctypes.c_uint32(nat.PUB_XY)],
                 [N], cid)]
    sec = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    lens = rng.integers(0, 129, N)
    off = np.zeros(N + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    L = int(off[N])
    msgs = rng.integers(0, 256, L, dtype=np.uint8)
    sig, pub = np.zeros((N, 64), np.uint8), np.zeros((N, 32), np.uint8)
    nat.call(lib.eb200_eddsa_sign_batch, N, sec, msgs, off, sig, pub, np.zeros(N, np.uint8))
    R, S = np.ascontiguousarray(sig[:, :32]), np.ascontiguousarray(sig[:, 32:])
    ed = nat.CURVE_ED25519
    calls += [
        Call(lib, "ed25519 eddsa_sign", (N,), lib.eb200_eddsa_sign_batch, lib.eb200_eddsa_sign_batch_dev,
             [sec, msgs, off], [sec, msgs, ctypes.c_uint64(L), off], [64 * N, 32 * N, N], ed),
        Call(lib, "ed25519 eddsa_verify_msgs", (N,), lib.eb200_eddsa_verify_batch_msgs, lib.eb200_eddsa_verify_batch_msgs_dev,
             [R, S, pub, msgs, off], [R, S, pub, msgs, ctypes.c_uint64(L), off], [N], ed)]
    kx, px = (rng.integers(0, 256, (N, 32), dtype=np.uint8) for _ in range(2))
    calls.append(Call(lib, "curve25519 mul", (N,), lib.eb200_x25519_mul_batch, lib.eb200_x25519_mul_batch_dev,
                      [kx, px], [kx, px], [32 * N, N], None))
    return calls


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return q[0], float(q[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_unkeyed_dev.json"))
    args = ap.parse_args()
    import torch
    from elliptic_b200 import _native as nat
    if not torch.cuda.is_available():
        raise SystemExit("bench_unkeyed_dev needs a CUDA device")
    lib = nat.init(0)
    name, power = gpu_info()
    calls = build_calls(lib, nat)
    stream = torch.cuda.Stream()
    rows = []
    for c in calls:
        for _ in range(args.warmup):
            c.run_host()
            c.run_dev(stream)
        host_ms, dev_ms, host_tm, dev_tm = [], [], None, None
        for _ in range(args.reps):
            host_ms.append(c.run_host())
            host_tm = nat.last_timing()
            dev_ms.append(c.run_dev(stream))
            dev_tm = nat.last_timing()
            assert c.equal(), c.label
        h, d = float(np.median(host_ms)), float(np.median(dev_ms))
        rows.append({"call": c.label, "items": c.lead[-1],
                     "host": {"wall_ms": h, "main_kernel_ms": host_tm["main_kernel_ms"], "launches": host_tm["launches"]},
                     "dev": {"dev_ms": d, "main_kernel_ms": dev_tm["main_kernel_ms"], "launches": dev_tm["launches"]},
                     "host_wall_vs_dev": h / d})
        print("%-28s host %8.3f ms   dev %8.3f ms   x%.2f" % (c.label, h, d, h / d), file=sys.stderr)
    doc = {"gpu": name, "power_limit_w": power, "reps": args.reps, "calls": rows}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(doc, f)
    print(json.dumps(doc))


if __name__ == "__main__":
    main()
