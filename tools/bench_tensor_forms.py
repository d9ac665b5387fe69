"""Time the tensor forms against the raw device-pointer calls and the packed host forms on one GPU; one JSON document.

Workloads, at 2^20 and 2^10 items: secp256k1 verify, keyed verify (one-format set of 64 keys), verify from DER, EdDSA
sign (64-byte messages), and keyed verify on a set of mixed wire formats (64 keys, {x, y} and compressed: two native
sets).  In each of --reps alternated rounds (after --warmup), on the same CUDA tensors:
  tensor  the `*_tensors` method
  raw     the `eb200_*_dev` call through ctypes with preallocated outputs and workspace (mixed set: one call per native
          set with the indices split beforehand, outside the timed region)
  packed  the `*_packed` method fed from the same tensors: `.cpu()` in, the result moved back to the device
Each time is the host clock around the call and a synchronisation of the device, so it includes the host-side work of
each form.  Outputs are asserted equal in every round; medians are reported with the GPU's name and power limit read
in the same run.

    python tools/bench_tensor_forms.py [--reps 7] [--warmup 2] [--out profiles/h100_tensor_forms.json]
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

M = 64


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return q[0], float(q[1])


def der_blob(r, s):
    def integer(b):
        b = b.lstrip(b"\0") or b"\0"
        return b"\x02" + bytes([len(b) + (b[0] >> 7)]) + (b"\0" if b[0] & 0x80 else b"") + b
    parts = []
    for ri, si in zip(r, s):
        body = integer(ri.tobytes()) + integer(si.tobytes())
        parts.append(b"\x30" + bytes([len(body)]) + body)
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in parts])
    return parts, np.frombuffer(b"".join(parts), np.uint8).copy(), off


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def raw(fn, *args):
    """A raw `_dev` call: tensors as device addresses, on the current stream."""
    import torch
    from elliptic_b200 import _native as nat
    cargs = [ctypes.c_void_p(a.data_ptr()) if hasattr(a, "data_ptr") else a for a in args]
    nat.check(fn(*cargs, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))


def workloads(lib, nat, n):
    import torch
    from gpu_keyset_items import gpu_items
    from elliptic_b200.ec import EC
    from elliptic_b200.eddsa import EDDSA
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    u8 = lambda *shape: torch.empty(shape, dtype=torch.uint8, device="cuda")   # noqa: E731
    cid, ln = nat.CURVE_SECP256K1, 32
    ec = EC("secp256k1")
    xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, M, n, seed=n)
    te, tr, ts, tq = cuda(e), cuda(r), cuda(s), cuda(xy[idx])
    ti64 = cuda(idx.astype(np.int64))
    ws_u = u8(lib.eb200_dev_workspace_bytes(cid, n))
    st = u8(n)
    out = []

    out.append(("secp256k1 verify",
                lambda: ec.verify_batch_tensors(te, tr, ts, tq),
                lambda: (raw(lib.eb200_ecdsa_verify_batch_dev, cid, n, te, tr, ts, tq, nat.PUB_XY, st, ws_u), st)[1],
                lambda: cuda(ec.verify_batch_packed(te.cpu().numpy(), tr.cpu().numpy(), ts.cpu().numpy(), tq.cpu().numpy()))))

    ks = ec.key_set([b"\x04" + xy[j].tobytes() for j in range(M)])
    h = ks._sets[0]
    ws_k = u8(lib.eb200_keyset_dev_workspace_bytes(h, n))
    ti32 = cuda(idx.astype(np.int32))
    out.append(("secp256k1 keyed verify",
                lambda: ks.verify_batch_tensors(te, tr, ts, ti64),
                lambda: (raw(lib.eb200_ecdsa_verify_batch_keyed_dev, h, n, te, tr, ts, ti32, st, ws_k), st)[1],
                lambda: cuda(ks.verify_batch_packed(te.cpu().numpy(), tr.cpu().numpy(), ts.cpu().numpy(), ti64.cpu().numpy()))))

    parts, blob, off = der_blob(r, s)
    tb, toff = cuda(blob), cuda(off.astype(np.int64))
    out.append(("secp256k1 verify from DER",
                lambda: ec.verify_batch_der_tensors(te, tb, toff, tq),
                lambda: (raw(lib.eb200_ecdsa_verify_batch_der_dev, cid, n, te, tb, blob.size, toff, tq, nat.PUB_XY, st, ws_u),
                         st)[1],
                lambda: cuda(ec.verify_batch_der_packed(
                    te.cpu().numpy(), [bytes(b) for b in np.split(tb.cpu().numpy(), toff.cpu().numpy()[1:-1])],
                    tq.cpu().numpy()))))

    ed = EDDSA()
    rng = np.random.default_rng(n)
    sec = cuda(rng.integers(0, 256, (n, 32), dtype=np.uint8))
    msgs = cuda(rng.integers(0, 256, 64 * n, dtype=np.uint8))
    moff = cuda(np.arange(0, 64 * (n + 1), 64, dtype=np.int64))
    ws_e = u8(lib.eb200_dev_workspace_bytes(nat.CURVE_ED25519, n))
    sig = u8(n, 64)
    out.append(("ed25519 EdDSA sign",
                lambda: ed.sign_batch_tensors(sec, msgs, moff)[0],
                lambda: (raw(lib.eb200_eddsa_sign_batch_dev, n, sec, msgs, 64 * n, moff, sig, None, st, ws_e), sig)[1],
                lambda: cuda(ed.sign_batch_packed(sec.cpu().numpy(), msgs.cpu().numpy(), moff.cpu().numpy()))))

    keys = [{"x": xy[j, :ln].tobytes().hex(), "y": xy[j, ln:].tobytes().hex()} if j % 2 else
            bytes([2 + (xy[j, -1] & 1)]) + xy[j, :ln].tobytes() for j in range(M)]
    mixed = ec.key_set(keys)
    assert len(mixed._sets) == 2
    where = mixed._where[idx]
    locs = [cuda(np.where(where[:, 0] == k, where[:, 1], M).astype(np.int32)) for k in range(2)]
    sel = [cuda(where[:, 0] == k) for k in range(2)]
    ws_m = u8(max(lib.eb200_keyset_dev_workspace_bytes(hh, n) for hh in mixed._sets))
    parts_st = [u8(n), u8(n)]

    def raw_mixed():
        for k, hh in enumerate(mixed._sets):
            raw(lib.eb200_ecdsa_verify_batch_keyed_dev, hh, n, te, tr, ts, locs[k], parts_st[k], ws_m)
        return parts_st

    out.append(("secp256k1 keyed verify, mixed formats",
                lambda: mixed.verify_batch_tensors(te, tr, ts, ti64),
                raw_mixed,
                lambda: cuda(mixed.verify_batch_packed(te.cpu().numpy(), tr.cpu().numpy(), ts.cpu().numpy(),
                                                       ti64.cpu().numpy()))))
    return out, (ks, mixed), sel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sizes", default="1048576,1024")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_tensor_forms.json"))
    args = ap.parse_args()
    import torch
    from elliptic_b200 import _native as nat
    if not torch.cuda.is_available():
        raise SystemExit("bench_tensor_forms needs a CUDA device")
    lib = nat.init(0)
    name, power = gpu_info()
    rows = []
    for n in (int(x) for x in args.sizes.split(",")):
        calls, sets, sel = workloads(lib, nat, n)
        for label, tensor, rawf, packed in calls:
            mixed = "mixed" in label

            def same(t_out, r_out, p_out):
                if mixed:
                    r_out = torch.where(sel[0], r_out[0], r_out[1])
                return bool((t_out == r_out).all()) and bool((t_out == p_out).all())

            for _ in range(args.warmup):
                assert same(tensor(), rawf(), packed()), label
            ms = {"tensor": [], "raw": [], "packed": []}
            for _ in range(args.reps):
                outs = {}
                for form, f in (("tensor", tensor), ("raw", rawf), ("packed", packed)):
                    t, o = timed(f)
                    ms[form].append(t)
                    outs[form] = o
                assert same(outs["tensor"], outs["raw"], outs["packed"]), label
            med = {k: float(np.median(v)) for k, v in ms.items()}
            rows.append({"workload": label, "items": n, "median_ms": med, "all_ms": ms,
                         "tensor_minus_raw_us": (med["tensor"] - med["raw"]) * 1e3,
                         "packed_over_tensor": med["packed"] / med["tensor"]})
            print("%-40s n=%-8d tensor %9.3f  raw %9.3f  packed %9.3f ms" % (label, n, med["tensor"], med["raw"],
                                                                             med["packed"]), file=sys.stderr)
        for s_ in sets:
            s_.close()
    doc = {"gpu": name, "power_limit_w": power, "reps": args.reps, "timing": "host clock around call + device sync",
           "rows": rows}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(doc, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": power, "rows": len(rows)}))


if __name__ == "__main__":
    main()
