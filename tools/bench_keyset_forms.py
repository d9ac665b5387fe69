"""Time the DER and device-pointer forms of the keyed ECDSA verify against their unkeyed counterparts on one GPU and
print one JSON line.

Per shape the items are valid signatures made by eb200_ecdsa_sign_batch over m keys (one in 64 damaged in e), with
their canonical DER, and the set is created at the given table width.  In each of --reps alternated rounds (after
--warmup), on the same items:
  keyed_der      eb200_ecdsa_verify_batch_keyed_der
  unkeyed_der    eb200_ecdsa_verify_batch_der, keys gathered
  keyed          eb200_ecdsa_verify_batch_keyed fed with r, s parsed from the DER on the host (the parse is not timed)
  keyed_dev      eb200_ecdsa_verify_batch_keyed_dev on torch tensors, timed with CUDA events on the caller's stream
  unkeyed_dev    eb200_ecdsa_verify_batch_dev, keys gathered on the device, timed the same way
wall_ms is the host clock around a host-pointer call (it returns synchronised); dev_ms the events around a
device-pointer call; main_kernel_ms comes from eb200_last_timing().  The statuses of all five are asserted equal in
every round.  Medians are reported.  Once per shape, the Python KeySet.verify_batch is timed on DER-hex signatures at
--host-items items, to put a number on the per-item host parse the keyed DER call avoids.

    python tools/bench_keyset_forms.py [--reps 10] [--warmup 2] [--host-items 16384] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

# (curve, id, len, items, keys, width)
SHAPES = [("secp256k1", 1, 32, 1 << 20, 4096, 8), ("p256", 2, 32, 1 << 20, 4096, 8)]


def canonical_der(r, s):
    def one(v):
        b = v.lstrip(b"\x00") or b"\x00"
        return b"\x00" + b if b[0] & 0x80 else b
    out = []
    for i in range(len(r)):
        ri, si = one(r[i].tobytes()), one(s[i].tobytes())
        body = b"\x02" + bytes([len(ri)]) + ri + b"\x02" + bytes([len(si)]) + si
        out.append(b"\x30" + bytes([len(body)]) + body)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-items", type=int, default=1 << 14)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from bench_keyset import gpu_query
    from elliptic_b200 import _native as nat
    from elliptic_b200.ec import EC, parse_der
    from gpu_keyset_items import gpu_items
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyset_forms: no CUDA device (there is no CPU path to measure)")
    lib = nat.init(0)
    name, watts = gpu_query()
    res = {"gpu": name, "power_limit_w": watts, "reps": a.reps, "shapes": []}
    for curve, cid, ln, n, m, W in SHAPES:
        xy, e, r, s, idx = gpu_items(lib, nat, cid, ln, m, n, seed=cid * 1000 + m % 997)
        pub = np.ascontiguousarray(xy[idx])
        ders = canonical_der(r, s)
        blob = np.frombuffer(b"".join(ders), np.uint8)
        off = np.zeros(n + 1, np.uint64)
        off[1:] = np.cumsum([len(d) for d in ders])
        kst, h = np.zeros(m, np.uint8), ctypes.c_void_p()
        nat.check(lib.eb200_keyset_create(cid, m, xy.ctypes.data, 0, W, kst.ctypes.data, ctypes.byref(h)))
        # host parse of the DER, as a caller of the fixed-width keyed call has to do it (timed once, not in the rounds)
        t = time.perf_counter()
        rs = [parse_der(d) for d in ders]
        host_parse_ms = (time.perf_counter() - t) * 1e3
        hr = np.frombuffer(b"".join(v[0].to_bytes(ln, "big") for v in rs), np.uint8).reshape(n, ln)
        hs = np.frombuffer(b"".join(v[1].to_bytes(ln, "big") for v in rs), np.uint8).reshape(n, ln)
        dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
        de, dr, ds, dpub = dev(e), dev(r), dev(s), dev(pub)
        didx = dev(idx.view(np.int32))
        dst = torch.empty(n, dtype=torch.uint8, device="cuda")
        wsk = torch.empty(lib.eb200_ecdsa_verify_keyed_workspace_bytes(h, n), dtype=torch.uint8, device="cuda")
        wsu = torch.empty(lib.eb200_ecdsa_verify_workspace_bytes(cid, n), dtype=torch.uint8, device="cuda")
        stream = torch.cuda.current_stream()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        out = {k: np.zeros(n, np.uint8) for k in ("keyed_der", "unkeyed_der", "keyed", "keyed_dev", "unkeyed_dev")}
        rows = {k: [] for k in out}
        for rep in range(a.warmup + a.reps):
            for kind in out:
                if kind.endswith("_dev"):
                    ev0.record(stream)
                    if kind == "keyed_dev":
                        rc = lib.eb200_ecdsa_verify_batch_keyed_dev(h, n, de.data_ptr(), dr.data_ptr(), ds.data_ptr(),
                                                                    didx.data_ptr(), dst.data_ptr(), wsk.data_ptr(),
                                                                    ctypes.c_void_p(stream.cuda_stream))
                    else:
                        rc = lib.eb200_ecdsa_verify_batch_dev(cid, n, de.data_ptr(), dr.data_ptr(), ds.data_ptr(),
                                                              dpub.data_ptr(), 0, dst.data_ptr(), wsu.data_ptr(),
                                                              ctypes.c_void_p(stream.cuda_stream))
                    nat.check(rc)
                    ev1.record(stream)
                    stream.synchronize()
                    t_ms = ev0.elapsed_time(ev1)
                    out[kind][:] = dst.cpu().numpy()
                else:
                    t = time.perf_counter()
                    if kind == "keyed_der":
                        nat.call(lib.eb200_ecdsa_verify_batch_keyed_der, h, n, e, blob, off, idx, out[kind])
                    elif kind == "unkeyed_der":
                        nat.call(lib.eb200_ecdsa_verify_batch_der, cid, n, e, blob, off, pub, 0, out[kind])
                    else:
                        nat.call(lib.eb200_ecdsa_verify_batch_keyed, h, n, e, hr, hs, idx, out[kind])
                    t_ms = (time.perf_counter() - t) * 1e3
                tm = nat.last_timing()
                if rep >= a.warmup:
                    rows[kind].append((tm["main_kernel_ms"], t_ms, tm["launches"]))
            ref = out["unkeyed_der"]
            assert all((v == ref).all() for v in out.values()) and ref.sum() == n - (n + 63) // 64, curve
        # the Python mirror's keyed verify on DER hex: its per-item host parse
        k = min(a.host_items, n)
        ec = EC(curve)
        ks = ec.key_set([{"x": xy[j, :ln].tobytes().hex(), "y": xy[j, ln:].tobytes().hex()} for j in range(m)])
        msgs = [e[i].tobytes().hex() for i in range(k)]
        sigs = [ders[i].hex() for i in range(k)]
        t = time.perf_counter()
        py = ks.verify_batch(msgs, sigs, idx[:k])
        py_ms = (time.perf_counter() - t) * 1e3
        assert (py == ref[:k]).all()
        ks.close()
        nat.check(lib.eb200_keyset_destroy(h))
        med = lambda kind, j: float(np.median([x[j] for x in rows[kind]]))
        shape = {"curve": curve, "items": n, "keys": m, "table_bits": W, "host_der_parse_ms": host_parse_ms,
                 "python_keyset_verify_batch_der_hex": {"items": k, "wall_ms": py_ms, "us_per_item": py_ms * 1e3 / k}}
        for kind in rows:
            shape[kind] = {"main_kernel_ms": med(kind, 0), ("dev_ms" if kind.endswith("_dev") else "wall_ms"): med(kind, 1),
                           "launches": int(rows[kind][0][2])}
        shape["keyed_der_vs_unkeyed_der_wall"] = med("unkeyed_der", 1) / med("keyed_der", 1)
        shape["keyed_dev_vs_unkeyed_dev"] = med("unkeyed_dev", 1) / med("keyed_dev", 1)
        res["shapes"].append(shape)
        del de, dr, ds, dpub, didx, dst, wsk, wsu
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
