#!/usr/bin/env python3
"""Device time of one large-k search (DESIGN §4.9) and its split into the path's three stages:

  FLAT      1M x 128, nq 100, k 16384
  IVF_FLAT  the C2 shape (1M x 128, nlist 1024, nprobe 32, nq 1000), k 5000
  IVF_PQ    1M x 128, m 16, nlist 1024, nprobe 64, nq 100, k 4096, refine_k 4 (fp32 store)

Stages, by kernel name in a torch.profiler trace of one search: keys (the contraction / the dense row scan), select
(select_rows_kernel), finalize (re-rank, segmented sorts, emission).  Next to each stage: the bytes the stage must move at
least (ALGORITHMIC: one pass over its inputs and outputs, not counting the select's repeated passes over L2-resident rows)
divided by its time.  The card name and power limit are read in the same run.  Prints one JSON line.

  python scripts/bench_large_k.py [--rows 1000000] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def stage_of(name):
    if "select_rows_kernel" in name:
        return "select"
    if "gemm" in name or "range_scan_kernel" in name or "row_norms" in name:
        return "keys"
    if "large_" in name or "Segmented" in name or "segment_offsets" in name or "max_abs" in name:
        return "finalize"
    return "other"


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return name, power


def measure(torch, fn, reps):
    fn()                                                  # warm-up: allocations, kernel attributes
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {"keys": 0.0, "select": 0.0, "finalize": 0.0, "other": 0.0}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0:
            split[stage_of(ev.name)] += ev.device_time / 1000.0
    return float(np.median(times)), split


def report(ms, split, bytes_):
    out = {"search_ms": round(ms, 3)}
    for s in ("keys", "select", "finalize"):
        t = split[s]
        out[f"{s}_ms"] = round(t, 3)
        out[f"{s}_algorithmic_GBps"] = round(bytes_[s] / (t * 1e-3) / 1e9, 1) if t > 0 else None
    out["other_ms"] = round(split["other"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    import knowhere_b200 as kb
    from knowhere_b200 import datagen
    n, d = args.rows, 128
    dev = torch.device("cuda", 0)
    xb = datagen.clustered_torch(n, d, 42, dev)
    gpu, power = card()
    res = {"gpu": gpu, "power_limit_w": power, "rows": n}

    # FLAT
    nq, k = 100, 16384
    K = k + 16
    xq = datagen.clustered_torch(nq, d, 43, dev)
    f = kb.Index("FLAT", "L2", d)
    f.add(xb)
    ms, split = measure(torch, lambda: f.search(xq, k), args.reps)
    assert f.last_stage_info()["engine"] == "large_k"
    res["flat"] = report(ms, split, {"keys": n * d * 4 + nq * n * 4, "select": nq * n * 4,
                                     "finalize": nq * K * (d * 4 + 48) + nq * k * 12})
    del f

    # IVF_FLAT, C2 shape
    nq, k, nlist, nprobe = 1000, 5000, 1024, 32
    xq = datagen.clustered_torch(nq, d, 44, dev)
    iv = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
    iv.build(xb)
    ms, split = measure(torch, lambda: iv.search(xq, k, {"nprobe": nprobe}), args.reps)
    scanned = iv.last_counters()["codes"]
    assert iv.last_stage_info()["engine"] == "large_k"
    res["ivf_flat_c2"] = report(ms, split, {"keys": scanned * (d * 4 + 8), "select": scanned * 8,
                                            "finalize": nq * k * 48 + nq * k * 12})
    del iv

    # IVF_PQ + refine
    nq, k, rk, nlist, nprobe = 100, 4096, 4, 1024, 64
    K = k * rk
    xq = datagen.clustered_torch(nq, d, 45, dev)
    pq = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": 16, "nbits": 8, "refine": True, "refine_type": "flat"})
    pq.build(xb)
    ms, split = measure(torch, lambda: pq.search(xq, k, {"nprobe": nprobe, "refine_k": rk}), args.reps)
    scanned = pq.last_counters()["codes"]
    assert pq.last_stage_info()["engine"] == "large_k"
    res["ivf_pq_refine"] = report(ms, split, {"keys": scanned * (16 + 4 + 8), "select": scanned * 8,
                                              "finalize": nq * K * (d * 4 + 48) + nq * k * 12})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
