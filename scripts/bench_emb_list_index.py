"""Emb-list (multi-vector) search on HNSW and IVF_FLAT (TokenANN, DESIGN §4.11): time per search and per stage, candidates
per list, the re-rank's useful FLOP/s, recall@k against the exact BruteForce emb-list search, and a torch.profiler
trace of one k = 100 search.  One JSON line per measurement; with --out the whole record also goes to that file.  Needs
an H100.

Workload (defaults): 20 000 documents of 32..256 rows of datagen.clustered (d = 128, ~2.9M rows), MAX_SIM_IP; HNSW
(M 16, efConstruction 100, built on the GPU) and IVF_FLAT (nlist 2048); 1000 query lists of 32 tokens, each token a row
of a random document plus noise, so that every list has true neighbours; k 10 and 100 at retrieval_ann_ratio 3."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import knowhere_b200 as kb  # noqa: E402
from knowhere_b200 import datagen  # noqa: E402

FP32_PEAK = 67e12   # H100 SXM data sheet, dense FP32 (a 700 W card)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:   # the measurement still names the device torch sees
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=20000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--nlist", type=int, default=2048)
    ap.add_argument("--ef", type=int, default=128)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--indexes", default="HNSW,IVF_FLAT")
    ap.add_argument("--out", default=None, help="also write the whole record to this JSON file")
    a = ap.parse_args()
    dev = "cuda"
    rng = np.random.default_rng(0)
    lens = rng.integers(32, 257, a.docs)
    xl = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = int(xl[-1])
    xb = datagen.clustered_torch(n, a.dim, 1, dev)
    pick = torch.as_tensor(rng.integers(0, n, a.lists * a.tokens), device=dev)
    xq = (xb[pick] + 0.3 * torch.randn(a.lists * a.tokens, a.dim, device=dev)).contiguous()
    ql = (np.arange(a.lists + 1) * a.tokens).astype(np.int64)
    rec = {"card": card(), "rows": n, "docs": a.docs, "dim": a.dim, "lists": a.lists, "tokens": a.tokens,
           "metric": "MAX_SIM_IP", "results": []}
    print(json.dumps({"card": rec["card"], "rows": n}), flush=True)

    gt = {}
    for k in (10, 100):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gi, _ = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, "MAX_SIM_IP")
        torch.cuda.synchronize()
        gt[k] = gi.cpu().numpy()
        print(json.dumps({"bruteforce_k": k, "ms": 1e3 * (time.perf_counter() - t0)}), flush=True)

    for itype in a.indexes.split(","):
        t0 = time.perf_counter()
        if itype == "HNSW":
            ix = kb.Index("HNSW", "IP", a.dim, {"M": 16, "efConstruction": 100})
            ix.add(xb)
            base_cfg = {"ef": a.ef}
        else:
            ix = kb.Index("IVF_FLAT", "IP", a.dim, {"nlist": a.nlist})
            ix.build(xb)
            base_cfg = {"nprobe": a.nprobe}
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        ix.set_emb_list(xl, "MAX_SIM_IP")
        ix.enable_kernel_timing(True)
        for k in (10, 100):
            cfg = dict(base_cfg, retrieval_ann_ratio=3.0)
            if itype == "HNSW":
                cfg["ef"] = max(a.ef, k)
            ix.search_emb_list(xq, ql, k, cfg)   # warm-up
            times, stages = [], []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                ids, dist, st = ix.search_emb_list(xq, ql, k, cfg, stats=True)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
                stages.append(ix.emb_list_stage_ms())
            med = {s: float(np.median([x[s] for x in stages])) for s in stages[0]}
            flop = 2.0 * a.dim * float(st[2])
            r = {"index": itype, "k": k, "cfg": cfg, "build_s": build_s, "search_ms_median": float(np.median(times)),
                 "search_ms_all": times, "stage_ms_median": med, "candidates_per_list": float(st[1]) / a.lists,
                 "token_row_distances": int(st[2]),
                 "rerank_useful_tflops": flop / (med["rerank"] * 1e-3) / 1e12 if med["rerank"] > 0 else None,
                 "rerank_share_of_fp32_datasheet_peak": flop / (med["rerank"] * 1e-3) / FP32_PEAK if med["rerank"] > 0 else None,
                 "recall_at_k_vs_bruteforce": datagen.recall(gt[k], ids.cpu().numpy())}
            rec["results"].append(r)
            print(json.dumps(r), flush=True)

        # one profiled run: device time per kernel
        cfg = dict(base_cfg, retrieval_ann_ratio=3.0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ix.search_emb_list(xq, ql, 100, cfg)
            torch.cuda.synchronize()
        ker = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" or getattr(ev, "self_device_time_total", 0) > 0:
                ker[ev.key[:80]] = getattr(ev, "self_device_time_total", getattr(ev, "self_cuda_time_total", 0)) / 1e3
        top = dict(sorted(ker.items(), key=lambda kv: -kv[1])[:12])
        rec["results"].append({"index": itype, "profile_k100_kernel_ms": top})
        print(json.dumps({"index": itype, "profile_k100_kernel_ms": top}), flush=True)

        del ix
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
