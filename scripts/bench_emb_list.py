#!/usr/bin/env python3
"""Emb-list BruteForce search (MAX_SIM, DESIGN §4.10) on ColBERT-like data, against a plain torch fp32 implementation.

Data (seeded, generated on the GPU): documents of uniformly drawn lengths, unit rows at d = 128, query lists of 32 tokens.
  --preset full   100000 documents of 32..512 tokens (about 27M rows), 1000 query lists
  --preset small    5000 documents of 32..512 tokens, 100 query lists
For MAX_SIM and MAX_SIM_L2 at k = 10 and k = 100: the median call time over --reps warm calls (device-resident inputs and
outputs, CUDA events), the filter kernel's device time (maxsim_filter_kernel in a torch.profiler trace of one more call),
useful TFLOP/s = 2 * query tokens * base tokens * d / time and its share of the data-sheet 3xTF32 ceiling (495 / 3
TFLOP/s, H100 SXM dense TF32 / 3 products), the HBM bytes the filter reads (base bytes x query chunks), and the stats
counters.  The baseline is torch with TF32 off: per chunk an fp32 matmul, a segment extremum (scatter_reduce), a sum over
each list's tokens and a topk; both must agree within the tests' error bound.  The card name and power limit are read in
the same run.  Prints one JSON line.

  python scripts/bench_emb_list.py [--preset full|small] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


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


def timed(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), out


def torch_maxsim(torch, X, xl, Q, ql, k, l2, lists_per_chunk=50, rows_per_chunk=1 << 20):
    """The plain torch baseline: fp32 matmuls (TF32 off), segment extremum, token sum, topk.  Returns (ids, scores)."""
    n_docs, n_lists = xl.numel() - 1, ql.numel() - 1
    doc = torch.repeat_interleave(torch.arange(n_docs, device=X.device), xl[1:] - xl[:-1])
    xn = (X * X).sum(1) if l2 else None
    out_i, out_s = [], []
    for l0 in range(0, n_lists, lists_per_chunk):
        l1 = min(n_lists, l0 + lists_per_chunk)
        q0, q1 = int(ql[l0]), int(ql[l1])
        Qc = Q[q0:q1]
        lst = torch.repeat_interleave(torch.arange(l1 - l0, device=X.device), ql[l0 + 1:l1 + 1] - ql[l0:l1])
        qn = (Qc * Qc).sum(1) if l2 else None
        ext = torch.full((n_docs, q1 - q0), float("inf") if l2 else -float("inf"), device=X.device)
        for r0 in range(0, X.shape[0], rows_per_chunk):
            s = X[r0:r0 + rows_per_chunk] @ Qc.T
            if l2:
                s = xn[r0:r0 + rows_per_chunk, None] + qn[None, :] - 2 * s
            idx = doc[r0:r0 + rows_per_chunk, None].expand(-1, q1 - q0)
            ext.scatter_reduce_(0, idx, s, "amin" if l2 else "amax")
        score = torch.zeros((l1 - l0, n_docs), device=X.device).index_add_(0, lst, ext.T)
        v, i = torch.topk(score, k, dim=1, largest=not l2)
        out_i.append(i)
        out_s.append(v)
    return torch.cat(out_i), torch.cat(out_s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="full", choices=["full", "small"])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import knowhere_b200 as kb
    torch.backends.cuda.matmul.allow_tf32 = False
    n_docs, n_lists = (100000, 1000) if a.preset == "full" else (5000, 100)
    d, qlen = 128, 32
    rng = np.random.default_rng(2026)
    xl = torch.as_tensor(np.concatenate([[0], np.cumsum(rng.integers(32, 513, n_docs))]), device="cuda")
    ql = torch.as_tensor(np.arange(n_lists + 1, dtype=np.int64) * qlen, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(7)
    X = torch.randn((int(xl[-1]), d), generator=g, device="cuda")
    X /= X.norm(dim=1, keepdim=True)
    Q = torch.randn((n_lists * qlen, d), generator=g, device="cuda")
    Q /= Q.norm(dim=1, keepdim=True)
    rows = X.shape[0]
    flop = 2.0 * Q.shape[0] * rows * d
    lds = (n_docs + 3) // 4 * 4
    name, power = card()
    res = dict(card=name, power_limit_w=power, preset=a.preset, n_docs=n_docs, base_rows=rows, n_lists=n_lists,
               query_tokens=Q.shape[0], d=d, useful_tflop=flop / 1e12, runs=[])
    from torch.profiler import ProfilerActivity, profile
    for metric in ("MAX_SIM", "MAX_SIM_L2"):
        l2 = metric == "MAX_SIM_L2"
        base_ms, (bi, bs) = timed(torch, lambda: torch_maxsim(torch, X, xl, Q, ql, 100, l2), max(1, a.reps // 2))
        for k in (10, 100):
            ms, (ids, dist, st) = timed(torch, lambda: kb.brute_force_search_emb_list(X, xl, Q, ql, k, metric, stats=True),
                                        a.reps)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                kb.brute_force_search_emb_list(X, xl, Q, ql, k, metric)
                torch.cuda.synchronize()
            filt_us = sum(e.device_time_total for e in prof.key_averages() if "maxsim_filter_kernel" in e.key)
            # agreement with the baseline: the k-th score (selection ties aside, the same documents score the same)
            # within a bound of 2 * 32 tokens * (d + 2) 2^-24 * 4 (unit rows, L2 distances up to 4) per list
            tol = 2 * qlen * (d + 2) * 2.0 ** -24 * 4
            dk = (dist[:, k - 1].double() - bs[:, k - 1].double()).abs().max().item()
            overlap = float(np.mean([len(set(x) & set(y)) / k for x, y in
                                     zip(ids.cpu().numpy(), bi[:, :k].cpu().numpy())]))
            chunks = -(-n_lists // max(1, min(n_lists, (64 << 20) // lds)))
            res["runs"].append(dict(
                metric=metric, k=k, median_ms=ms, filter_ms=filt_us / 1e3,
                useful_tflops_call=flop / ms / 1e9, useful_tflops_filter=flop / (filt_us / 1e3) / 1e9 if filt_us else None,
                share_of_3xtf32_ceiling_filter=(flop / (filt_us / 1e3) / 1e9) / (495.0 / 3) if filt_us else None,
                filter_hbm_bytes=rows * d * 4 * chunks, query_chunks=chunks, stats=[int(v) for v in st],
                torch_fp32_ms=base_ms, speedup_vs_torch=base_ms / ms, kth_score_max_abs_diff=dk, kth_tol=tol,
                agree=bool(dk <= tol), id_overlap=overlap))
            print(json.dumps(res["runs"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
