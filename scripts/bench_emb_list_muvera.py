"""Emb-list search with the MUVERA strategy against TokenANN on the same index type (DESIGN §4.11, §6): time per search and
per stage (encode + base search, candidates, re-rank, select: device events), candidates per list, and recall@10 against
the exact BruteForce emb-list search.  TokenANN runs in the same call over a sweep of its base search key, so that the
two can be compared at matched recall.  One JSON line per measurement, the card's name and power limit first; with --out
the whole record also goes to that file.  Needs an H100.

Workload: the documents of scripts/bench_emb_list_index.py (20 000 documents of 32..256 rows of datagen.clustered,
d = 128, MAX_SIM_IP) on IVF_FLAT (nlist 2048), and 1000 query lists of 32 tokens in two forms:
  tokens    each token a row of a random document plus noise (bench_emb_list_index.py's queries): a list matches
            single tokens of many documents;
  document  the tokens of a list are rows of one random document plus noise: a list describes one document, the case
            MUVERA's one encoding per list is made for.
MUVERA at its defaults (P 4, R 7: E = 14 336) builds IVF_FLAT over the 20 000 encoded documents."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import knowhere_b200 as kb  # noqa: E402
from knowhere_b200 import datagen  # noqa: E402
from bench_emb_list_index import card  # noqa: E402


def timed(ix, xq, ql, k, cfg, reps):
    ix.search_emb_list(xq, ql, k, cfg)   # warm-up
    times, stages = [], []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ids, _, st = ix.search_emb_list(xq, ql, k, cfg, stats=True)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        stages.append(ix.emb_list_stage_ms())
    med = {s: float(np.median([x[s] for x in stages])) for s in stages[0]}
    return ids, st, float(np.median(times)), times, med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=20000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--lists", type=int, default=1000)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--nlist", type=int, default=2048)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--projections", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--muvera-nprobe", default="32,128")
    ap.add_argument("--muvera-ratio", default="3,10")
    ap.add_argument("--tokenann-nprobe", default="4,8,16,32")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the whole record to this JSON file")
    a = ap.parse_args()
    dev = "cuda"
    rng = np.random.default_rng(0)
    lens = rng.integers(32, 257, a.docs)
    xl = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = int(xl[-1])
    xb = datagen.clustered_torch(n, a.dim, 1, dev)
    pick = torch.as_tensor(rng.integers(0, n, a.lists * a.tokens), device=dev)
    queries = {"tokens": xb[pick]}
    doc = rng.integers(0, a.docs, a.lists).repeat(a.tokens)
    queries["document"] = xb[torch.as_tensor(xl[doc] + rng.integers(0, 1 << 30, doc.size) % lens[doc], device=dev)]
    for m in queries:
        queries[m] = (queries[m] + 0.3 * torch.randn(a.lists * a.tokens, a.dim, device=dev)).contiguous()
    ql = (np.arange(a.lists + 1) * a.tokens).astype(np.int64)
    rec = {"card": card(), "rows": n, "docs": a.docs, "dim": a.dim, "lists": a.lists, "tokens": a.tokens, "k": a.k,
           "metric": "MAX_SIM_IP", "index": "IVF_FLAT", "reps": a.reps, "results": []}
    print(json.dumps({"card": rec["card"], "rows": n}), flush=True)
    gt = {m: kb.brute_force_search_emb_list(xb, xl, xq, ql, a.k, "MAX_SIM_IP")[0].cpu().numpy() for m, xq in queries.items()}

    def report(r):
        rec["results"].append(r)
        print(json.dumps(r), flush=True)

    for strategy in ("muvera", "tokenann"):
        cfg = {"nlist": a.nlist}
        if strategy == "muvera":
            cfg.update(emb_list_strategy="muvera", muvera_num_projections=a.projections, muvera_num_repeats=a.repeats)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix = kb.Index("IVF_FLAT", "IP", a.dim, cfg)
        if strategy == "tokenann":
            ix.train(xb)
        ix.add(xb)
        ix.set_emb_list(xl, "MAX_SIM_IP")
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        ix.enable_kernel_timing(True)
        sweep = ([(int(p), float(r)) for p in a.muvera_nprobe.split(",") for r in a.muvera_ratio.split(",")]
                 if strategy == "muvera" else [(int(p), 3.0) for p in a.tokenann_nprobe.split(",")])
        for mode, xq in queries.items():
            for nprobe, ratio in sweep:
                scfg = {"nprobe": nprobe, "retrieval_ann_ratio": ratio}
                ids, st, med_ms, all_ms, stages = timed(ix, xq, ql, a.k, scfg, a.reps)
                report({"strategy": strategy, "queries": mode, "cfg": scfg, "build_s": build_s, "search_ms_median": med_ms,
                        "search_ms_all": all_ms, "stage_ms_median": stages, "candidates_per_list": float(st[1]) / a.lists,
                        "recall_at_10_vs_bruteforce": datagen.recall(gt[mode], ids.cpu().numpy())})
        del ix
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
