#!/usr/bin/env python3
"""BASELINE configs[4] (C5): IVF_PQ IP, 100M x 96 int8, m=48 nbits=8 nlist=65536 nprobe=128, batch=10000, inverted lists
sharded across the GPUs of one box (one process per GPU, NCCL communicator owned by libknowhere_b200.so).

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port P \
      scripts/bench_c5.py --rows 100000000 --steps 10 --warmup 3

int8 data: the reference widens int8 to fp32 up front (src/index/index_node_data_mock_wrapper.cc:24-60); here the typed
entry points widen each chunk on the device.  Every rank regenerates the same synthetic rows chunk by chunk (seeded), assigns
all of them (wgmma contraction against the 65536 centroids) and keeps the codes of the lists it owns (l % world).
Rank 0 trains (k-means on 256 x nlist sampled rows, PQ on 65536) and broadcasts the quantizers.
Prints ONE JSON line (rank 0): queries/s (device-resident batch, collective search), e2e with host buffers, recall@10 vs
exact brute force on a sample of the queries, roofline of the filter kernel, per-stage breakdown.
--rows / --nlist scale the problem down for smoke runs (e.g. 10M / 6553 on 2 GPUs).
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def gen_chunk(torch, datagen, start, count, d, dev, scale):
    """rows [start, start+count) of the synthetic base as int8 (deterministic per chunk)"""
    x = datagen.clustered_torch(count, d, 42 + 7919 * (start // count + 1), dev, n_clusters=50000)
    return torch.clamp(torch.round(x * scale), -127, 127).to(torch.int8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--nlist", type=int, default=65536)
    ap.add_argument("--nprobe", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=2_000_000)
    ap.add_argument("--gt-queries", type=int, default=500)
    args = ap.parse_args()

    import torch
    import torch.distributed as dist

    import knowhere_b200 as kb
    from knowhere_b200 import datagen
    sys.path.insert(0, ROOT)
    from bench import ClockSampler, make_comm, peaks, peaks_tensor, recall_of

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("NCCL_DEBUG", "WARN")
        dist.init_process_group("nccl", device_id=dev)
    n, d, m, k, nq = args.rows, 96, 48, 10, args.nq
    nlist, nprobe, chunk = args.nlist, args.nprobe, min(args.chunk, args.rows)
    assert n % chunk == 0
    stream = torch.cuda.current_stream().cuda_stream
    scale = 127.0 / 14.0   # the mixture's values stay within ~ +-14

    # ---- quantizers: rank 0 trains on a sample, everybody receives them
    t0 = time.time()
    cfgb = {"nlist": nlist, "m": m, "nbits": 8}
    ix = kb.Index("IVF_PQ", "IP", d, cfgb, device=local_rank)
    ix.set_stream(stream)
    if world > 1:
        ix.set_shard(rank, world)
    cent = torch.empty((nlist, d), dtype=torch.float32, device=dev)
    pq = torch.empty((m, 256, d // m), dtype=torch.float32, device=dev)
    if rank == 0:
        n_train = min(n, 256 * nlist)
        per = max(1, n_train // (n // chunk))
        parts = []
        for c0 in range(0, n, chunk):
            xc = gen_chunk(torch, datagen, c0, chunk, d, dev, scale)
            sel = torch.randperm(chunk, device=dev, generator=torch.Generator(device=dev).manual_seed(c0 + 1))[:per]
            parts.append(xc[sel].contiguous())
        xt = torch.cat(parts)
        t = kb.Index("IVF_PQ", "IP", d, cfgb, device=local_rank)
        t.set_stream(stream)
        t.train(xt)
        c_h, pq_h = t.ivf_export_centroids(m)
        cent.copy_(torch.from_numpy(c_h))
        pq.copy_(torch.from_numpy(pq_h))
        del t, xt, parts
    if world > 1:
        dist.broadcast(cent, 0)
        dist.broadcast(pq, 0)
    torch.cuda.synchronize()
    t_train = time.time() - t0
    kb._check(kb.lib().kb2_ivf_import_begin(ix.h, nlist, cent.data_ptr(), pq.data_ptr()))

    # ---- add: every rank encodes the stream; seal keeps the owned lists
    t0 = time.time()
    for c0 in range(0, n, chunk):
        ix.add(gen_chunk(torch, datagen, c0, chunk, d, dev, scale))
    torch.cuda.synchronize()
    t_add = time.time() - t0
    comm = make_comm(kb, dist, rank, world, local_rank) if world > 1 else None
    if comm is not None:
        ix.set_comm(comm)

    xq = torch.clamp(torch.round(datagen.clustered_torch(nq, d, 43, dev, n_clusters=50000) * scale), -127, 127).to(torch.int8)
    ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
    dis = torch.empty((nq, k), dtype=torch.float32, device=dev)
    cfg = {"nprobe": nprobe}
    t0 = time.time()
    ix.search(xq, k, cfg, out=(ids, dis))      # first search seals the lists
    torch.cuda.synchronize()
    t_seal = time.time() - t0

    # ---- ground truth on a sample of the queries: exact IP over the whole base, chunk by chunk (every rank takes a slice
    #      of the chunks; partial top-k merged on rank 0 through gloo-free NCCL gathers of small tensors)
    ngt = min(args.gt_queries, nq)
    xq_f = xq[:ngt].to(torch.float32).contiguous()
    best_i = torch.full((ngt, k), -1, dtype=torch.int64, device=dev)
    best_d = torch.full((ngt, k), -3.0e38, dtype=torch.float32, device=dev)
    my_chunks = [c0 for j, c0 in enumerate(range(0, n, chunk)) if j % world == rank]
    for c0 in my_chunks:
        xc = gen_chunk(torch, datagen, c0, chunk, d, dev, scale).to(torch.float32)
        gi, gd = kb.brute_force_search(xc, xq_f, k, "IP", device=local_rank, stream=stream)
        ci = torch.stack([best_i, gi + c0])
        cd = torch.stack([best_d, gd])
        best_i, best_d = kb.merge_topk(ci, cd, "IP", device=local_rank, stream=stream)
        del xc
    if world > 1:
        gi_all = torch.empty((world, ngt, k), dtype=torch.int64, device=dev)
        gd_all = torch.empty((world, ngt, k), dtype=torch.float32, device=dev)
        dist.all_gather_into_tensor(gi_all, best_i)
        dist.all_gather_into_tensor(gd_all, best_d)
        best_i, best_d = kb.merge_topk(gi_all, gd_all, "IP", device=local_rank, stream=stream)
    torch.cuda.synchronize()
    recall = recall_of(best_i.cpu().numpy(), ids[:ngt].cpu().numpy())

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        ix.search(xq, k, cfg, out=(ids, dis))
    ix.enable_kernel_timing(True)
    sampler = ClockSampler(local_rank) if rank == 0 else None
    barrier()
    if os.environ.get("KB2_PROFILE"):       # ncu --profile-from-start off: capture only the timed steps
        torch.cuda.cudart().cudaProfilerStart()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kernel_ms, stage_ms, comm_ms = [], [], []
    e0.record()
    for _ in range(args.steps):
        ix.search(xq, k, cfg, out=(ids, dis))
        info = ix.last_stage_info()
        kernel_ms.append(info["kernel_ms"]); stage_ms.append(info["stage_ms"]); comm_ms.append(info["comm_ms"])
    e1.record()
    barrier()
    if os.environ.get("KB2_PROFILE"):
        torch.cuda.cudart().cudaProfilerStop()
    clocks = sampler.stop() if sampler else None
    ms_total = e0.elapsed_time(e1)
    ctr = ix.last_counters()
    pairs_codes = torch.tensor([float(ctr["codes"]), float(ctr["survivors"]), ms_total], device=dev, dtype=torch.float64)
    if world > 1:
        tmax = torch.tensor([ms_total], device=dev)
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        ms_total = float(tmax.item())
        allc = [torch.zeros_like(pairs_codes) for _ in range(world)]
        dist.all_gather(allc, pairs_codes)
        codes_all = sum(float(c[0]) for c in allc)
    else:
        codes_all = float(ctr["codes"])

    # ---- end to end with host buffers
    xq_h = xq.cpu().numpy()
    ids_h = np.empty((nq, k), np.int64)
    dis_h = np.empty((nq, k), np.float32)
    ix.enable_kernel_timing(False)
    for _ in range(2):
        ix.search(xq_h, k, cfg, out=(ids_h, dis_h))
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        ix.search(xq_h, k, cfg, out=(ids_h, dis_h))
    barrier()
    e2e_s = time.perf_counter() - t0
    if world > 1:
        t = torch.tensor([e2e_s], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e_s = float(t.item())

    if rank == 0:
        peak, peak_src = peaks()
        tpeak, tsrc = peaks_tensor()
        k_ms = statistics.mean(kernel_ms)
        qps = nq * args.steps / (ms_total / 1e3)
        alg_bytes_all = codes_all * m        # SURVEY 8(d): probed codes x 48 B, all shards
        out = {
            "metric": "queries/sec, IVF_PQ IP 100Mx96 int8 m48 nlist65536 nprobe128 (BASELINE configs[4])",
            "value": qps, "unit": "queries/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_total / args.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "f32 (int8 inputs widened on the device)", "data": "synthetic",
            "config": {"workload": f"IVF_PQ IP {n}x{d} int8, nlist={nlist}, m={m}, nbits=8, nprobe={nprobe}, batch={nq}, k={k}",
                       "recall_at_10_pure_adc": recall, "recall_queries": ngt,
                       "sharding": f"lists l % {world}, collectives inside the library" if world > 1 else "single GPU",
                       "train_s": round(t_train, 1), "add_s": round(t_add, 1), "seal_and_first_search_s": round(t_seal, 1)},
            "e2e": {"value": nq * args.steps / e2e_s, "unit": "queries/s", "h2d_bytes_per_step": nq * d,
                    "d2h_bytes_per_step": nq * k * 12},
            "clocks": clocks,
            "roofline": {"bound": "tensor", "kernel": "ivfpq_tc_filter_kernel<3,2>", "kernel_ms_rank0": k_ms,
                         "achieved": ctr["codes"] * 2.0 * d / (k_ms / 1e3) / 1e12, "peak": tpeak, "unit": "TFLOP/s",
                         "frac": ctr["codes"] * 2.0 * d / (k_ms / 1e3) / 1e12 / tpeak, "peak_source": tsrc,
                         "engine": ix.last_stage_info()["engine"],
                         "hbm_algorithmic": {"bytes_per_batch_all_shards": alg_bytes_all,
                                             "bytes_per_query": alg_bytes_all / nq,
                                             "achieved_gbs_per_gpu": alg_bytes_all / world / (ms_total / args.steps / 1e3) / 1e9,
                                             "frac_of_hbm_peak_per_gpu": alg_bytes_all / world / (ms_total / args.steps / 1e3) / 1e9 / peak,
                                             "peak_gbs": peak, "peak_source": peak_src}},
            "stage_breakdown_rank0_ms": {"list_scan_stage": statistics.mean(stage_ms), "filter_kernel": k_ms,
                                         "collectives_and_merge": statistics.mean(comm_ms)},
            "survivors_rank0": ctr["survivors"], "queries_redone_rank0": ctr["flagged"],
        }
        print(json.dumps(out))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
