#!/usr/bin/env python3
"""Per-role cycle accounting of the IVF_PQ filter kernel (ivfpq_tc_filter_kernel, knowhere_b200/csrc/kb2_ivfpq_tc.cuh).

  python scripts/filter_stalls.py [--workload ivf_pq_10m] [--refine-k 4] [--lib PATH]

Builds the library with -DKB2_FILTER_STALLS into a temporary directory (or takes a library built that way with --lib),
loads it through KB2_LIB, builds the workload's index as bench.py does and runs one search.  With the macro set, each
CTA of the filter kernel prints the clock64() cycles that one thread of each group spent in the waits and phases of
its role, summed over the role's two groups.  The script prints every phase as a share of the role's cycles, median
and max over the CTAs, then one JSON line.  The instrumented kernel is slower than the default build; the shares say
where a role waits, not how long the default build takes.
"""
import argparse
import ctypes
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build_lib(out_dir):
    from knowhere_b200 import _build
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    lib = os.path.join(out_dir, "libknowhere_b200_stalls.so")
    cmd = [nvcc] + _build.NVCC_FLAGS + ["-DKB2_FILTER_STALLS", "-o", lib] + _build.UNITS + ["-lgomp", "-ldl"]
    subprocess.run(cmd, check=True)
    return lib


def captured_stdout(fn):
    """run fn() with file descriptor 1 (where device printf goes) sent to a temporary file; return its text"""
    libc = ctypes.CDLL(None)
    sys.stdout.flush()
    libc.fflush(None)
    saved = os.dup(1)
    with tempfile.TemporaryFile("w+") as f:
        os.dup2(f.fileno(), 1)
        try:
            fn()
        finally:
            libc.fflush(None)
            os.dup2(saved, 1)
            os.close(saved)
        f.seek(0)
        return f.read()


def parse(text):
    rows = []
    for line in text.splitlines():
        if not line.startswith("KB2STALL "):
            continue
        f = dict(kv.split("=", 1) for kv in line.split()[1:])
        rows.append({"dec": [int(v) for v in f["dec"].split(",")], "cons": [int(v) for v in f["cons"].split(",")]})
    return rows


def shares(rows):
    """per CTA: each phase over the role's total cycles.  The slots are those listed at the end of
    ivfpq_tc_filter_kernel; decode and stage_b are reported without the a_empty and b_free waits that they contain."""
    per = {"consumers": {}, "decoders": {}}
    for r in rows:
        d, c = r["dec"], r["cons"]
        dec = {"a_empty": d[1], "b_free": d[2], "decode": d[3] - d[1], "stage_b": d[4] - d[2], "write_meta": d[5]}
        cons = {"meta_full": c[1], "b_full": c[2], "a_full": c[3], "wgmma_wait": c[4], "flush": c[5],
                "wgmma_issue": c[6], "sign_test": c[7]}
        cons["other"] = c[0] - sum(cons.values())
        dec["other"] = d[0] - sum(dec.values())
        for role, vals, tot in (("decoders", dec, d[0]), ("consumers", cons, c[0])):
            for k, v in vals.items():
                per[role].setdefault(k, []).append(v / max(tot, 1))
    return {role: {k: {"median": statistics.median(v), "max": max(v)} for k, v in ph.items()} for role, ph in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ivf_pq_10m", choices=["ivf_pq_10m", "ivf_pq_1m"])
    ap.add_argument("--refine-k", type=int, default=4, help="refine_k of the search (bench.py calibrates 4 on ivf_pq_10m)")
    ap.add_argument("--lib", default=None, help="a library already built with -DKB2_FILTER_STALLS")
    args = ap.parse_args()

    tmp = tempfile.mkdtemp(prefix="kb2_stalls_")
    try:
        os.environ["KB2_LIB"] = args.lib or build_lib(tmp)
        import torch

        import knowhere_b200 as kb
        from bench import WORKLOADS, build_index
        from knowhere_b200 import datagen

        wl = WORKLOADS[args.workload]
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(0)
        stream = torch.cuda.current_stream().cuda_stream
        xb = datagen.clustered_torch(wl["n"], wl["d"], 42, dev)
        xq = datagen.clustered_torch(wl["nq"], wl["d"], 43, dev)
        ix = build_index(kb, torch, None, wl, xb, 0, 1, stream)
        cfg = dict(wl["search"], refine_k=args.refine_k)

        def step():
            ix.search(xq, wl["k"], cfg)
            torch.cuda.synchronize()

        captured_stdout(step)             # warm-up: module load, list sealing
        rows = parse(captured_stdout(step))
        if ix.last_stage_info()["engine"] != "tc" or not rows:
            raise SystemExit("the search did not run the instrumented filter kernel (engine "
                             f"{ix.last_stage_info()['engine']}, {len(rows)} CTA lines): is the library built with -DKB2_FILTER_STALLS?")
        sh = shares(rows)
        print(f"{args.workload}: filter kernel, {len(rows)} CTAs, share of each role's cycles (median / max over CTAs)")
        for role in ("consumers", "decoders"):
            for k, v in sh[role].items():
                print(f"  {role:9s} {k:12s} {v['median']:6.3f} / {v['max']:6.3f}")
        print(json.dumps({"workload": args.workload, "ctas": len(rows), "shares": sh,
                          "gpu": torch.cuda.get_device_name(0)}))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
