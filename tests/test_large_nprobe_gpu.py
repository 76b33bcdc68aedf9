"""IVF_FLAT and IVF_PQ Search, RangeSearch and AnnIterator with nprobe above 1008 (up to 65536), GPU.

Above 1008 probes the coarse stage selects each query's probes with the large-k selection, no scan CTA holds more than
1024 of them, and the queries run in groups whose probe arrays fit a fixed scratch (DESIGN §4.9.1).  The results follow
the rules every IVF search follows: probes in (dis0, list id) order, rows in storage order, (distance, id) order of the
result, -1 / +-FLT_MAX padding.  IVF_FLAT at nprobe = nlist is checked against the float64 brute-force oracle, IVF_PQ
against the compiled reference's IndexIVFPQ over the same imported quantizers and codes.  Indexes are imported, so nlist
can exceed what training on these corpora allows (rows / 39).
"""
import os
import subprocess

import numpy as np
import pytest

from knowhere_b200 import datagen
from tests.test_exact_oracle_gpu import _bits, _with_env, check_topk, flat_oracle, pq_oracle
from tests.test_range_oracle_gpu import (_ids_to_list, check_range, heuristic_model, in_window, per_query, probe_order,
                                         window_of)
from tests.util import assert_topk_parity

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ imported indexes
def _centroids(xb, nlist, seed, metric):
    """nlist rows of the corpus (repeated with a small perturbation when nlist exceeds it) as the coarse centroids"""
    rng = np.random.default_rng(seed)
    base = xb / np.linalg.norm(xb, axis=1, keepdims=True) if metric == "COSINE" else xb
    n = base.shape[0]
    pick = rng.choice(n, min(nlist, n), replace=False)
    cent = base[pick]
    if nlist > n:
        extra = base[rng.choice(n, nlist - n)] + 0.05 * rng.standard_normal((nlist - n, base.shape[1]))
        cent = np.concatenate([cent, extra])
    return np.ascontiguousarray(cent, np.float32)


def _pq_codebook(xb, cent, m, seed):
    """256 residuals of sampled rows against their nearest centroid, per sub-quantizer: [m][256][dsub]"""
    rng = np.random.default_rng(seed)
    X = torch.as_tensor(xb, device="cuda")
    C = torch.as_tensor(cent, device="cuda")
    a = torch.cat([torch.cdist(X[i:i + 8192], C).argmin(1) for i in range(0, X.shape[0], 8192)]).cpu().numpy()
    pick = rng.choice(xb.shape[0], 256, replace=False)
    res = xb[pick] - cent[a[pick]]
    d = xb.shape[1]
    return np.ascontiguousarray(res.reshape(256, m, d // m).transpose(1, 0, 2), np.float32)


def _import(kb, kind, metric, xb, cent, pq=None, cfg=None):
    """centroids (and PQ codebook) imported, rows assigned, encoded and laid out on the GPU by add()"""
    ix = kb.Index(kind, metric, xb.shape[1], dict({"nlist": cent.shape[0]}, **(cfg or {})))
    kb._check(kb.lib().kb2_ivf_import_begin(ix.h, cent.shape[0], cent.ctypes.data, None if pq is None else pq.ctypes.data))
    ix.add(xb)
    return ix


_cache = {}


def _flat_index(kb, metric, nlist, n=20000, d=64, nq=64):
    key = ("flat", metric, nlist, n, d, nq)
    if key not in _cache:
        xb, xq = datagen.clustered(n, d, 201), datagen.clustered(nq, d, 202)
        ix = _import(kb, "IVF_FLAT", metric, xb, _centroids(xb, nlist, 203, metric))
        _cache[key] = (ix, xb, xq) + flat_oracle(xb, xq, metric)
    return _cache[key]


# ------------------------------------------------------------------------------------------------ exact through IVF
@pytest.mark.parametrize("engine", ["scan", "tc"])
@pytest.mark.parametrize("nlist", [2048, 65536])
@pytest.mark.parametrize("metric", ["L2", "IP", "COSINE"])
def test_ivf_flat_all_lists_is_exact(kb, metric, nlist, engine):
    """nprobe = nlist scans every row with direct differences: the top-k is the float64 brute-force top-k.  At nlist
    65536 most of the 20000 rows' lists hold one row and most lists are empty."""
    ix, xb, xq, D, B = _flat_index(kb, metric, nlist)
    n = xb.shape[0]
    for k in (1, 10, 100, 1000):
        ids, dist = _with_env("KB2_FLAT_ENGINE", engine, lambda: ix.search(xq, k, {"nprobe": nlist}))
        check_topk(ids, dist, D, B, np.arange(n), metric, what=f"IVF_FLAT nlist {nlist} {engine} k={k}")


# ------------------------------------------------------------------------------------------------ IVF_PQ vs the reference
PQ_GEOMS = [pytest.param(16, 128, id="m16xdsub8"), pytest.param(48, 96, id="m48xdsub2")]


def _pq_index(kb, ref, m, d, refine_type=None, nlist=8192, n=40000):
    key = ("pq", m, d, refine_type, nlist, n)
    if key not in _cache:
        xb = datagen.clustered(n, d, 211)
        cent = _centroids(xb, nlist, 212, "L2")
        pq = _pq_codebook(xb, cent, m, 213)
        cfg = {"m": m, "nbits": 8}
        if refine_type:
            cfg.update(refine=True, refine_type=refine_type)
        ix = _import(kb, "IVF_PQ", "L2", xb, cent, pq, cfg)
        r = ref.RefIvf("IVF_PQ", d, 0, nlist, m, 8, refine=refine_type is not None)
        r.import_state(cent, pq, [(l,) + ix.ivf_export_list(l, m) for l in range(nlist)], raw=xb)
        _cache[key] = (ix, r, xb)
    return _cache[key]


@pytest.mark.parametrize("nprobe", [1009, 4096, 8192])
@pytest.mark.parametrize("m,d", PQ_GEOMS)
def test_ivfpq_matches_reference(kb, ref, m, d, nprobe):
    """ids and ADC distances against IndexIVFPQ over the same state: 64 queries through the query-major LUT kernels and
    512 through the list-major tensor-core engine"""
    ix, r, _ = _pq_index(kb, ref, m, d)
    xq = datagen.clustered(512, d, 214)
    k = 10
    I0, D0 = r.search(xq, k, nprobe)
    ids, dist = _with_env("KB2_PQ_ENGINE", "lut", lambda: ix.search(xq[:64].copy(), k, {"nprobe": nprobe}))
    assert ix.last_stage_info()["engine"] == "scan"
    assert_topk_parity(ids, dist, I0[:64], D0[:64], rtol=1e-4, atol=1e-3, what=f"IVF_PQ m{m} lut nprobe {nprobe}",
                       max_tie_rows=64)
    ids, dist = ix.search(xq, k, {"nprobe": nprobe})
    assert ix.last_stage_info()["engine"] == "tc"
    assert_topk_parity(ids, dist, I0, D0, rtol=1e-4, atol=1e-3, what=f"IVF_PQ m{m} tc nprobe {nprobe}", max_tie_rows=512)


@pytest.mark.parametrize("refine_type", ["flat", "fp16", "bf16"])
@pytest.mark.parametrize("nprobe", [1009, 8192])
def test_ivfpq_refine_matches_reference(kb, ref, refine_type, nprobe):
    """refine_k 4 against IndexIVFPQ + IndexRefineFlat: the fp32 store gives the reference's ids and distances; the
    16-bit stores re-rank the same candidates with rounded rows, so ids agree up to near ties and distances to the
    rounding"""
    ix, r, _ = _pq_index(kb, ref, 16, 128, refine_type)
    xq = datagen.clustered(64, 128, 215)
    k = 10
    I0, D0 = r.search(xq, k, nprobe, refine_k=4.0)
    ids, dist = ix.search(xq, k, {"nprobe": nprobe, "refine_k": 4})
    if refine_type == "flat":
        assert_topk_parity(ids, dist, I0, D0, what=f"IVF_PQ refine nprobe {nprobe}")
    else:
        same = np.mean([len(set(a) & set(b)) / k for a, b in zip(ids, I0)])
        assert same >= 0.95, f"{refine_type} refine overlap {same}"
        hit = ids == I0
        np.testing.assert_allclose(dist[hit], D0[hit], rtol=2e-2, atol=1e-2)


def test_ivfpq_large_batch_groups_match_single_queries(kb, ref):
    """nprobe = nlist = 65536 (the largest accepted) on 40000 rows: 1000 queries need two query groups; every row of
    the batch equals the search of that query alone, and the whole batch matches the reference"""
    ix, r, _ = _pq_index(kb, ref, 16, 128, nlist=65536)
    xq = datagen.clustered(1000, 128, 216)
    k = 10
    ids, dist = ix.search(xq, k, {"nprobe": 65536})
    for i in (0, 1, 788, 789, 999):
        a, b = ix.search(xq[i:i + 1].copy(), k, {"nprobe": 65536})
        assert np.array_equal(a[0], ids[i]) and np.array_equal(b[0].view(np.uint32), dist[i].view(np.uint32)), f"q{i}"
    I0, D0 = r.search(xq, k, 65536)
    assert_topk_parity(ids, dist, I0, D0, rtol=1e-4, atol=1e-3, what="IVF_PQ nprobe 65536 nq 1000", max_tie_rows=1000)


# ------------------------------------------------------------------------------------------------ continuity at 1008
def test_rows_scanned_at_1008_and_1009(kb, ref):
    """query-major LUT path: one more probe scans exactly each query's 1009th list in addition"""
    ix, r, _ = _pq_index(kb, ref, 16, 128)
    xq = datagen.clustered(64, 128, 217)
    lens = np.array([kb.lib().kb2_ivf_list_size(ix.h, l) for l in range(8192)], np.int64)
    probes, _ = r.coarse(xq, 1009)
    codes = []
    for nprobe in (1008, 1009):
        _with_env("KB2_PQ_ENGINE", "lut", lambda: ix.search(xq, 10, {"nprobe": nprobe}))
        assert ix.last_stage_info()["engine"] == "scan"
        codes.append(ix.last_counters()["codes"])
    assert codes[1] - codes[0] == int(lens[probes[:, 1008]].sum())


# ------------------------------------------------------------------------------------------------ RangeSearch
def _range_model(off, list_of, order, metric, radius, max_empty):
    ids, dist = off
    if max_empty <= 0:
        keep = np.isin(list_of[ids], order) & in_window(dist, metric, radius)
        return ids[keep], dist[keep], len(order)
    ids, dist, cut, _ = heuristic_model(off, list_of, order, metric, radius, None, max_empty)
    return ids, dist, cut


@pytest.mark.parametrize("max_empty", [0, 2])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_ivf_flat_range_many_probes(kb, metric, max_empty):
    """RangeSearch at nprobe 4096 and nlist (8192) follows range_search_preassigned: the index's own hits with every
    list probed and the heuristic off, restricted to the probed lists and cut after max_empty consecutive empty
    probes, equal the result exactly.  The unrestricted result passes the float64 oracle."""
    nlist = 8192
    ix, xb, xq, D, B = _flat_index(kb, metric, nlist, nq=100)
    n = xb.shape[0]
    cent = ix.ivf_export_centroids(0)[0]
    list_of = _ids_to_list(ix, 4 * xb.shape[1], nlist, n)
    radius = window_of(D, metric, 0.002, 0.02)[0]
    full = ix.range_search(xq, radius, None, {"nprobe": nlist, "max_empty_result_buckets": 0})
    assert check_range(*full, D, B, np.arange(n), metric, radius, what=f"IVF_FLAT range nprobe {nlist}") > 0
    off = per_query(*full)
    order, tie = probe_order(cent, xq, metric)
    for nprobe in (4096, nlist):
        on = per_query(*ix.range_search(xq, radius, None, {"nprobe": nprobe, "max_empty_result_buckets": max_empty}))
        checked = 0
        for i in range(xq.shape[0]):
            ids, dist, cut = _range_model(off[i], list_of, order[i, :nprobe], metric, radius, max_empty)
            # a near tie between consecutive probes can reorder them: it matters at the last probe scanned, and with the
            # heuristic on anywhere up to the cut
            if tie[i, nprobe - 1:nprobe].any() or (max_empty > 0 and tie[i, :cut].any()):
                continue
            checked += 1
            key = dist if metric == "L2" else -dist
            o = np.lexsort((ids, key))
            assert np.array_equal(on[i][0], ids[o]) and np.array_equal(on[i][1], dist[o]), \
                f"nprobe {nprobe} max_empty {max_empty} q{i}: {on[i][0].size} hits, the model keeps {ids.size}"
        assert checked >= 0.3 * xq.shape[0], checked


# ------------------------------------------------------------------------------------------------ edges
@pytest.mark.parametrize("keep", [1.0, 0.5, 0.0], ids=["no-bitset", "half", "all-filtered"])
def test_bitsets_many_probes(kb, keep):
    ix, xb, xq, D, B = _flat_index(kb, "L2", 2048)
    n = xb.shape[0]
    valid = np.random.default_rng(218).random(n) < keep
    bits = None if keep == 1.0 else _bits(~valid)
    for k in (10, 1500):
        ids, dist = ix.search(xq, k, {"nprobe": 2048}, bitset=bits)
        check_topk(ids, dist, D, B, np.arange(n), "L2", valid=valid, what=f"bitset keep {keep} k={k}")


@pytest.mark.parametrize("nq", [1, 64])
def test_large_k_many_probes(kb, nq):
    """k up to 16384 with nprobe 2048 (the large-k path over more than 1008 probes)"""
    ix, xb, xq, D, B = _flat_index(kb, "L2", 2048)
    for k in (2000, 16384):
        ids, dist = ix.search(xq[:nq].copy(), k, {"nprobe": 2048})
        assert ix.last_stage_info()["engine"] == "large_k"
        check_topk(ids, dist, D[:nq], B[:nq], np.arange(xb.shape[0]), "L2", what=f"k={k} nq={nq}")


def test_nq1_and_clamp(kb):
    """one query; nprobe 65536 on nlist 2048 is clamped and gives the nprobe = 2048 result bit for bit"""
    ix, xb, xq, D, B = _flat_index(kb, "IP", 2048)
    a = ix.search(xq[:1].copy(), 10, {"nprobe": 2048})
    check_topk(*a, D[:1], B[:1], np.arange(xb.shape[0]), "IP", what="nq=1")
    b = ix.search(xq[:1].copy(), 10, {"nprobe": 65536})
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def _status(kb, fn):
    try:
        fn()
    except kb.KnowhereError as e:
        return e.status, str(e)
    return 0, ""


def test_nprobe_range_and_sharded_limit(kb):
    ix, xb, xq, _, _ = _flat_index(kb, "L2", 2048)
    assert _status(kb, lambda: ix.search(xq, 10, {"nprobe": 65537}))[0] == 3
    assert _status(kb, lambda: ix.range_search(xq, 1.0, None, {"nprobe": 65537}))[0] == 3
    small = _import(kb, "IVF_FLAT", "L2", xb, _centroids(xb, 64, 219, "L2"))
    assert _status(kb, lambda: small.search(xq, 10, {"nprobe": 65537}))[0] == 3
    # a list-sharded handle keeps the limit of one coarse window
    sh = kb.Index("IVF_FLAT", "L2", xb.shape[1], {"nlist": 2048})
    sh.set_shard(0, 2)
    cent = _centroids(xb, 2048, 203, "L2")
    kb._check(kb.lib().kb2_ivf_import_begin(sh.h, 2048, cent.ctypes.data, None))
    sh.add(xb)
    sh.search(xq, 10, {"nprobe": 1008})
    st, msg = _status(kb, lambda: sh.search(xq, 10, {"nprobe": 1009}))
    assert st == 3 and "nprobe too large for the GPU path (max 1008)" in msg


# ------------------------------------------------------------------------------------------------ AnnIterator (C++)
def test_ann_iterator_ivfpq_nprobe_4096(tmp_path):
    exe = tmp_path / "test_large_nprobe"
    subprocess.run(["g++", "-std=c++17", "-O2", f"-I{ROOT}/include", os.path.join(ROOT, "tests", "cpp", "test_large_nprobe.cc"),
                    "-o", str(exe), f"-L{ROOT}/knowhere_b200", "-l:libknowhere_b200.so",
                    f"-Wl,-rpath,{ROOT}/knowhere_b200"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "iterator ok" in r.stdout
