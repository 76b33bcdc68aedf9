"""Search with a candidate window above 1024 entries (k > 1008 on FLAT / BruteForce / HNSW's exact branch, k (x refine_k)
> 1024 on IVF_FLAT / IVF_PQ) up to 16384: the large-k path of DESIGN §4.9, checked against the float64 oracle of
test_exact_oracle_gpu (check_topk: exact ids up to the oracle's error bound, (distance, id) order, padding)."""
import os
import subprocess

import numpy as np
import pytest

from knowhere_b200 import datagen
from tests.test_exact_oracle_gpu import _bits, check_topk, flat_oracle, pq_oracle
from tests.util import assert_topk_parity

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _custom_ids(n, seed):
    return np.random.default_rng(seed).permutation(n).astype(np.int64) * 3 + 11


# ------------------------------------------------------------------------------------------------ FLAT / BruteForce
FLAT_CASES = [
    # nq, n, d, k
    pytest.param(8, 40000, 128, 1009, id="k1009"),
    pytest.param(8, 40000, 128, 4096, id="k4096"),
    pytest.param(8, 40000, 128, 16384, id="k16384"),
    pytest.param(2000, 40000, 128, 2000, id="two_chunks"),     # key matrix in two chunks: running best set merged once
    pytest.param(16, 20000, 17, 1500, id="d17-fp32"),          # d % 4 != 0: fp32 contraction, whole-warp re-rank
    pytest.param(8, 20000, 1536, 1200, id="d1536"),
    pytest.param(4, 10000, 64, 16384, id="n_lt_k-padding"),
]


@pytest.mark.parametrize("custom", [False, True], ids=["rowids", "customids"])
@pytest.mark.parametrize("metric", ["L2", "IP", "COSINE"])
@pytest.mark.parametrize("nq,n,d,k", FLAT_CASES)
def test_flat_large_k_exact(kb, nq, n, d, k, metric, custom):
    xb = datagen.uniform(n, d, 1000 + d)
    xq = datagen.uniform(nq, d, 2000 + d)
    labels = _custom_ids(n, 5) if custom else np.arange(n, dtype=np.int64)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb, labels if custom else None)
    ids, dist = ix.search(xq, k)
    assert ix.last_stage_info()["engine"] == "large_k"
    c = ix.last_counters()
    assert c["codes"] == nq * n and c["pairs"] == nq
    sample = np.arange(nq) if nq <= 64 else np.random.default_rng(3).choice(nq, 24, replace=False)
    D, B = flat_oracle(xb, xq[sample], metric)
    om = "IP" if metric == "COSINE" else metric
    check_topk(ids[sample], dist[sample], D, B, labels, om, what=f"FLAT {metric} k={k}")
    if not custom:
        bi, bd = kb.brute_force_search(xb, xq, k, metric)
        assert np.array_equal(bi, ids) and np.array_equal(bd, dist)


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_bruteforce_large_k_device_tensors(kb, metric):
    n, nq, d, k = 30000, 12, 128, 3000
    xb = datagen.uniform(n, d, 51)
    xq = datagen.uniform(nq, d, 52)
    bi, bd = kb.brute_force_search(torch.from_numpy(xb).cuda(), torch.from_numpy(xq).cuda(), k, metric)
    assert bi.is_cuda and bd.is_cuda
    D, B = flat_oracle(xb, xq, metric)
    check_topk(bi.cpu().numpy(), bd.cpu().numpy(), D, B, np.arange(n), metric, what="BruteForce device")
    hi, hd = kb.brute_force_search(xb, xq, k, metric)
    assert np.array_equal(hi, bi.cpu().numpy()) and np.array_equal(hd, bd.cpu().numpy())


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("keep,k", [(3000, 5000), (30000, 16384)])
def test_flat_large_k_bitset(kb, metric, keep, k):
    n, nq, d = 50000, 6, 64
    xb = datagen.uniform(n, d, 31)
    xq = datagen.uniform(nq, d, 32)
    mask = np.ones(n, bool)                       # True = filtered out
    mask[np.random.default_rng(keep).choice(n, keep, replace=False)] = False
    labels = _custom_ids(n, 9)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb, labels)
    ids, dist = ix.search(xq, k, bitset=_bits(mask))
    D, B = flat_oracle(xb, xq, metric)
    check_topk(ids, dist, D, B, labels, metric, valid=~mask, what=f"FLAT bitset keep={keep} k={k}")


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_flat_large_k_translated_data(kb, metric):
    """Rows 1000 + N(0, 1): the norm-expanded keys cancel, finalize cannot certify the window, and the queries are redone
    from the directly accumulated key rows of range_scan_kernel's dense mode."""
    n, nq, d, k = 20000, 16, 128, 2000
    rng = np.random.default_rng(7)
    xb = (1000.0 + rng.standard_normal((n, d))).astype(np.float32)
    xq = (1000.0 + rng.standard_normal((nq, d))).astype(np.float32)
    mask = rng.random(n) < 0.3
    D, B = flat_oracle(xb, xq, metric)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb)
    for bits, valid in ((None, None), (_bits(mask), ~mask)):
        ids, dist = ix.search(xq, k, bitset=bits)
        if metric == "L2":
            assert ix.last_counters()["flagged"] > 0
        check_topk(ids, dist, D, B, np.arange(n), metric, valid=valid, what="FLAT translated large k")


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_flat_large_k_ties_keep_lowest_positions(kb, metric):
    """One row copied to 1400 positions, queries next to it, k = 1200: the tie group crosses the k-th rank and the kept
    copies are the lowest positions (DESIGN §4.6)."""
    n, d, ndup, k = 20000, 64, 1400, 1200
    rng = np.random.default_rng(3)
    xb = datagen.uniform(n, d, 3)
    pos = np.sort(rng.choice(n, ndup, replace=False))
    xb[pos] = xb[pos[0]] * (4.0 if metric == "IP" else 1.0)
    xq = (xb[pos[0]] + 0.01 * rng.standard_normal((4, d))).astype(np.float32)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb)
    ids, dist = ix.search(xq, k)
    D, B = flat_oracle(xb, xq, metric)
    check_topk(ids, dist, D, B, np.arange(n), metric, what="FLAT ties large k")
    for i in range(xq.shape[0]):
        assert np.array_equal(ids[i], pos[:k]), "tied copies must be taken in position order"
        assert (dist[i] == dist[i, 0]).all()


# ------------------------------------------------------------------------------------------------ IVF
@pytest.fixture(scope="module")
def ivf_flat_data():
    n, nq, d = 20000, 12, 64
    plain = (datagen.clustered(n, d, 81), datagen.clustered(nq, d, 82))
    rng = np.random.default_rng(83)
    shifted = ((1000.0 + rng.standard_normal((n, d))).astype(np.float32),
               (1000.0 + rng.standard_normal((nq, d))).astype(np.float32))
    return {"clustered": plain, "translated": shifted}


@pytest.mark.parametrize("data", ["clustered", "translated"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_ivf_flat_large_k_all_lists_is_exact(kb, ivf_flat_data, data, metric):
    xb, xq = ivf_flat_data[data]
    n, d = xb.shape
    nlist = 32
    ix = kb.Index("IVF_FLAT", metric, d, {"nlist": nlist})
    ix.build(xb)
    D, B = flat_oracle(xb, xq, metric)
    for k in (1009, 5000, 16384):
        ids, dist = ix.search(xq, k, {"nprobe": nlist})
        if k > 1024:                             # IVF: the window is k itself (k 1009 stays on the scan kernels)
            assert ix.last_stage_info()["engine"] == "large_k"
            c = ix.last_counters()
            assert c["codes"] == xq.shape[0] * n and c["pairs"] == xq.shape[0] * nlist
        check_topk(ids, dist, D, B, np.arange(n), metric, what=f"IVF_FLAT {data} k={k}")


PQ_GEOMS = [(16, 128), (32, 128), (48, 96)]


@pytest.fixture(scope="module")
def pq_indexes(kb):
    cache = {}

    def get(m, d, metric, nlist=32, n=20000, nq=12):
        key = (m, d, metric, nlist, n, nq)
        if key not in cache:
            xb = datagen.clustered(n, d, 91)
            xq = datagen.clustered(nq, d, 92)
            ix = kb.Index("IVF_PQ", metric, d, {"nlist": nlist, "m": m, "nbits": 8})
            ix.build(xb)
            cache[key] = (ix, xb, xq) + pq_oracle(ix, xq, m, metric)
        return cache[key]
    return get


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("m,d", PQ_GEOMS, ids=["m16d128", "m32d128", "m48d96"])
def test_ivfpq_large_k_matches_adc_oracle(kb, pq_indexes, m, d, metric):
    ix, _, xq, D, B, labels = pq_indexes(m, d, metric)
    for k in (1009, 4096, 16384):
        ids, dist = ix.search(xq, k, {"nprobe": 32})
        assert (ix.last_stage_info()["engine"] == "large_k") == (k > 1024)
        check_topk(ids, dist, D, B, labels, metric, what=f"IVF_PQ m{m} k={k}")


@pytest.mark.parametrize("refine_type", ["flat", "fp16", "bf16"])
def test_ivfpq_large_k_refine(kb, refine_type):
    n, nq, d, m, nlist, k = 20000, 8, 128, 16, 32, 2000
    xb = datagen.clustered(n, d, 101)
    xq = datagen.clustered(nq, d, 102)
    ix = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m, "refine": True, "refine_type": refine_type})
    ix.build(xb)
    ids, dist = ix.search(xq, k, {"nprobe": nlist, "refine_k": 4})
    assert ix.last_stage_info()["engine"] == "large_k"
    # the refine store answers exactly like fp32 rows holding its rounded values
    tdt = {"flat": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}[refine_type]
    xr = torch.from_numpy(xb).to(tdt).to(torch.float32).numpy()
    D, B = flat_oracle(xr, xq, "L2")
    for i in range(nq):
        assert (ids[i] >= 0).all() and np.unique(ids[i]).size == k
        err = np.abs(dist[i].astype(np.float64) - D[i, ids[i]])
        assert (err <= B[i, ids[i]]).all(), f"q{i}: refined distances are not exact"
        key = dist[i].astype(np.float64)
        assert ((key[1:] > key[:-1]) | ((key[1:] == key[:-1]) & (ids[i, 1:] > ids[i, :-1]))).all()
    gt = np.argsort(D, axis=1)[:, :k]
    assert datagen.recall(gt, ids) > 0.9
    with pytest.raises(kb.KnowhereError) as e:
        ix.search(xq, 16385, {"nprobe": nlist, "refine_k": 1})
    assert e.value.status == 1
    # k * refine_k = 16385
    with pytest.raises(kb.KnowhereError) as e:
        ix.search(xq, 3277, {"nprobe": nlist, "refine_k": 5.0001})
    assert e.value.status == 1


def test_large_k_prefix_stability(kb, pq_indexes):
    """The first 1000 entries of a k = 3000 search are the k = 1000 search (what AnnIterator relies on), with a bitset
    and nprobe < nlist."""
    n, d = 20000, 128
    xb = datagen.clustered(n, d, 91)
    xq = datagen.clustered(20, d, 92)
    mask = np.random.default_rng(5).random(n) < 0.3
    bits = _bits(mask)
    f = kb.Index("FLAT", "L2", d)
    f.add(xb)
    iv = kb.Index("IVF_FLAT", "L2", d, {"nlist": 64})
    iv.build(xb)
    pq, _, _, _, _, _ = pq_indexes(16, 128, "L2", nlist=32)
    for name, ix, cfg in (("FLAT", f, {}), ("IVF_FLAT", iv, {"nprobe": 16}), ("IVF_PQ", pq, {"nprobe": 8})):
        i_s, d_s = ix.search(xq, 1000, cfg, bitset=bits)
        i_l, d_l = ix.search(xq, 3000, cfg, bitset=bits)
        assert ix.last_stage_info()["engine"] == "large_k"
        assert not np.isin(i_l[i_l >= 0], np.nonzero(mask)[0]).any()
        assert_topk_parity(i_l[:, :1000], d_l[:, :1000], i_s, d_s, what=f"{name} prefix")


def test_ivfpq_large_k_batch_shapes(kb, pq_indexes):
    """k 2048: one query (the iterator's pattern), five queries (probes split over many CTAs), and a batch run in query
    groups (200000 rows with nprobe = nlist: about 650 query rows fit the scratch budget).  Every batch gives each query
    the answer it gets alone."""
    ix, _, xq, D, B, labels = pq_indexes(16, 128, "L2")
    k = 2048
    one_i, one_d = ix.search(xq[:1].copy(), k, {"nprobe": 32})
    check_topk(one_i, one_d, D[:1], B[:1], labels, "L2", what="IVF_PQ nq=1")
    five_i, five_d = ix.search(xq[:5].copy(), k, {"nprobe": 32})
    check_topk(five_i, five_d, D[:5], B[:5], labels, "L2", what="IVF_PQ nq=5")
    assert np.array_equal(five_i[:1], one_i) and np.array_equal(five_d[:1], one_d)

    n, d, nlist, nq = 200000, 128, 64, 1500
    xb = datagen.clustered(n, d, 93)
    xq2 = datagen.clustered(nq, d, 94)
    big = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": 16, "nbits": 8})
    big.build(xb)
    bi, bd = big.search(xq2, k, {"nprobe": nlist})
    for s in (slice(0, 3), slice(700, 703), slice(nq - 3, nq)):
        si, sd = big.search(xq2[s].copy(), k, {"nprobe": nlist})
        assert np.array_equal(si, bi[s]) and np.array_equal(sd, bd[s])
    D2, B2, l2 = pq_oracle(big, xq2[-4:], 16, "L2")
    check_topk(bi[-4:], bd[-4:], D2, B2, l2, "L2", what="IVF_PQ grouped batch")


def test_large_k_path_selection_and_errors(kb):
    n, d = 20000, 64
    xb = datagen.uniform(n, d, 7)
    xq = datagen.uniform(4, d, 8)
    f = kb.Index("FLAT", "L2", d)
    f.add(xb)
    iv = kb.Index("IVF_FLAT", "L2", d, {"nlist": 16})
    iv.build(xb)
    f.search(xq, 1008)
    assert f.last_stage_info()["engine"] == "scan"
    f.search(xq, 1009)
    assert f.last_stage_info()["engine"] == "large_k"
    iv.search(xq, 1024, {"nprobe": 4})
    assert iv.last_stage_info()["engine"] != "large_k"
    iv.search(xq, 1025, {"nprobe": 4})
    assert iv.last_stage_info()["engine"] == "large_k"
    for ix, cfg in ((f, {}), (iv, {"nprobe": 4})):
        with pytest.raises(kb.KnowhereError) as e:
            ix.search(xq, 16385, cfg)
        assert e.value.status == 1 and "16384" in str(e.value)
    with pytest.raises(kb.KnowhereError) as e:
        kb.brute_force_search(xb, xq, 16385, "L2")
    assert e.value.status == 1


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_hnsw_exact_branch_large_k(kb, metric):
    n, nq, d, k = 3000, 10, 32, 2000
    xb = datagen.uniform(n, d, 21)
    xq = datagen.uniform(nq, d, 22)
    ix = kb.Index("HNSW", metric, d, {"M": 8, "efConstruction": 40})
    ix.build(xb)
    ids, dist = ix.search(xq, k)                 # k >= n / 2: exact branch
    D, B = flat_oracle(xb, xq, metric)
    check_topk(ids, dist, D, B, np.arange(n), metric, what="HNSW exact branch k=2000")


def test_ann_iterator_past_1008(tmp_path):
    """AnnIterator over an IVF_FLAT index walks 5000 results: distinct ids, monotone distances, the first 1008 equal to
    Search(k = 1008)."""
    exe = tmp_path / "test_large_k"
    subprocess.run(["g++", "-std=c++17", "-O2", f"-I{ROOT}/include", os.path.join(ROOT, "tests", "cpp", "test_large_k.cc"),
                    "-o", str(exe), f"-L{ROOT}/knowhere_b200", "-l:libknowhere_b200.so",
                    f"-Wl,-rpath,{ROOT}/knowhere_b200"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "iterator ok" in r.stdout
