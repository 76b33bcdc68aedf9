"""HNSW beam search with max(ef, k) beyond the four-queries-per-CTA kernels, up to 16384: hnsw_wide_kernel (one query per
CTA, DESIGN §4.7).  Parity cases search the reference's own graph (RefHnsw.export -> hnsw_import), as test_hnsw_gpu does."""
import functools
import os
import subprocess

import numpy as np
import pytest

from knowhere_b200 import datagen
from tests.util import recall_at_k

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MAX = np.finfo(np.float32).max


@functools.lru_cache(maxsize=8)
def _ref_graph(n, d, M, metric, seed=42):
    from oracle import ref
    xb = datagen.clustered(n, d, seed)
    h = ref.RefHnsw(d, M, metric, 100)
    h.add(xb)
    return xb, h, h.export()


def _imported(kb, ref, n, d, M, metric):
    xb, h, g = _ref_graph(n, d, M, metric)
    ix = kb.Index("HNSW", "L2" if metric == 0 else "IP", d, {"M": M, "efConstruction": 100})
    ix.hnsw_import(xb, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    return xb, h, ix


def _engine(ix):
    return ix.last_stage_info()["engine"]


def _against_reference(ids, dist, I0, D0, stats, stats0, k, tol, by_position=True):
    """by_position=False: the bar is on each row's id set.  A filtered traversal that evaluates one node more or less than
    the reference's (an fp32 near tie against the valid pool's back) adds or drops one id, which shifts every later
    position of that row."""
    if k <= 10:
        same_rows = (ids == I0).all(axis=1).mean()
        print(f"identical rows {same_rows:.3f}")
        assert same_rows > 0.9
    else:
        same_pos = (ids == I0).mean()
        common = np.mean([len(np.intersect1d(a[a >= 0], b[b >= 0])) / max(1, int((b >= 0).sum())) for a, b in zip(ids, I0)])
        first = [int(np.argmax(a != b)) for a, b in zip(ids, I0) if (a != b).any()]
        print(f"identical (row, position) ids {same_pos:.4f}, common ids per row {common:.4f}, "
              f"rows that differ {len(first)} (first differing positions {sorted(first)[:8]})")
        assert (same_pos if by_position else common) >= 0.99
    eq = ids == I0
    np.testing.assert_allclose(dist[eq], D0[eq], rtol=1e-4, atol=1e-4)
    (ndis, nhops), (ndis0, nhops0) = stats, stats0
    print(f"ndis {ndis} / {ndis0}, nhops {nhops} / {nhops0}")
    assert abs(ndis - ndis0) <= tol * ndis0 and abs(nhops - nhops0) <= tol * nhops0


# ---------------------------------------------------------------------------------------------------------------- (a)
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("n,d,ef,k", [(30000, 128, 5000, 10), (30000, 128, 5000, 5000), (12000, 768, 4000, 10)])
def test_wide_kernel_bit_identical_to_warp_kernel(kb, ref, metric, n, d, ef, k):
    """An all-zeros bitset is the plain search: the plain search runs hnsw_search_kernel, the filtered one (its pool
    needs twice the shared memory) runs hnsw_wide_kernel; ids, distances and the work counters must be equal."""
    xb, h, ix = _imported(kb, ref, n, d, 16, metric)
    xq = datagen.clustered(48, d, 43)
    ids0, dist0 = ix.search(xq, k, {"ef": ef})
    assert _engine(ix) == "scan"
    st0 = ix.hnsw_last_stats()
    zero = np.zeros((n + 7) // 8, np.uint8)
    ids1, dist1 = ix.search(xq, k, {"ef": ef}, bitset=zero)
    assert _engine(ix) == "hnsw_wide"
    st1 = ix.hnsw_last_stats()
    assert np.array_equal(ids0, ids1)
    assert np.array_equal(dist0.view(np.uint32), dist1.view(np.uint32))
    assert st0 == st1


# ---------------------------------------------------------------------------------------------------------------- (b)
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("ef,k", [(8192, 10), (8192, 2000), (16384, 8192)])
def test_wide_plain_parity(kb, ref, metric, ef, k):
    n, d = 50000, 64
    xb, h, ix = _imported(kb, ref, n, d, 16, metric)
    xq = datagen.clustered(32, d, 43)
    I0, D0, st0 = h.search(xq, k, ef)
    ids, dist = ix.search(xq, k, {"ef": ef})
    assert _engine(ix) == "hnsw_wide"
    _against_reference(ids, dist, I0, D0, ix.hnsw_last_stats(), st0, k, 0.02)
    gt, _ = ref.flat_search(xb, xq, k, metric)
    r0, r1 = recall_at_k(gt, I0), recall_at_k(gt, ids)
    print(f"recall@{k}: reference {r0:.4f}, gpu {r1:.4f}")
    assert r1 >= r0 - 0.005


# ---------------------------------------------------------------------------------------------------------------- (c)
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("frac", [0.1, 0.5, 0.9])
def test_wide_filtered_parity(kb, ref, metric, frac):
    """Two pools and the kAlpha budget; an invalid neighbour is admitted against the valid pool's back as it stands after
    the valid neighbours of the earlier link slots were inserted."""
    n, d, ef, k = 50000, 64, 8192, 1000
    xb, h, ix = _imported(kb, ref, n, d, 16, metric)
    xq = datagen.clustered(32, d, 43)
    mask = np.random.default_rng(7).random(n) < frac
    bits = np.packbits(mask, bitorder="little")
    I0, D0, st0 = h.search_filtered(xq, k, ef, bits, n)
    ids, dist = ix.search(xq, k, {"ef": ef, "disable_fallback_brute_force": True}, bitset=bits)
    assert _engine(ix) == "hnsw_wide"
    assert not mask[ids[ids >= 0]].any()
    _against_reference(ids, dist, I0, D0, ix.hnsw_last_stats(), st0, k, 0.001, by_position=False)
    gt, _ = ref.flat_search(xb[~mask], xq, k, metric)
    gt = np.nonzero(~mask)[0][gt]
    assert recall_at_k(gt, ids) >= recall_at_k(gt, I0) - 0.005


@functools.lru_cache(maxsize=2)
def _int_graph(metric, n=30000, d=32):
    from oracle import ref
    rng = np.random.default_rng(11)
    xb = rng.integers(0, 16, (n, d)).astype(np.float32)
    xq = rng.integers(0, 16, (24, d)).astype(np.float32)
    h = ref.RefHnsw(d, 16, metric, 100)
    h.add(xb)
    return xb, xq, h, h.export()


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("frac,ef,k", [(0.0, 8192, 2000), (0.2, 6000, 3000), (0.5, 8192, 1000), (0.9, 4000, 500)])
def test_wide_exact_arithmetic_bit_identical_to_reference(kb, ref, metric, frac, ef, k):
    """Small-integer vectors: every distance is exact in fp32 whatever the summation order, so the reference searcher and
    the wide kernel see the same keys, and the same traversal must give the same ids, distances, ndis and nhops, bit for
    bit.  This checks the filtered admission rule (a filtered neighbour at slot j against the valid pool's back after the
    valid neighbours of slots < j) and the invalid pool's merge, on data full of exact ties."""
    xb, xq, h, g = _int_graph(metric)
    n, d = xb.shape
    ix = kb.Index("HNSW", "L2" if metric == 0 else "IP", d, {"M": 16, "efConstruction": 100})
    ix.hnsw_import(xb, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    if frac == 0.0:
        I0, D0, st0 = h.search(xq, k, ef)
        ids, dist = ix.search(xq, k, {"ef": ef})
    else:
        mask = np.random.default_rng(13).random(n) < frac
        bits = np.packbits(mask, bitorder="little")
        I0, D0, st0 = h.search_filtered(xq, k, ef, bits, n)
        ids, dist = ix.search(xq, k, {"ef": ef, "disable_fallback_brute_force": True}, bitset=bits)
    assert _engine(ix) == "hnsw_wide"
    print(f"identical (row, position) ids {(ids == I0).mean():.4f}, ndis {ix.hnsw_last_stats()} / {st0}")
    assert np.array_equal(ids, I0)
    assert np.array_equal(dist.view(np.uint32), D0.view(np.uint32))
    assert ix.hnsw_last_stats() == st0


# ---------------------------------------------------------------------------------------------------------------- (d)
def test_wide_filtered_large_dim(kb, ref):
    n, d, ef, k = 6000, 4096, 3000, 100
    xb, h, ix = _imported(kb, ref, n, d, 16, 0)
    xq = datagen.clustered(16, d, 43)
    mask = np.random.default_rng(5).random(n) < 0.5
    bits = np.packbits(mask, bitorder="little")
    I0, D0, st0 = h.search_filtered(xq, k, ef, bits, n)
    ids, dist = ix.search(xq, k, {"ef": ef, "disable_fallback_brute_force": True}, bitset=bits)
    assert _engine(ix) == "hnsw_wide"
    assert not mask[ids[ids >= 0]].any()
    _against_reference(ids, dist, I0, D0, ix.hnsw_last_stats(), st0, k, 0.001, by_position=False)


# ---------------------------------------------------------------------------------------------------------------- (e)
def _exact(xb, xq, ids, metric):
    """float64 distances of the returned rows"""
    x = xb[ids].astype(np.float64)
    q = xq.astype(np.float64)[:, None, :]
    return ((x - q) ** 2).sum(-1) if metric == "L2" else (x * q).sum(-1)


@functools.lru_cache(maxsize=1)
def _own_index_40k():
    import knowhere_b200 as kb
    n, d = 40000, 32
    xb = datagen.clustered(n, d, 17)
    ix = kb.Index("HNSW", "L2", d, {"M": 16, "efConstruction": 100})
    ix.build(xb)
    return xb, ix


def test_wide_k_equals_ef_16384(kb):
    xb, ix = _own_index_40k()
    xq = datagen.clustered(8, xb.shape[1], 18)
    k = 16384
    ids, dist = ix.search(xq, k, {"ef": k})
    assert _engine(ix) == "hnsw_wide"
    assert (ids >= 0).all()
    for row in ids:
        assert len(np.unique(row)) == k
    assert (np.diff(dist, axis=1) >= 0).all()
    np.testing.assert_allclose(dist, _exact(xb, xq, ids, "L2"), rtol=1e-4, atol=1e-3)
    # two identical calls give identical results
    ids2, dist2 = ix.search(xq, k, {"ef": k})
    assert np.array_equal(ids, ids2) and np.array_equal(dist.view(np.uint32), dist2.view(np.uint32))


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_wide_custom_ids(kb, metric):
    n, d, k, ef = 12000, 32, 3000, 6000
    xb = datagen.clustered(n, d, 23)
    labels = (np.random.default_rng(1).permutation(n) * 7 + 1000).astype(np.int64)
    ix = kb.Index("HNSW", metric, d, {"M": 16, "efConstruction": 80})
    ix.build(xb, ids=labels)
    xq = datagen.clustered(6, d, 24)
    ids, dist = ix.search(xq, k, {"ef": ef, "disable_fallback_brute_force": True},
                          bitset=np.zeros((n + 7) // 8, np.uint8))
    assert _engine(ix) == "hnsw_wide"
    row_of = {int(l): i for i, l in enumerate(labels)}
    assert (ids >= 0).all()
    rows = np.vectorize(row_of.__getitem__)(ids)
    np.testing.assert_allclose(dist, _exact(xb, xq, rows, metric), rtol=1e-4, atol=1e-3)
    assert (np.diff(dist, axis=1) >= 0).all() if metric == "L2" else (np.diff(dist, axis=1) <= 0).all()


def _two_component_index(kb, n_a=2000, n_b=10000, d=16, deg=16):
    """one level, a ring graph per component: only the entry point's component (rows [0, n_a)) is reachable"""
    n = n_a + n_b
    xb = datagen.clustered(n, d, 31)
    nb = np.empty((n, deg), np.int32)
    for lo, cnt in ((0, n_a), (n_a, n_b)):
        r = np.arange(cnt)
        for j in range(deg):
            step = (j // 2 + 1) * (1 if j % 2 == 0 else -1)
            nb[lo:lo + cnt, j] = lo + (r + step) % cnt
    ix = kb.Index("HNSW", "L2", d, {"M": deg // 2, "efConstruction": 40})
    ix.hnsw_import(xb, np.ones(n, np.int32), (np.arange(n + 1) * deg).astype(np.int64), nb.reshape(-1),
                   np.array([0, deg], np.int32), 0, 0)
    return xb, ix


def test_wide_padding_and_short_row_fallback(kb, ref):
    xb, ix = _two_component_index(kb)
    n, n_a = xb.shape[0], 2000
    xq = datagen.clustered(4, xb.shape[1], 32)
    # plain: 2000 reachable rows, k = 4000
    ids, dist = ix.search(xq, 4000, {"ef": 8192})
    assert _engine(ix) == "hnsw_wide"
    assert (ids[:, :n_a] >= 0).all() and (ids[:, :n_a] < n_a).all() and (ids[:, n_a:] == -1).all()
    assert (dist[:, n_a:] == FLT_MAX).all()
    # filtered, fallback disabled: fewer than k valid rows are reachable; the row is padded
    mask = np.random.default_rng(9).random(n) < 0.5
    bits = np.packbits(mask, bitorder="little")
    k = 2000
    ids, dist = ix.search(xq, k, {"ef": 8192, "disable_fallback_brute_force": True}, bitset=bits)
    assert _engine(ix) == "hnsw_wide"
    for i in range(len(xq)):
        real = ids[i] >= 0
        cnt = int(real.sum())
        assert 0 < cnt < k and real[:cnt].all() and not real[cnt:].any()
        assert (ids[i, :cnt] < n_a).all() and not mask[ids[i, :cnt]].any()
        assert (dist[i, cnt:] == FLT_MAX).all()
    # with the fallback the short rows (k > 1008) are completed by the exact scan of the valid rows
    ids, dist = ix.search(xq, k, {"ef": 8192}, bitset=bits)
    assert ix.last_counters()["flagged"] == len(xq)
    assert (ids >= 0).all() and not mask[ids].any()
    gt, gd = ref.flat_search(xb[~mask], xq, k, 0)
    gt = np.nonzero(~mask)[0][gt]
    assert recall_at_k(gt, ids) >= 0.999
    np.testing.assert_allclose(dist, gd, rtol=1e-4, atol=1e-4)


def test_wide_filtered_on_a_shard(kb):
    """A graph-partition shard searched on its own (rank 1 of 2, no communicator) addresses the caller's bitset from its
    first global row, on the wide path as on the warp path."""
    n, d, k = 24000, 32, 500
    xb = datagen.clustered(n, d, 41)
    xq = datagen.clustered(8, d, 42)
    mask = np.random.default_rng(3).random(n) < 0.5
    bits = np.packbits(mask, bitorder="little")
    ix = kb.Index("HNSW", "L2", d, {"M": 16, "efConstruction": 80})
    ix.set_shard(1, 2)
    ix.build(xb)
    lo = n // 2
    for ef, engine in ((1000, "scan"), (6000, "hnsw_wide")):
        ids, dist = ix.search(xq, k, {"ef": ef, "disable_fallback_brute_force": True}, bitset=bits)
        assert _engine(ix) == engine
        assert (ids >= lo).all() and (ids < n).all()
        assert not mask[ids].any()
        np.testing.assert_allclose(dist, _exact(xb, xq, ids, "L2"), rtol=1e-4, atol=1e-3)


# ---------------------------------------------------------------------------------------------------------------- (f)
def test_wide_errors(kb):
    xb, ix = _own_index_40k()
    xq = datagen.clustered(2, xb.shape[1], 18)
    with pytest.raises(kb.KnowhereError) as e:
        ix.search(xq, 10, {"ef": 16385})
    assert e.value.status == 3 and "16384" in str(e.value)
    with pytest.raises(kb.KnowhereError) as e:
        ix.search(xq, 10, {"ef": 16385}, bitset=np.zeros((xb.shape[0] + 7) // 8, np.uint8))
    assert e.value.status == 3 and "16384" in str(e.value)
    with pytest.raises(kb.KnowhereError) as e:
        ix.search(xq, 100, {"ef": 50})                   # ef < k is still rejected
    assert e.value.status == 3
    # a dimension the one-query-per-CTA layout cannot hold at this ef: the message names the largest one
    n, d = 64, 28000
    big = datagen.uniform(n, d, 3)
    ix2 = kb.Index("HNSW", "L2", d, {"M": 4, "efConstruction": 16})
    ix2.build(big)
    with pytest.raises(kb.KnowhereError) as e:
        ix2.search(big[:1].copy(), 10, {"ef": 16384})
    assert e.value.status == 3 and "at most" in str(e.value)


# ---------------------------------------------------------------------------------------------------------------- (g)
def test_ann_iterator_hnsw_12000(tmp_path):
    """The C++ AnnIterator doubles k (and ef) up to 16384; on HNSW the refills past 4096 run hnsw_wide_kernel."""
    exe = tmp_path / "test_hnsw_iterator"
    subprocess.run(["g++", "-std=c++17", "-O2", f"-I{ROOT}/include", os.path.join(ROOT, "tests", "cpp", "test_hnsw_iterator.cc"),
                    "-o", str(exe), f"-L{ROOT}/knowhere_b200", "-l:libknowhere_b200.so",
                    f"-Wl,-rpath,{ROOT}/knowhere_b200"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "iterator ok" in r.stdout
