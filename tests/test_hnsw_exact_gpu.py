"""HNSW warp kernels (hnsw_search_kernel, four queries per CTA) against the reference searcher, bit for bit.  The vectors
are small integers, so every distance is exact in fp32 whatever the summation order: on the reference's own graph
(RefHnsw.export -> hnsw_import) the same traversal must give the same ids, distance bits and ndis / nhops.  This pins
the plain one-pool traversal, the filtered two-pool traversal with its kAlpha budget, and range search."""
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
N, NQ = 20000, 200


@functools.lru_cache(maxsize=4)
def _int_graph(metric, d):
    from oracle import ref
    rng = np.random.default_rng(23 + d)
    xb = rng.integers(0, 16, (N, d)).astype(np.float32)
    xq = rng.integers(0, 16, (NQ, d)).astype(np.float32)
    h = ref.RefHnsw(d, 16, metric, 100)
    h.add(xb)
    return xb, xq, h, h.export()


def _imported(kb, metric, d):
    xb, xq, h, g = _int_graph(metric, d)
    ix = kb.Index("HNSW", "L2" if metric == 0 else "IP", d, {"M": 16, "efConstruction": 100})
    ix.hnsw_import(xb, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    return xb, xq, h, ix


def _bits(frac, seed=13):
    mask = np.random.default_rng(seed).random(N) < frac
    return mask, np.packbits(mask, bitorder="little")


def _identical(ix, ids, dist, I0, D0, st0):
    assert ix.last_stage_info()["engine"] == "scan"
    print(f"identical (row, position) ids {(ids == I0).mean():.4f}, ndis/nhops {ix.hnsw_last_stats()} / {st0}")
    assert np.array_equal(ids, I0)
    assert np.array_equal(dist.view(np.uint32), D0.view(np.uint32))
    assert ix.hnsw_last_stats() == st0


# d = 30: rows are not float4-aligned, so the keys take the scalar path instead of the four-row batch
@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("d,ef,k", [(32, 16, 10), (32, 128, 50), (32, 1000, 100), (30, 128, 50)])
def test_plain_search_bit_identical_to_reference(kb, ref, metric, d, ef, k):
    xb, xq, h, ix = _imported(kb, metric, d)
    I0, D0, st0 = h.search(xq, k, ef)
    ids, dist = ix.search(xq, k, {"ef": ef})
    _identical(ix, ids, dist, I0, D0, st0)


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("frac", [0.2, 0.5, 0.9])
@pytest.mark.parametrize("d,ef,k", [(32, 64, 10), (32, 500, 100), (30, 64, 10)])
def test_filtered_search_bit_identical_to_reference(kb, ref, metric, frac, d, ef, k):
    xb, xq, h, ix = _imported(kb, metric, d)
    mask, bits = _bits(frac)
    I0, D0, st0 = h.search_filtered(xq, k, ef, bits, N)
    ids, dist = ix.search(xq, k, {"ef": ef, "disable_fallback_brute_force": True}, bitset=bits)
    assert not mask[ids[ids >= 0]].any()
    _identical(ix, ids, dist, I0, D0, st0)


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("frac", [None, 0.3])
@pytest.mark.parametrize("d", [32, 30])
def test_range_search_same_hits_as_reference(kb, ref, metric, frac, d):
    """Each query's set of (id, distance bits) is the reference's.  Distances are integers, so a radius halfway between
    two of them leaves no hit on the boundary."""
    ef = 32
    xb, xq, h, ix = _imported(kb, metric, d)
    mask, bits = _bits(frac) if frac is not None else (np.zeros(N, bool), None)
    gt, gd = ref.flat_search(xb, xq, 40, metric)
    radius = float(np.median(gd[:, 25])) + (0.5 if metric == 0 else -0.5)
    lims0, ids0, dis0 = h.range_search(xq, radius, ef, bits, N if bits is not None else 0)
    lims, ids, dis = ix.range_search(xq, radius, config={"ef": ef}, bitset=bits)
    assert lims[-1] > 0
    for i in range(len(xq)):
        a = set(zip(ids0[lims0[i]:lims0[i + 1]].tolist(), dis0[lims0[i]:lims0[i + 1]].view(np.uint32).tolist()))
        b = set(zip(ids[lims[i]:lims[i + 1]].tolist(), dis[lims[i]:lims[i + 1]].view(np.uint32).tolist()))
        assert a == b, f"query {i}: {len(a - b)} hits only in the reference, {len(b - a)} only here"
    assert not mask[ids].any()
