"""Row -> id labels of the dense indexes.  With custom ids, search and range search return, per query, the ids of the rows
that the same search without ids returns, and a KB2I round trip keeps the bytes and the results.  GPU_CAGRA takes no
custom ids; that refusal and the refusals around range search and emb-lists are pinned by status and message."""
import numpy as np
import pytest

import knowhere_b200 as kb

pytestmark = pytest.mark.gpu
N, D, NQ, K = 2000, 32, 24, 10
INVALID_ARGS, NOT_IMPLEMENTED = 1, 7

# IVF_PQ m=16 (dim 32): one 16-sub-quantizer group, the G > 0 scan kernels; m=8: the generic kernel
CASES = {
    "FLAT": ("FLAT", {}, {}),
    "IVF_FLAT": ("IVF_FLAT", {"nlist": 16}, {"nprobe": 4}),
    "IVF_PQ_m16": ("IVF_PQ", {"nlist": 16, "m": 16}, {"nprobe": 4}),
    "IVF_PQ_m8": ("IVF_PQ", {"nlist": 16, "m": 8}, {"nprobe": 4}),
    "HNSW": ("HNSW", {"M": 16, "efConstruction": 64}, {"ef": 64}),
}


def _data():
    rng = np.random.default_rng(11)
    X = rng.standard_normal((N, D)).astype(np.float32)
    Q = rng.standard_normal((NQ, D)).astype(np.float32)
    ids = (rng.permutation(N) * 7 + 1_000_003).astype(np.int64)   # not the rows, not a permutation of them
    return X, Q, ids


def _pair(name, X, ids):
    """(index with custom ids, the same index with the rows as ids)"""
    t, build, _ = CASES[name]
    a = kb.Index(t, "L2", D, build)
    a.build(X, ids)
    b = kb.Index(t, "L2", D, build)
    if t == "HNSW":
        # the host build is multi-threaded: the identity index imports the graph of the first one
        g = a.hnsw_export()
        b.hnsw_import(X, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    else:
        b.build(X)
    return a, b


def _range(ix, Q, radius, cfg):
    lims, rid, rdist = ix.range_search(Q, radius, None, cfg)
    return [(rid[lims[i]:lims[i + 1]], rdist[lims[i]:lims[i + 1]]) for i in range(len(Q))]


def _results(ix, Q, radius, cfg):
    return ix.search(Q, K, cfg), _range(ix, Q, radius, cfg)


def _assert_mapped(got, want, ids):
    """got: results of the custom-id index; want: those of the identity index, mapped through ids"""
    (gi, gd), grange = got
    (wi, wd), wrange = want
    np.testing.assert_array_equal(gi, np.where(wi >= 0, ids[np.maximum(wi, 0)], -1))
    np.testing.assert_array_equal(gd, wd)
    for (a_ids, a_dist), (b_ids, b_dist) in zip(grange, wrange):
        np.testing.assert_array_equal(a_ids, ids[b_ids])
        np.testing.assert_array_equal(a_dist, b_dist)


@pytest.mark.parametrize("name", list(CASES))
def test_custom_ids_map_rows(name):
    X, Q, ids = _data()
    a, b = _pair(name, X, ids)
    cfg = CASES[name][2]
    want = _results(b, Q, 0.0, cfg)
    # a radius that keeps about the K nearest rows of each query
    radius = float(np.median(want[0][1][:, K // 2]))
    want = _results(b, Q, radius, cfg)
    assert sum(len(r[0]) for r in want[1]) > 0
    got = _results(a, Q, radius, cfg)
    _assert_mapped(got, want, ids)

    blob = a.serialize()
    c = kb.Index.deserialize(blob)
    assert c.serialize() == blob
    (ci, cd), crange = _results(c, Q, radius, cfg)
    np.testing.assert_array_equal(ci, got[0][0])
    np.testing.assert_array_equal(cd, got[0][1])
    for (c_ids, c_dist), (g_ids, g_dist) in zip(crange, got[1]):
        np.testing.assert_array_equal(c_ids, g_ids)
        np.testing.assert_array_equal(c_dist, g_dist)


def _refusal(fn):
    with pytest.raises(kb.KnowhereError) as e:
        fn()
    return e.value.status, str(e.value).split(": ", 1)[1]


def test_refusals():
    X, Q, ids = _data()
    cagra = kb.Index("GPU_CAGRA", "L2", D, {"intermediate_graph_degree": 32, "graph_degree": 16})
    assert _refusal(lambda: cagra.add(X, ids)) == (NOT_IMPLEMENTED, "GPU_CAGRA: custom ids are not implemented")
    # RangeSearch is refused before the empty-index and nq == 0 checks
    for q in (Q, Q[:0]):
        assert _refusal(lambda: cagra.range_search(q, 1.0)) == (NOT_IMPLEMENTED, "RangeSearch is not implemented on GPU_CAGRA")

    hnsw = kb.Index("HNSW", "L2", D, CASES["HNSW"][1])
    hnsw.build(X, ids)
    assert _refusal(lambda: hnsw.set_emb_list(np.array([0, N // 2, N]), "MAX_SIM_L2")) == (
        NOT_IMPLEMENTED, "emb-lists with custom ids")

    for t in ("SPARSE_INVERTED_INDEX", "SPARSE_WAND"):
        sx = kb.Index(t, "IP", 0)
        assert _refusal(lambda: sx.range_search(Q, 0.5)) == (
            INVALID_ARGS, t + " holds sparse rows: search it with kb2_index_range_search_sparse")
