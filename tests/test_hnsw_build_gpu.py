"""The device HNSW build (build_graph_gpu: hnsw_search_kernel in build mode, hnsw_select_kernel, the pair sort,
hnsw_link_kernel) against tests/hnsw_build_model.py.  On small-integer data every key is exact in fp32, so the graph must
equal the model's bit for bit, exact ties included.  On float data builds must be reproducible and structurally sound."""
import numpy as np
import pytest

from knowhere_b200 import datagen
from tests import hnsw_build_model as bm

pytestmark = pytest.mark.gpu

# n, d, M, efConstruction: each reaches a different path of the three kernels
SHAPES = [
    (3000, 32, 8, 32),     # baseline; the last batches (~600 nodes) contend on hub rows
    (3000, 30, 8, 48),     # d % 4 != 0: scalar hnsw_key in search, select and link
    (2500, 36, 4, 16),     # many levels, rows of 8 / 4, lanes partly idle in hnsw_key4
    (4000, 128, 16, 64),   # hnsw_key4 / hnsw_key2
    (3000, 64, 32, 40),    # 2M = 64 > efConstruction sets the beam; 65-candidate re-shrinks
    (1500, 260, 8, 24),    # several float4 per lane
]


def _int_rows(n, d, seed):
    """clustered rows scaled to small integers: |x| <= 8, so every key is an exact fp32 integer and exact ties occur"""
    return np.ascontiguousarray(np.clip(np.round(datagen.clustered(n, d, seed) * 0.25), -8, 8), np.float32)


def _gpu_build(kb, X, metric, M, efc):
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("KB2_HNSW_BUILD", "gpu")
        ix = kb.Index("HNSW", metric, X.shape[1], {"M": M, "efConstruction": efc})
        ix.build(X)
    return ix


@pytest.fixture(scope="module")
def model_graphs():
    cache = {}

    def get(X, key, M, efc, metric):
        if key not in cache:
            cache[key] = bm.build(X, M, efc, metric)
        return cache[key]
    return get


def _first_mismatch(gm, gg):
    """the differing row the earliest batch wrote: (level, batch, node, model row, device row)"""
    off, cum, lv = gm["offsets"], gm["cum"], gm["levels"] - 1
    bad = []
    for v in range(len(lv)):
        for L in range(lv[v] + 1):
            a, b = off[v] + cum[L], off[v] + cum[L + 1]
            if not np.array_equal(gm["neighbors"][a:b], gg["neighbors"][a:b]):
                bad.append((gm["writer"].get((v, L), (L, -1))[1], L, v, gm["neighbors"][a:b], gg["neighbors"][a:b]))
    bad.sort(key=lambda t: t[0])
    return len(bad), bad[0]


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("n,d,M,efc", SHAPES)
def test_gpu_build_equals_model(kb, model_graphs, n, d, M, efc, metric):
    X = _int_rows(n, d, n + d)
    gm = model_graphs(X, (n, d, M, efc, metric), M, efc, metric)
    gg = _gpu_build(kb, X, metric, M, efc).hnsw_export()
    for f in ("levels", "offsets", "cum"):
        np.testing.assert_array_equal(gg[f], gm[f], err_msg=f)
    assert (gg["entry_point"], gg["max_level"]) == (gm["entry_point"], gm["max_level"])
    if not np.array_equal(gg["neighbors"], gm["neighbors"]):
        nbad, (bi, L, v, rm, rg) = _first_mismatch(gm, gg)
        pytest.fail(f"{nbad} rows differ; first written by batch {bi} on level {L}: node {v}\n"
                    f"  model  {rm.tolist()}\n  device {rg.tolist()}")


def _check_structure(g):
    """every row of every level: compact, ids in range, no self-links or duplicates, neighbours on that level; every node
    but the entry point has a link on each of its levels"""
    lv, off, cum, nb = g["levels"] - 1, g["offsets"], g["cum"], g["neighbors"]
    n = len(lv)
    for L in range(g["max_level"] + 1):
        nodes = np.nonzero(lv >= L)[0]
        cap = cum[L + 1] - cum[L]
        rows = nb[(off[nodes] + cum[L])[:, None] + np.arange(cap)[None, :]]
        live = rows >= 0
        assert (live[:, 1:] <= live[:, :-1]).all(), f"level {L}: a row is not compact"
        assert (rows >= -1).all() and (rows < n).all(), f"level {L}: id out of range"
        assert not (rows == nodes[:, None]).any(), f"level {L}: self-link"
        srt = np.sort(np.where(live, rows, -1 - np.arange(cap)[None, :]), axis=1)
        assert not (srt[:, 1:] == srt[:, :-1]).any(), f"level {L}: duplicate link"
        assert (lv[rows[live]] >= L).all(), f"level {L}: link to a node below the level"
        empty = nodes[~live[:, 0]]
        assert set(empty.tolist()) <= {g["entry_point"]}, f"level {L}: nodes without links {empty[:10].tolist()}"


@pytest.mark.parametrize("n,d,metric", [(100000, 128, "L2"), (100000, 128, "IP"), (30000, 768, "COSINE")])
def test_gpu_build_is_deterministic(kb, n, d, metric):
    M, efc = 16, 100
    X = datagen.clustered(n, d, 21)
    g1 = _gpu_build(kb, X, metric, M, efc)
    launches = g1.last_counters()["launches"]
    g1 = g1.hnsw_export()
    g2 = _gpu_build(kb, X, metric, M, efc).hnsw_export()
    for f in ("levels", "offsets", "cum", "neighbors"):
        np.testing.assert_array_equal(g1[f], g2[f], err_msg=f)
    assert (g1["entry_point"], g1["max_level"]) == (g2["entry_point"], g2["max_level"])
    lay = bm.layout(n, M)
    np.testing.assert_array_equal(g1["levels"], lay["levels"])
    sched = bm.schedule(lay["levels"] - 1, lay["order"])
    assert launches == 4 * len(sched)   # search, select, pair sort, link per batch
    if n > 4 * bm.BUILD_BATCH:
        assert any(nb == bm.BUILD_BATCH for _, _, nb in sched)
    _check_structure(g1)


def test_short_candidate_lists_kept_whole(kb, monkeypatch):
    """Eight collinear points, M = 4, efConstruction 16: no node ever has 8 = max_size candidates on level 0, so every
    list is kept whole (K/impl/HNSW.cpp:290-292) and level 0 is the complete graph K8.  Pruning instead would keep only
    the nearest point on each side.  Device batches all have size 1 here."""
    pos = [0, 3, 7, 12, 18, 25, 33, 42]
    X = np.array([[p, 0, 0, 0] for p in pos], np.float32)
    monkeypatch.setenv("KB2_HNSW_BUILD", "gpu")
    ix = kb.Index("HNSW", "L2", 4, {"M": 4, "efConstruction": 16})
    ix.build(X)
    g = ix.hnsw_export()
    off, cum, nb = g["offsets"], g["cum"], g["neighbors"]
    assert cum[1] == 8
    for v in range(8):
        row = nb[off[v] + cum[0]: off[v] + cum[1]]
        assert sorted(row[row >= 0].tolist()) == [u for u in range(8) if u != v], f"node {v}: {row.tolist()}"
    np.testing.assert_array_equal(nb, bm.build(X, 4, 16, "L2")["neighbors"])
