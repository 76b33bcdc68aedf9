"""GPU_CAGRA with build_algo NN_DESCENT (DESIGN §4.12): the device NN-descent graph against the numpy model of
tests/cagra_nnd_model.py on small-integer data, where every key is exact in fp32; then determinism, quality, round trips
and errors on real-valued data."""
import functools

import numpy as np
import pytest

from knowhere_b200 import datagen
from tests import cagra_model as cm
from tests import cagra_nnd_model as nm
from tests.util import recall_at_k

pytestmark = pytest.mark.gpu
NND = {"build_algo": "NN_DESCENT"}


@functools.lru_cache(maxsize=None)
def _data(n, d, seed=5):
    rng = np.random.default_rng(seed)
    X = rng.integers(-8, 9, (n, d)).astype(np.float32)
    Q = rng.integers(-8, 9, (40, d)).astype(np.float32)
    return X, Q


@functools.lru_cache(maxsize=None)
def _model(n, d, m, metric):
    X, _ = _data(n, d)
    return nm.nn_descent(X, m, 20, metric, history=True)


def _hook(kb, X, metric, cfg):
    import torch
    ids, keys, iters, upd, ms = kb.debug_cagra_knn_graph(torch.from_numpy(X).cuda(), metric, cfg)
    return ids.cpu().numpy().astype(np.int64), keys.cpu().numpy(), iters, upd.tolist(), ms


def _graph(ix):
    g = ix.hnsw_export()
    return g["neighbors"].reshape(-1, int(g["cum"][1])).astype(np.int64)


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("n,d,m", [(3000, 32, 64), (5000, 30, 48)])
@pytest.mark.parametrize("niter", [1, 3, 20])
def test_hook_equals_model(kb, metric, n, d, m, niter):
    """n above the 4096-row chunk of the exact graph and d not a multiple of 4 included"""
    X, _ = _data(n, d)
    _, _, iters20, upd20, hist = _model(n, d, m, metric)
    t = min(niter, iters20)
    ids0, keys0, _ = hist[t - 1]
    ids, keys, iters, upd, ms = _hook(kb, X, metric, dict(NND, intermediate_graph_degree=m, graph_degree=m // 2,
                                                                      nn_descent_niter=niter))
    assert iters == t and upd == upd20[:t]
    np.testing.assert_array_equal(ids, ids0)
    np.testing.assert_array_equal(keys.view(np.uint32), keys0.view(np.uint32))
    assert ms > 0


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_build_and_search_equal_model(kb, metric):
    n, d, igd, gd = 3000, 32, 64, 32
    X, Q = _data(n, d)
    G0 = _model(n, d, igd, metric)[0]
    P = cm.prune(G0, cm.detour_counts(G0), gd)
    G_want = cm.merge_rows(P, cm.reverse_lists(P, n))
    ix = kb.Index("GPU_CAGRA", metric, d, dict(NND, intermediate_graph_degree=igd, graph_degree=gd))
    ix.build(X)
    G = _graph(ix)
    np.testing.assert_array_equal(G, G_want)
    filtered = np.random.default_rng(3).random(n) < 0.3
    for f in (None, filtered):
        cfg = {"itopk_size": 64, "search_width": 2}
        bits = None if f is None else np.packbits(f, bitorder="little")
        ids, dist = ix.search(Q, 10, cfg, bitset=bits)
        ids0, dist0, stats0 = cm.search(X, G, Q, 10, 64, 2, 0, 1, metric, f)
        np.testing.assert_array_equal(ids, ids0)
        np.testing.assert_array_equal(dist.view(np.uint32), dist0.view(np.uint32))
        assert ix.hnsw_last_stats() == stats0


@pytest.mark.parametrize("n", [1, 2, 50])
def test_small_n_equals_exact_build(kb, n):
    X, Q = _data(3000, 32)
    X = X[:n]
    graphs = []
    for cfg in ({}, NND):
        ix = kb.Index("GPU_CAGRA", "L2", 32, dict(cfg, intermediate_graph_degree=64, graph_degree=32))
        ix.build(X)
        graphs.append(_graph(ix))
    np.testing.assert_array_equal(graphs[1], graphs[0])
    np.testing.assert_array_equal(graphs[0], cm.build(X, 64, 32, "L2"))


@functools.lru_cache(maxsize=None)
def _real(n, d, metric):
    X = datagen.clustered(n, d, 11)
    Q = datagen.clustered(1000, d, 12)
    if metric == "IP":
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    return X, Q


def test_determinism_and_keys_on_real_data(kb):
    X, _ = _real(100000, 128, "L2")
    blobs = []
    for _ in range(2):
        ix = kb.Index("GPU_CAGRA", "L2", 128, NND)
        ix.build(X)
        blobs.append(ix.serialize())
    assert blobs[0] == blobs[1]
    ids, keys, iters, upd, _ = _hook(kb, X, "L2", NND)
    ids2, keys2, _, upd2, _ = _hook(kb, X, "L2", NND)
    np.testing.assert_array_equal(ids, ids2)
    np.testing.assert_array_equal(keys.view(np.uint32), keys2.view(np.uint32))
    assert upd == upd2 and 1 <= iters <= 20
    rows = np.arange(0, len(X), 97)
    for i in rows:
        r = ids[i]
        assert len(np.unique(r)) == len(r) and i not in r
        assert (np.lexsort((r, keys[i])) == np.arange(len(r))).all()
        x64 = X[r].astype(np.float64)
        want = ((x64 - X[i].astype(np.float64)) ** 2).sum(-1)
        # keys are |u|^2 + |v|^2 - 2<u, v> in fp32 with a 3xTF32 product: within fp32 rounding of the norms
        scale = (x64 ** 2).sum(-1) + float((X[i].astype(np.float64) ** 2).sum())
        assert (np.abs(keys[i] - want) <= 1e-5 * scale + 1e-6).all()


def _g0_recall(ids, exact):
    return float(np.mean([len(np.intersect1d(a, b)) for a, b in zip(ids, exact)]) / ids.shape[1])


@pytest.mark.parametrize("n,d,metric,slack", [(100000, 128, "L2", 0.02), (100000, 768, "IP", 0.05)])
def test_quality(kb, n, d, metric, slack):
    X, Q = _real(n, d, metric)
    flat = kb.Index("FLAT", metric, d)
    flat.build(X)
    gt, _ = flat.search(Q, 10)
    if metric == "L2":
        ids, _, iters, upd, _ = _hook(kb, X, metric, NND)
        exact, _, _, _, _ = _hook(kb, X, metric, {})
        r0 = _g0_recall(ids, exact)
        print(f"NN-descent G0 recall {n}x{d} {metric}: {r0:.4f} after {iters} iterations, updates {upd}")
        assert r0 >= 0.90
    rec = []
    for cfg in ({}, NND):
        ix = kb.Index("GPU_CAGRA", metric, d, cfg)
        ix.build(X)
        rec.append(recall_at_k(gt, ix.search(Q, 10, {"itopk_size": 128})[0]))
    print(f"GPU_CAGRA {n}x{d} {metric} recall@10 at itopk 128: exact graph {rec[0]:.4f}, NN-descent {rec[1]:.4f}")
    assert rec[1] >= rec[0] - slack


def test_round_trips(kb):
    X, Q = _data(3000, 32)
    ix = kb.Index("GPU_CAGRA", "IP", 32, dict(NND, intermediate_graph_degree=64, graph_degree=32))
    ix.build(X)
    cfg = {"itopk_size": 64, "search_width": 2}
    ids, dist = ix.search(Q, 10, cfg)
    for back in (kb.Index.deserialize(ix.serialize()), kb.Index.deserialize_faiss(ix.serialize_faiss())):
        np.testing.assert_array_equal(back.hnsw_export()["neighbors"], ix.hnsw_export()["neighbors"])
    back = kb.Index.deserialize(ix.serialize())
    a, b = back.search(Q, 10, cfg)
    np.testing.assert_array_equal(a, ids)
    np.testing.assert_array_equal(b.view(np.uint32), dist.view(np.uint32))


def test_errors(kb):
    from knowhere_b200 import KnowhereError
    for niter in (0, 1001):
        with pytest.raises(KnowhereError) as e:
            kb.Index("GPU_CAGRA", "L2", 32, dict(NND, nn_descent_niter=niter))
        assert e.value.status == 3
    # lower case selects NN-descent too; other values, or niter out of range without NN_DESCENT, build the exact graph
    with pytest.raises(KnowhereError):
        kb.Index("GPU_CAGRA", "L2", 32, {"build_algo": "nn_descent", "nn_descent_niter": 0})
    X, _ = _data(3000, 32)
    exact = kb.Index("GPU_CAGRA", "L2", 32, {"intermediate_graph_degree": 32, "graph_degree": 16})
    exact.build(X)
    for cfg in ({"build_algo": "IVF_PQ"}, {"build_algo": "AUTO", "nn_descent_niter": 0}):
        ix = kb.Index("GPU_CAGRA", "L2", 32, dict(cfg, intermediate_graph_degree=32, graph_degree=16))
        ix.build(X)
        np.testing.assert_array_equal(_graph(ix), _graph(exact))
