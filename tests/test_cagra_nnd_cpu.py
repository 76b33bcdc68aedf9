"""GPU_CAGRA's NN-descent intermediate graph (DESIGN §4.12) in the numpy model of tests/cagra_nnd_model.py, checked
against its definition and the exact k-NN graph.  No GPU needed."""
import numpy as np

from tests import cagra_model as cm
from tests import cagra_nnd_model as nm


def _ints(n, d, seed):
    return np.random.default_rng(seed).integers(-8, 9, (n, d)).astype(np.float32)


def test_init_lists_are_distinct_and_self_free():
    for n, m in ((2, 1), (7, 6), (50, 49), (300, 40), (1000, 128)):
        ids = nm.init_ids(n, m)
        for i, row in enumerate(ids):
            assert len(set(row.tolist())) == m and i not in row and ((row >= 0) & (row < n)).all()


def test_hash_matches_scalar_definition():
    src, tgt, t = 12345, 678, 3
    want = cm.splitmix64(cm.splitmix64(t) ^ ((src << 32) | tgt)) >> 32
    assert int(nm.nnd_hash(src, tgt, t)) == want


def test_rows_are_distinct_best_first_and_self_free():
    X = _ints(400, 16, 1)
    for metric in ("L2", "IP"):
        ids, keys, iters, upd = nm.nn_descent(X, 24, 5, metric)
        assert ids.shape == (400, 24) and 1 <= iters <= 5 and len(upd) == iters
        for i in range(len(X)):
            assert len(set(ids[i].tolist())) == 24 and i not in ids[i]
            order = np.lexsort((ids[i], keys[i]))
            np.testing.assert_array_equal(order, np.arange(24))
            np.testing.assert_array_equal(keys[i], nm.pair_keys(X, [i], ids[i], metric)[0])


def test_full_lists_equal_exact_graph():
    """m = n - 1: every list holds every other row, so the result is the exact k-NN graph"""
    for n in (2, 3, 50):
        X = _ints(n, 8, n)
        for metric in ("L2", "IP"):
            ids = nm.nn_descent(X, n - 1, 20, metric)[0]
            np.testing.assert_array_equal(ids, cm.knn_graph(X, n - 1, metric))


def test_kth_key_never_worsens_and_counts_match_flags():
    X = _ints(600, 16, 2)
    for metric in ("L2", "IP"):
        _, _, iters, upd, hist = nm.nn_descent(X, 32, 8, metric, history=True)
        assert len(hist) == iters == len(upd)
        prev = None
        for t, (ids, keys, new) in enumerate(hist):
            assert upd[t] == int(new.sum())
            if prev is not None:
                assert (keys <= prev).all()
            prev = keys.copy()
        assert upd[-1] <= nm.DELTA * 600 * 32 or iters == 8


def test_converges_to_exact_graph_on_easy_case():
    rng = np.random.default_rng(4)
    X = rng.standard_normal((500, 8)).astype(np.float32)
    ids, _, iters, upd = nm.nn_descent(X, 16, 20, "L2")
    exact = cm.knn_graph(X, 16, "L2")
    recall = np.mean([len(set(a) & set(b)) / 16 for a, b in zip(ids.tolist(), exact.tolist())])
    assert recall >= 0.99, (recall, iters, upd)


def test_build_runs_steps_2_to_5_on_nnd_graph():
    X = _ints(200, 8, 5)
    G = nm.build(X, 24, 12, "L2")
    G0 = nm.nn_descent(X, 24, 20, "L2")[0]
    P = cm.prune(G0, cm.detour_counts(G0), 12)
    np.testing.assert_array_equal(G, cm.merge_rows(P, cm.reverse_lists(P, 200)))
    assert nm.build(X[:1], 64, 32, "L2").tolist() == [[-1]]
