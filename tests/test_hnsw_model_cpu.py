"""tests/hnsw_model.py against the reference's own searcher (kref_hnsw_search) on the reference's own graph, on
small-integer data where every key is exact in fp32: ids, distance bits, ndis and nhops.  No GPU needed."""
import numpy as np
import pytest

from tests import hnsw_model as hm


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_model_equals_reference_searcher(ref, metric):
    rng = np.random.default_rng(5)
    X = rng.integers(-8, 9, (2000, 32)).astype(np.float32)
    Q = rng.integers(-8, 9, (30, 32)).astype(np.float32)
    h = ref.RefHnsw(32, 16, 0 if metric == "L2" else 1, 100)
    h.add(X)
    g = h.export()
    assert g["max_level"] >= 1   # the greedy descent is exercised too
    for ef in (16, 64):
        I0, D0, st0 = h.search(Q, 10, ef, nthreads=1)
        I, D, st = hm.search(X, g, Q, 10, ef, metric)
        np.testing.assert_array_equal(I, I0)
        np.testing.assert_array_equal(D.view(np.uint32), D0.view(np.uint32))
        assert st == st0
