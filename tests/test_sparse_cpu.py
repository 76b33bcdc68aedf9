"""CPU checks of the sparse model (tests/sparse_model.py) against its definition and the reference's formulas."""
import numpy as np
import pytest

from knowhere_b200 import datagen
from tests import sparse_model as sm


def _nth_element_threshold(values, ratio):
    # get_query_drop_threshold (inverted_index.h:151-162) restated: size_t truncation of a float product, nth_element
    drop_count = int(np.float32(ratio) * np.float32(len(values)))
    if drop_count == 0:
        return 0.0
    return float(sorted(float(np.float32(v)) for v in values)[drop_count])


@pytest.mark.parametrize("ratio", [0.0, 0.01, 0.1, 0.3, 0.5, 0.9, 0.99])
@pytest.mark.parametrize("nnz", [1, 2, 3, 7, 40, 333])
def test_drop_threshold_matches_get_query_drop_threshold(ratio, nnz):
    rng = np.random.default_rng(nnz)
    vals = rng.integers(0, 5, nnz).astype(np.float32)   # ties included
    assert float(sm.drop_threshold(vals, ratio)) == _nth_element_threshold(vals, ratio)


def test_drop_count_zero_keeps_everything():
    # 0.3 * 3 = 0.9 truncates to 0: no threshold, every entry (zero values too) is kept
    post = sm.Postings((np.array([0, 3], np.int64), np.array([1, 2, 3], np.uint32), np.ones(3, np.float32)))
    kept = sm.kept_entries(post, np.array([1, 2, 3], np.uint32), np.array([0.0, 5.0, 1.0], np.float32), 0.3)
    assert [t for t, _ in kept] == [1, 2, 3]
    kept = sm.kept_entries(post, np.array([1, 2, 3], np.uint32), np.array([0.0, 5.0, 1.0], np.float32), 0.34)
    assert [t for t, _ in kept] == [2, 3]


def test_bm25_params_and_formula_match_scorer():
    # BM25IndexScorer (scorer.h:81-104): p1 = k1 + 1, p2 = k1 (1 - b), p3 = k1 b / avgdl; score = qval p1 tf / (tf + p2 + p3 len)
    k1, b, avgdl = 1.2, 0.75, 100.0
    p1, p2, p3 = sm.bm25_params(k1, b, avgdl)
    f = np.float32
    assert p1 == f(f(k1) + f(1)) and p2 == f(f(k1) * f(f(1) - f(b))) and p3 == f(f(f(k1) * f(b)) / f(avgdl))
    assert sm.bm25_params(k1, b, 0.25)[2] == f(f(k1) * f(b))   # avgdl below 1 counts as 1
    base = (np.array([0, 2, 3], np.int64), np.array([4, 9, 4], np.uint32), np.array([3.0, 1.0, 2.0], np.float32))
    post = sm.Postings(base)
    s = sm.scores(post, np.array([4], np.uint32), np.array([0.7], np.float32), "BM25", bm25=(k1, b, avgdl))
    for r, tf, L in ((0, 3.0, 4.0), (1, 2.0, 2.0)):
        want = f(f(f(f(0.7) * p1) * f(tf)) / f(f(f(tf) + p2) + f(p3 * f(L))))
        assert s[r] == want
        assert abs(float(s[r]) - 0.7 * (k1 + 1) * tf / (tf + k1 * (1 - b + b * L / avgdl))) < 1e-6


@pytest.mark.parametrize("metric", ["IP", "BM25"])
def test_model_agrees_with_float64_oracle(metric):
    if metric == "IP":
        base, queries = datagen.sparse_splade(3000, 30, 5, vocab=2000), datagen.sparse_splade(20, 10, 6, vocab=2000)
        bm25 = None
    else:
        base, avgdl = datagen.sparse_bm25_docs(3000, 7, vocab=5000, mean_len=30)
        queries, bm25 = datagen.sparse_bm25_queries(20, 3000, 8, vocab=5000), (1.2, 0.75, avgdl)
    post = sm.Postings(base)
    i32, d32 = sm.search(base, queries, 50, metric, bm25=bm25, post=post)
    i64, d64 = sm.search(base, queries, 50, metric, bm25=bm25, dtype=np.float64, post=post)
    np.testing.assert_allclose(d32, d64, rtol=1e-5, atol=1e-6)
    same = np.mean([len(set(a) & set(b)) / 50 for a, b in zip(i32, i64)])
    assert same >= 0.98


def test_row_sums_are_sequential_float32():
    vals = np.array([1e8, 1.0, 1.0, -0.0, 3.0], np.float32)
    post = sm.Postings((np.array([0, 3, 3, 5], np.int64), np.array([0, 1, 2, 0, 1], np.uint32), vals))
    f = np.float32
    assert post.row_sum[0] == f(f(f(1e8) + f(1)) + f(1)) and post.row_sum[1] == 0 and post.row_sum[2] == 3
