"""CPU tests of the IVF build model (tests/ivf_build_model.py): its generator is the standard's std::mt19937_64, and each of
its checkers rejects a result made wrong on purpose, so the bounds the GPU tests use are not vacuous."""
import shutil
import subprocess

import numpy as np
import pytest

from tests import ivf_build_model as ibm

CPP = r"""
#include <cstdio>
#include <random>
#include <utility>
#include <vector>
int main() {
    for (unsigned long long seed : {1234ull, 1241ull}) {
        std::mt19937_64 rng(seed);
        for (int i = 0; i < 700; i++) std::printf("%llu\n", (unsigned long long)rng());
    }
    std::mt19937_64 rng(1234);   // kmeans_train's partial Fisher-Yates shuffle
    std::vector<int> perm(1000);
    for (int i = 0; i < 1000; i++) perm[i] = i;
    for (long i = 0; i < 300; i++) std::swap(perm[i], perm[i + (long)(rng() % (unsigned long long)(1000 - i))]);
    for (int i = 0; i < 300; i++) std::printf("%d\n", perm[i]);
    return 0;
}
"""


def test_mt19937_64_standard_value():
    rng = ibm.MT19937_64()
    for _ in range(9999):
        rng()
    assert rng() == 9981545732273789042


def test_mt19937_64_matches_cpp(tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    src = tmp_path / "mt.cc"
    src.write_text(CPP)
    exe = tmp_path / "mt"
    subprocess.run(["g++", "-std=c++17", "-O1", str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = []
    for seed in (ibm.KMEANS_SEED, ibm.PQ_SAMPLE_SEED):
        rng = ibm.MT19937_64(seed)
        want += [rng() for _ in range(700)]
    want += ibm.partial_shuffle(1000, 300, ibm.MT19937_64(1234)).tolist()
    assert out == want


def test_kmeans_draws():
    # subsample then init from one stream; the init of a subsampled set indexes the sample
    d = ibm.KMeansDraws(5000, 4)
    assert d.sample is not None and d.nt == 1024 and len(np.unique(d.sample)) == 1024
    rng = ibm.MT19937_64(1234)
    assert (d.sample == ibm.partial_shuffle(5000, 1024, rng)).all()
    assert (d.init == ibm.partial_shuffle(1024, 4, rng)).all()
    # nothing is split when nt <= k
    d = ibm.KMeansDraws(16, 16)
    assert d.sample is None and d.split([16] + [0] * 15) == []
    # all rows in cluster 0: k - 1 splits, the counts halved in order, every pair's donor populated
    d = ibm.KMeansDraws(1000, 8)
    pairs = d.split([1000] + [0] * 7)
    assert [p[0] for p in pairs] == list(range(1, 8)) and pairs[0] == (1, 0)
    C = ibm.apply_splits(np.full((8, 3), 3.0, np.float32), pairs[:1])
    assert C[1].tolist() == [3 * (1 + 2 ** -10), 3 * (1 - 2 ** -10), 3 * (1 + 2 ** -10)]
    assert C[0].tolist() == [3 * (1 - 2 ** -10), 3 * (1 + 2 ** -10), 3 * (1 - 2 ** -10)]
    assert ibm.match_nlist(64, 1000) == 25 and ibm.match_nlist(64, 39 * 64) == 64 and ibm.match_nlist(8, 10) == 1


def _float_case(seed=0, n=400, d=8, k=16, offset=0.0):
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((n, d)) + offset).astype(np.float32)
    C = (rng.standard_normal((k, d)) + offset).astype(np.float32)
    return X, C


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("offset", [0.0, 300.0])
def test_fp32_keys_pass_and_a_moved_row_fails(metric, offset):
    X, C = _float_case(offset=offset)
    # an fp32 evaluation of the norm-expanded keys passes the rule
    x32, c32 = X.astype(np.float32), C.astype(np.float32)
    k32 = -(x32 @ c32.T) if metric == "IP" else ((x32 * x32).sum(1)[:, None] + (c32 * c32).sum(1)[None] - 2 * (x32 @ c32.T))
    ibm.check_assignment(X, C, np.argmin(k32, 1), metric, tf32=False)
    A = ibm.exact_assign(X, C, metric)
    ibm.check_assignment(X, C, A, metric, tf32=True)
    # a row moved to its second-nearest list, where the gap exceeds the bound, is rejected
    K, B = ibm.keys_and_bounds(X, C, metric, tf32=True)
    second = np.argsort(K, 1, kind="stable")[:, 1]
    r = np.arange(len(X))
    gap_ok = K[r, second] > K[r, A] + B[r, second] + B[r, A]
    assert gap_ok.any()
    i = int(np.nonzero(gap_ok)[0][0])
    bad = A.copy()
    bad[i] = second[i]
    with pytest.raises(AssertionError, match="wrong list"):
        ibm.check_assignment(X, C, bad, metric, tf32=True)


def test_integer_ties_go_to_the_lowest_list():
    X = np.array([[1, 2], [0, 0], [3, 3]], np.float32)
    C = np.array([[0, 0], [1, 2], [1, 2], [0, 0]], np.float32)
    assert ibm.exact_assign(X, C, "L2").tolist() == [1, 0, 1]
    ibm.check_assignment(X, C, [1, 0, 1], "L2", tf32=False, exact=True)
    with pytest.raises(AssertionError):
        ibm.check_assignment(X, C, [2, 0, 1], "L2", tf32=False, exact=True)


def test_moved_code_fails():
    rng = np.random.default_rng(1)
    M, dsub = 4, 3
    R = rng.standard_normal((300, M * dsub)).astype(np.float32)
    pqc = rng.standard_normal((M, 256, dsub)).astype(np.float32)
    codes = ibm.pq_encode(R, pqc)
    ibm.check_codes(R, pqc, codes)
    K, B = ibm.pq_keys_and_bounds(R, pqc)
    second = np.argsort(K, -1, kind="stable")[..., 1]
    gap = np.take_along_axis(K, second[..., None], -1)[..., 0] - np.take_along_axis(K, codes[..., None], -1)[..., 0]
    i, m = np.argwhere(gap > 1e-3)[0]
    bad = codes.copy()
    bad[i, m] = second[i, m]
    with pytest.raises(AssertionError, match="nearest codeword"):
        ibm.check_codes(R, pqc, bad)
    # integer residuals and a duplicated codeword: the lowest code wins
    Ri = np.array([[2, -1]], np.float32)
    pqi = np.zeros((1, 256, 2), np.float32)
    pqi[0, 7] = pqi[0, 9] = [2, -1]
    assert ibm.pq_encode(Ri, pqi).tolist() == [[7]]
    with pytest.raises(AssertionError):
        ibm.check_codes(Ri, pqi, [[9]], exact=True)


def test_shifted_centroid_fails():
    rng = np.random.default_rng(2)
    X = (rng.random((60, 5)) * 10 + 1).astype(np.float32)       # positive: the mean is the mean of |x|
    A = np.concatenate([[0, 0], rng.integers(1, 6, 58)])       # cluster 0 holds 2 points
    C, mean, cnt, mabs = ibm.lloyd_means(X, A, np.zeros((6, 5), np.float32))
    assert cnt[0] == 2
    ibm.check_means(C, mean, cnt, mabs)                        # the fp32 update is within the bound
    bad = C.copy()
    v = bad[0].astype(np.float64)
    j = int(np.argmax(np.spacing(bad[0]) / v))                 # the coordinate where 4 ulp is the largest share
    for _ in range(4):
        bad[0, j] = np.nextafter(bad[0, j], np.float32(np.inf))
    with pytest.raises(AssertionError, match="not the mean"):
        ibm.check_means(bad, mean, cnt, mabs)
    # integer data: the update is exact, and one ulp is caught
    Xi = np.array([[1, 2], [2, 2], [4, 7]], np.float32)
    Ci, _, cnti, mi = ibm.lloyd_means(Xi, np.array([0, 0, 0]), np.zeros((2, 2), np.float32))
    third = np.float32(1) / np.float32(3)
    assert Ci[0].tolist() == [np.float32(7) * third, np.float32(11) * third]
    assert Ci[1].tolist() == [0, 0] and cnti.tolist() == [3, 0]
    bad = Ci.copy()
    bad[0, 0] = np.nextafter(bad[0, 0], np.float32(0))
    ibm.check_means(Ci, Ci, cnti, mi, exact=True)
    with pytest.raises(AssertionError):
        ibm.check_means(bad, Ci, cnti, mi, exact=True)


def test_layout_faults_fail():
    A = np.array([2, 0, 2, 1, 0, 2, 2])
    labels = np.arange(100, 107)
    lists = [labels[r] for r in ibm.layout(A, 3)]
    assert [x.tolist() for x in lists] == [[101, 104], [103], [100, 102, 105, 106]]
    assert (ibm.check_layout(lists, labels) == A).all()
    swapped = [x.copy() for x in lists]
    swapped[2][[1, 2]] = swapped[2][[2, 1]]
    with pytest.raises(AssertionError, match="insertion order"):
        ibm.check_layout(swapped, labels)
    dropped = [x.copy() for x in lists]
    dropped[2] = dropped[2][:-1]
    with pytest.raises(AssertionError, match="in no list"):
        ibm.check_layout(dropped, labels)


def test_owner_table():
    assert ibm.owner_table([5, 9, 9, 1, 0], 2).tolist() == [0, 0, 1, 1, 1]
    assert ibm.owner_table([3, 3, 3], 1).tolist() == [0, 0, 0]
    assert ibm.owner_table([0, 0, 0, 0], 3).tolist() == [0, 0, 0, 0]   # empty lists add no load
