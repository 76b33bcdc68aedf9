"""GPU_CAGRA's definition (DESIGN §4.12) in the numpy model of tests/cagra_model.py, checked by hand and against the
literal definitions.  No GPU needed."""
import numpy as np

from tests import cagra_model as cm

# a hand-checked intermediate graph of 5 rows, m = 3
G0 = np.array([[1, 2, 3],
               [0, 2, 4],
               [1, 0, 3],
               [2, 4, 0],
               [3, 1, 2]])


def test_splitmix64_seeds():
    # the first outputs of splitmix64 from state 0
    assert [cm.splitmix64(j) for j in range(3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    assert cm.splitmix64(0) % 3000 == 0xE220A8397B1DCDAF % 3000


def test_detour_counts_by_hand():
    det = cm.detour_counts(G0)
    # row 2: G0[2][1] = 0 is G0[G0[2][0]][0] = G0[1][0]; row 4: G0[4][2] = 2 is in G0[3][0:2] and in G0[1][0:2]
    np.testing.assert_array_equal(det, [[0, 0, 0], [0, 0, 0], [0, 1, 0], [0, 0, 1], [0, 0, 2]])


def test_detour_counts_match_definition():
    rng = np.random.default_rng(3)
    n, m = 40, 9
    G = np.array([rng.choice(np.delete(np.arange(n), i), m, replace=False) for i in range(n)])
    det = cm.detour_counts(G)
    for i in range(n):
        for b in range(m):
            want = sum(1 for a in range(b) if G[i][b] in G[G[i][a]][:b])
            assert det[i, b] == want


def test_prune_reverse_merge_by_hand():
    det = cm.detour_counts(G0)
    P = cm.prune(G0, det, 2)
    np.testing.assert_array_equal(P, [[1, 2], [0, 2], [1, 3], [2, 4], [3, 1]])
    P3 = cm.prune(G0, det, 3)
    np.testing.assert_array_equal(P3, [[1, 2, 3], [0, 2, 4], [1, 3, 0], [2, 4, 0], [3, 1, 2]])
    R = cm.reverse_lists(P3, 5)
    assert R == [[1, 2, 3], [0, 2, 4], [3, 0, 1, 4], [4, 2, 0], [3, 1]]
    np.testing.assert_array_equal(cm.merge_rows(P3, R), [[1, 2, 3], [0, 2, 4], [1, 3, 0], [2, 4, 0], [3, 1, 2]])
    # a row whose reverse list replaces the tail of its pruned list: P[0][0:2], then R[0] until g = 4
    P4 = np.array([[1, 2, 3, 4], [0, 2, 3, 4], [0, 1, 3, 4], [0, 1, 2, 4], [0, 1, 2, 3]])
    R4 = [[3, 4, 1, 2], [], [], [], []]
    np.testing.assert_array_equal(cm.merge_rows(P4, R4)[0], [1, 2, 3, 4])
    R4 = [[4, 9, 1], [], [], [], []]
    np.testing.assert_array_equal(cm.merge_rows(P4, R4)[0], [1, 2, 4, 9])


def test_build_rows_are_distinct_and_exclude_self():
    rng = np.random.default_rng(0)
    X = rng.integers(-4, 5, (120, 8)).astype(np.float32)
    for metric in ("L2", "IP"):
        G = cm.build(X, 24, 12, metric)
        assert G.shape == (120, 12)
        for i, row in enumerate(G):
            assert len(set(row.tolist())) == 12 and i not in row and (row >= 0).all()
    # clamped degrees
    assert cm.build(X[:1], 64, 32, "L2").tolist() == [[-1]]
    np.testing.assert_array_equal(cm.build(X[:2], 64, 32, "L2"), [[1], [0]])


def test_search_model_finds_exact_neighbours_with_a_full_pool():
    rng = np.random.default_rng(1)
    X = rng.integers(-4, 5, (300, 8)).astype(np.float32)
    Q = rng.integers(-4, 5, (5, 8)).astype(np.float32)
    G = cm.build(X, 32, 16, "L2")
    ids, dist, (ndis, nhops) = cm.search(X, G, Q, 10, itopk=320, width=4)
    ids0, dist0 = cm.exact(X, Q, 10, "L2")
    np.testing.assert_array_equal(dist, dist0)
    assert ndis <= 5 * 300 and nhops > 0
    # max_iterations bounds the parents: seeds, then at most width parents per iteration
    _, _, (_, nh) = cm.search(X, G, Q[:1], 10, itopk=64, width=2, max_iter=3)
    assert nh <= 6
