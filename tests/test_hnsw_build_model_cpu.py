"""tests/hnsw_build_model.py on what can be checked without a GPU: the level draw against a compiled std::mt19937 program,
the batch schedule, and selection / reverse links on hand-made collinear integer points, where the heuristic keeps the
nearest point on each side and every key is exact."""
import subprocess

import numpy as np
import pytest

from tests import hnsw_build_model as bm
from tests import hnsw_model as hm

LEVELS_CC = r"""
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
int main(int argc, char** argv) {
    const int n = atoi(argv[1]);
    std::mt19937 rng(12345);
    std::uniform_real_distribution<double> uni(0.0, 1.0);
    const double mult = 1.0 / std::log((double)atoi(argv[2]));
    for (int i = 0; i < n; i++) { double u = uni(rng); if (u <= 0) u = 1e-12; printf("%d\n", (int)(-std::log(u) * mult)); }
}
"""


@pytest.mark.parametrize("M", [4, 16, 32])
def test_levels_equal_std_mt19937(tmp_path, M):
    src, exe = tmp_path / "levels.cc", tmp_path / "levels"
    src.write_text(LEVELS_CC)
    subprocess.run(["g++", "-std=c++17", "-O2", str(src), "-o", str(exe)], check=True)
    n = 20000
    out = subprocess.run([str(exe), str(n), str(M)], capture_output=True, text=True, check=True).stdout
    want = np.array(out.split(), np.int32)
    got = bm.levels(n, M)
    np.testing.assert_array_equal(got, want)
    assert want.max() >= 2   # upper levels are drawn, not only level 0


def test_layout():
    g = bm.layout(5000, 8)
    lv = g["levels"] - 1
    assert (np.diff(lv[g["order"]]) <= 0).all() and g["entry_point"] == g["order"][0] and lv[g["entry_point"]] == g["max_level"]
    for a, b in zip(g["order"][:-1], g["order"][1:]):   # stable: ties keep the row order
        assert lv[a] > lv[b] or a < b
    assert list(g["cum"][:3]) == [0, 16, 24] and len(g["cum"]) == g["max_level"] + 2
    assert (np.diff(g["offsets"]) == g["cum"][g["levels"]]).all()


def test_schedule():
    n = 200000
    lv = bm.levels(n, 16)
    order = np.argsort(-lv, kind="stable")
    sched = bm.schedule(lv, order)
    assert max(nb for _, _, nb in sched) == bm.BUILD_BATCH
    for L in range(int(lv.max()), -1, -1):
        mine = [(s, nb) for l, s, nb in sched if l == L]
        cnt = int((lv >= L).sum())
        assert sum(nb for _, nb in mine) == cnt - 1
        pos = 1
        for s, nb in mine:
            assert s == pos and 1 <= nb <= bm.BUILD_BATCH and nb <= max(1, s // 4)
            if s < 8:
                assert nb == 1
            pos += nb
    assert [l for l, _, _ in sched] == sorted((l for l, _, _ in sched), reverse=True)


def _line(pos):
    """points on the x axis of R^2 (d = 2)"""
    return np.array([[p, 0] for p in pos], np.float32)


# eight points, M = 4: levels 0 1 2 0 0 0 0 0 (the first eight draws), so level 0 holds eight nodes in rows of 8
POS8 = [0, 3, 7, 12, 18, 25, 33, 42]


def test_short_lists_kept_whole_k8():
    """Every node sees at most 7 < 8 candidates: the keep-all rule links each to all others, and no row ever fills."""
    assert list(bm.levels(8, 4)) == [0, 1, 2, 0, 0, 0, 0, 0]
    g = bm.build(_line(POS8), 4, 16, "L2")
    off, cum, nb = g["offsets"], g["cum"], g["neighbors"]
    for v in range(8):
        row = nb[off[v] + cum[0]: off[v] + cum[1]]
        assert sorted(row[row >= 0].tolist()) == [u for u in range(8) if u != v]
        assert (row[7:] == -1).all()
    assert nb[off[1] + cum[1]: off[1] + cum[2]].tolist() == [2, -1, -1, -1]   # level 1: nodes 1 and 2
    assert nb[off[2] + cum[1]: off[2] + cum[2]].tolist() == [1, -1, -1, -1]


def test_ninth_point_is_pruned():
    """A ninth point sees 8 = max_size candidates, so the heuristic applies (the rule is count < max_size): on a line it
    keeps the nearest point on each side, in pool order; the two gain it as a reverse link in their free slot."""
    assert bm.levels(9, 4)[8] == 0
    g = bm.build(_line(POS8 + [20]), 4, 16, "L2")
    off, cum, nb = g["offsets"], g["cum"], g["neighbors"]
    assert g["order"][-1] == 8
    assert nb[off[8] + cum[0]: off[8] + cum[1]].tolist() == [4, 5] + [-1] * 6   # 18 (key 4), then 25 (key 25)
    for s in (4, 5):
        row = nb[off[s] + cum[0]: off[s] + cum[1]]
        assert row[7] == 8 and sorted(row[:7].tolist()) == [u for u in range(8) if u != s]
    for s in (0, 1, 2, 3, 6, 7):
        assert 8 not in nb[off[s] + cum[0]: off[s] + cum[1]]


def test_full_row_reshrinks():
    """s at 0 with a full row of 8 at 2..9: a new node at -6 gives 9 candidates; 2 (key 4) is kept, 3..9 lie behind it,
    -6 (key 36) is on the other side and kept."""
    X = _line([0, 2, 3, 4, 5, 6, 7, 8, 9, -6])
    K = bm.key_matrix(X, "L2")
    row = list(range(1, 9))
    assert bm.add_link(K, 0, row, 9, 8) == [1, 9]
    assert bm.add_link(K, 0, row[:7], 9, 8) == row[:7] + [9]   # room: appended, not pruned


def test_ties_by_key_then_id_in_link_and_by_pool_order_in_select():
    # link: a = (3, 4) and b = (5, 0) are both at key 25 from s = 0 and 20 from each other, so only the first of the two
    # in (key, id) order survives a re-shrink; with the new node as a or as b it is always the lower id
    X = np.array([[0, 0], [3, 4], [5, 0], [-1, 0], [-2, 0], [-3, 0], [-4, 0], [-6, 0], [-7, 0]], np.float32)
    K = bm.key_matrix(X, "L2")
    assert K[0, 1] == K[0, 2] == 25 and K[1, 2] == 20
    full = [3, 4, 5, 6, 7, 8]   # cap 7 with one of a, b: the other arrives
    assert bm.add_link(K, 0, full + [2], 1, 7) == [3, 1]
    assert bm.add_link(K, 0, full + [1], 2, 7) == [3, 1]
    # select: the pool is ascending by key with ties in pool order; the first of the tied pair is kept, whatever its id
    assert bm.select(K, 0, [3, 4, 2, 1], 3) == [3, 2]
    assert bm.select(K, 0, [3, 4, 1, 2], 3) == [3, 1]
    assert bm.select(K, 0, [0, 3, 2, 1], 3) == [3, 2]      # itself skipped: 3 = max_size candidates are pruned
    assert bm.select(K, 0, [0, 3, 2, 1], 4) == [3, 2, 1]   # 3 < 4: all kept


def test_descent_skips_unlinked_nodes():
    """the greedy descent scores nodes not yet linked on the beam level as +inf, so it stays on linked ones"""
    g = bm.layout(8, 4)
    g["neighbors"] = np.full(int(g["offsets"][-1]), -1, np.int32)
    off, cum = g["offsets"], g["cum"]
    g["neighbors"][off[2] + cum[1]] = 1   # level 1: 2 -> 1
    keys = [9.0, 0.0, 5.0, 9, 9, 9, 9, 9]
    assert hm.descend(g, lambda v: keys[v], 2, 5.0, 2, 0)[:2] == (1, 0.0)
    allowed = [k if r < 1 else np.inf for r, k in zip([2, 1, 0, 3, 4, 5, 6, 7], keys)]
    assert hm.descend(g, lambda v: allowed[v], 2, 5.0, 2, 0)[:2] == (2, 5.0)
