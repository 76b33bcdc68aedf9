"""numpy model of the device HNSW build (HnswIndex::add and build_graph_gpu, with hnsw_search_kernel in build mode,
hnsw_select_kernel and hnsw_link_kernel, kb2_hnsw.cuh), as DESIGN §4.8 defines it.  Plain code of the definition, not a
port of the kernels.

  * levels: std::mt19937(12345), std::uniform_real_distribution<double>(0, 1) (libstdc++ generate_canonical: two 32-bit
    words a, b per draw, u = (a + b 2^32) / 2^64), u <= 0 -> 1e-12, level = int(-log(u) * (1.0 / log(M)));
  * order: stable sort by level, descending; entry_point = order[0]; cum = 0, 2M, then M per upper level;
  * schedule: for L = max_level .. 0, the nodes order[1 : count(level >= L)] in batches of
    min(16384, max(1, inserted / 4), rest), inserted counting the entry point;
  * candidates of a batch node q on level L: greedy descent from max_level to L + 1 (first strict minimum, nodes not yet
    linked on L score +inf), then the pop-list beam of tests/hnsw_model.py on L with cap max(efConstruction, 2M);
  * selection: the pool in order without q; fewer than nlinks(L) are all kept, else the heuristic (keep c unless a kept
    s has key(c, s) < key(c, q)) up to nlinks(L); the row is the kept nodes in pool order, -1 padded;
  * reverse links, after the whole batch has selected: per target s, the arrivals in batch order; a row with room gets
    the new node appended, a full row is re-selected from members + new node sorted by (key to s, id) with the
    heuristic up to its capacity (K/impl/HNSW.cpp:311-354 add_link, with the kept nodes in ascending order).

Nodes of one batch see the graph as the previous batch left it.  Keys are computed in float64 and rounded to float32,
so on small-integer data they are exactly the device's keys whatever its summation order."""
import math

import numpy as np

from tests import hnsw_model as hm

BUILD_BATCH = 16384   # HnswIndex::kBuildBatch


def levels(n, M):
    """level of every row (0-based), std::mt19937(12345) as HnswIndex::add draws it"""
    bg = np.random.MT19937(0)
    bg._legacy_seeding(12345)
    raw = bg.random_raw(2 * n).astype(np.float64)
    u = (raw[0::2] + raw[1::2] * 2.0 ** 32) / 2.0 ** 64
    u = np.minimum(u, np.nextafter(1.0, 0.0))
    mult = 1.0 / math.log(M)
    return np.array([int(-math.log(x if x > 0 else 1e-12) * mult) for x in u], np.int32)


def layout(n, M):
    """levels (+1, as exported), order, cum, offsets, entry_point, max_level"""
    lv = levels(n, M)
    order = np.argsort(-lv, kind="stable").astype(np.int32)
    top = int(lv.max())
    cum = np.array([0, 2 * M] + [2 * M + M * i for i in range(1, top + 1)], np.int32)
    offsets = np.zeros(n + 1, np.int64)
    offsets[1:] = np.cumsum(cum[lv + 1])
    return dict(levels=lv + 1, order=order, cum=cum, offsets=offsets, entry_point=int(order[0]), max_level=top)


def schedule(lv, order):
    """[(level, start, size)] of every batch in launch order: order[start : start + size] is inserted on level"""
    n = len(lv)
    maxb = min(BUILD_BATCH, n)
    out = []
    for L in range(int(lv.max()), -1, -1):
        cnt = int((lv >= L).sum())
        inserted = 1
        while inserted < cnt:
            nb = min(maxb, max(1, inserted // 4), cnt - inserted)
            out.append((L, inserted, nb))
            inserted += nb
    return out


def key_matrix(X, metric):
    """fp32 keys between all rows: squared L2, or minus the inner product (exact float64 on small-integer data)"""
    X = X.astype(np.float64)
    G = X @ X.T
    if metric == "L2":
        sq = np.einsum("ij,ij->i", X, X)
        G = sq[:, None] + sq[None, :] - 2.0 * G
    else:
        G = -G
    return G.astype(np.float32)


def heuristic(K, centre, cands, cap):
    """shrink_neighbor_list (K/impl/HNSW.cpp:231-272): cands ascending by key to centre; keep c unless a kept s has
    key(c, s) < key(c, centre), stop at cap"""
    out = []
    for c in cands:
        kc = K[centre, c]
        if all(not (K[c, s] < kc) for s in out):
            out.append(c)
            if len(out) >= cap:
                break
    return out


def select(K, q, pool, cap):
    """hnsw_select_kernel: the neighbours of q from its beam pool (ascending by key to q)"""
    cands = [int(c) for c in pool if c != q]
    return cands if len(cands) < cap else heuristic(K, q, cands, cap)


def add_link(K, s, row, q, cap):
    """hnsw_link_kernel for one arrival: s's live links after q is added to them"""
    if len(row) < cap:
        return row + [int(q)]
    cands = sorted(row + [int(q)], key=lambda c: (K[s, c], c))
    return heuristic(K, s, cands, cap)


def build(X, M, ef_construction, metric):
    """the graph build_graph_gpu leaves, as hnsw_export returns it, plus 'order' and 'writer': {(node, level): (level,
    batch index)} of the batch that last wrote each row that was ever written"""
    n = len(X)
    g = layout(n, M)
    lv, order, cum, off = g["levels"] - 1, g["order"], g["cum"], g["offsets"]
    K = key_matrix(X, metric)
    nbr = np.full(int(off[-1]), -1, np.int32)
    g["neighbors"] = nbr
    writer = {}
    rank = np.empty(n, np.int64)
    rank[order] = np.arange(n)
    ef = max(ef_construction, 2 * M)
    inf = np.float32(np.inf)

    def set_row(v, L, ids, tag):
        cap = int(cum[L + 1] - cum[L])
        base = int(off[v] + cum[L])
        nbr[base:base + cap] = -1
        nbr[base:base + len(ids)] = ids
        writer[(int(v), L)] = tag

    for bi, (L, start, nb) in enumerate(schedule(lv, order)):
        cap = int(cum[L + 1] - cum[L])
        batch = order[start:start + nb]
        sel = []
        for q in batch:
            kq = K[q]
            allowed = np.where(rank < start, kq, inf)
            nearest, d_nearest, _, _ = hm.descend(g, lambda v: allowed[v], g["entry_point"], kq[g["entry_point"]],
                                                  g["max_level"], L)
            _, pool, _, _ = hm.beam(g, lambda v: kq[v], nearest, d_nearest, ef, L)
            sel.append(select(K, q, pool, cap))
        for q, s_list in zip(batch, sel):
            set_row(q, L, s_list, (L, bi))
        for q, s_list in zip(batch, sel):   # per target, the arrivals in batch order
            for s in s_list:
                set_row(s, L, add_link(K, s, hm.row_links(g, s, L), q, cap), (L, bi))
    g["writer"] = writer
    return g
