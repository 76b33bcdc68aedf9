"""numpy restatement of the reference's HNSW searcher without a filter (v2_hnsw_searcher::search,
K/impl/HnswSearcher.h:116-432, with NeighborSetPopList, K/impl/Neighbor.h:46-150), for graphs in the HNSW layout.

Keys are computed in float64 and rounded to float32 (squared L2, or minus the inner product), so on small-integer data
they equal the fp32 keys of every searcher.  Returns ids, distances (IP sign restored) and the summed (ndis, nhops).

descend and beam are the two halves of a search; tests/hnsw_build_model.py runs them in build mode (a beam on an upper
level, a descent restricted to the nodes already linked)."""
import bisect

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def _key(X, v, q, metric):
    x = X[v].astype(np.float64)
    k = ((x - q) ** 2).sum() if metric == "L2" else -(x @ q)
    return float(np.float32(k))


def row_links(g, v, level):
    """the live links of v on level, up to the first -1"""
    nb, off, cum = g["neighbors"], g["offsets"], g["cum"]
    out = []
    for j in range(off[v] + cum[level], off[v] + cum[level + 1]):
        if nb[j] < 0:
            break
        out.append(int(nb[j]))
    return out


def descend(g, key, nearest, d_nearest, top, bottom):
    """greedy_update_nearest on levels top .. bottom + 1: first strict minimum over the link slots, until no change.
    key(v) is the key of node v to the query.  Returns (nearest, d_nearest, ndis, nhops)."""
    ndis = nhops = 0
    for level in range(top, bottom, -1):
        while True:
            prev = nearest
            row = row_links(g, prev, level)
            for v in row:
                dv = key(v)
                if dv < d_nearest:
                    nearest, d_nearest = v, dv
            ndis += len(row)
            nhops += 1
            if nearest == prev:
                break
    return nearest, d_nearest, ndis, nhops


def beam(g, key, entry, d_entry, cap, level=0):
    """the pop-list beam of capacity cap on level from one entry node.  Returns the sorted pool (dist, ids) and
    (ndis, nhops)."""
    ndis = nhops = 0
    dist, ids, checked = [d_entry], [entry], [False]
    visited = {entry}
    cur = 0
    while cur < len(dist):
        node = ids[cur]
        checked[cur] = True
        cur += 1
        while cur < len(dist) and checked[cur]:
            cur += 1
        nhops += 1
        for v in row_links(g, node, level):
            if v in visited:
                continue
            visited.add(v)
            ndis += 1
            dv = key(v)
            pos = bisect.bisect_right(dist, dv)   # upper_bound: after every equal key
            if pos >= cap:
                continue
            dist.insert(pos, dv)
            ids.insert(pos, v)
            checked.insert(pos, False)
            del dist[cap:], ids[cap:], checked[cap:]
            if pos < cur:
                cur = pos
    return dist, ids, ndis, nhops


def search_one(X, g, q, k, ef, metric):
    """g: dict with levels, offsets, neighbors, cum, entry_point, max_level (kb2_hnsw_export / RefHnsw.export)"""
    q = np.asarray(q, np.float64)
    key = lambda v: _key(X, v, q, metric)   # noqa: E731
    ep = int(g["entry_point"])
    nearest, d_nearest, ndis, nhops = descend(g, key, ep, key(ep), int(g["max_level"]), 0)
    dist, ids, a, b = beam(g, key, nearest, d_nearest, max(ef, k))
    ndis += a
    nhops += b
    n = min(k, len(dist))
    out_i = np.full(k, -1, np.int64)
    out_d = np.full(k, FLT_MAX if metric == "L2" else -FLT_MAX, np.float32)
    out_i[:n] = ids[:n]
    out_d[:n] = dist[:n] if metric == "L2" else [-d for d in dist[:n]]
    return out_i, out_d, ndis, nhops


def search(X, g, Q, k, ef, metric):
    I = np.empty((len(Q), k), np.int64)
    D = np.empty((len(Q), k), np.float32)
    ndis = nhops = 0
    for r, q in enumerate(Q):
        I[r], D[r], a, b = search_one(X, g, q, k, ef, metric)
        ndis += a
        nhops += b
    return I, D, (ndis, nhops)
