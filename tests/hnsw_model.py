"""numpy restatement of the reference's HNSW searcher without a filter (v2_hnsw_searcher::search,
K/impl/HnswSearcher.h:116-432, with NeighborSetPopList, K/impl/Neighbor.h:46-150), for graphs in the HNSW layout.

Keys are computed in float64 and rounded to float32 (squared L2, or minus the inner product), so on small-integer data
they equal the fp32 keys of every searcher.  Returns ids, distances (IP sign restored) and the summed (ndis, nhops)."""
import bisect

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def _key(X, v, q, metric):
    x = X[v].astype(np.float64)
    k = ((x - q) ** 2).sum() if metric == "L2" else -(x @ q)
    return float(np.float32(k))


def search_one(X, g, q, k, ef, metric):
    """g: dict with levels, offsets, neighbors, cum, entry_point, max_level (kb2_hnsw_export / RefHnsw.export)"""
    q = np.asarray(q, np.float64)
    nb, off, cum = g["neighbors"], g["offsets"], g["cum"]

    def links(v, level):
        out = []
        for j in range(off[v] + cum[level], off[v] + cum[level + 1]):
            if nb[j] < 0:
                break
            out.append(int(nb[j]))
        return out

    ndis = nhops = 0
    nearest = int(g["entry_point"])
    d_nearest = _key(X, nearest, q, metric)
    for level in range(int(g["max_level"]), 0, -1):   # greedy_update_nearest: first strict minimum, until no change
        while True:
            prev = nearest
            row = links(prev, level)
            for v in row:
                dv = _key(X, v, q, metric)
                if dv < d_nearest:
                    nearest, d_nearest = v, dv
            ndis += len(row)
            nhops += 1
            if nearest == prev:
                break
    cap = max(ef, k)
    dist, ids, checked = [d_nearest], [nearest], [False]
    visited = {nearest}
    cur = 0
    while cur < len(dist):
        node = ids[cur]
        checked[cur] = True
        cur += 1
        while cur < len(dist) and checked[cur]:
            cur += 1
        nhops += 1
        for v in links(node, 0):
            if v in visited:
                continue
            visited.add(v)
            ndis += 1
            dv = _key(X, v, q, metric)
            pos = bisect.bisect_right(dist, dv)   # upper_bound: after every equal key
            if pos >= cap:
                continue
            dist.insert(pos, dv)
            ids.insert(pos, v)
            checked.insert(pos, False)
            del dist[cap:], ids[cap:], checked[cap:]
            if pos < cur:
                cur = pos
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
