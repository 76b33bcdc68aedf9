"""numpy model of GPU_CAGRA's build and search, as defined in DESIGN §4.12.

Keys are computed in float64 and rounded to float32: on small-integer data every key is exact in fp32, so the device must
reproduce this model bit for bit.  The key of a row is its squared L2 distance, or minus its inner product."""
import numpy as np

M64 = (1 << 64) - 1
FLT_MAX = float(np.finfo(np.float32).max)


def splitmix64(j):
    """seed j of every query"""
    z = ((j + 1) * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def keys(X, q, metric):
    X = np.asarray(X, np.float64)
    q = np.asarray(q, np.float64)
    k = ((X - q) ** 2).sum(-1) if metric == "L2" else -(X @ q)
    return k.astype(np.float32)


def best_first(k):
    """positions of the keys k in (key, id) order"""
    return np.lexsort((np.arange(len(k)), k))


# ------------------------------------------------------------------------------------------------------------- build
def knn_graph(X, m, metric):
    """step 1: the m nearest rows of each row, best first, ties by ascending id, the row itself removed (or the last
    entry dropped when the row is not among the m + 1 nearest)"""
    n = len(X)
    G0 = np.empty((n, m), np.int64)
    for i in range(n):
        lst = best_first(keys(X, X[i], metric))[:m + 1]
        hit = np.nonzero(lst == i)[0]
        G0[i] = np.delete(lst, hit[0]) if len(hit) else lst[:m]
    return G0


def detour_counts(G0, n=None):
    """step 2: detour(i, b) = #{a < b : G0[i][b] in G0[G0[i][a]][0:b]}"""
    nrow, m = G0.shape
    n = nrow if n is None else n
    det = np.zeros((nrow, m), np.int64)
    rank = np.full(n, -1, np.int64)
    A = np.arange(m)[:, None]
    C = np.arange(m)[None, :]
    for i in range(nrow):
        rank[G0[i]] = np.arange(m)
        B = rank[G0[G0[i]]]   # B[a, c]: rank in G0[i] of G0[G0[i][a]][c], or -1
        ok = (B > A) & (B > C)
        det[i] = np.bincount(B[ok], minlength=m)
        rank[G0[i]] = -1
    return det


def prune(G0, det, g):
    """step 3: the g entries of each row with the smallest (detour, position)"""
    m = G0.shape[1]
    P = np.empty((len(G0), g), np.int64)
    for i in range(len(G0)):
        P[i] = G0[i][np.lexsort((np.arange(m), det[i]))[:g]]
    return P


def reverse_lists(P, n):
    """step 4: R[v] = the sources i of the edges i -> v = P[i][p], ordered by (p, i)"""
    g = P.shape[1]
    src = np.repeat(np.arange(len(P)), g)
    slot = np.tile(np.arange(g), len(P))
    v = P.reshape(-1)
    order = np.lexsort((src, slot, v))
    R = [[] for _ in range(n)]
    for e in order:
        R[v[e]].append(int(src[e]))
    return R


def merge_rows(P, R):
    """step 5: P[i][0:g/2], then R[i], then P[i][g/2:], each id once, up to g ids"""
    n, g = P.shape
    out = np.empty((n, g), np.int64)
    for i in range(n):
        row = [int(x) for x in P[i][:g // 2]]
        seen = set(row)
        for x in list(R[i]) + [int(x) for x in P[i][g // 2:]]:
            if len(row) >= g:
                break
            if x not in seen:
                row.append(x)
                seen.add(x)
        out[i] = row
    return out


def build(X, igd, gd, metric):
    """the graph of n rows (n x max(g, 1), -1 padded when n = 1)"""
    n = len(X)
    m = min(igd, n - 1)
    g = min(gd, m)
    if g == 0:
        return np.full((n, 1), -1, np.int64)
    G0 = knn_graph(X, m, metric)
    P = prune(G0, detour_counts(G0), g)
    return merge_rows(P, reverse_lists(P, n))


# ------------------------------------------------------------------------------------------------------------ search
def search_one(X, graph, q, itopk, width, max_iter, nrs, metric):
    """the pool T of one query after the search: [(key, id)], plus ndis and nhops"""
    n, g = graph.shape
    s = min(n, max(1, nrs * width * g))
    visited = set()
    pool = []   # [key, id, expanded]
    ndis = nhops = 0

    def absorb(cand):
        nonlocal pool, ndis
        ndis += len(cand)
        if not cand:
            return
        ks = keys(X[cand], q, metric)
        pool = sorted(pool + [[float(k), int(v), False] for k, v in zip(ks, cand)], key=lambda e: (e[0], e[1]))[:itopk]

    seeds = []
    for j in range(s):
        r = splitmix64(j) % n
        if r not in visited:
            visited.add(r)
            seeds.append(r)
    absorb(seeds)
    it = 0
    while max_iter == 0 or it < max_iter:
        parents = [e for e in pool if not e[2]][:width]
        if not parents:
            break
        for e in parents:
            e[2] = True
        nhops += len(parents)
        cand = []
        for e in parents:
            for v in graph[e[1]]:
                v = int(v)
                if v >= 0 and v not in visited:
                    visited.add(v)
                    cand.append(v)
        absorb(cand)
        it += 1
    return [(e[0], e[1]) for e in pool], ndis, nhops


def exact(X, Q, k, metric, filtered=None):
    """exact top-k, ties by ascending id, padded with -1 and +-FLT_MAX"""
    nq = len(Q)
    ids = np.full((nq, k), -1, np.int64)
    dist = np.full((nq, k), FLT_MAX if metric == "L2" else -FLT_MAX, np.float32)
    for r, q in enumerate(Q):
        kk = keys(X, q, metric)
        order = best_first(kk)
        if filtered is not None:
            order = order[~filtered[order]]
        order = order[:k]
        ids[r, :len(order)] = order
        dist[r, :len(order)] = kk[order] if metric == "L2" else -kk[order]
    return ids, dist


def search(X, graph, Q, k, itopk, width, max_iter=0, nrs=1, metric="L2", filtered=None):
    """the index's search: HNSW's exact-branch rule, the graph search, and the exact completion of short rows.
    filtered: bool[n], True = filtered out.  Returns ids, dist, (ndis, nhops)."""
    n = len(X)
    n_filtered = 0 if filtered is None else int(filtered.sum())
    n_valid = n - n_filtered
    bf = k >= n * 0.5
    if filtered is not None:
        bf = bf or n_filtered >= n * 0.93 or k >= n_valid * 0.5
    if bf:
        ids, dist = exact(X, Q, k, metric, filtered)
        return ids, dist, (len(Q) * n_valid, 0)
    nq = len(Q)
    ids = np.full((nq, k), -1, np.int64)
    dist = np.full((nq, k), FLT_MAX if metric == "L2" else -FLT_MAX, np.float32)
    ndis = nhops = 0
    for r, q in enumerate(Q):
        pool, a, b = search_one(X, graph, q, itopk, width, max_iter, nrs, metric)
        ndis += a
        nhops += b
        res = [e for e in pool if filtered is None or not filtered[e[1]]][:k]
        if len(res) < min(k, n_valid):
            ids[r:r + 1], dist[r:r + 1] = exact(X, q[None], k, metric, filtered)
            continue
        for c, (kk, v) in enumerate(res):
            ids[r, c] = v
            dist[r, c] = kk if metric == "L2" else -kk
    return ids, dist, (ndis, nhops)
