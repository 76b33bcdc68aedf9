"""numpy restatement of the sparse search definition (DESIGN §4.13), in float32 with the device's rounding order, plus a
float64 oracle.  numpy only: every float32 operation below is one correctly rounded IEEE operation, as the device's
__fmul_rn / __fadd_rn / __fdiv_rn are.

Row sets are CSR triples (indptr int64 [n + 1], indices uint32, values float32)."""
import numpy as np

F32 = np.float32


def drop_threshold(values, ratio):
    """get_query_drop_threshold (reference inverted_index.h:151-162): c = (size_t)(float(ratio) * float(nnz)); 0 when c is
    0, else the value at 0-based position c of the values in ascending order (nth_element)."""
    values = np.asarray(values, F32)
    c = int(F32(ratio) * F32(values.size))
    if c == 0:
        return F32(0)
    c = min(c, values.size - 1)
    return np.partition(values, c)[c]


def bm25_params(k1, b, avgdl):
    """p1 = k1 + 1, p2 = k1 (1 - b), p3 = k1 b / max(avgdl, 1) in float32 (BM25IndexScorer, scorer.h:81-104)"""
    k1, b, avgdl = F32(k1), F32(b), F32(avgdl)
    return k1 + F32(1), k1 * (F32(1) - b), (k1 * b) / max(avgdl, F32(1))


class Postings:
    """term -> (rows, values) of a CSR row set, and the float32 row sums L_r in index order"""

    def __init__(self, csr):
        indptr, indices, values = csr
        self.n = indptr.size - 1
        rows = np.repeat(np.arange(self.n, dtype=np.int64), np.diff(indptr))
        order = np.lexsort((rows, indices))
        t, r, v = indices[order], rows[order], values[order]
        self.terms, start = np.unique(t, return_index=True)
        end = np.append(start[1:], t.size)
        self.lists = {int(x): (r[a:e], v[a:e]) for x, a, e in zip(self.terms, start, end)}
        # sequential float32 sums in index order: step j adds every row's j-th value
        lens = np.diff(indptr)
        self.row_sum = np.zeros(self.n, F32)
        for j in range(int(lens.max()) if self.n else 0):
            live = np.nonzero(lens > j)[0]
            self.row_sum[live] = self.row_sum[live] + values[indptr[live] + j]
        self.row_sum64 = np.zeros(self.n)
        np.add.at(self.row_sum64, rows, values.astype(np.float64))


def kept_entries(post, q_idx, q_val, ratio):
    """the kept (term, weight) entries of one query, in query order"""
    thr = drop_threshold(q_val, ratio) if ratio > 0 else F32(0)
    return [(int(t), F32(w)) for t, w in zip(q_idx, q_val) if w >= thr and int(t) in post.lists]


def scores(post, q_idx, q_val, metric="IP", ratio=0.0, bm25=None, dtype=F32):
    """s(q, r) for every row.  dtype float32: the definition's rounding; float64: the oracle (bm25 = (k1, b, avgdl))."""
    s = np.zeros(post.n, dtype)
    if metric == "BM25":
        k1, b, avgdl = bm25
        if dtype == F32:
            p1, p2, p3 = bm25_params(k1, b, avgdl)
        else:
            p1, p2, p3 = k1 + 1.0, k1 * (1.0 - b), k1 * b / max(avgdl, 1.0)
        L = post.row_sum if dtype == F32 else post.row_sum64
    for t, w in kept_entries(post, q_idx, q_val, ratio):
        r, v = post.lists[t]
        v = v.astype(dtype)
        w = dtype(w)
        if metric == "IP":
            c = w * v
        else:
            c = ((w * dtype(p1)) * v) / ((v + dtype(p2)) + (dtype(p3) * L[r]))
        s[r] = s[r] + c.astype(dtype)
    return s


def candidates(s, bitset=None):
    ok = s > 0
    if bitset is not None:
        bits = np.unpackbits(np.asarray(bitset, np.uint8), bitorder="little")[:s.size].astype(bool)
        ok &= ~bits
    return np.nonzero(ok)[0]


def topk(s, k, bitset=None):
    """ids, dist of the k best candidates by (s descending, row ascending), padded with -1 / -FLT_MAX"""
    c = candidates(s, bitset)
    order = np.lexsort((c, -s[c].astype(np.float64)))[:k]
    ids = np.full(k, -1, np.int64)
    dist = np.full(k, -np.finfo(np.float32).max, np.float32)
    ids[:order.size] = c[order]
    dist[:order.size] = s[c[order]]
    return ids, dist


def search(base, queries, k, metric="IP", ratio=0.0, bm25=None, bitset=None, dtype=F32, post=None):
    """[nq, k] ids and distances of the definition (dtype float32) or of the float64 oracle"""
    post = post or Postings(base)
    qp, qi, qv = queries
    nq = qp.size - 1
    ids = np.empty((nq, k), np.int64)
    dist = np.empty((nq, k), np.float32 if dtype == F32 else np.float64)
    for q in range(nq):
        s = scores(post, qi[qp[q]:qp[q + 1]], qv[qp[q]:qp[q + 1]], metric, ratio, bm25, dtype)
        ids[q], d = topk(s, k, bitset)
        dist[q] = d
    return ids, dist


def range_search(base, queries, radius, range_filter=None, metric="IP", ratio=0.0, bm25=None, bitset=None, post=None):
    """(lims, ids, dist): candidates with radius < s <= range_filter, best first, ties by row"""
    post = post or Postings(base)
    qp, qi, qv = queries
    nq = qp.size - 1
    lims, ids, dist = [0], [], []
    for q in range(nq):
        s = scores(post, qi[qp[q]:qp[q + 1]], qv[qp[q]:qp[q + 1]], metric, ratio, bm25)
        c = candidates(s, bitset)
        c = c[s[c] > F32(radius)]
        if range_filter is not None:
            c = c[s[c] <= F32(range_filter)]
        order = np.lexsort((c, -s[c].astype(np.float64)))
        ids.append(c[order])
        dist.append(s[c[order]])
        lims.append(lims[-1] + c.size)
    cat = (lambda a, t: np.concatenate(a).astype(t) if a else np.empty(0, t))
    return np.array(lims, np.int64), cat(ids, np.int64), cat(dist, np.float32)
