"""Seeded synthetic data (SURVEY §8d).

`uniform` reproduces the reference unit tests' GenDataSet distribution (tests/ut/utils.h:41-50:
uniform_real(0,100)); `clustered` is the structured low-rank mixture needed for PQ recall:
z ~ N(mu_c, I_r), x = z B + 0.05 eps."""
import numpy as np


def uniform(n, d, seed):
    rng = np.random.default_rng(seed)
    return (rng.random((n, d), dtype=np.float32) * 100.0).astype(np.float32)


def clustered(n, d, seed, r=16, n_clusters=None, struct_seed=7):
    n_clusters = n_clusters or max(16, int(1000 * n / 200000))
    srng = np.random.default_rng(struct_seed)
    mu = srng.standard_normal((n_clusters, r)).astype(np.float32) * 3.0
    B = srng.standard_normal((r, d)).astype(np.float32)
    rng = np.random.default_rng(seed)
    c = rng.integers(0, n_clusters, n)
    z = mu[c] + rng.standard_normal((n, r)).astype(np.float32)
    x = z @ B + 0.05 * rng.standard_normal((n, d)).astype(np.float32)
    return np.ascontiguousarray(x, np.float32)


def clustered_torch(n, d, seed, device, r=16, n_clusters=None, struct_seed=7, chunk=1 << 20):
    """Same mixture generated on the GPU (torch is plumbing here: device memory + RNG)."""
    import torch
    n_clusters = n_clusters or max(16, int(1000 * n / 200000))
    g = torch.Generator(device=device)
    g.manual_seed(struct_seed)
    mu = torch.randn((n_clusters, r), generator=g, device=device) * 3.0
    B = torch.randn((r, d), generator=g, device=device)
    g.manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device=device)
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        c = torch.randint(0, n_clusters, (m,), generator=g, device=device)
        z = mu[c] + torch.randn((m, r), generator=g, device=device)
        out[s:s + m] = z @ B + 0.05 * torch.randn((m, d), generator=g, device=device)
    return out


def recall(gt_ids, ids):
    """size(gt ∩ res) / (nq*k)  (reference tests/ut/utils.h:110-133)."""
    hit = 0
    for a, b in zip(gt_ids, ids):
        hit += len(set(a.tolist()) & set(b.tolist()) - {-1})
    return hit / float(gt_ids.shape[0] * gt_ids.shape[1])


def _csr_from_pairs(rows, terms, vals, n):
    """CSR (indptr int64, indices uint32, values float32) of (row, term, value) triples: sorted by (row, term), the first
    of each duplicate (row, term) kept"""
    key = (rows.astype(np.int64) << 32) | terms.astype(np.int64)
    order = np.argsort(key, kind="stable")
    key, vals = key[order], vals[order]
    keep = np.ones(key.size, bool)
    keep[1:] = key[1:] != key[:-1]
    key, vals = key[keep], vals[keep]
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(key >> 32, minlength=n), out=indptr[1:])
    return indptr, (key & 0xFFFFFFFF).astype(np.uint32), np.ascontiguousarray(vals, np.float32)


def _zipf_terms(rng, count, vocab, s):
    """`count` term ranks in [0, vocab) with P(rank r) proportional to (r + 1)^-s"""
    cdf = np.cumsum(np.arange(1, vocab + 1, dtype=np.float64) ** -s)
    return np.minimum(np.searchsorted(cdf, rng.random(count) * cdf[-1]), vocab - 1)


def sparse_splade(n, nnz, seed, vocab=30522, s=1.0):
    """SPLADE-like learned sparse rows: about `nnz` nonzeros per row over a vocabulary of `vocab` term ids with Zipf(s)
    term frequencies, positive log-normal weights.  Returns CSR (indptr, indices, values)."""
    rng = np.random.default_rng(seed)
    # Poisson draw counts; repeated draws of a frequent term merge, which costs about a quarter of them at s = 1
    lens = np.maximum(rng.poisson(nnz * 4 / 3, n), 1)
    rows = np.repeat(np.arange(n, dtype=np.int64), lens)
    terms = _zipf_terms(rng, rows.size, vocab, s)
    vals = rng.lognormal(-1.0, 0.6, rows.size).astype(np.float32)
    return _csr_from_pairs(rows, terms, vals, n)


def _hashed(ranks, seed):
    # an odd multiplier is a bijection of the 32-bit ids: distinct ranks keep distinct hashed ids
    return ((ranks.astype(np.uint64) * np.uint64(2654435761) + np.uint64(seed * 40503 + 1)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def sparse_bm25_docs(n, seed, vocab=200000, mean_len=100, s=1.05, hash_seed=11):
    """BM25-like documents: integer term counts (a term drawn k times has value k) of about `mean_len` Zipf(s) draws per
    row over `vocab` terms, with hashed uint32 term ids.  Returns (CSR, average row sum)."""
    rng = np.random.default_rng(seed)
    lens = np.maximum(rng.poisson(mean_len, n), 1)
    rows = np.repeat(np.arange(n, dtype=np.int64), lens)
    ranks = _zipf_terms(rng, rows.size, vocab, s)
    key = (rows << 32) | ranks
    uk, cnt = np.unique(key, return_counts=True)
    indptr, idx, vals = _csr_from_pairs(uk >> 32, _hashed(uk & 0xFFFFFFFF, hash_seed), cnt.astype(np.float32), n)
    return (indptr, idx, vals), float(vals.sum(dtype=np.float64) / n)


def sparse_bm25_queries(nq, n_docs, seed, vocab=200000, s=1.05, hash_seed=11):
    """BM25 queries of 4-8 distinct Zipf(s) terms over the same hashed ids as sparse_bm25_docs, each weighted by its IDF
    log(1 + (N - df + 0.5) / (df + 0.5)) with df taken from the Zipf frequencies of a collection of n_docs rows."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(4, 9, nq)
    rows = np.repeat(np.arange(nq, dtype=np.int64), lens)
    ranks = _zipf_terms(rng, rows.size, vocab, s)
    p = (np.arange(1, vocab + 1, dtype=np.float64) ** -s)
    p /= p.sum()
    df = np.minimum(n_docs * (1.0 - np.exp(-100.0 * p[ranks])), n_docs)
    idf = np.log1p((n_docs - df + 0.5) / (df + 0.5)).astype(np.float32)
    return _csr_from_pairs(rows, _hashed(ranks, hash_seed), idf, nq)
