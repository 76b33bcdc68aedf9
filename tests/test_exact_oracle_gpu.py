"""Exact top-k of FLAT, BruteForce, IVF_FLAT and IVF_PQ against a float64 oracle (GPU).

The oracle computes every distance in float64 (direct sum((q-x)^2) for L2, sum(q*x) for IP, IP of rows normalised in
float64 for COSINE, and the ADC distance |q - c_l - r^|^2 / <q, c_l + r^> rebuilt from the index's exported state for
IVF_PQ).  `check_topk` is the one acceptance rule used by every case:

1. returned ids are distinct, belong to the index and are not filtered out by the bitset;
2. each returned distance matches the oracle within (n_terms + 2) * 2^-24 * sum|terms| of its own operands;
3. rows are in (distance, id) order;
4. nothing is missed: every valid row whose oracle distance beats the k-th returned one by more than twice the bound
   is in the result;
5. when fewer than k valid rows exist, exactly those are returned and the tail is -1 / +-FLT_MAX.

Each FLAT case names the selection / finalize path its shape reaches (thresholds in kb2_index.cuh dense_candidates and
launch_finalize, 132 SMs).
"""
import os

import numpy as np
import pytest

from knowhere_b200 import datagen

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
FLT_MAX = float(np.finfo(np.float32).max)
DEV = "cuda"


# ------------------------------------------------------------------------------------------------ oracle
def _t(a):
    return torch.as_tensor(np.asarray(a, np.float64), device=DEV)


def flat_oracle(xb, xq, metric):
    """(dist, bound) [nq, n] float64 numpy.  L2: direct sum((q-x)^2), sum|terms| = the distance itself.
    IP: sum(q*x), sum|terms| = sum|q*x|.  COSINE: IP of float64-normalised rows; the index normalises in fp32, which
    perturbs each operand by about (d+2) ulp, so the bound is tripled."""
    X, Q = _t(xb), _t(xq)
    nq, d = Q.shape
    n = X.shape[0]
    if metric == "COSINE":
        X = X / X.norm(dim=1, keepdim=True)
        Q = Q / Q.norm(dim=1, keepdim=True)
    D = torch.empty((nq, n), dtype=torch.float64, device=DEV)
    S = torch.empty_like(D)
    if metric == "L2":
        bq = max(1, min(nq, (1 << 25) // max(1, min(n, 8192) * d)))
        for q0 in range(0, nq, bq):
            for r0 in range(0, n, 8192):
                diff = Q[q0:q0 + bq, None, :] - X[None, r0:r0 + 8192, :]
                D[q0:q0 + bq, r0:r0 + 8192] = diff.square().sum(-1)
        S.copy_(D)
    else:
        D.copy_(Q @ X.T)
        S.copy_(Q.abs() @ X.abs().T)
    scale = 3.0 if metric == "COSINE" else 1.0
    B = scale * (d + 2) * U * S
    return D.cpu().numpy(), B.cpu().numpy()


def check_topk(ids, dist, D, B, labels, metric, valid=None, what=""):
    """The acceptance rule (module docstring).  D, B: [nq, n] oracle distance / error bound per row (row = position in
    `labels`); valid: [n] bool, False for rows filtered out by the bitset."""
    ids, dist = np.asarray(ids), np.asarray(dist)
    labels = np.asarray(labels, np.int64)
    nq, k = ids.shape
    n = labels.size
    valid = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    n_valid = int(valid.sum())
    sgn = 1.0 if metric == "L2" else -1.0          # key = sgn * distance, smaller is better
    order = np.argsort(labels, kind="stable")
    sl = labels[order]
    assert np.unique(sl).size == n, "labels must be distinct"
    for i in range(nq):
        msg = f"{what} q{i}"
        got = ids[i]
        m = min(k, n_valid)
        # 5. padding
        assert (got[m:] == -1).all(), f"{msg}: {n_valid} valid rows but ids past {m} are {got[m:][:8]}"
        assert (dist[i, m:] == sgn * FLT_MAX).all(), f"{msg}: padding distances {dist[i, m:][:8]}"
        g = got[:m]
        assert (g >= 0).all(), f"{msg}: -1 among the first {m} results: {got}"
        # 1. ids valid
        assert np.unique(g).size == m, f"{msg}: duplicate ids {g}"
        p = np.searchsorted(sl, g)
        assert (p < n).all() and (sl[np.minimum(p, n - 1)] == g).all(), f"{msg}: ids not in the index {g}"
        rows = order[p]
        assert valid[rows].all(), f"{msg}: filtered rows returned {g[~valid[rows]]}"
        # 2. distances
        od, ob = D[i, rows], B[i, rows]
        err = np.abs(dist[i, :m].astype(np.float64) - od)
        bad = np.nonzero(err > ob)[0]
        assert bad.size == 0, (f"{msg}: distance of id {g[bad[0]]} is {dist[i, bad[0]]!r}, oracle {od[bad[0]]!r}, "
                               f"bound {ob[bad[0]]:.3g}")
        # 3. order by (distance, id)
        key = sgn * dist[i, :m].astype(np.float64)
        ok = (key[1:] > key[:-1]) | ((key[1:] == key[:-1]) & (g[1:] > g[:-1]))
        assert ok.all(), f"{msg}: not in (distance, id) order at rank {int(np.argmin(ok))}"
        # 4. nothing missed
        if m == n_valid:
            continue
        kth = key[-1]
        kth_b = ob[-1]
        okey = sgn * D[i]
        must = valid & (okey < kth - 2.0 * np.maximum(B[i], kth_b))
        missing = np.setdiff1d(labels[must], g)
        assert missing.size == 0, (f"{msg}: {missing.size} true neighbours missing, e.g. id {missing[0]} at oracle "
                                   f"{sgn * okey[np.nonzero(labels == missing[0])[0][0]]!r}, k-th returned {dist[i, -1]!r}")


def _bits(mask):
    return np.packbits(mask, bitorder="little")


def _with_env(name, value, fn):
    old = os.environ.get(name)
    os.environ[name] = value
    try:
        return fn()
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


# ------------------------------------------------------------------------------------------------ FLAT / BruteForce
FLAT_CASES = [
    # nq, n, d, k
    pytest.param(100, 10000, 128, 10, id="select_keys-warpfin4"),       # Ksel 32: select_keys_kernel, finalize_warp<4>
    pytest.param(5, 20000, 64, 10, id="nsplit39-ctafin"),                # nsplit 39: 1248 partials, CTA finalize
    pytest.param(1, 50000, 128, 1, id="nsplit97-ctafin"),                # nsplit 97: 3104 partials, CTA finalize
    pytest.param(200, 20000, 128, 112, id="hist_fast-warpfin8"),         # Ksel 128, 2*K_need = 256: histogram fast path, warp<8>
    pytest.param(200, 20000, 128, 113, id="hist_levels-ctafin"),         # Ksel 256, K_need 129: level-wise histogram, CTA finalize
    pytest.param(40, 100, 32, 64, id="hist_whole_slice"),                # 100 keys <= K_cap 128: "whole slice fits"
    pytest.param(64, 30000, 36, 500, id="ksel1024"),                     # Ksel 1024
    pytest.param(16, 30000, 128, 1008, id="ksel1024-kmax"),              # Ksel 1024, k at the limit, 7 slices
    pytest.param(2000, 40000, 128, 10, id="two_chunks"),                 # key matrix in two chunks of 33536 columns
    pytest.param(4096, 150000, 32, 500, id="ten_chunks-reduce"),         # ten chunks: reduce_partials_kernel after eight
    pytest.param(50, 8000, 1536, 10, id="d1536-ctafin"),                 # d > 1024: no warp finalize
    pytest.param(5000, 3000, 17, 7, id="d17-fp32"),                      # d % 4 != 0: fp32 CUDA-core contraction
]


def _custom_ids(n, seed):
    # distinct, not monotone in the row position
    return (np.random.default_rng(seed).permutation(n).astype(np.int64) * 3 + 11)


@pytest.mark.parametrize("custom", [False, True], ids=["rowids", "customids"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("nq,n,d,k", FLAT_CASES)
def test_flat_exact(kb, nq, n, d, k, metric, custom):
    xb = datagen.uniform(n, d, 1000 + d)
    xq = datagen.uniform(nq, d, 2000 + d)
    labels = _custom_ids(n, 5) if custom else np.arange(n, dtype=np.int64)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb, labels if custom else None)
    ids, dist = ix.search(xq, k)
    assert ix.last_counters()["flagged"] == 0, "no query of ordinary data needs the exact redo scan"
    sample = np.arange(nq) if nq <= 2000 else np.random.default_rng(3).choice(nq, 128, replace=False)
    D, B = flat_oracle(xb, xq[sample], metric)
    check_topk(ids[sample], dist[sample], D, B, labels, metric, what=f"FLAT {metric}")
    if not custom and nq <= 2000:
        bi, bd = kb.brute_force_search(xb, xq, k, metric)
        assert np.array_equal(bi, ids) and np.array_equal(bd, dist)


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("d,k,custom,filtered", [
    pytest.param(128, 10, False, False, id="d128-k10"),               # redo finalized by finalize_warp<4>
    pytest.param(128, 100, False, False, id="d128-k100"),             # ... by finalize_warp<8>
    pytest.param(128, 500, True, True, id="d128-k500-ids-bitset"),    # ... by the CTA finalize; bitset and labels in the redo
    pytest.param(1536, 10, True, False, id="d1536-k10-ids"),          # d > 1024: CTA finalize
])
def test_flat_translated_data(kb, metric, d, k, custom, filtered):
    """Rows 1000 + N(0, 1): the norm-expanded key |q|^2 + |x|^2 - 2 q.x cancels catastrophically, so the exact re-rank
    of the best k + 16 approximate keys alone misses true neighbours.  Finalize cannot certify those queries and they
    are redone by flat_exact_scan_kernel with directly accumulated distances, then finalized again through `qlist`."""
    n, nq = 20000, (200 if d <= 1024 else 100)
    rng = np.random.default_rng(7)
    xb = (1000.0 + rng.standard_normal((n, d))).astype(np.float32)
    xq = (1000.0 + rng.standard_normal((nq, d))).astype(np.float32)
    labels = _custom_ids(n, 8) if custom else np.arange(n, dtype=np.int64)
    mask = (rng.random(n) < 0.5) if filtered else np.zeros(n, bool)     # True = filtered out
    bits = _bits(mask) if filtered else None
    D, B = flat_oracle(xb, xq, metric)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb, labels if custom else None)
    ids, dist = ix.search(xq, k, bitset=bits)
    if metric == "L2":
        assert ix.last_counters()["flagged"] == nq, "the key error exceeds every distance gap here"
    check_topk(ids, dist, D, B, labels, metric, valid=~mask, what="FLAT translated")
    bi, bd = kb.brute_force_search(xb, xq, k, metric, bitset=bits)
    check_topk(bi, bd, D, B, np.arange(n), metric, valid=~mask, what="BruteForce translated")


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_hnsw_fallback_translated_data(kb, metric):
    """HNSW's exact fallback ranks by the same norm-expanded keys as FLAT and is certified the same way.  Rows
    1000 + N(0, 1), reached through both of its triggers: a bitset that keeps about 5 % of the rows, and k >= n / 2."""
    n, nq, d = 20000, 200, 128
    rng = np.random.default_rng(12)
    xb = (1000.0 + rng.standard_normal((n, d))).astype(np.float32)
    xq = (1000.0 + rng.standard_normal((nq, d))).astype(np.float32)
    D, B = flat_oracle(xb, xq, metric)
    mask = rng.random(n) >= 0.05                                        # True = filtered out
    ix = kb.Index("HNSW", metric, d, {"M": 8, "efConstruction": 40})
    ix.build(xb)
    ids, dist = ix.search(xq, 10, bitset=_bits(mask))
    check_topk(ids, dist, D, B, np.arange(n), metric, valid=~mask, what="HNSW filtered fallback")
    n2, k2 = 2000, 1000
    small = kb.Index("HNSW", metric, d, {"M": 8, "efConstruction": 40})
    small.build(xb[:n2])
    ids, dist = small.search(xq, k2)
    check_topk(ids, dist, D[:, :n2], B[:, :n2], np.arange(n2), metric, what="HNSW k >= n/2 fallback")


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("keep,k", [(0, 10), (5, 10), (100, 500), (700, 1008)])
def test_flat_sparse_bitset(kb, metric, keep, k):
    """Bitsets that leave fewer than k rows (padding) or none at all."""
    n, nq, d = 20000, 30, 64
    xb = datagen.uniform(n, d, 31)
    xq = datagen.uniform(nq, d, 32)
    mask = np.ones(n, bool)                       # True = filtered out
    mask[np.random.default_rng(keep).choice(n, keep, replace=False)] = False
    labels = _custom_ids(n, 9)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb, labels)
    ids, dist = ix.search(xq, k, bitset=_bits(mask))
    D, B = flat_oracle(xb, xq, metric)
    check_topk(ids, dist, D, B, labels, metric, valid=~mask, what=f"FLAT bitset keep={keep}")


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_flat_half_bitset_large_k(kb, metric):
    n, nq, d, k = 30000, 64, 36, 500
    xb = datagen.uniform(n, d, 41)
    xq = datagen.uniform(nq, d, 42)
    mask = np.random.default_rng(1).random(n) < 0.5
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb)
    ids, dist = ix.search(xq, k, bitset=_bits(mask))
    D, B = flat_oracle(xb, xq, metric)
    check_topk(ids, dist, D, B, np.arange(n), metric, valid=~mask, what="FLAT half bitset")


def _dup_setup(n=20000, d=64, ndup=300, seed=3):
    """Rows uniform in [0, 100); one row copied to `ndup` random positions among the first 544 rows, queries close to
    that row.  With 4 queries dense_candidates cuts the 20000 columns into 39 slices of 544 rows, so all copies sit in
    slice 0: they tie bit for bit, there are more of them than K_cap = 128, and select_keys_hist_kernel drains the tied
    bin (shift == 0)."""
    rng = np.random.default_rng(seed)
    xb = datagen.uniform(n, d, seed)
    pos = np.sort(rng.choice(544, ndup, replace=False))
    xb[pos] = xb[pos[0]]
    xq = (xb[pos[0]] + 0.01 * rng.standard_normal((4, d))).astype(np.float32)
    return xb, xq, pos


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("custom", [False, "monotone", "permuted"])
def test_flat_exact_ties(kb, metric, custom):
    """DESIGN §4.6: rows whose distances tie exactly are taken in position (insertion) order; the k + 16 rows kept for
    the exact re-rank are output in (distance, id) order.  With ids that grow with the position the smallest ids win.
    The re-ranked window ends inside the tie group, so a dropped copy ties with the k-th result and finalize cannot
    certify the query: it is redone by flat_exact_scan_kernel, whose selection also breaks ties by position.
    (test_coarse_tie_drain_keeps_positions shows the equal-key drain's own output.)"""
    k = 100
    xb, xq, pos = _dup_setup()
    n = xb.shape[0]
    if custom == "monotone":
        labels = np.arange(n, dtype=np.int64) * 5 + 2
    elif custom == "permuted":
        labels = _custom_ids(n, 4)
    else:
        labels = np.arange(n, dtype=np.int64)
    if metric == "IP":
        # the duplicated row must be the best IP match: scale it up
        xb[pos] = xb[pos[0]] * 4.0
        xq = xb[pos[0]][None, :].repeat(4, 0) + 0.01
        xq = xq.astype(np.float32)
    ix = kb.Index("FLAT", metric, xb.shape[1])
    ix.add(xb, None if custom is False else labels)
    ids, dist = ix.search(xq, k)
    assert ix.last_counters()["flagged"] == xq.shape[0]
    D, B = flat_oracle(xb, xq, metric)
    check_topk(ids, dist, D, B, labels, metric, what="FLAT ties")
    tied = labels[pos]
    for i in range(xq.shape[0]):
        assert np.isin(ids[i], tied).all(), "the duplicated row is the nearest: all k results must be copies of it"
        assert (dist[i] == dist[i, 0]).all(), "copies of one row must get bit-identical distances"
        if custom == "permuted":
            window = tied[: k + 16]                  # first k + 16 copies in position order
            assert np.isin(ids[i], window).all()
            assert (np.diff(ids[i]) > 0).all()
        else:
            assert np.array_equal(ids[i], np.sort(tied)[:k])


def test_coarse_tie_drain_keeps_positions(kb):
    """The IVF coarse quantizer ranks centroids through dense_candidates without the FLAT certification, so its probes
    show the equal-key drain of select_keys_hist_kernel directly.  300 of 600 centroids are one vector and the query is
    that vector.  With nprobe 100 (K_need 116, K_cap 128, one 600-column slice) the 300 tied keys fill the first bin of
    every histogram level and the drain (shift == 0) takes 116 of them in position order; finalize keeps those and
    probes the 100 with the smallest ids.  Each list holds one row, nearer to the query the later its list, so the
    result names exactly the lists probed: the 91st to 100th copies in position order, the 100th first."""
    d, nlist, ndup, nprobe, k = 32, 600, 300, 100, 10
    rng = np.random.default_rng(11)
    cent = (rng.random((nlist, d)) * 100.0).astype(np.float32)
    pos = np.sort(rng.choice(nlist, ndup, replace=False))
    cent[pos] = cent[pos[0]]
    rows = cent.copy()
    rows[:, 0] += (0.02 - 0.01 * np.arange(nlist) / nlist).astype(np.float32)   # distinct offsets, shrinking with the list
    lists = [(l, np.array([l], np.int64), rows[l:l + 1]) for l in range(nlist)]
    ix = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
    ix.ivf_import(cent, None, lists)
    xq = cent[pos[:1]].copy()
    ids, dist = ix.search(xq, k, {"nprobe": nprobe})
    want = pos[:nprobe][::-1][:k]
    assert np.array_equal(ids[0], want), f"probed lists are not the first {nprobe} copies in position order: {ids[0]}"
    np.testing.assert_array_equal(dist[0], ((rows[want] - xq[0]) ** 2).sum(1, dtype=np.float32))


def test_bruteforce_device_tensors(kb):
    n, nq, d, k = 20000, 100, 128, 10
    xb = datagen.uniform(n, d, 51)
    xq = datagen.uniform(nq, d, 52)
    bi, bd = kb.brute_force_search(torch.from_numpy(xb).cuda(), torch.from_numpy(xq).cuda(), k, "L2")
    assert bi.is_cuda and bd.is_cuda
    D, B = flat_oracle(xb, xq, "L2")
    check_topk(bi.cpu().numpy(), bd.cpu().numpy(), D, B, np.arange(n), "L2", what="BruteForce device")
    hi, hd = kb.brute_force_search(xb, xq, k, "L2")
    assert np.array_equal(hi, bi.cpu().numpy()) and np.array_equal(hd, bd.cpu().numpy())


@pytest.mark.parametrize("nq,n,d,k", [(100, 10000, 128, 10), (200, 20000, 128, 113), (50, 8000, 1536, 10)])
def test_cosine_exact(kb, nq, n, d, k):
    xb = datagen.clustered(n, d, 61) + 1.0
    xq = datagen.clustered(nq, d, 62) + 1.0
    D, B = flat_oracle(xb, xq, "COSINE")
    ix = kb.Index("FLAT", "COSINE", d)
    ix.add(xb)
    ids, dist = ix.search(xq, k)
    check_topk(ids, dist, D, B, np.arange(n), "IP", what="FLAT COSINE")
    bi, bd = kb.brute_force_search(xb, xq, k, "COSINE")
    check_topk(bi, bd, D, B, np.arange(n), "IP", what="BruteForce COSINE")


@pytest.mark.parametrize("dtype", ["int8", "float16", "bfloat16"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_flat_typed_ingest_exact(kb, dtype, metric):
    """int8 / fp16 / bf16 rows and queries are widened exactly to fp32: the oracle sees the widened values."""
    n, nq, d, k = 20000, 64, 96, 20
    xb = datagen.clustered(n, d, 71)
    xq = datagen.clustered(nq, d, 72)
    if dtype == "int8":
        s = 127.0 / np.abs(xb).max()
        tb = torch.from_numpy(np.clip(np.round(xb * s), -127, 127).astype(np.int8))
        tq = torch.from_numpy(np.clip(np.round(xq * s), -127, 127).astype(np.int8))
    else:
        tb = torch.from_numpy(xb).to(getattr(torch, dtype))
        tq = torch.from_numpy(xq).to(getattr(torch, dtype))
    wb, wq = tb.to(torch.float32).numpy(), tq.to(torch.float32).numpy()
    ix = kb.Index("FLAT", metric, d)
    ix.add(tb)
    ids, dist = ix.search(tq, k)
    D, B = flat_oracle(wb, wq, metric)
    check_topk(ids, dist, D, B, np.arange(n), metric, what=f"FLAT {dtype}")
    f = kb.Index("FLAT", metric, d)
    f.add(wb)
    fi, fd = f.search(wq, k)
    assert np.array_equal(ids, fi) and np.array_equal(dist, fd)


# ------------------------------------------------------------------------------------------------ IVF_FLAT
@pytest.fixture(scope="module")
def ivf_flat_data():
    n, nq, d = 20000, 200, 64
    plain = (datagen.clustered(n, d, 81), datagen.clustered(nq, d, 82))
    rng = np.random.default_rng(83)
    shifted = ((1000.0 + rng.standard_normal((n, d))).astype(np.float32),
               (1000.0 + rng.standard_normal((nq, d))).astype(np.float32))
    return {"clustered": plain, "translated": shifted}


@pytest.mark.parametrize("engine", ["scan", "tc"])
@pytest.mark.parametrize("data", ["clustered", "translated"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_ivf_flat_all_lists_is_exact(kb, ivf_flat_data, engine, data, metric):
    """With nprobe = nlist IVF_FLAT scans every row with direct differences: the result is the exact top-k."""
    xb, xq = ivf_flat_data[data]
    n, d = xb.shape
    nlist = 32
    ix = kb.Index("IVF_FLAT", metric, d, {"nlist": nlist})
    ix.build(xb)
    D, B = flat_oracle(xb, xq, metric)
    for k in (1, 10, 113, 500, 1008):
        ids, dist = _with_env("KB2_FLAT_ENGINE", engine, lambda: ix.search(xq, k, {"nprobe": nlist}))
        check_topk(ids, dist, D, B, np.arange(n), metric, what=f"IVF_FLAT {engine} {data} k={k}")


# ------------------------------------------------------------------------------------------------ IVF_PQ
def pq_oracle(ix, xq, m, metric):
    """ADC distance of every stored row, rebuilt in float64 from the index's exported state.  Returns (D, B, labels).
    L2: |q - c_l - r^|^2 with terms dis0 = |q - c_l|^2, t1 = sum(r^^2 + 2 c_l r^) and the tables sum(-2 q r^).
    IP: <q, c_l> + <q, r^>.  Bound: (d + m + 2) * 2^-24 * sum|terms|."""
    cent, pq = ix.ivf_export_centroids(m)
    nlist, d = cent.shape
    dsub = d // m
    labs, recs, cids = [], [], []
    for l in range(nlist):
        ids, codes = ix.ivf_export_list(l, m)
        if ids.size == 0:
            continue
        r = pq[np.arange(m)[None, :], codes.astype(np.int64)]          # [len, m, dsub]
        recs.append(r.reshape(ids.size, d))
        labs.append(ids)
        cids.append(np.full(ids.size, l))
    R, C, Q = _t(np.concatenate(recs)), _t(cent), _t(xq)
    li = torch.as_tensor(np.concatenate(cids), device=DEV)
    labels = np.concatenate(labs)
    CL = C[li]
    if metric == "L2":
        X = CL + R
        D = torch.empty((Q.shape[0], X.shape[0]), dtype=torch.float64, device=DEV)
        for r0 in range(0, X.shape[0], 4096):
            D[:, r0:r0 + 4096] = (Q[:, None, :] - X[None, r0:r0 + 4096, :]).square().sum(-1)
        dis0 = ((Q[:, None, :] - C[None, :, :]).square().sum(-1))[:, li]
        t1 = (R.square() + 2.0 * (CL * R).abs()).sum(1)
        S = dis0 + t1[None, :] + 2.0 * (Q.abs() @ R.abs().T)
    else:
        D = Q @ (CL + R).T
        S = (Q.abs() @ CL.abs().T) + (Q.abs() @ R.abs().T)
    B = (d + m + 2) * U * S
    return D.cpu().numpy(), B.cpu().numpy(), labels


PQ_GEOMS = [(16, 128), (32, 128), (48, 96)]


@pytest.fixture(scope="module")
def pq_indexes(kb):
    cache = {}

    def get(m, d, metric, nlist=32, n=20000, nq=200):
        key = (m, d, metric, nlist, n, nq)
        if key not in cache:
            xb = datagen.clustered(n, d, 91)
            xq = datagen.clustered(nq, d, 92)
            ix = kb.Index("IVF_PQ", metric, d, {"nlist": nlist, "m": m, "nbits": 8})
            ix.build(xb)
            cache[key] = (ix, xq) + pq_oracle(ix, xq, m, metric)
        return cache[key]
    return get


@pytest.mark.parametrize("k", [1, 10, 100, 129, 500, 1008])
@pytest.mark.parametrize("engine", ["lut", "tc"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("m,d", PQ_GEOMS, ids=["m16d128", "m32d128", "m48d96"])
def test_ivfpq_all_lists_matches_adc_oracle(kb, pq_indexes, m, d, metric, engine, k):
    ix, xq, D, B, labels = pq_indexes(m, d, metric)
    ids, dist = _with_env("KB2_PQ_ENGINE", engine, lambda: ix.search(xq, k, {"nprobe": 32}))
    check_topk(ids, dist, D, B, labels, metric, what=f"IVF_PQ m{m} {engine} k={k}")


@pytest.mark.parametrize("m,d", PQ_GEOMS, ids=["m16d128", "m32d128", "m48d96"])
def test_ivfpq_small_batch_split_probes(kb, pq_indexes, m, d):
    """Five queries: each query's probes are split over many CTAs (nsplit = min(nprobe, 2 * SMs / nq))."""
    ix, xq, D, B, labels = pq_indexes(m, d, "L2")
    for k in (10, 500):
        ids, dist = ix.search(xq[:5].copy(), k, {"nprobe": 32})
        check_topk(ids, dist, D[:5], B[:5], labels, "L2", what=f"IVF_PQ m{m} nq=5 k={k}")


@pytest.mark.parametrize("m,d", PQ_GEOMS, ids=["m16d128", "m32d128", "m48d96"])
def test_ivfpq_refine_k16(kb, m, d):
    """refine_k 16 at k = 10 (160 refine candidates): results are the exact distances of the refined rows."""
    n, nq, nlist, k = 20000, 100, 32, 10
    xb = datagen.clustered(n, d, 101)
    xq = datagen.clustered(nq, d, 102)
    ix = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m, "refine": True, "refine_type": "flat"})
    ix.build(xb)
    D, B = flat_oracle(xb, xq, "L2")
    ids, dist = ix.search(xq, k, {"nprobe": nlist, "refine_k": 16})
    assert (ids >= 0).all()
    for i in range(nq):
        assert np.unique(ids[i]).size == k
        err = np.abs(dist[i].astype(np.float64) - D[i, ids[i]])
        assert (err <= B[i, ids[i]]).all(), f"q{i}: refined distances are not exact"
        assert (np.diff(dist[i]) >= 0).all()
    # the refined top-10 of 160 ADC candidates recovers (nearly) all of the exact top-10 on this data
    gt = np.argsort(D, axis=1)[:, :k]
    assert datagen.recall(gt, ids) > 0.9


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_ivfpq_tc_large_batch_tail_finalize(kb, pq_indexes, metric):
    """1200 queries (> 8 x 132) through the tensor-core engine at k = 128: finalize_warp_kernel takes the rows of at most
    256 candidates and the CTA finalize's tail pass (row_loop_nq) walks the rest.  KB2_TC_P0=1 lets phase A see only the
    query's nearest list, which holds about 78 codes (256 lists of 20000 rows), fewer than k: those queries get no bound,
    are flagged and redone by the LUT kernel into full 2048-entry rows, which only the tail pass can finalize."""
    ix, xq, D, B, labels = pq_indexes(16, 128, metric, nlist=256, nq=1200)
    ids, dist = _with_env("KB2_TC_P0", "1",
                          lambda: _with_env("KB2_PQ_ENGINE", "tc", lambda: ix.search(xq, 128, {"nprobe": 256})))
    c = ix.last_counters()
    assert ix.last_stage_info()["engine"] == "tc"
    assert c["flagged"] > 0, c
    check_topk(ids, dist, D, B, labels, metric, what=f"IVF_PQ tc nq=1200 {metric}")


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_ivfpq_tc_redo_through_generic_kernel(kb, pq_indexes, metric):
    """m48 at k = 1008: the skewed LUT kernel does not fit, so the tensor-core engine's redo pass runs
    ivfpq_scan_generic_kernel over the flagged queries only.  KB2_TC_P0=1 lets phase A see only the nearest list, which
    holds fewer than 1008 codes for most queries: they get no bound and are flagged."""
    ix, xq, D, B, labels = pq_indexes(48, 96, metric)
    ids, dist = _with_env("KB2_TC_P0", "1",
                          lambda: _with_env("KB2_PQ_ENGINE", "tc", lambda: ix.search(xq, 1008, {"nprobe": 32})))
    c = ix.last_counters()
    assert ix.last_stage_info()["engine"] == "tc"
    assert c["flagged"] > 0, c
    check_topk(ids, dist, D, B, labels, metric, what=f"IVF_PQ m48 tc redo k=1008 {metric}")


@pytest.mark.parametrize("engine", ["lut", "tc"])
def test_ivfpq_many_probes_k1000(kb, pq_indexes, engine):
    """nprobe 160 (> 145) at k = 1000 with 300 queries (one CTA per query, so all 160 probes in one CTA): the skewed LUT
    kernel's probe arrays no longer fit next to its tables."""
    ix, xq, D, B, labels = pq_indexes(16, 128, "L2", nlist=160, nq=300)
    ids, dist = _with_env("KB2_PQ_ENGINE", engine, lambda: ix.search(xq, 1000, {"nprobe": 160}))
    check_topk(ids, dist, D, B, labels, "L2", what=f"IVF_PQ nprobe 160 k=1000 {engine}")


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("m,d", [(16, 128), (48, 96)], ids=["m16d128", "m48d96"])
def test_ivfpq_short_empty_and_repeated_lists(kb, m, d, metric):
    """Imported lists: four empty, four shorter than k, and one holding 60 copies of a single code (exact ties)."""
    n, nq, nlist, k = 12000, 100, 32, 50
    xb = datagen.clustered(n, d, 111)
    xq = datagen.clustered(nq, d, 112)
    src = kb.Index("IVF_PQ", metric, d, {"nlist": nlist, "m": m})
    src.build(xb)
    cent, pq = src.ivf_export_centroids(m)
    lists = []
    for l in range(nlist):
        ids, codes = src.ivf_export_list(l, m)
        if l < 4:
            continue
        if l < 8:
            ids, codes = ids[:3], codes[:3]
        if l == 8 and ids.size > 60:
            codes = codes.copy()
            codes[:60] = codes[0]
        lists.append((l, ids, codes))
    for engine in ("lut", "tc"):
        ix = kb.Index("IVF_PQ", metric, d, {"nlist": nlist, "m": m})
        ix.ivf_import(cent, pq, lists)
        D, B, labels = pq_oracle(ix, xq, m, metric)
        ids, dist = _with_env("KB2_PQ_ENGINE", engine, lambda: ix.search(xq, k, {"nprobe": nlist}))
        check_topk(ids, dist, D, B, labels, metric, what=f"IVF_PQ crafted lists {engine}")


def test_ivfpq_bf16_ingest_matches_widened_fp32(kb):
    nb, d, nlist, m = 20000, 96, 32, 48
    xb = torch.from_numpy(datagen.clustered(nb, d, 42)).to(torch.bfloat16)
    xq = torch.from_numpy(datagen.clustered(64, d, 43)).to(torch.bfloat16)
    a = kb.Index("IVF_PQ", "IP", d, {"nlist": nlist, "m": m})
    a.build(xb)
    b = kb.Index("IVF_PQ", "IP", d, {"nlist": nlist, "m": m})
    b.build(xb.to(torch.float32).numpy())
    ra = a.search(xq, 10, {"nprobe": 8})
    rb = b.search(xq.to(torch.float32).numpy(), 10, {"nprobe": 8})
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
