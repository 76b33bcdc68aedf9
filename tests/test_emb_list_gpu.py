"""Emb-list (multi-vector) BruteForce search with the MAX_SIM metrics (DESIGN §4.10) against a float64 oracle (GPU).

The oracle computes every query-token x base-token distance in float64 on the GPU (sum(q*x) for IP, sum((q-x)^2) for L2,
IP of rows normalised in float64 for COSINE), the extremum over each document and the sum over each query list.  Its
bound for one score is the sum over the list's tokens of the largest per-distance bound of test_exact_oracle_gpu over the
document's vectors, plus the fp32 rounding of the token sum.  `check_emb` is the acceptance rule of every case, check_topk
adapted to emb-lists:

1. ids are distinct, valid documents, not empty and not filtered out;
2. each returned score is within its bound of the oracle;
3. rows are in (score, id) order, larger first for IP / COSINE, smaller first for L2;
4. nothing is missed: every valid document beating the k-th returned one by more than twice the bound is in the result;
5. padding is exactly -1 with FLT_MIN (std::numeric_limits<float>::min(); IP, COSINE) or FLT_MAX (L2), and an empty
   query list gets a whole row of it.

Paths: d % 4 == 0 runs the tensor-core filter (maxsim_filter_kernel), the K = k + 16 selection, the exact re-rank and
certification; k >= 1009 has K > 1024 (the same path, no other selection kernel exists here); d % 4 != 0 runs the exact
all-documents mode for every list (stats[2] == n_lists); data with a large common offset under MAX_SIM_L2 makes the filter's
bound too wide to certify and runs the exact redo of those lists (stats[2] > 0).  Documents longer than 128 rows span
several filter tiles, query lists longer than 128 tokens several query blocks.  The candidate re-rank and the
all-documents mode both run maxsim_rerank_kernel; test_rerank_shapes takes each across its row tiles and token blocks.
"""
import os
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)
DEV = "cuda"
METRICS = ["MAX_SIM", "MAX_SIM_COSINE", "MAX_SIM_IP", "MAX_SIM_L2"]


def _lims(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


def _data(lengths, d, seed, offset=0.0, scale=1.0):
    x = np.random.default_rng(seed).standard_normal((int(np.sum(lengths)), d)).astype(np.float32)
    return (x * scale + offset).astype(np.float32), _lims(lengths)


def oracle(xb, xl, xq, ql, metric):
    """(score, bound) [n_lists, n_docs] float64 numpy; score is NaN for an empty document or query list."""
    X = torch.as_tensor(np.asarray(xb, np.float64), device=DEV)
    Q = torch.as_tensor(np.asarray(xq, np.float64), device=DEV)
    cos = metric in ("MAX_SIM", "MAX_SIM_COSINE")
    l2 = metric == "MAX_SIM_L2"
    if cos:
        X = X / X.norm(dim=1, keepdim=True)
        Q = Q / Q.norm(dim=1, keepdim=True)
    d = X.shape[1]
    n_docs, n_lists = len(xl) - 1, len(ql) - 1
    doc = torch.as_tensor(np.repeat(np.arange(n_docs), np.diff(xl)), device=DEV)
    lst = torch.as_tensor(np.repeat(np.arange(n_lists), np.diff(ql)), device=DEV)
    nqr = Q.shape[0]
    ext = torch.full((n_docs, nqr), np.inf if l2 else -np.inf, dtype=torch.float64, device=DEV)
    bnd = torch.zeros((n_docs, nqr), dtype=torch.float64, device=DEV)
    scale = 3.0 if cos else 1.0
    for r0 in range(0, X.shape[0], 4096):
        Xc = X[r0:r0 + 4096]
        if l2:
            D = torch.cdist(Xc, Q, compute_mode="donot_use_mm_for_euclid_dist").square()
            S = D
        else:
            D = Xc @ Q.T
            S = Xc.abs() @ Q.abs().T
        idx = doc[r0:r0 + 4096, None].expand(-1, nqr)
        ext.scatter_reduce_(0, idx, D, "amin" if l2 else "amax")
        bnd.scatter_reduce_(0, idx, scale * (d + 2) * U * S, "amax")
    score = torch.zeros((n_lists, n_docs), dtype=torch.float64, device=DEV).index_add_(0, lst, ext.T)
    mag = torch.zeros_like(score).index_add_(0, lst, ext.T.abs())
    ntok = torch.as_tensor(np.diff(ql), dtype=torch.float64, device=DEV)[:, None]
    bound = torch.zeros_like(score).index_add_(0, lst, bnd.T) + (ntok + 2) * U * mag
    score[:, torch.as_tensor(np.diff(xl) == 0, device=DEV)] = np.nan
    score[torch.as_tensor(np.diff(ql) == 0, device=DEV)] = np.nan
    return score.cpu().numpy(), bound.cpu().numpy()


def check_emb(ids, dist, score, bound, metric, valid=None, what=""):
    ids, dist = np.asarray(ids), np.asarray(dist)
    n_lists, k = ids.shape
    n_docs = score.shape[1]
    l2 = metric == "MAX_SIM_L2"
    sgn = 1.0 if l2 else -1.0
    pad = FLT_MAX if l2 else FLT_MIN
    valid = np.ones(n_docs, bool) if valid is None else np.asarray(valid, bool)
    for i in range(n_lists):
        msg = f"{what} list {i}"
        ok_docs = valid & ~np.isnan(score[i])
        m = min(k, int(ok_docs.sum()))
        got = ids[i]
        assert (got[m:] == -1).all(), f"{msg}: {ok_docs.sum()} valid documents but ids past {m} are {got[m:][:8]}"
        assert (dist[i, m:] == np.float32(pad)).all(), f"{msg}: padding {dist[i, m:][:8]}"
        g = got[:m]
        assert np.unique(g).size == m and (g >= 0).all() and (g < n_docs).all(), f"{msg}: bad ids {g[:16]}"
        assert ok_docs[g].all(), f"{msg}: empty or filtered documents returned {g[~ok_docs[g]]}"
        err = np.abs(dist[i, :m].astype(np.float64) - score[i, g])
        bad = np.nonzero(err > bound[i, g])[0]
        assert bad.size == 0, (f"{msg}: score of doc {g[bad[0]]} is {dist[i, bad[0]]!r}, oracle {score[i, g[bad[0]]]!r}, "
                               f"bound {bound[i, g[bad[0]]]:.3g}")
        key = sgn * dist[i, :m].astype(np.float64)
        order_ok = (key[1:] > key[:-1]) | ((key[1:] == key[:-1]) & (g[1:] > g[:-1]))
        assert order_ok.all(), f"{msg}: not in (score, id) order at rank {int(np.argmin(order_ok))}"
        if m == 0 or m == int(ok_docs.sum()):
            continue
        okey = sgn * np.where(ok_docs, score[i], np.nan)
        must = ok_docs & (okey < key[-1] - 2.0 * np.maximum(bound[i], bound[i, g[-1]]))
        missing = np.setdiff1d(np.nonzero(must)[0], g)
        assert missing.size == 0, f"{msg}: {missing.size} documents missing, e.g. {missing[0]} at {score[i, missing[0]]!r}"


# documents: 1 token, mixed lengths up to several 128-row tiles, empty ones in the middle
DOC_LEN = np.array([1, 7, 0, 130, 33, 1, 300, 0, 0, 64, 128, 129, 5, 1, 1, 1, 257, 40, 0, 90] * 8)
# query lists: 1 token, 32, longer than a query block (300 > 128), an empty one in the middle
Q_LEN = np.array([1, 32, 300, 0, 5, 32, 129, 2])


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", [128, 768, 17])
def test_metrics_and_dims(kb, metric, d):
    xb, xl = _data(DOC_LEN, d, 1)
    xq, ql = _data(Q_LEN, d, 2)
    k = 10
    ids, dist, st = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, metric, stats=True)
    S, B = oracle(xb, xl, xq, ql, metric)
    check_emb(ids, dist, S, B, metric, what=f"{metric} d={d}")
    assert st[0] == len(Q_LEN)
    if d == 128:
        assert st[1] == len(Q_LEN) * (k + 16) and st[2] == 0, st   # ordinary data: every list certified
    elif d % 4:
        assert st[2] == len(Q_LEN), st                              # exact all-documents mode
    assert (ids[3] == -1).all() and (dist[3] == np.float32(FLT_MAX if metric == "MAX_SIM_L2" else FLT_MIN)).all()


def test_metric_names_case_insensitive(kb):
    xb, xl = _data(DOC_LEN[:20], 32, 3)
    xq, ql = _data(Q_LEN[:3], 32, 4)
    a = kb.brute_force_search_emb_list(xb, xl, xq, ql, 5, "max_sim_ip")
    b = kb.brute_force_search_emb_list(xb, xl, xq, ql, 5, "MAX_SIM_IP")
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    c = kb.brute_force_search_emb_list(xb, xl, xq, ql, 5, "MAX_SIM")
    e = kb.brute_force_search_emb_list(xb, xl, xq, ql, 5, "Max_Sim_Cosine")
    assert np.array_equal(c[0], e[0]) and np.array_equal(c[1], e[1])


@pytest.mark.parametrize("metric", ["MAX_SIM_IP", "MAX_SIM_L2"])
@pytest.mark.parametrize("k", [1, 10, 1009, 16384])
@pytest.mark.parametrize("keep", [1.0, 0.5, 0.0])
def test_k_and_bitsets(kb, metric, k, keep):
    """k = 1 and 10, k >= 1009 (K above 1024) and k = 16384, which is more than the unfiltered documents (padding)."""
    n_docs = 2500
    lens = np.random.default_rng(5).integers(0, 40, n_docs)
    xb, xl = _data(lens, 64, 6)
    xq, ql = _data(np.array([3, 32, 1, 140]), 64, 7)
    filt = np.random.default_rng(8).random(n_docs) >= keep      # True = filtered out
    bits = np.packbits(filt, bitorder="little")
    ids, dist = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, metric, bitset=bits)
    S, B = oracle(xb, xl, xq, ql, metric)
    check_emb(ids, dist, S, B, metric, valid=~filt, what=f"k={k} keep={keep}")
    if keep == 0.0:
        assert (ids == -1).all()


def test_short_bitset_rejected_then_usable(kb):
    xb, xl = _data(DOC_LEN[:40], 32, 9)
    xq, ql = _data(Q_LEN[:2], 32, 10)
    with pytest.raises(kb.KnowhereError) as e:
        kb.brute_force_search_emb_list(xb, xl, xq, ql, 3, "MAX_SIM_IP", bitset=np.zeros(2, np.uint8))   # 16 < 40 bits
    assert e.value.status == 1
    ids, _ = kb.brute_force_search_emb_list(xb, xl, xq, ql, 3, "MAX_SIM_IP", bitset=np.zeros(5, np.uint8))
    assert (ids >= 0).all()


def test_several_query_chunks(kb):
    """n_docs x n_lists above the 64M-entry score budget: the lists run in two chunks."""
    n_docs, n_lists, d = 70000, 1000, 32
    xb, xl = _data(np.random.default_rng(11).integers(1, 4, n_docs), d, 12)
    xq, ql = _data(np.random.default_rng(13).integers(1, 3, n_lists), d, 14)
    ids, dist, st = kb.brute_force_search_emb_list(xb, xl, xq, ql, 10, "MAX_SIM_IP", stats=True)
    sample = np.random.default_rng(15).choice(n_lists, 40, replace=False)
    sample.sort()
    S, B = oracle(xb, xl, xq, ql, "MAX_SIM_IP")
    check_emb(ids[sample], dist[sample], S[sample], B[sample], "MAX_SIM_IP", what="chunks")
    assert st[0] == n_lists and st[2] == 0


@pytest.mark.parametrize("metric", ["MAX_SIM", "MAX_SIM_L2"])
def test_host_device_and_repeat_bits(kb, metric):
    xb, xl = _data(DOC_LEN, 128, 16)
    xq, ql = _data(Q_LEN, 128, 17)
    hi, hd = kb.brute_force_search_emb_list(xb, xl, xq, ql, 20, metric)
    hi2, hd2 = kb.brute_force_search_emb_list(xb, xl, xq, ql, 20, metric)
    t = lambda a: torch.from_numpy(a).cuda()
    di, dd = kb.brute_force_search_emb_list(t(xb), t(xl), t(xq), t(ql), 20, metric)
    mi, md = kb.brute_force_search_emb_list(t(xb), xl, xq, t(ql), 20, metric)   # mixed host / device inputs
    assert di.is_cuda and dd.is_cuda
    for i, dist in ((hi2, hd2), (di.cpu().numpy(), dd.cpu().numpy()), (mi, md)):
        assert np.array_equal(hi, i) and np.array_equal(hd.view(np.uint32), dist.view(np.uint32))


def test_fallback_large_offset_l2(kb):
    """A large common offset: the filter's |q|^2 + |x|^2 - 2<q, x> cancels, the bound is too wide to certify, and the
    uncertified lists are redone exactly over every document."""
    lens = np.random.default_rng(18).integers(1, 60, 600)
    xb, xl = _data(lens, 64, 19, offset=200.0, scale=0.05)
    xq, ql = _data(np.array([8, 16, 32, 4]), 64, 20, offset=200.0, scale=0.05)
    ids, dist, st = kb.brute_force_search_emb_list(xb, xl, xq, ql, 10, "MAX_SIM_L2", stats=True)
    assert st[2] > 0, st
    S, B = oracle(xb, xl, xq, ql, "MAX_SIM_L2")
    check_emb(ids, dist, S, B, "MAX_SIM_L2", what="offset")


# the re-rank's shapes: documents of 0, 1, 128, 129 and 300 rows (several 128-row tiles), query lists of 0, 1 and 200
# tokens (several 32-token blocks)
RR_DOC_LEN = np.concatenate([[0, 1, 129, 300, 0, 128], np.random.default_rng(27).integers(0, 60, 200)])
RR_Q_LEN = np.array([200, 1, 37, 0, 5, 64])


@pytest.mark.parametrize("metric,offset", [("MAX_SIM_IP", 0.0), ("MAX_SIM_L2", 0.0), ("MAX_SIM_L2", 200.0)])
@pytest.mark.parametrize("d", [30, 128, 768])
@pytest.mark.parametrize("keep", [1.0, 0.5])
def test_rerank_shapes(kb, metric, offset, d, keep):
    """d = 30 re-ranks every document of every list with scalar loads; d = 128 and 768 re-rank the filter's candidates
    with float4 loads, and with the large common offset under MAX_SIM_L2 also every document of the uncertified lists.
    With keep = 0.5 half the documents are filtered out and skipped inside each all-documents row."""
    xb, xl = _data(RR_DOC_LEN, d, 28 + d, offset=offset, scale=0.05 if offset else 1.0)
    xq, ql = _data(RR_Q_LEN, d, 29 + d, offset=offset, scale=0.05 if offset else 1.0)
    filt = np.random.default_rng(30).random(len(RR_DOC_LEN)) >= keep
    k = 10
    ids, dist, st = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, metric, bitset=np.packbits(filt, bitorder="little"),
                                                   stats=True)
    S, B = oracle(xb, xl, xq, ql, metric)
    check_emb(ids, dist, S, B, metric, valid=~filt, what=f"{metric} d={d} offset={offset} keep={keep}")
    if d % 4:
        assert st[1] == 0 and st[2] == len(RR_Q_LEN), st           # all-documents mode
    else:
        assert st[1] == len(RR_Q_LEN) * (k + 16), st                # the filter's candidates
        assert st[2] > 0 or offset == 0, st                         # the redo of uncertified lists


@pytest.mark.parametrize("metric,single", [("MAX_SIM_IP", "IP"), ("MAX_SIM_L2", "L2")])
def test_single_vector_lists_match_bruteforce(kb, metric, single):
    n, nq, d, k = 3000, 20, 64, 10
    xb, xl = _data(np.ones(n, np.int64), d, 21)
    xq, ql = _data(np.ones(nq, np.int64), d, 22)
    ids, dist = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, metric)
    bi, bd = kb.brute_force_search(xb, xq, k, single)
    S, B = oracle(xb, xl, xq, ql, metric)
    check_emb(ids, dist, S, B, metric, what="single")
    same = ids == bi
    assert same.mean() >= 0.99, same.mean()
    rows = np.arange(nq)[:, None].repeat(k, 1)
    assert (np.abs(dist - bd) <= B[rows, np.maximum(ids, 0)] + B[rows, np.maximum(bi, 0)]).all()


def test_self_query_l2(kb):
    """Each document as its own query list under MAX_SIM_L2 comes back first at distance 0 (test_bruteforce.cc:57-77)."""
    lens = np.random.default_rng(23).integers(1, 200, 64)
    xb, xl = _data(lens, 128, 24)
    ids, dist = kb.brute_force_search_emb_list(xb, xl, xb, xl, 5, "MAX_SIM_L2")
    assert (ids[:, 0] == np.arange(64)).all() and (dist[:, 0] == 0).all()


def test_errors_and_recovery(kb):
    xb, xl = _data(DOC_LEN[:20], 32, 25)
    xq, ql = _data(Q_LEN[:3], 32, 26)

    def status(*a, **kw):
        with pytest.raises(kb.KnowhereError) as e:
            kb.brute_force_search_emb_list(*a, **kw)
        return e.value.status

    bad_start = xl.copy(); bad_start[0] = 1
    bad_dec = xl.copy(); bad_dec[3] = bad_dec[2] - 1
    assert status(xb, bad_start, xq, ql, 5, "MAX_SIM_IP") == 1
    assert status(xb, bad_dec, xq, ql, 5, "MAX_SIM_IP") == 1
    assert status(xb, xl[:-1], xq, ql, 5, "MAX_SIM_IP") == 1          # does not end at the row count
    assert status(xb, xl, xq, ql[:-1], 5, "MAX_SIM_IP") == 1
    assert status(xb, xl, xq, ql, 16385, "MAX_SIM_IP") == 1
    assert status(xb, xl, xq, ql, 0, "MAX_SIM_IP") == 1
    assert status(xb, xl, xq, ql, 5, "MAX_SIM_HAMMING") == 5
    assert status(xb, xl, xq, ql, 5, "MAX_SIM_JACCARD") == 5
    assert status(xb, xl, xq, ql, 5, "L2") == 5
    L = kb.lib()
    ids = np.empty((3, 5), np.int64)
    dis = np.empty((3, 5), np.float32)
    p = lambda a: a.ctypes.data
    assert L.kb2_bruteforce_search_emb_list(None, p(xl), len(xl) - 1, 32, 4, p(xq), p(ql), 3, 5, None, 0, p(ids), p(dis),
                                            None, 0, None) == 1
    assert L.kb2_bruteforce_search_emb_list(p(xb), p(xl), len(xl) - 1, 0, 4, p(xq), p(ql), 3, 5, None, 0, p(ids), p(dis),
                                            None, 0, None) == 1
    assert L.kb2_bruteforce_search_emb_list(p(xb), p(xl), 0, 32, 4, p(xq), p(ql), 3, 5, None, 0, p(ids), p(dis),
                                            None, 0, None) == 1
    i2, d2 = kb.brute_force_search_emb_list(xb, xl, xq, ql, 5, "MAX_SIM_IP")
    S, B = oracle(xb, xl, xq, ql, "MAX_SIM_IP")
    check_emb(i2, d2, S, B, "MAX_SIM_IP", what="after errors")


def test_cpp_mirror(tmp_path):
    """BruteForce::Search / SearchWithBuf<fp32> with EMB_LIST_OFFSET on both DataSets (tests/cpp/test_emb_list.cc)."""
    exe = tmp_path / "test_emb_list"
    subprocess.run(["g++", "-std=c++17", "-O2", f"-I{ROOT}/include", os.path.join(ROOT, "tests", "cpp", "test_emb_list.cc"),
                    "-o", str(exe), f"-L{ROOT}/knowhere_b200", "-l:libknowhere_b200.so",
                    f"-Wl,-rpath,{ROOT}/knowhere_b200"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "emb_list ok" in r.stdout
