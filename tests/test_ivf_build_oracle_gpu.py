"""IVF_FLAT / IVF_PQ construction against the float64 model of tests/ivf_build_model.py (GPU).

The search oracles take an index's exported centroids, codebooks and lists as given; these tests check the contents
themselves: k-means step by step (kb2_debug_kmeans), train() as the composition of those k-means runs, the coarse
assignment and the PQ codes add() stores, the sealed list layout and the rows behind it.

Two levels of check:
* bit-exact, on small-integer data (values in [-8, 8]): every key is exact in fp32 on both contractions, so initial
  centroids, assignments (first minimum on ties), the first Lloyd step with its splits, and the codes equal the model;
* within the bound, on float data: every list and code choice passes the rule of ibm.check_assignment / check_codes,
  and every updated centroid is the mean of its points within (cnt + 1) u mean|x|.

The assignment a k-means step used is observed without a second hook: C_t is imported into an IVF_FLAT of k lists with
the same metric and the same training rows are added in the same order; add() runs assign_nearest with the same rows,
k, chunking and contraction, so its exported lists are that assignment.  Each case names the branch of assign_nearest
it reaches (ibm.uses_wgmma: the wgmma 3xTF32 kernel when k >= 512, d % 4 == 0 and the batch has >= 1024 rows, the fp32
CUDA-core gemm_keys_kernel otherwise); the test asserts the shape condition, not a run-time switch.
"""
import ctypes
import functools

import numpy as np
import pytest

from knowhere_b200 import datagen
from tests import ivf_build_model as ibm

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

METRIC = {"L2": 0, "IP": 1}
U = ibm.U


# ------------------------------------------------------------------------------------------------ data
def _ints(n, d, seed, lo=-8, hi=8):
    return np.random.default_rng(seed).integers(lo, hi + 1, (n, d)).astype(np.float32)


def _dups(n, d, seed, distinct=20):
    """integer rows drawn from `distinct` rows: initial centroids tie and clusters empty"""
    base = _ints(distinct, d, seed)
    return np.ascontiguousarray(base[np.random.default_rng(seed + 1).integers(0, distinct, n)])


def _same(n, d, seed):
    return np.tile(_ints(1, d, seed), (n, 1))


def _few_1d(n, d, seed):
    return np.random.default_rng(seed).integers(0, 4, (n, 1)).astype(np.float32)


def _clustered(n, d, seed):
    return datagen.clustered(n, d, seed)


def _uniform(n, d, seed):
    return datagen.uniform(n, d, seed)


def _offset(n, d, seed):
    """rows with a large common offset: the norm-expanded keys cancel"""
    return (datagen.clustered(n, d, seed) + np.float32(1000.0)).astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _assert_bits(a, b, what):
    a, b = _bits(a), _bits(b)
    assert a.shape == b.shape, f"{what}: shapes {a.shape} vs {b.shape}"
    bad = np.argwhere(a != b)
    assert bad.size == 0, f"{what}: {len(bad)} values differ, first at {tuple(bad[0])}"


# ------------------------------------------------------------------------------------------------ library access
def _hook(kb, X, k, metric, niter, seed=ibm.KMEANS_SEED):
    """kb2_debug_kmeans over the rows X (copied to the device): the k x d centroids after niter Lloyd iterations"""
    L = kb.lib()
    L.kb2_debug_kmeans.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                   ctypes.c_uint64, ctypes.c_void_p, ctypes.c_int]
    n, d = X.shape
    x = torch.from_numpy(np.ascontiguousarray(X, np.float32)).cuda()
    out = torch.full((k, d), float("nan"), dtype=torch.float32, device="cuda")
    kb._check(L.kb2_debug_kmeans(x.data_ptr(), n, d, k, METRIC[metric], niter, seed, out.data_ptr(), 0))
    return out.cpu().numpy()


def _import(kb, kind, metric, C, pq=None, cfg=None):
    """an index whose quantizers are C (and pq), with no rows"""
    k, d = C.shape
    cfg = dict(cfg or {}, nlist=k)
    ix = kb.Index(kind, metric, d, cfg)
    C = np.ascontiguousarray(C, np.float32)
    pq = None if pq is None else np.ascontiguousarray(pq, np.float32)
    kb._check(kb.lib().kb2_ivf_import_begin(ix.h, k, C.ctypes.data, None if pq is None else pq.ctypes.data))
    return ix


def _code_size(ix, m):
    return m if ix.type == "IVF_PQ" else ix.dim * 4


def _lists(ix, m=0):
    """[(ids, codes)] of every list in scan order"""
    return [ix.ivf_export_list(l, _code_size(ix, m)) for l in range(ix.ivf_nlist())]


def _list_of_row(lists, n):
    A = np.full(n, -1, np.int64)
    for l, (ids, _) in enumerate(lists):
        A[ids] = l
    assert (A >= 0).all()
    return A


def _assign(kb, C, X, metric):
    """the lists add() gives the rows X against the centroids C (imported into an IVF_FLAT of len(C) lists)"""
    ix = _import(kb, "IVF_FLAT", metric, C)
    ix.add(np.ascontiguousarray(X, np.float32))
    lists = _lists(ix)
    ibm.check_layout([ids for ids, _ in lists], np.arange(len(X)), what="assignment index")
    return _list_of_row(lists, len(X))


def _counts(kb, C, X, metric):
    """the list sizes add() gives the rows X against the centroids C"""
    ix = _import(kb, "IVF_FLAT", metric, C)
    ix.add(np.ascontiguousarray(X, np.float32))
    return np.array([kb.lib().kb2_ivf_list_size(ix.h, l) for l in range(len(C))], np.int64)


def _assert_same_lists(a, b, what):
    assert len(a) == len(b), f"{what}: {len(a)} vs {len(b)} lists"
    for l, ((ia, ca), (ib, cb)) in enumerate(zip(a, b)):
        assert np.array_equal(ia, ib), f"{what}: list {l} ids differ"
        assert np.array_equal(ca, cb), f"{what}: list {l} codes differ"


def _status(fn):
    import knowhere_b200 as kb
    try:
        fn()
    except kb.KnowhereError as e:
        return e.status
    return 0


# ------------------------------------------------------------------------------------------------ a. k-means steps
STEPS = (0, 1, 2, 3, 4, 24)
KM_CASES = [
    # data, n, d, k, metric, bit-exact, wgmma
    pytest.param(_ints, 3000, 1, 256, "L2", True, False, id="d1-int"),
    pytest.param(_ints, 3000, 2, 256, "L2", True, False, id="d2-int"),
    pytest.param(_ints, 3000, 3, 256, "IP", True, False, id="d3-int-ip"),
    pytest.param(_ints, 3000, 4, 256, "L2", True, False, id="d4-int"),
    pytest.param(_clustered, 3000, 8, 256, "L2", False, False, id="d8-clustered"),
    pytest.param(_clustered, 3000, 31, 64, "IP", False, False, id="d31-clustered-ip"),
    pytest.param(_uniform, 3000, 33, 64, "L2", False, False, id="d33-uniform"),
    pytest.param(_clustered, 4000, 128, 100, "L2", False, False, id="d128-clustered"),
    pytest.param(_ints, 600, 8, 1, "L2", True, False, id="k1-subsample-int"),
    pytest.param(_clustered, 5000, 16, 8, "IP", False, False, id="k8-subsample-ip"),
    pytest.param(_ints, 2048, 8, 511, "L2", True, False, id="k511-int"),
    pytest.param(_ints, 2048, 8, 512, "L2", True, True, id="k512-int-wgmma"),
    pytest.param(_ints, 2048, 8, 512, "IP", True, True, id="k512-int-wgmma-ip"),
    pytest.param(_offset, 2048, 32, 512, "L2", False, True, id="k512-offset-wgmma"),
    pytest.param(_dups, 300, 4, 300, "L2", True, False, id="k=n-dups"),
    pytest.param(_dups, 2000, 8, 256, "L2", True, False, id="dups"),
    pytest.param(_same, 1000, 4, 16, "L2", True, False, id="identical-rows"),
    pytest.param(_few_1d, 2000, 1, 16, "L2", True, False, id="1d-four-values"),
]


@pytest.mark.parametrize("data,n,d,k,metric,exact,wgmma", KM_CASES)
def test_kmeans_steps(kb, data, n, d, k, metric, exact, wgmma):
    """kmeans_train one Lloyd step at a time (kb2_debug_kmeans with niter = t): the subsample and init rows
    (gather_rows_kernel), the assignment (assign_nearest: gemm_keys_kernel or the wgmma gemm_keys_tc_kernel, then
    argmin_rows_kernel), the update (histogram_kernel, cub radix sort, kmeans_reduce_kernel, whose lanes-per-point
    geometry d = 3 leaves a masked lane) and the empty-cluster split (kmeans_split_kernel), with the split draws replayed
    from the GPU's own counts.  On integer data C_0, A_0 and C_1 equal the model bit for bit."""
    X = data(n, d, 11)
    draws = ibm.KMeansDraws(n, k)
    Xt = X if draws.sample is None else np.ascontiguousarray(X[draws.sample])
    assert ibm.uses_wgmma(len(Xt), d, k) == wgmma
    C = [_hook(kb, X, k, metric, t) for t in range(max(STEPS) + 2)]
    _assert_bits(C[0], Xt[draws.init], "C_0 = the init rows")
    for t in range(max(STEPS) + 1):
        if t not in STEPS:
            draws.split(_counts(kb, C[t], Xt, metric))   # every step's draws keep the generator in step with the device's
            continue
        A = _assign(kb, C[t], Xt, metric)
        pairs = draws.split(np.bincount(A, minlength=k))
        what = f"step {t}"
        ibm.check_assignment(Xt, C[t], A, metric, wgmma, exact=exact and t == 0, what=what)
        Cm, mean, cnt, mabs = ibm.lloyd_means(Xt, A, C[t])
        if exact and t == 0:
            _assert_bits(C[1], ibm.apply_splits(Cm, pairs), "C_1 = means and splits of A_0")
            continue
        # populated clusters: the mean within its bound; empty ones unsplit (nt <= k): unchanged; split ones: the
        # donor's value times 1 +- 2^-10
        Cs, tol = ibm.apply_splits(mean, pairs, ibm.mean_tolerance(cnt, mabs))
        err = np.abs(C[t + 1].astype(np.float64) - Cs)
        bad = np.argwhere(err > tol)
        assert bad.size == 0, (f"{what}: centroid {bad[0][0]} (count {cnt[bad[0][0]]}, split pairs {pairs[:4]}) is "
                               f"{C[t + 1][tuple(bad[0])]!r}, model {Cs[tuple(bad[0])]!r}")


def test_kmeans_all_identical_rows_split_every_step(kb):
    """all rows identical: every step puts every row in cluster 0 (first minimum among equal keys) until the splits
    separate the centroids, and each step splits every empty cluster (kmeans_split_kernel, pairs applied in order)."""
    X = _same(1000, 4, 3)
    draws = ibm.KMeansDraws(1000, 16)
    C0 = _hook(kb, X, 16, "L2", 0)
    A = _assign(kb, C0, X, "L2")
    assert (A == 0).all()
    pairs = draws.split(np.bincount(A, minlength=16))
    assert [p[0] for p in pairs] == list(range(1, 16))
    _assert_bits(_hook(kb, X, 16, "L2", 1), ibm.apply_splits(ibm.lloyd_means(X, A, C0)[0], pairs), "C_1")


# ------------------------------------------------------------------------------------------------ b. train()
def _pq_sample(X):
    n = len(X)
    if n <= ibm.PQ_SAMPLE_ROWS:
        return X
    return np.ascontiguousarray(X[ibm.partial_shuffle(n, ibm.PQ_SAMPLE_ROWS, ibm.MT19937_64(ibm.PQ_SAMPLE_SEED))])


TRAIN_CASES = [
    # kind, metric, n, d, nlist, m
    pytest.param("IVF_FLAT", "L2", 6000, 32, 64, 0, id="flat-l2"),
    pytest.param("IVF_FLAT", "IP", 20000, 32, 16, 0, id="flat-ip-subsample"),
    pytest.param("IVF_FLAT", "COSINE", 6000, 32, 64, 0, id="flat-cosine"),
    pytest.param("IVF_FLAT", "L2", 1000, 16, 64, 0, id="flat-nlist-reduced"),
    pytest.param("IVF_FLAT", "L2", 40000, 8, 1024, 0, id="flat-wgmma"),
    pytest.param("IVF_PQ", "L2", 3000, 32, 16, 8, id="pq-l2"),
    pytest.param("IVF_PQ", "IP", 3000, 48, 16, 16, id="pq-ip-dsub3"),
    pytest.param("IVF_PQ", "L2", 70000, 16, 32, 4, id="pq-l2-pq-sample"),
]


@pytest.mark.parametrize("kind,metric,n,d,nlist,m", TRAIN_CASES)
def test_train_is_the_documented_composition(kb, kind, metric, n, d, nlist, m):
    """IvfIndex::train: nlist reduced to max(1, n / 39) when nlist * 39 > n; the coarse centroids are
    kmeans_train(rows, nlist, metric, 25, 1234) (COSINE: the normalised rows the index stores, with IP); PQ codebook m is
    kmeans_train(fp32 residual slice m of the PQ sample, 256, L2, 25, 1234) (slice_residual_kernel), the sample drawn
    with seed 1234 + 7 when n > 65536 and each row's residual taken against its own list (assign_nearest)."""
    X = _clustered(n, d, 5)
    cfg = {"nlist": nlist}
    if m:
        cfg["m"] = m
    ix = kb.Index(kind, metric, d, cfg)
    ix.train(X)
    nl = ibm.match_nlist(nlist, n)
    assert ix.ivf_nlist() == nl
    C, pq = ix.ivf_export_centroids(m)
    hm = metric
    rows = X
    if metric == "COSINE":
        st = kb.Index("IVF_FLAT", "COSINE", d, {"nlist": 1})
        st.build(X)
        (ids, codes), = _lists(st)
        rows = np.empty_like(X)
        rows[ids] = codes.view(np.float32).reshape(-1, d)
        hm = "IP"
    _assert_bits(C, _hook(kb, rows, nl, hm, ibm.KMEANS_NITER), "coarse centroids")
    if not m:
        return
    S = _pq_sample(rows)
    A = _assign(kb, C, S, hm)
    R = ibm.residuals(S, C, A)
    dsub = d // m
    for j in range(m):
        sub = np.ascontiguousarray(R[:, j * dsub:(j + 1) * dsub])
        _assert_bits(pq[j], _hook(kb, sub, 256, "L2", ibm.KMEANS_NITER), f"PQ codebook {j}")


# ------------------------------------------------------------------------------------------------ c. coarse assignment
@functools.lru_cache(maxsize=None)
def _trained_flat(kb, metric, n, d, nlist, seed):
    ix = kb.Index("IVF_FLAT", metric, d, {"nlist": nlist})
    ix.train(_clustered(n, d, seed))
    return ix.ivf_export_centroids()[0]


def _stored_rows(lists, n, d):
    out = np.full((n, d), np.nan, np.float32)
    for ids, codes in lists:
        out[ids] = codes.view(np.float32).reshape(-1, d)
    return out


def _check_adds(kb, metric, C, batches, exact=False):
    """add() the batches in turn to an IVF_FLAT over C; each batch's rows pass the rule on its own contraction"""
    k, d = C.shape
    ix = _import(kb, "IVF_FLAT", metric, C)
    for b in batches:
        ix.add(b)
    X = np.concatenate(batches)
    lists = _lists(ix)
    ibm.check_layout([ids for ids, _ in lists], np.arange(len(X)), what="lists")
    A = _list_of_row(lists, len(X))
    stored = _stored_rows(lists, len(X), d)
    hm = "IP" if metric == "COSINE" else metric
    s = 0
    for b in batches:
        tc = ibm.uses_wgmma(len(b), d, k)
        sl = slice(s, s + len(b))
        rows = stored[sl] if metric == "COSINE" else X[sl]
        ibm.check_assignment(rows, C, A[sl], hm, tc, exact=exact, what=f"batch of {len(b)} ({'wgmma' if tc else 'fp32'})")
        s += len(b)
    return [ibm.uses_wgmma(len(b), d, k) for b in batches]


@pytest.mark.parametrize("metric", ["L2", "IP", "COSINE"])
def test_add_assignment_fp32(kb, metric):
    """trained quantizer, nlist 256 < 512: gemm_keys_kernel + argmin_rows_kernel"""
    C = _trained_flat(kb, metric, 12000, 32, 256, 1)
    assert _check_adds(kb, metric, C, [_clustered(4000, 32, 2)]) == [False]


@pytest.mark.parametrize("metric", ["L2", "IP", "COSINE"])
def test_add_assignment_wgmma(kb, metric):
    """trained quantizer, nlist 1024, d % 4 == 0, 3000 rows: the wgmma 3xTF32 gemm_keys_tc_kernel"""
    C = _trained_flat(kb, metric, 45000, 32, 1024, 3)
    assert _check_adds(kb, metric, C, [_clustered(3000, 32, 4)]) == [True]


def test_add_assignment_d_not_multiple_of_4(kb):
    """d = 30 with 600 lists and 2000 rows stays on gemm_keys_kernel (its scalar loads)"""
    C = _clustered(600, 30, 6)
    assert _check_adds(kb, "L2", C, [_clustered(2000, 30, 7)]) == [False]


def test_add_assignment_chunks_and_tail(kb):
    """65536 imported lists: assign_nearest's key matrix holds 1024 rows, so 5000 rows run in four chunks and a tail of
    904, all on the wgmma kernel"""
    C = _offset(65536, 8, 8)
    assert _check_adds(kb, "L2", C, [_offset(5000, 8, 9)]) == [True]


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_add_assignment_switches_by_batch_size(kb, metric):
    """1024 lists: batches of 700 and 300 rows run gemm_keys_kernel, a batch of 2000 the wgmma kernel; each row passes
    the rule of the contraction its batch took"""
    C = _clustered(1024, 32, 10)
    X = _clustered(3000, 32, 11)
    assert _check_adds(kb, metric, C, [X[:700], X[700:2700], X[2700:]]) == [False, True, False]


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_add_assignment_integer_ties(kb, metric):
    """integer centroids with duplicates: rows at equal keys go to the lowest list id, on gemm_keys_kernel (500 rows)
    and on the wgmma kernel (2000 rows) alike (argmin_rows_kernel keeps the first minimum)"""
    C = _dups(600, 8, 12, distinct=100)
    X = _ints(2500, 8, 13)
    assert _check_adds(kb, metric, C, [X[:2000], X[2000:]], exact=True) == [True, False]


# ------------------------------------------------------------------------------------------------ d. PQ codes
PQ_SHAPES = [(8, 16), (16, 8), (32, 4), (48, 2), (64, 1), (16, 3)]


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("m,dsub", PQ_SHAPES)
def test_pq_codes(kb, m, dsub, metric):
    """pq_encode_kernel over a trained IVF_PQ: every code of every row is the nearest codeword of its residual against
    its own list; read back through both code layouts (layout_codes_kernel for m = 16, 32, 48, layout_codes_plain_kernel
    for m = 8, 64)"""
    d = m * dsub
    X = _clustered(2000, d, 14)
    ix = kb.Index("IVF_PQ", metric, d, {"nlist": 16, "m": m})
    ix.build(X)
    C, pq = ix.ivf_export_centroids(m)
    lists = _lists(ix, m)
    ibm.check_layout([ids for ids, _ in lists], np.arange(len(X)))
    A = _list_of_row(lists, len(X))
    ibm.check_assignment(X, C, A, metric, False)
    for l, (ids, codes) in enumerate(lists):
        if len(ids):
            ibm.check_codes(ibm.residuals(X[ids], C, A[ids]), pq, codes, what=f"list {l}")


@pytest.mark.parametrize("m", [16, 8])
def test_pq_codes_integer_ties(kb, m):
    """imported integer centroids and codebooks with duplicate codewords: assignment and codes equal the model bit for
    bit, the lowest code on ties (pq_encode_kernel's lane-ascending scan and shuffle tie-break)"""
    d, nlist = 32, 8
    dsub = d // m
    C = _dups(nlist, d, 15, distinct=5)
    rng = np.random.default_rng(16)
    pq = rng.integers(-4, 5, (m, 256, dsub)).astype(np.float32)
    pq[:, 128:] = pq[:, :128]                  # every codeword twice
    X = _ints(1500, d, 17)
    ix = _import(kb, "IVF_PQ", "L2", C, pq, {"m": m})
    ix.add(X)
    lists = _lists(ix, m)
    A = _list_of_row(lists, len(X))
    assert (A == ibm.exact_assign(X, C, "L2")).all()
    codes = np.zeros((len(X), m), np.int64)
    for ids, c in lists:
        codes[ids] = c
    want = ibm.pq_encode(ibm.residuals(X, C, A), pq)
    assert (want < 128).all() and np.array_equal(codes, want)


# ------------------------------------------------------------------------------------------------ e. lists and rows
@pytest.mark.parametrize("metric", ["L2", "IP", "COSINE"])
def test_lists_labels_and_rows(kb, metric):
    """seal(): place_rows_kernel after a stable cub radix sort by list; the stored rows (gather_rows_kernel) and
    get_vector_by_ids.  One add(), three add() calls, custom ids, and add() after an ivf_import of the first rows all
    give the lists the model's layout gives."""
    n, d, nlist = 6000, 32, 64
    X = _clustered(n, d, 18)
    if metric == "COSINE":
        X[[5, 77]] = 0.0
    one = kb.Index("IVF_FLAT", metric, d, {"nlist": nlist})
    one.build(X)
    C = one.ivf_export_centroids()[0]
    lists = _lists(one)
    A = ibm.check_layout([ids for ids, _ in lists], np.arange(n), what="one add")
    stored = _stored_rows(lists, n, d)
    if metric == "COSINE":
        X64 = X.astype(np.float64)
        nrm = np.linalg.norm(X64, axis=1, keepdims=True)
        unit = np.divide(X64, nrm, out=np.zeros_like(X64), where=nrm > 0)
        assert np.abs(stored - unit).max() <= 3 * (d + 2) * U
        assert (stored[[5, 77]] == 0).all()
    else:
        _assert_bits(stored, X, "stored rows")
        _assert_bits(one.get_vector_by_ids(np.arange(n)[::-1].copy()), X[::-1], "get_vector_by_ids")
    ibm.check_assignment(stored if metric == "COSINE" else X, C, A, "IP" if metric == "COSINE" else metric, False)
    # several add() calls
    three = _import(kb, "IVF_FLAT", metric, C)
    for s in (slice(0, 1000), slice(1000, 4500), slice(4500, n)):
        three.add(np.ascontiguousarray(X[s]))
    _assert_same_lists(_lists(three), lists, "three add() calls")
    # custom ids: the same lists under the labels
    ids = (np.random.default_rng(19).permutation(n) * 7 + 1000).astype(np.int64)
    cu = _import(kb, "IVF_FLAT", metric, C)
    cu.add(X, ids)
    cl = _lists(cu)
    assert (ibm.check_layout([i for i, _ in cl], ids, what="custom ids") == A).all()
    for (a, ca), (b, cb) in zip(cl, lists):
        assert np.array_equal(a, ids[b]) and np.array_equal(ca, cb)
    # add() after an import of the first 2500 rows' lists
    h = 2500
    part = kb.Index("IVF_FLAT", metric, d, {"nlist": nlist})
    imp = [(l, ids_l[ids_l < h], codes_l[ids_l < h]) for l, (ids_l, codes_l) in enumerate(lists)]
    part.ivf_import(C, None, imp)
    part.add(np.ascontiguousarray(X[h:]))
    _assert_same_lists(_lists(part), lists, "add() after ivf_import")


@functools.lru_cache(maxsize=None)
def _pq_quantizers(kb, m):
    ix = kb.Index("IVF_PQ", "L2", 192, {"nlist": 32, "m": m})
    ix.train(_clustered(8000, 192, 20))
    return ix.ivf_export_centroids(m)


@pytest.mark.parametrize("kind,m,refine", [
    ("IVF_FLAT", 0, None), ("IVF_PQ", 16, None), ("IVF_PQ", 48, "flat"), ("IVF_PQ", 64, "fp16"), ("IVF_PQ", 16, "bf16"),
    ("IVF_PQ", 64, "bf16")])
def test_add_after_search_equals_one_add(kb, kind, m, refine):
    """unseal() (unlayout_codes_kernel for both code layouts, the 16-bit refine store widened and narrowed again) then
    add(): the exported lists and the search results at nprobe = nlist equal one big add() bit for bit"""
    d, n = 192, 6000
    X = _clustered(n, d, 21)
    Q = _clustered(50, d, 22)
    if kind == "IVF_FLAT":
        C, pq = _trained_flat(kb, "L2", 8000, d, 32, 20), None
    else:
        C, pq = _pq_quantizers(kb, m)
    cfg = {"m": m} if m else {}
    if refine:
        cfg.update(refine=True, refine_type=refine)
    one = _import(kb, kind, "L2", C, pq, cfg)
    one.add(X)
    two = _import(kb, kind, "L2", C, pq, cfg)
    scfg = {"nprobe": 32, "refine_k": 2} if refine else {"nprobe": 32}
    for s in (slice(0, 2000), slice(2000, 2001), slice(2001, n)):
        two.add(np.ascontiguousarray(X[s]))
        two.search(Q, 10, scfg)
    ra, rb = one.search(Q, 10, scfg), two.search(Q, 10, scfg)
    _assert_same_lists(_lists(two, m), _lists(one, m), "add() after search")
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(_bits(ra[1]), _bits(rb[1]))


@pytest.mark.parametrize("kind,world", [("IVF_FLAT", 2), ("IVF_PQ", 3)])
def test_shard_lists_follow_the_owner_table(kb, kind, world):
    """set_shard on one GPU (no communicator): seal() gives each rank the lists of the greedy size-balanced owner table,
    and the shards' lists together are the unsharded index's"""
    d, n, m = 192, 6000, 16
    X = _clustered(n, d, 23)
    if kind == "IVF_FLAT":
        C, pq, cfg = _trained_flat(kb, "L2", 8000, d, 32, 20), None, {}
    else:
        (C, pq), cfg = _pq_quantizers(kb, m), {"m": m}
    full = _import(kb, kind, "L2", C, pq, cfg)
    full.add(X)
    fl = _lists(full, m)
    owner = ibm.owner_table([len(ids) for ids, _ in fl], world)
    seen = np.zeros(len(fl), np.int64)
    for r in range(world):
        sh = kb.Index(kind, "L2", d, dict(cfg, nlist=len(C)))
        sh.set_shard(r, world)
        Cc = np.ascontiguousarray(C, np.float32)
        kb._check(kb.lib().kb2_ivf_import_begin(sh.h, len(C), Cc.ctypes.data, None if pq is None else pq.ctypes.data))
        sh.add(X)
        for l, (ids, codes) in enumerate(_lists(sh, m)):
            if owner[l] == r:
                assert np.array_equal(ids, fl[l][0]) and np.array_equal(codes, fl[l][1]), f"rank {r} list {l}"
                seen[l] += 1
            else:
                assert len(ids) == 0, f"rank {r} holds list {l} of rank {owner[l]}"
    assert (seen == 1).all()


# ------------------------------------------------------------------------------------------------ f. typed ingest
@pytest.mark.parametrize("kind", ["IVF_FLAT", "IVF_PQ"])
@pytest.mark.parametrize("dtype", ["float16", "bfloat16", "int8"])
def test_typed_build_equals_widened_fp32(kb, kind, dtype):
    """kb2_index_train_typed / add_typed (widen_kernel, then the fp32 build): centroids, codebooks and lists equal the
    fp32 build of the widened values bit for bit"""
    n, d, nlist, m = 5000, 32, 32, 8
    X = _clustered(n, d, 24)
    if dtype == "int8":
        t = torch.from_numpy(np.clip(np.round(X * (127.0 / np.abs(X).max())), -127, 127).astype(np.int8))
    else:
        t = torch.from_numpy(X).to(getattr(torch, dtype))
    w = t.to(torch.float32).numpy()
    cfg = {"nlist": nlist, "m": m} if kind == "IVF_PQ" else {"nlist": nlist}
    mm = m if kind == "IVF_PQ" else 0
    a = kb.Index(kind, "L2", d, cfg)
    a.build(t)
    b = kb.Index(kind, "L2", d, cfg)
    b.build(w)
    (ca, pa), (cb, pb) = a.ivf_export_centroids(mm), b.ivf_export_centroids(mm)
    _assert_bits(ca, cb, "centroids")
    if mm:
        _assert_bits(pa, pb, "codebooks")
    _assert_same_lists(_lists(a, mm), _lists(b, mm), "lists")


# ------------------------------------------------------------------------------------------------ g. refusals
def test_refusals_leave_the_index_usable(kb):
    """IvfIndex::train / add and kmeans_train refuse by status; a refused train() leaves nlist as configured, so a later
    train() builds what a fresh index builds"""
    d, nlist, m = 32, 16, 8
    X = _clustered(3000, d, 25)

    def fresh(kind, cfg):
        ix = kb.Index(kind, "L2", d, cfg)
        ix.build(X)
        return ix

    pq_cfg = {"nlist": nlist, "m": m}
    want = fresh("IVF_PQ", pq_cfg)
    want_c = want.ivf_export_centroids(m)
    # n < 256 rows for nbits = 8, then the same index trained properly
    ix = kb.Index("IVF_PQ", "L2", d, pq_cfg)
    assert _status(lambda: ix.train(X[:200].copy())) == 1
    assert not ix.is_trained() and ix.ivf_nlist() == nlist
    ix.build(X)
    got_c = ix.ivf_export_centroids(m)
    _assert_bits(got_c[0], want_c[0], "centroids after a refused train")
    _assert_bits(got_c[1], want_c[1], "codebooks after a refused train")
    _assert_same_lists(_lists(ix, m), _lists(want, m), "lists after a refused train")
    # an empty training set, and add() before train()
    for kind, cfg, mm in (("IVF_FLAT", {"nlist": nlist}, 0), ("IVF_PQ", pq_cfg, m)):
        ref = want if kind == "IVF_PQ" else fresh(kind, cfg)
        ix = kb.Index(kind, "L2", d, cfg)
        assert _status(lambda: ix.train(np.zeros((0, d), np.float32))) == 1
        assert _status(lambda: ix.add(X[:10].copy())) == 8
        assert ix.count() == 0 and not ix.is_trained()
        ix.build(X)
        _assert_same_lists(_lists(ix, mm), _lists(ref, mm), f"{kind} after refusals")
    # dim % m != 0 at creation; nbits != 8 at train()
    assert _status(lambda: kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": 5})) == 1
    ix = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m, "nbits": 4})
    assert _status(lambda: ix.train(X)) == 7
    assert not ix.is_trained() and ix.ivf_nlist() == nlist
    assert _status(lambda: ix.add(X[:10].copy())) == 8
    # the hook: n < k, a metric other than L2 / IP
    assert _status(lambda: _hook(kb, X[:10], 16, "L2", 1)) == 1
    L = kb.lib()
    x = torch.from_numpy(X).cuda()
    out = torch.empty((16, d), dtype=torch.float32, device="cuda")
    assert L.kb2_debug_kmeans(x.data_ptr(), len(X), d, 16, 2, 1, 1234, out.data_ptr(), 0) == 5
    _assert_bits(_hook(kb, X, 16, "L2", 3), _hook(kb, X, 16, "L2", 3), "hook after refusals")
