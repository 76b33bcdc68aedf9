"""Emb-list (multi-vector) search on HNSW and IVF_FLAT indexes: the reference's TokenANN strategy (DESIGN §4.11).

Expected results come from a numpy restatement of TokenANN applied to the reference's own stage-1 search: each query
token's vec_topk = min(max(int32(fp32(k) * fp32(ratio)), 1), rows) hits, the distinct documents of a list's hits as its
candidates, their MaxSim scores in float64, the k best by (score, document id), padded with id -1 and -FLT_MAX (IP) or
FLT_MAX (L2).  HNSW runs on small-integer vectors, where every distance and every score is exact in fp32, so ids and
distance bits must be equal.  The re-rank is the BruteForce re-rank: with every document a candidate, the result is the
BruteForce emb-list result, ids and distance bits.
"""
import functools
import os
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from tests.test_emb_list_gpu import oracle  # noqa: E402  (float64 MaxSim scores and their bounds)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MAX = float(np.finfo(np.float32).max)
NAMES = {0: ("L2", "MAX_SIM_L2"), 1: ("IP", "MAX_SIM_IP")}


def _lims(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


def vec_topk(k, ratio, n):
    return int(min(max(int(np.float32(k) * np.float32(ratio)), 1), n))


def token_ann(I, xb, xl, xq, ql, k, metric, doc_valid=None):
    """TokenANN over stage-1 ids I [tokens, vec_topk]: (ids, dist) [n_lists, k] and the candidate count"""
    doc_of_row = np.repeat(np.arange(len(xl) - 1), np.diff(xl))
    n_lists = len(ql) - 1
    ids = np.full((n_lists, k), -1, np.int64)
    dist = np.full((n_lists, k), FLT_MAX if metric == 0 else -FLT_MAX, np.float32)
    ncand = 0
    for l in range(n_lists):
        hits = I[ql[l]:ql[l + 1]].ravel()
        cand = np.unique(doc_of_row[hits[hits >= 0]])
        if doc_valid is not None:
            assert doc_valid[cand].all(), "stage 1 returned a filtered row"
        ncand += cand.size
        if cand.size == 0:
            continue
        Q = xq[ql[l]:ql[l + 1]].astype(np.float64)
        sc = np.empty(cand.size)
        for i, c in enumerate(cand):
            X = xb[xl[c]:xl[c + 1]].astype(np.float64)
            if metric == 0:
                sc[i] = ((Q[:, None, :] - X[None, :, :]) ** 2).sum(-1).min(1).sum()
            else:
                sc[i] = (Q @ X.T).max(1).sum()
        order = np.lexsort((cand, sc if metric == 0 else -sc))[:k]
        ids[l, :order.size] = cand[order]
        dist[l, :order.size] = sc[order]
    return ids, dist, ncand


# ---------------------------------------------------------------- HNSW, bit-exact against the reference's stage 1
DOCS = 1000


@functools.lru_cache(maxsize=4)
def _int_corpus(metric, d):
    from oracle import ref
    rng = np.random.default_rng(5 + d + 100 * metric)
    xl = _lims(rng.integers(0, 41, DOCS))
    xb = rng.integers(0, 16, (int(xl[-1]), d)).astype(np.float32)
    qlen = np.concatenate([[0, 40, 33, 1, 0], rng.integers(0, 41, 15)])
    ql = _lims(qlen)
    xq = rng.integers(0, 16, (int(ql[-1]), d)).astype(np.float32)
    h = ref.RefHnsw(d, 16, metric, 100)
    h.add(xb)
    return xb, xl, xq, ql, h, h.export()


def _hnsw_index(kb, metric, d):
    xb, xl, xq, ql, h, g = _int_corpus(metric, d)
    ix = kb.Index("HNSW", NAMES[metric][0], d, {"M": 16, "efConstruction": 100})
    ix.hnsw_import(xb, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    ix.set_emb_list(xl, NAMES[metric][1])
    return ix


def _same(ids, dist, I0, D0):
    assert np.array_equal(ids, I0), f"ids differ in {np.argwhere(ids != I0)[:5].tolist()}"
    assert np.array_equal(dist.view(np.uint32), D0.view(np.uint32))


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("d", [32, 30])
@pytest.mark.parametrize("k", [1, 10, 100])
@pytest.mark.parametrize("ratio", [0.35, 1.0, 3.0])
def test_hnsw_bit_exact_against_reference(kb, ref, metric, d, k, ratio):
    xb, xl, xq, ql, h, _ = _int_corpus(metric, d)
    ix = _hnsw_index(kb, metric, d)
    ef = k + 20   # below vec_topk at ratio 3: the beam is max(ef, vec_topk)
    vt = vec_topk(k, ratio, len(xb))
    I, _, _ = h.search(xq, vt, max(ef, vt))
    I0, D0, ncand = token_ann(I, xb, xl, xq, ql, k, metric)
    ids, dist, st = ix.search_emb_list(xq, ql, k, {"ef": ef, "retrieval_ann_ratio": ratio}, stats=True)
    _same(ids, dist, I0, D0)
    assert st[0] == len(ql) - 1 and st[1] == ncand


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("ef", [21, 35])
def test_hnsw_plain_search_with_odd_ef(kb, ref, metric, ef):
    """stage 1 searches with ef = max(ef, vec_topk), often odd: the warp kernel's per-warp shared regions stay 16-byte
    aligned whatever ef is"""
    xb, xl, xq, ql, h, g = _int_corpus(metric, 32)
    ix = kb.Index("HNSW", NAMES[metric][0], 32, {"M": 16, "efConstruction": 100})
    ix.hnsw_import(xb, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    I0, D0, _ = h.search(xq, 10, ef)
    ids, dist = ix.search(xq, 10, {"ef": ef})
    _same(ids, dist, I0, D0)


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("frac", [0.2, 0.5, 0.9])
@pytest.mark.parametrize("d,k,ratio", [(32, 10, 3.0), (30, 100, 1.0)])
def test_hnsw_filtered_bit_exact_against_reference(kb, ref, metric, frac, d, k, ratio):
    xb, xl, xq, ql, h, _ = _int_corpus(metric, d)
    ix = _hnsw_index(kb, metric, d)
    doc_mask = np.random.default_rng(17).random(DOCS) < frac
    row_mask = np.repeat(doc_mask, np.diff(xl))
    ef = k + 20
    vt = vec_topk(k, ratio, len(xb))
    I, _, _ = h.search_filtered(xq, vt, max(ef, vt), np.packbits(row_mask, bitorder="little"), len(xb))
    I0, D0, _ = token_ann(I, xb, xl, xq, ql, k, metric, doc_valid=~doc_mask)
    cfg = {"ef": ef, "retrieval_ann_ratio": ratio, "disable_fallback_brute_force": True}
    ids, dist = ix.search_emb_list(xq, ql, k, cfg, bitset=np.packbits(doc_mask, bitorder="little"))
    assert not doc_mask[ids[ids >= 0]].any()
    _same(ids, dist, I0, D0)


# ---------------------------------------------------------------- IVF_FLAT against the same restatement of its own stage 1
@functools.lru_cache(maxsize=2)
def _ivf_corpus(metric):
    from oracle import ref
    rng = np.random.default_rng(31 + metric)
    d, nlist = 64, 32
    xl = _lims(rng.integers(1, 30, 600))
    xb = rng.standard_normal((int(xl[-1]), d)).astype(np.float32)
    ql = _lims(np.concatenate([[0, 12], rng.integers(1, 40, 10)]))
    xq = rng.standard_normal((int(ql[-1]), d)).astype(np.float32)
    r = ref.RefIvf("IVF_FLAT", d, metric, nlist)
    r.train(xb)
    r.add(xb)
    return xb, xl, xq, ql, r.centroids(), list(r.lists())


def _ivf(kb, metric):
    xb, xl, xq, ql, cent, lists = _ivf_corpus(metric)
    ix = kb.Index("IVF_FLAT", NAMES[metric][0], xb.shape[1], {"nlist": len(cent)})
    ix.ivf_import(cent, None, lists)
    return ix


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("nprobe", [4, 32])
def test_ivf_flat_matches_restatement(kb, ref, metric, nprobe):
    xb, xl, xq, ql, cent, _ = _ivf_corpus(metric)
    k, ratio = 10, 3.0
    plain = _ivf(kb, metric)
    I, _ = plain.search(xq, vec_topk(k, ratio, len(xb)), {"nprobe": nprobe})
    I0, D0, _ = token_ann(I, xb, xl, xq, ql, k, metric)
    ix = _ivf(kb, metric)
    ix.set_emb_list(xl, NAMES[metric][1])
    ids, dist = ix.search_emb_list(xq, ql, k, {"nprobe": nprobe, "retrieval_ann_ratio": ratio})
    assert np.array_equal(ids, I0)
    # each score within the float64 oracle's bound (test_emb_list_gpu.py)
    S, B = oracle(xb, xl, xq, ql, NAMES[metric][1])
    for l in range(len(ql) - 1):
        g = ids[l][ids[l] >= 0]
        err = np.abs(dist[l, :g.size].astype(np.float64) - S[l, g])
        assert (err <= B[l, g]).all(), f"list {l}: score error {err.max()} beyond the bound"


@pytest.mark.parametrize("metric", [0, 1])
def test_ivf_flat_exact_stage1_equals_bruteforce(kb, ref, metric):
    """nprobe = nlist and vec_topk = rows: every non-empty document is a candidate, and IVF_FLAT's rows, read through
    pos_of_row, give the BruteForce emb-list result: ids and score bits"""
    xb, xl, xq, ql, cent, _ = _ivf_corpus(metric)
    assert xl[-1] <= 16384
    ix = _ivf(kb, metric)
    ix.set_emb_list(xl, NAMES[metric][1])
    k = 20
    ids, dist = ix.search_emb_list(xq, ql, k, {"nprobe": len(cent), "retrieval_ann_ratio": 1e6})
    bi, bd = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, NAMES[metric][1])
    v = ids >= 0
    assert np.array_equal(v, bi >= 0)
    assert np.array_equal(ids[v], bi[v])
    assert np.array_equal(dist[v].view(np.uint32), bd[v].view(np.uint32))


@pytest.mark.parametrize("metric,chunks", [(0, 1), (1, 1), (0, 2), (1, 2)], ids=["0", "1", "0-2chunks", "1-2chunks"])
def test_exact_branch_equals_bruteforce(kb, metric, chunks):
    """vec_topk = rows: HNSW takes its exact branch and every non-empty document is a candidate, so the result is the
    BruteForce emb-list result, ids and score bits"""
    rng = np.random.default_rng(7 + metric)
    d = 64
    xl = _lims(np.concatenate([[0, 3], rng.integers(0, 40, 500)]))
    xb = rng.standard_normal((int(xl[-1]), d)).astype(np.float32)
    assert xl[-1] <= 16384
    # chunks = 2: 32 + 5 + 0 + 150 + 24 * 40 = 1147 tokens x vec_topk = rows (10 089 at L2, 9 923 at IP) make 11.4 to 11.6 M
    # stage-1 entries, above the 8 M (2^23) of one chunk: a chunk takes at most 845 of the tokens, so two chunks
    ql = _lims([32, 5, 0, 150] + [40] * 24 * (chunks - 1))
    assert chunks == 1 or ql[-1] * xl[-1] > 8 << 20
    xq = rng.standard_normal((int(ql[-1]), d)).astype(np.float32)
    ix = kb.Index("HNSW", NAMES[metric][0], d, {"M": 16, "efConstruction": 64})
    ix.add(xb)
    ix.set_emb_list(xl, NAMES[metric][1])
    k = 20
    ids, dist = ix.search_emb_list(xq, ql, k, {"retrieval_ann_ratio": 1e6})
    bi, bd = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, NAMES[metric][1])
    v = ids >= 0
    assert np.array_equal(v, bi >= 0)
    assert np.array_equal(ids[v], bi[v])
    assert np.array_equal(dist[v].view(np.uint32), bd[v].view(np.uint32))
    assert (ids[2] == -1).all()   # empty query list


def test_cosine_within_bound_of_bruteforce(kb):
    rng = np.random.default_rng(3)
    d = 48
    xl = _lims(rng.integers(1, 30, 300))
    xb = rng.standard_normal((int(xl[-1]), d)).astype(np.float32)
    ql = _lims([10, 20, 3])
    xq = rng.standard_normal((int(ql[-1]), d)).astype(np.float32)
    ix = kb.Index("HNSW", "COSINE", d, {"M": 16, "efConstruction": 64})
    ix.add(xb)
    ix.set_emb_list(xl, "MAX_SIM_COSINE")
    ids, dist = ix.search_emb_list(xq, ql, 10, {"retrieval_ann_ratio": 1e6})
    bi, bd = kb.brute_force_search_emb_list(xb, xl, xq, ql, 10, "MAX_SIM_COSINE")
    assert (ids == bi).mean() > 0.95
    np.testing.assert_allclose(dist, bd, rtol=1e-5, atol=1e-4 * 20)


# ---------------------------------------------------------------- contract
def test_filtering_padding_and_large_k(kb, ref):
    xb, xl, xq, ql, _, _ = _int_corpus(0, 32)
    ix = _hnsw_index(kb, 0, 32)
    all_bits = np.packbits(np.ones(DOCS, bool), bitorder="little")
    ids, dist = ix.search_emb_list(xq, ql, 5, bitset=all_bits)
    assert (ids == -1).all() and (dist == np.float32(FLT_MAX)).all()
    mask = np.random.default_rng(1).random(DOCS) < 0.5
    ids, _ = ix.search_emb_list(xq, ql, 50, {"ef": 60}, bitset=np.packbits(mask, bitorder="little"))
    assert not mask[ids[ids >= 0]].any()
    # more k than candidates: the row pads
    ids, dist, st = ix.search_emb_list(xq, ql, 500, {"ef": 500, "retrieval_ann_ratio": 0.01}, stats=True)
    assert (ids[:, -1] == -1).all() and (ids[1, 0] >= 0)
    # k = 16384: vec_topk = 16384 is at least half the ~20k rows, so stage 1 takes HNSW's exact branch; k exceeds the
    # candidates, so every candidate comes back, each with its exact score (integer data: float64 is exact)
    ids, dist, st = ix.search_emb_list(xq[:ql[2]], ql[:3], 16384, {"ef": 16384, "retrieval_ann_ratio": 1.0}, stats=True)
    assert (ids[0] == -1).all()   # list 0 is empty
    g = ids[1][ids[1] >= 0]
    assert g.size == st[1] > 0 and np.unique(g).size == g.size and (ids[1, g.size:] == -1).all()
    Q = xq[ql[1]:ql[2]].astype(np.float64)
    sc = np.array([((Q[:, None, :] - xb[xl[c]:xl[c + 1]][None].astype(np.float64)) ** 2).sum(-1).min(1).sum() for c in g])
    assert np.array_equal(dist[1, :g.size], sc.astype(np.float32))
    assert (np.diff(sc) >= 0).all()


def test_deterministic_host_device_and_serialize(kb, ref):
    xb, xl, xq, ql, _, _ = _int_corpus(1, 32)
    ix = _hnsw_index(kb, 1, 32)
    cfg = {"ef": 64, "retrieval_ann_ratio": 2.0}
    i1, d1 = ix.search_emb_list(xq, ql, 10, cfg)
    i2, d2 = ix.search_emb_list(xq, ql, 10, cfg)
    assert np.array_equal(i1, i2) and np.array_equal(d1.view(np.uint32), d2.view(np.uint32))
    i3, d3 = ix.search_emb_list(torch.as_tensor(xq, device="cuda"), torch.as_tensor(ql, device="cuda"), 10, cfg)
    assert np.array_equal(i1, i3.cpu().numpy()) and np.array_equal(d1.view(np.uint32), d3.cpu().numpy().view(np.uint32))
    ix2 = kb.Index.deserialize(ix.serialize())
    assert np.array_equal(ix2.emb_list_offsets(), xl)
    i4, d4 = ix2.search_emb_list(xq, ql, 10, cfg)
    assert np.array_equal(i1, i4) and np.array_equal(d1.view(np.uint32), d4.view(np.uint32))
    # an IVF_FLAT blob without the section still loads as a plain index
    xb2, xl2, xq2, ql2, _, _ = _ivf_corpus(0)
    plain = _ivf(kb, 0)
    again = kb.Index.deserialize(plain.serialize())
    with pytest.raises(kb.KnowhereError):
        again.emb_list_offsets()
    again.set_emb_list(xl2, "MAX_SIM_L2")
    a, _ = again.search_emb_list(xq2, ql2, 5, {"nprobe": 8})
    b, _ = kb.Index.deserialize(again.serialize()).search_emb_list(xq2, ql2, 5, {"nprobe": 8})
    assert np.array_equal(a, b)


def test_error_statuses(kb, ref):
    xb, xl, xq, ql, _, _ = _int_corpus(0, 32)
    d = 32

    def status(f):
        with pytest.raises(kb.KnowhereError) as e:
            f()
        return e.value.status

    ix = kb.Index("HNSW", "L2", d, {"M": 16})
    ix.add(xb)
    assert status(lambda: ix.set_emb_list(xl, "MAX_SIM_IP")) == 5
    assert status(lambda: ix.set_emb_list(xl, "MAX_SIM_COSINE")) == 5
    bad = xl.copy()
    bad[-1] += 1
    assert status(lambda: ix.set_emb_list(bad, "MAX_SIM_L2")) == 1
    bad = xl.copy()
    bad[3], bad[4] = bad[4] + 1, bad[3]
    assert status(lambda: ix.set_emb_list(bad, "MAX_SIM_L2")) == 1
    assert status(lambda: ix.search_emb_list(xq, ql, 5)) == 31   # no offsets attached
    flat = kb.Index("FLAT", "L2", d)
    flat.add(xb)
    assert status(lambda: flat.set_emb_list(xl, "MAX_SIM_L2")) == 5
    ix.set_emb_list(xl, "MAX_SIM_L2")
    assert status(lambda: ix.add(xb[:10])) == 7
    assert status(lambda: ix.search(xq, 5)) == 31
    assert status(lambda: ix.range_search(xq, 1.0)) == 31
    assert status(lambda: ix.search_emb_list(xq, ql, 5, {"retrieval_ann_ratio": 0})) == 31
    assert status(lambda: ix.search_emb_list(xq, ql, 5, {"ef": 4})) == 3
    assert status(lambda: ix.search_emb_list(xq, ql, 5, bitset=np.zeros(DOCS // 8 - 4, np.uint8))) == 1
    assert status(lambda: ix.search_emb_list(xq, ql, 0)) == 1
    # the rows cannot change under the offsets: graph and list imports are refused like add
    g = _int_corpus(0, 32)[5]
    assert status(lambda: ix.hnsw_import(xb[:100], g["levels"][:100], g["offsets"][:101], g["neighbors"], g["cum"],
                                         0, 0)) == 7
    ids, _ = ix.search_emb_list(xq, ql, 5, {"ef": 16})   # the handle still searches its own rows
    assert (ids[1] >= 0).all()
    xb2, xl2, _, _, cent, lists = _ivf_corpus(0)
    iv = _ivf(kb, 0)
    iv.set_emb_list(xl2, "MAX_SIM_L2")
    assert status(lambda: iv.ivf_import(cent, None, lists)) == 7


def test_ivf_pq_rejected(kb):
    rng = np.random.default_rng(0)
    x = rng.standard_normal((3000, 32)).astype(np.float32)
    ix = kb.Index("IVF_PQ", "L2", 32, {"nlist": 16, "m": 8, "nbits": 8})
    ix.build(x)
    with pytest.raises(kb.KnowhereError) as e:
        ix.set_emb_list(_lims([1000, 2000]), "MAX_SIM_L2")
    assert e.value.status == 5


def test_cpp_mirror(tmp_path):
    """B200IndexNode Build / Search / Serialize / Deserialize with emb-lists (tests/cpp/test_emb_list_index.cc)."""
    exe = tmp_path / "test_emb_list_index"
    subprocess.run(["g++", "-std=c++17", "-O2", f"-I{ROOT}/include", os.path.join(ROOT, "tests", "cpp", "test_emb_list_index.cc"),
                    "-o", str(exe), f"-L{ROOT}/knowhere_b200", "-l:libknowhere_b200.so",
                    f"-Wl,-rpath,{ROOT}/knowhere_b200"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ok")
