"""Emb-list search with the MUVERA strategy on HNSW and IVF_FLAT (DESIGN §4.11).

The encoder is held to the numpy model of tests/muvera_model.py: the projections to the C++ standard library's draws, and
the encodings bit for bit wherever no token of the item lies within fp32 rounding of a hyperplane.  The search is held
to the definition: with an exact stage 1 (IVF_FLAT probing every list, HNSW with ef >= n_docs) the candidates are the
ann_k documents whose encodings score best (ties within the fp32 bound), and the result is the BruteForce MaxSim result
(kb2_bruteforce_search_emb_list) restricted to those candidates, ids and distance bits.
"""
import os
import subprocess

import numpy as np
import pytest

from tests import muvera_model as mm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EL = {"L2": "MAX_SIM_L2", "IP": "MAX_SIM_IP", "COSINE": "MAX_SIM_COSINE"}
FLT_MAX = float(np.finfo(np.float32).max)


def _lims(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


def corpus(seed, n_docs, d, nq=24, maxlen=16):
    """clustered token rows: documents of one topic each (document 3 empty, 5 of one token); query lists are noisy
    tokens of one document"""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((16, d)).astype(np.float32)
    lens = rng.integers(1, maxlen, n_docs)
    lens[3], lens[5] = 0, 1
    xl = _lims(lens)
    topic = rng.integers(0, 16, n_docs)
    xb = (centers[np.repeat(topic, lens)] + 0.7 * rng.standard_normal((int(xl[-1]), d))).astype(np.float32)
    qlens = rng.integers(1, 12, nq)
    ql = _lims(qlens)
    src = rng.choice(np.flatnonzero(lens > 0), nq)
    rows = np.concatenate([rng.integers(xl[s], xl[s + 1], n) for s, n in zip(src, qlens)])
    xq = (xb[rows] + 0.3 * rng.standard_normal((len(rows), d))).astype(np.float32)
    return xb, xl, xq, ql


def muvera_index(kb, typ, metric, xb, xl, P=4, R=7, S=42, **build):
    cfg = {"emb_list_strategy": "muvera", "muvera_num_projections": P, "muvera_num_repeats": R, "muvera_seed": S}
    cfg.update(build)
    ix = kb.Index(typ, metric, xb.shape[1], cfg)
    ix.train(xb)
    ix.add(xb)
    ix.set_emb_list(xl, EL[metric])
    return ix


def bf_scores(kb, xb, xl, xq, ql, metric):
    """[n_lists] dicts document -> BruteForce MaxSim distance (every document with rows)"""
    n_docs = len(xl) - 1
    ids, dist = kb.brute_force_search_emb_list(xb, xl, xq, ql, n_docs, EL[metric])
    return [{int(i): v for i, v in zip(ids[l], dist[l]) if i >= 0} for l in range(len(ql) - 1)]


def expected_from_candidates(scores, cands, k, metric):
    """the k best of the candidates by (BruteForce distance, id), padded as the emb-list search pads"""
    ids = np.full(k, -1, np.int64)
    dist = np.full(k, FLT_MAX if metric == "L2" else -FLT_MAX, np.float32)
    c = sorted((int(x) for x in cands if int(x) in scores), key=lambda i: (scores[i] if metric == "L2" else -scores[i], i))[:k]
    ids[:len(c)] = c
    dist[:len(c)] = [scores[i] for i in c]
    return ids, dist


def fde_scores(kb, xb, xl, xq, ql, P, R, S, metric):
    """float64 scores (larger is better) of every (query list, document) pair from the device encodings, and their
    fp32 summation bounds"""
    _, D = kb.debug_muvera_encode(xb, xl, P, R, S, mean=True)
    _, Q = kb.debug_muvera_encode(xq, ql, P, R, S, mean=False)
    D, Q = D.astype(np.float64), Q.astype(np.float64)
    E = D.shape[1]
    g = 2 * E * 2.0 ** -24
    if metric == "COSINE":
        D = D / np.maximum(np.linalg.norm(D, axis=1, keepdims=True), 1e-30)
        Q = Q / np.maximum(np.linalg.norm(Q, axis=1, keepdims=True), 1e-30)
    if metric == "L2":
        s = -((Q[:, None, :] - D[None, :, :]) ** 2).sum(-1)
        b = np.broadcast_to(g * ((np.abs(Q) + np.abs(D).max(0)) ** 2).sum(-1)[:, None] + 1e-6, s.shape)
    else:
        s = Q @ D.T
        b = g * (np.abs(Q) @ np.abs(D).T) + 1e-6
    return s, b


def check_candidates(got, s, b, ann):
    """got: a list's stage-1 documents; s / b: that list's scores and bounds over all documents"""
    got = got[got >= 0]
    assert len(got) == ann and len(set(got.tolist())) == ann, got
    kth = np.sort(s)[::-1][ann - 1]
    assert (s[got] >= kth - 2 * b[got]).all(), "a candidate scores below the ann_k-th best by more than the bound"
    must = np.flatnonzero(s > kth + 2 * b)
    assert set(must.tolist()) <= set(got.tolist()), "a document scoring above the ann_k-th best is missing"


# ---------------------------------------------------------------- the encoder
@pytest.mark.parametrize("P,R,d", [(4, 7, 128), (3, 5, 30), (7, 2, 20), (1, 1, 8), (3, 2, 200)])
def test_encoder_matches_the_model(kb, P, R, d):
    xb, xl, xq, ql = corpus(11 + d, 200, d)
    proj, D = kb.debug_muvera_encode(xb, xl, P, R, 42, mean=True)
    assert np.array_equal(proj, mm.projections(P, R, d, 42)), "projections differ from std::normal_distribution draws"
    _, Q = kb.debug_muvera_encode(xq, ql, P, R, 42, mean=False)
    for x, lims, got, mean in ((xb, xl, D, True), (xq, ql, Q, False)):
        want, amb = mm.encode(x, lims, proj, mean)
        assert amb.sum() <= 3, f"{amb.sum()} ambiguous tokens: the data should have a handful at most"
        bad_items = {int(np.searchsorted(lims, t, side="right")) - 1 for t in np.flatnonzero(amb)}
        for i in range(len(lims) - 1):
            if i not in bad_items:
                assert np.array_equal(got[i].view(np.uint32), want[i].view(np.uint32)), f"item {i} differs (mean={mean})"
    assert not D[3].any(), "an empty document encodes to zeros"


# ---------------------------------------------------------------- end to end, exact stage 1
EXACT = [(m, t, 1) for m in ("L2", "IP", "COSINE") for t in ("IVF_FLAT", "HNSW")] + [("IP", "IVF_FLAT", 2),
                                                                                     ("COSINE", "IVF_FLAT", 2)]


@pytest.mark.parametrize("metric,typ,chunks", EXACT, ids=[f"{m}-{t}" + ("-2chunks" if c > 1 else "") for m, t, c in EXACT])
def test_exact_stage1_then_bruteforce_rerank(kb, metric, typ, chunks):
    P, R, S, n_docs, k, ratio, d, nq = 3, 5, 7, 300, 10, 3.0, 32, 24
    if chunks > 1:
        # E = R * 2^P * d = 8 * 32 * 64 = 16 384 floats per encoded list: a chunk takes at most 16 M (2^24) / 16 384 =
        # 1 024 lists, so 1 100 lists span two chunks
        P, R, d, nq = 5, 8, 64, 1100
    xb, xl, xq, ql = corpus(21, n_docs, d, nq=nq)
    build = {"nlist": 4} if typ == "IVF_FLAT" else {"M": 16, "efConstruction": 200}
    ix = muvera_index(kb, typ, metric, xb, xl, P, R, S, **build)
    search = {"nprobe": 4} if typ == "IVF_FLAT" else {"ef": 512}
    ann = mm.ann_k(k, ratio, n_docs)
    cand, _ = ix.search_emb_list(xq, ql, ann, dict(search, emb_list_rerank=False))
    s, b = fde_scores(kb, xb, xl, xq, ql, P, R, S, metric)
    scores = bf_scores(kb, xb, xl, xq, ql, metric)
    ids, dist, st = ix.search_emb_list(xq, ql, k, dict(search, retrieval_ann_ratio=ratio), stats=True)
    n_cand = 0
    for l in range(len(ql) - 1):
        check_candidates(cand[l], s[l], b[l], ann)
        I0, D0 = expected_from_candidates(scores[l], cand[l], k, metric)
        n_cand += int(sum(1 for c in cand[l] if c >= 0 and xl[c + 1] > xl[c]))
        assert np.array_equal(ids[l], I0), (l, ids[l], I0)
        assert np.array_equal(dist[l].view(np.uint32), D0.view(np.uint32)), (l, dist[l], D0)
    assert st[0] == len(ql) - 1 and st[1] == n_cand


# ---------------------------------------------------------------- recall on the reference test's grid
# measured on an H100 80GB HBM3 (700 W), ratio 3, filter rates 0 / 0.5 / 0.9: (3, 5) IVF_FLAT 0.542 / 0.750 / 0.983, HNSW
# 0.541 / 0.744 / 0.939; (4, 3) IVF_FLAT 0.508 / 0.723 / 0.977, HNSW 0.508 / 0.725 / 0.973.  The floors leave a margin.
RECALL_FLOOR = {(3, 5): {0.0: 0.50, 0.5: 0.70, 0.9: 0.90}, (4, 3): {0.0: 0.47, 0.5: 0.68, 0.9: 0.90}}


@pytest.mark.parametrize("P,R", [(3, 5), (4, 3)])
@pytest.mark.parametrize("typ", ["IVF_FLAT", "HNSW"])
def test_recall_against_bruteforce(kb, P, R, typ):
    n_docs, k = 2000, 10
    xb, xl, xq, ql = corpus(31, n_docs, 32, nq=64)
    build = {"nlist": 16} if typ == "IVF_FLAT" else {"M": 16, "efConstruction": 200}
    ix = muvera_index(kb, typ, "IP", xb, xl, P, R, **build)
    search = {"nprobe": 8} if typ == "IVF_FLAT" else {"ef": 64}
    rng = np.random.default_rng(4)
    got = {}
    for rate in (0.0, 0.5, 0.9):
        filt = rng.random(n_docs) < rate
        bits = np.packbits(filt.astype(np.uint8), bitorder="little")
        gt, _ = kb.brute_force_search_emb_list(xb, xl, xq, ql, k, "MAX_SIM_IP", bitset=bits if rate else None)
        ids, _ = ix.search_emb_list(xq, ql, k, dict(search, retrieval_ann_ratio=3), bitset=bits if rate else None)
        assert not filt[ids[ids >= 0]].any(), "a filtered document was returned"
        hits = sum(len(set(ids[l][ids[l] >= 0]) & set(gt[l][gt[l] >= 0])) for l in range(len(ql) - 1))
        recall = hits / max(1, int((gt >= 0).sum()))
        print(f"MUVERA {typ} P={P} R={R} filter={rate}: recall@10 {recall:.3f}")
        got[rate] = recall
    for rate, recall in got.items():
        assert recall >= RECALL_FLOOR[(P, R)][rate], (typ, P, R, rate, recall)


# ---------------------------------------------------------------- the defaults: E = 7 * 16 * 128 = 14336
def test_defaults_at_d128_on_ivf_flat(kb):
    n_docs, k = 600, 5
    xb, xl, xq, ql = corpus(41, n_docs, 128, nq=16)
    ix = kb.Index("IVF_FLAT", "IP", 128, {"emb_list_strategy": "muvera", "nlist": 8})
    ix.add(xb)
    ix.set_emb_list(xl, "MAX_SIM_IP")
    meta = ix.meta()
    assert meta["emb_list_strategy"] == "muvera" and meta["muvera_encoded_dim"] == 14336
    assert (meta["muvera_num_projections"], meta["muvera_num_repeats"], meta["muvera_seed"]) == (4, 7, 42)
    assert meta["rows"] == xl[-1] == ix.count()
    cand, _ = ix.search_emb_list(xq, ql, 15, {"nprobe": 8, "emb_list_rerank": False})
    s, b = fde_scores(kb, xb, xl, xq, ql, 4, 7, 42, "IP")
    scores = bf_scores(kb, xb, xl, xq, ql, "IP")
    ids, dist = ix.search_emb_list(xq, ql, k, {"nprobe": 8})
    for l in range(len(ql) - 1):
        check_candidates(cand[l], s[l], b[l], 15)
        I0, D0 = expected_from_candidates(scores[l], cand[l], k, "IP")
        assert np.array_equal(ids[l], I0) and np.array_equal(dist[l].view(np.uint32), D0.view(np.uint32))


# ---------------------------------------------------------------- without re-rank: the base search as it is
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_without_rerank_is_the_base_search(kb, metric):
    P, R, S, n_docs = 3, 4, 5, 50
    xb, xl, xq, ql = corpus(51, n_docs, 16)
    ix = muvera_index(kb, "IVF_FLAT", metric, xb, xl, P, R, S, nlist=2)
    _, D = kb.debug_muvera_encode(xb, xl, P, R, S, mean=True)
    _, Q = kb.debug_muvera_encode(xq, ql, P, R, S, mean=False)
    base = kb.Index("IVF_FLAT", metric, D.shape[1], {"nlist": 2})
    base.train(D)
    base.add(D)
    k = 64   # > n_docs: ann_k = n_docs, then padding
    I0, D0 = base.search(Q, n_docs, {"nprobe": 2})
    ids, dist = ix.search_emb_list(xq, ql, k, {"nprobe": 2, "emb_list_rerank": False})
    assert np.array_equal(ids[:, :n_docs], I0)
    assert np.array_equal(dist[:, :n_docs].view(np.uint32), D0.view(np.uint32))
    assert (ids[:, n_docs:] == -1).all()
    assert (dist[:, n_docs:] == (np.inf if metric == "L2" else -np.inf)).all()


# ---------------------------------------------------------------- edge cases
def test_edge_cases(kb):
    n_docs = 40
    xb, xl, xq, ql = corpus(61, n_docs, 16, nq=6)
    ix = muvera_index(kb, "HNSW", "L2", xb, xl, 3, 3, M=8, efConstruction=64)
    scores = bf_scores(kb, xb, xl, xq, ql, "L2")
    # k > n_docs: every document with rows, best first, then padding
    ids, dist = ix.search_emb_list(xq, ql, 50, {"ef": 64, "retrieval_ann_ratio": 3})
    for l in range(len(ql) - 1):
        I0, D0 = expected_from_candidates(scores[l], np.arange(n_docs), 50, "L2")
        assert np.array_equal(ids[l], I0) and np.array_equal(dist[l].view(np.uint32), D0.view(np.uint32))
    # an empty query list: a whole row of padding
    ql2 = np.array([0, 0, int(ql[1])], np.int64)
    ids, dist = ix.search_emb_list(xq[:ql[1]], ql2, 5, {"ef": 64})
    assert (ids[0] == -1).all() and (dist[0] == FLT_MAX).all() and (ids[1] >= 0).all()
    # every document filtered out
    bits = np.full((n_docs + 7) // 8, 0xFF, np.uint8)
    ids, dist = ix.search_emb_list(xq, ql, 5, {"ef": 64}, bitset=bits)
    assert (ids == -1).all() and (dist == FLT_MAX).all()
    # no query list
    ids, _ = ix.search_emb_list(xq[:0], np.zeros(1, np.int64), 5, {"ef": 64})
    assert ids.shape == (0, 5)


# ---------------------------------------------------------------- persistence
@pytest.mark.parametrize("typ,metric", [("HNSW", "IP"), ("IVF_FLAT", "COSINE")])
def test_serialize_round_trip(kb, typ, metric):
    xb, xl, xq, ql = corpus(71, 120, 24)
    build = {"nlist": 4} if typ == "IVF_FLAT" else {"M": 16, "efConstruction": 100}
    ix = muvera_index(kb, typ, metric, xb, xl, 3, 4, 9, **build)
    cfg = {"nprobe": 2} if typ == "IVF_FLAT" else {"ef": 32}
    a = ix.search_emb_list(xq, ql, 7, cfg)
    ix2 = kb.Index.deserialize(ix.serialize())
    b = ix2.search_emb_list(xq, ql, 7, cfg)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
    assert ix2.meta()["muvera_encoded_dim"] == 4 * 8 * 24 and ix2.count() == xl[-1]
    assert np.array_equal(ix2.emb_list_offsets(), xl)


# ---------------------------------------------------------------- refusals
def _status(kb, f):
    with pytest.raises(kb.KnowhereError) as e:
        f()
    return e.value.status


def test_refusals(kb):
    xb, xl, xq, ql = corpus(81, 30, 8, nq=3)
    mv = {"emb_list_strategy": "muvera"}
    assert _status(kb, lambda: kb.Index("HNSW", "L2", 8, {"emb_list_strategy": "lemur"})) == 7
    assert _status(kb, lambda: kb.Index("HNSW", "L2", 8, {"emb_list_strategy": "colbert"})) == 1
    # an empty strategy is TokenANN; types without emb-lists do not read the strategy keys
    assert "emb_list_strategy" not in kb.Index("IVF_FLAT", "L2", 8, {"emb_list_strategy": ""}).meta()
    for typ in ("FLAT", "GPU_CAGRA"):
        kb.Index(typ, "L2", 8, {"emb_list_strategy": "lemur", "muvera_num_repeats": 99})
    for key, bad in (("muvera_num_projections", 0), ("muvera_num_projections", 8), ("muvera_num_repeats", 0),
                     ("muvera_num_repeats", 33), ("muvera_seed", 2 ** 31)):
        assert _status(kb, lambda: kb.Index("IVF_FLAT", "L2", 8, dict(mv, **{key: bad}))) == 3, key
    # FLAT and IVF_PQ: refused at the attach, as for TokenANN
    for typ, extra in (("FLAT", {}), ("IVF_PQ", {"m": 2, "nlist": 2})):
        ix = kb.Index(typ, "L2", 8, dict(mv, **extra))
        ix.train(np.tile(xb, (10, 1)))
        ix.add(xb)
        assert _status(kb, lambda: ix.set_emb_list(xl, "MAX_SIM_L2")) == 5, typ
    # custom ids and a sharded handle: KB2_NOT_IMPLEMENTED at the attach
    ix = kb.Index("HNSW", "L2", 8, mv)
    ix.add(xb, ids=np.arange(len(xb), dtype=np.int64) + 100)
    assert _status(kb, lambda: ix.set_emb_list(xl, "MAX_SIM_L2")) == 7
    ix = kb.Index("IVF_FLAT", "L2", 8, dict(mv, nlist=2))
    ix.set_shard(0, 2)
    ix.add(xb)
    assert _status(kb, lambda: ix.set_emb_list(xl, "MAX_SIM_L2")) == 7
    # metric pairing, offsets
    ix = kb.Index("HNSW", "L2", 8, mv)
    ix.add(xb)
    assert _status(kb, lambda: ix.set_emb_list(xl, "MAX_SIM_IP")) == 5
    assert _status(kb, lambda: ix.set_emb_list(xl[:-1], "MAX_SIM_L2")) == 1
    # before the attach: no plain or emb-list search, no serialisation
    assert _status(kb, lambda: ix.search(xq, 3)) == 31
    assert _status(kb, lambda: ix.range_search(xq, 1.0)) == 31
    assert _status(kb, lambda: ix.search_emb_list(xq, ql, 3)) == 31
    assert _status(kb, lambda: ix.serialize()) == 1
    ix.set_emb_list(xl, "MAX_SIM_L2")
    # the documents are attached once, also on a deserialised handle
    assert _status(kb, lambda: ix.set_emb_list(xl, "MAX_SIM_L2")) == 7
    assert _status(kb, lambda: kb.Index.deserialize(ix.serialize()).set_emb_list(xl, "MAX_SIM_L2")) == 7
    # after the attach: as TokenANN
    assert _status(kb, lambda: ix.search(xq, 3)) == 31
    assert _status(kb, lambda: ix.range_search(xq, 1.0)) == 31
    assert _status(kb, lambda: ix.add(xb)) == 7
    assert _status(kb, lambda: ix.train(xb)) == 7
    assert _status(kb, lambda: ix.hnsw_export()) == 7
    assert _status(kb, lambda: ix.serialize_faiss()) == 7
    assert _status(kb, lambda: ix.search_emb_list(xq, ql, 3, {"retrieval_ann_ratio": 0})) == 31
    assert _status(kb, lambda: ix.search_emb_list(xq, ql, 3, {"ef": 2})) == 3


# ---------------------------------------------------------------- the C++ mirror
def test_cpp_build_search_serialize(tmp_path):
    exe = tmp_path / "test_emb_list_muvera"
    subprocess.run(["g++", "-std=c++17", "-O2", f"-I{ROOT}/include", os.path.join(ROOT, "tests", "cpp", "test_emb_list_muvera.cc"),
                    "-o", str(exe), f"-L{ROOT}/knowhere_b200", "-l:libknowhere_b200.so",
                    f"-Wl,-rpath,{ROOT}/knowhere_b200"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "muvera ok" in r.stdout
