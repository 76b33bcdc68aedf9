"""SPARSE_INVERTED_INDEX / SPARSE_WAND and the sparse BruteForce on the GPU, held bit for bit (ids and distance bits) to
the numpy model of the definition (tests/sparse_model.py, DESIGN §4.13)."""
import os

import numpy as np
import pytest

from knowhere_b200 import datagen
from tests import sparse_model as sm
from tests.util import assert_topk_parity

pytestmark = pytest.mark.gpu

TILE = 16384
K1, B = 1.2, 0.75


def _near_2_32(csr, vocab=30522):
    # an increasing map of the term ids onto [2^32 - 3 * vocab, 2^32): row order is kept, the largest id is 2^32 - 1
    ip, ix, val = csr
    return ip, (np.uint64(0xFFFFFFFF) - np.uint64(3) * (np.uint64(vocab - 1) - ix.astype(np.uint64))).astype(np.uint32), val


def _with_edge_queries(q, absent):
    """q plus an empty query and a query whose terms no row holds"""
    qp, qi, qv = q
    return (np.concatenate([qp, [qp[-1], qp[-1] + len(absent)]]).astype(np.int64),
            np.concatenate([qi, np.asarray(absent, np.uint32)]), np.concatenate([qv, np.ones(len(absent), np.float32)]))


def _data(vocab, n, seed):
    base = datagen.sparse_splade(n, 24, seed)
    queries = datagen.sparse_splade(14, 12, seed + 100)
    absent = [30522, 40000]
    if vocab == "hashed":
        base, queries = _near_2_32(base), _near_2_32(queries)
        absent = [5, 7]
    return base, _with_edge_queries(queries, absent)


def _bitset(n, frac, seed):
    rng = np.random.default_rng(seed)
    return np.packbits(rng.random(n) < frac, bitorder="little")


def _build_cfg(metric, base):
    if metric == "IP":
        return {}
    ip, _, val = base
    return {"bm25_k1": K1, "bm25_b": B, "bm25_avgdl": float(val.sum(dtype=np.float64) / (ip.size - 1))}


def _same_bits(got, want, what):
    ids, dist = got
    mi, md = want
    assert np.array_equal(ids, mi), f"{what}: ids differ"
    assert np.array_equal(np.asarray(dist, np.float32).view(np.uint32), md.view(np.uint32)), f"{what}: distance bits differ"


@pytest.mark.parametrize("vocab", ["splade", "hashed"])
@pytest.mark.parametrize("n", [3000, TILE, 3 * TILE + 777])
@pytest.mark.parametrize("metric", ["IP", "BM25"])
@pytest.mark.parametrize("itype", ["SPARSE_INVERTED_INDEX", "SPARSE_WAND"])
def test_search_matches_model_bit_for_bit(kb, itype, metric, n, vocab):
    base, queries = _data(vocab, n, seed=n % 97 + (vocab == "hashed"))
    cfg = _build_cfg(metric, base)
    ix = kb.Index(itype, metric, 0, cfg)
    ix.add_sparse(base)
    post = sm.Postings(base)
    bm25 = (K1, B, cfg["bm25_avgdl"]) if metric == "BM25" else None
    cases = [(10, 0.0, None), (10, 0.3, None), (10, 0.9, None), (10, 0.0, 0.5), (10, 0.0, 0.99), (1, 0.0, None),
             (1008, 0.0, 0.5), (1009, 0.0, None)]
    if n == 3 * TILE + 777:
        cases += [(4096, 0.3, 0.5), (16384, 0.0, None)]
    for k, ratio, frac in cases:
        bits = None if frac is None else _bitset(n, frac, k)
        got = ix.search_sparse(queries, k, dict(cfg, drop_ratio_search=ratio), bitset=bits)
        want = sm.search(base, queries, k, metric, ratio, bm25, bits, post=post)
        _same_bits(got, want, f"{itype} {metric} n={n} {vocab} k={k} ratio={ratio} bitset={frac}")
        assert (got[0][-2:] == -1).all()   # the empty query and the all-absent query: padding only
        assert ix.last_stage_info()["engine"] == ("sparse" if k + 16 <= 1024 else "large_k")
    c = ix.last_counters()
    assert c["pairs"] > 0 and c["code_bytes"] == 8 * c["pairs"]


@pytest.mark.parametrize("metric", ["IP", "BM25"])
def test_range_search_matches_model(kb, metric):
    base, queries = _data("splade", 2 * TILE + 5, 3)
    cfg = _build_cfg(metric, base)
    ix = kb.Index("SPARSE_INVERTED_INDEX", metric, 0, cfg)
    ix.add_sparse(base)
    post = sm.Postings(base)
    bm25 = (K1, B, cfg["bm25_avgdl"]) if metric == "BM25" else None
    s10 = ix.search_sparse(queries, 10, cfg)[1][0]
    radius, top = float(s10[9]), float(s10[2])
    for rf, ratio, frac in [(None, 0.0, None), (top, 0.0, None), (top, 0.3, 0.5), (None, 0.0, 0.99)]:
        bits = None if frac is None else _bitset(base[0].size - 1, frac, 9)
        lims, ids, dist = ix.range_search_sparse(queries, radius * 0.5, rf, dict(cfg, drop_ratio_search=ratio), bitset=bits)
        ml, mi, md = sm.range_search(base, queries, radius * 0.5, rf, metric, ratio, bm25, bits, post=post)
        assert np.array_equal(lims, ml) and np.array_equal(ids, mi)
        assert np.array_equal(dist.view(np.uint32), md.view(np.uint32))
    assert lims[-1] > 0


@pytest.mark.parametrize("metric", ["IP", "BM25"])
def test_two_adds_equal_one_and_round_trip(kb, metric, tmp_path):
    base, queries = _data("splade", TILE + 300, 4)
    cfg = _build_cfg(metric, base)
    ip, ix_, val = base
    cut = 7001
    first = (ip[:cut + 1], ix_[:ip[cut]], val[:ip[cut]])
    second = (ip[cut:] - ip[cut], ix_[ip[cut]:], val[ip[cut]:])
    one = kb.Index("SPARSE_INVERTED_INDEX", metric, 0, cfg)
    one.add_sparse(base)
    two = kb.Index("SPARSE_INVERTED_INDEX", metric, 0, cfg)
    two.add_sparse(first)
    two.add_sparse(second)
    blob = one.serialize()
    assert two.serialize() == blob
    scfg = dict(cfg, drop_ratio_search=0.3)
    want = one.search_sparse(queries, 100, scfg)
    _same_bits(two.search_sparse(queries, 100, scfg), want, "two adds")
    back = kb.Index.deserialize(blob)
    assert back.serialize() == blob
    path = os.path.join(tmp_path, "sparse.kb2i")
    with open(path, "wb") as f:
        f.write(blob)
    again = kb.Index.deserialize_from_file(path)
    assert again.serialize() == blob
    for h in (back, again):
        _same_bits(h.search_sparse(queries, 100, scfg), want, "round trip")
        m = h.meta()
        assert m["type"] == "SPARSE_INVERTED_INDEX" and m["metric_type"] == metric and m["dim"] == 0
        assert m["rows"] == ip.size - 1 and m["nnz"] == int(ip[-1]) and m["sparse_dim"] == int(ix_.max()) + 1
        assert h.dim == 0 and not h.has_raw_data() and h.is_trained()


@pytest.mark.parametrize("metric", ["IP", "BM25"])
def test_bruteforce_equals_index_and_torch_inputs(kb, metric):
    import torch
    base, queries = _data("hashed", TILE + 1234, 5)
    cfg = _build_cfg(metric, base)
    ix = kb.Index("SPARSE_WAND", metric, 0, cfg)
    ix.add_sparse(base)
    bits = _bitset(base[0].size - 1, 0.5, 1)
    want = ix.search_sparse(queries, 64, cfg, bitset=bits)
    _same_bits(kb.brute_force_search_sparse(base, queries, 64, metric, cfg, bitset=bits), want, "BruteForce")
    dev = [tuple(torch.from_numpy(a.astype(np.int64) if a.dtype == np.uint32 else a).cuda() for a in c) for c in (base, queries)]
    tbits = torch.from_numpy(bits).cuda()
    ids, dist = kb.brute_force_search_sparse(dev[0], dev[1], 64, metric, cfg, bitset=tbits)
    _same_bits((ids.cpu().numpy(), dist.cpu().numpy()), want, "BruteForce, torch device inputs")
    ix2 = kb.Index("SPARSE_WAND", metric, 0, cfg)
    ix2.add_sparse(dev[0])
    ids, dist = ix2.search_sparse(dev[1], 64, cfg, bitset=tbits)
    _same_bits((ids.cpu().numpy(), dist.cpu().numpy()), want, "index, torch device inputs")
    assert ix2.serialize() == ix.serialize()


def _status(fn):
    import knowhere_b200 as kb
    with pytest.raises(kb.KnowhereError) as e:
        fn()
    return e.value.status


def test_refusals_and_validation(kb):
    base, queries = _data("splade", 500, 6)
    ip, ix_, val = base
    bm = _build_cfg("BM25", base)
    assert _status(lambda: kb.Index("SPARSE_INVERTED_INDEX", "L2", 0)) == 5
    assert _status(lambda: kb.Index("SPARSE_WAND", "COSINE", 0)) == 5
    assert _status(lambda: kb.Index("FLAT", "BM25", 8)) == 5
    assert _status(lambda: kb.Index("SPARSE_INVERTED_INDEX", "BM25", 0, {"bm25_k1": 1.2, "bm25_b": 0.75})) == 1
    assert _status(lambda: kb.Index("SPARSE_INVERTED_INDEX", "BM25", 0, dict(bm, bm25_k1=3.5))) == 3
    assert _status(lambda: kb.Index("SPARSE_INVERTED_INDEX", "BM25", 0, dict(bm, bm25_b=-0.1))) == 3
    assert _status(lambda: kb.Index("SPARSE_INVERTED_INDEX", "IP", 0, {"inverted_index_algo": "NOPE"})) == 1
    assert _status(lambda: kb.Index("SPARSE_INVERTED_INDEX", "IP", 0, {"quant_type": "u16"})) == 1
    assert _status(lambda: kb.Index("SPARSE_INVERTED_INDEX", "BM25", 0, dict(bm, quant_type="fp16"))) == 1
    for algo in ["taat_naive", "DAAT_WAND", "DAAT_MAXSCORE", "BLOCK_MAX_MAXSCORE", "BLOCK_MAX_WAND", "SINDI"]:
        kb.Index("SPARSE_WAND", "IP", 0, {"inverted_index_algo": algo, "quant_type": "fp32", "drop_ratio_build": 0.2,
                                           "inverted_index_codec": "block_streamvbyte", "block_max_block_size": 64,
                                           "sindi_window_size": 4096})
    sx = kb.Index("SPARSE_INVERTED_INDEX", "BM25", 0, bm)
    assert _status(lambda: sx.search_sparse(queries, 5, bm)) == 6   # empty index
    sx.add_sparse(base)
    dense = kb.Index("FLAT", "IP", 8)
    x = np.zeros((4, 8), np.float32)
    for f in (lambda: sx.train(x), lambda: sx.add(x), lambda: sx.search(x, 5), lambda: sx.range_search(x, 0.5),
              lambda: dense.add_sparse(base), lambda: dense.search_sparse(queries, 5),
              lambda: dense.range_search_sparse(queries, 0.5)):
        assert _status(f) == 1
    assert _status(lambda: kb.Index("SPARSE_WAND", "IP", 0).set_shard(0, 2)) == 7
    assert _status(lambda: sx.set_emb_list(np.array([0, ip.size - 1]), "MAX_SIM_IP")) == 7
    assert _status(lambda: sx.get_vector_by_ids(np.array([0]))) == 7
    assert _status(lambda: sx.serialize_faiss()) == 7
    # search keys
    nob = {k: v for k, v in bm.items() if k != "bm25_avgdl"}
    assert _status(lambda: sx.search_sparse(queries, 5, nob)) == 1
    assert _status(lambda: sx.search_sparse(queries, 5, dict(bm, bm25_k1=1.5))) == 16
    assert _status(lambda: sx.search_sparse(queries, 5, dict(bm, bm25_b=0.5))) == 16
    assert _status(lambda: sx.search_sparse(queries, 5, dict(bm, drop_ratio_search=1.0))) == 3
    assert _status(lambda: sx.search_sparse(queries, 5, dict(bm, metric_type="IP"))) == 5
    assert _status(lambda: sx.search_sparse(queries, 0, bm)) == 1
    assert _status(lambda: sx.search_sparse(queries, 16385, bm)) == 1
    sx.search_sparse(queries, 5, dict(bm, bm25_k1=K1, bm25_b=B, search_algo="DAAT_WAND", dim_max_score_ratio=1.1,
                                      refine_factor=3, bulk_query_nnz_threshold=5))
    assert _status(lambda: kb.brute_force_search_sparse(base, queries, 5, "L2")) == 5
    assert _status(lambda: kb.brute_force_search_sparse(base, queries, 5, "BM25", {"bm25_k1": 1.0})) == 1
    # malformed rows and queries, host and device
    import torch
    bad = [
        (np.array([0, 2, 1], np.int64), np.array([1, 2], np.uint32), np.ones(2, np.float32)),    # indptr decreases
        (np.array([1, 2], np.int64), np.array([1, 2], np.uint32), np.ones(2, np.float32)),       # indptr[0] != 0
        (np.array([0, 2], np.int64), np.array([2, 1], np.uint32), np.ones(2, np.float32)),       # unsorted
        (np.array([0, 2], np.int64), np.array([2, 2], np.uint32), np.ones(2, np.float32)),       # duplicate
        (np.array([0, 2], np.int64), np.array([1, 2], np.uint32), np.array([1, -1], np.float32)),
        (np.array([0, 2], np.int64), np.array([1, 2], np.uint32), np.array([1, np.nan], np.float32)),
        (np.array([0, 2], np.int64), np.array([1, 2], np.uint32), np.array([np.inf, 1], np.float32)),
    ]
    for csr in bad:
        dev = tuple(torch.from_numpy(a.astype(np.int64) if a.dtype == np.uint32 else a).cuda() for a in csr)
        for c in (csr, dev):
            assert _status(lambda: sx.add_sparse(c)) == 1
            assert _status(lambda: sx.search_sparse(c, 5, bm)) == 1
            assert _status(lambda: kb.brute_force_search_sparse(c, queries, 5, "IP")) == 1
    assert sx.count() == ip.size - 1


def test_splade_200k_parity_with_float64_oracle(kb):
    base = datagen.sparse_splade(200000, 120, 21)
    queries = datagen.sparse_splade(24, 40, 22)
    ix = kb.Index("SPARSE_INVERTED_INDEX", "IP", 0)
    ix.add_sparse(base)
    ids, dist = ix.search_sparse(queries, 100)
    ri, rd = sm.search(base, queries, 100, "IP", dtype=np.float64)
    assert_topk_parity(ids, dist, ri, rd, rtol=1e-5, what="SPLADE 200k")


def test_reduced_partial_slots_and_chunked_large_k(kb):
    # k = 1008 keeps 1024 entries per tile in 8 slots per query: ten tiles pass through reduce_partials_kernel.  k = 1009
    # over 4100 queries gives one-tile key chunks, so the running best set of select_rows_kernel merges three chunks.
    base = datagen.sparse_splade(9 * TILE + 123, 24, 31)
    queries = datagen.sparse_splade(12, 12, 32)
    ix = kb.Index("SPARSE_INVERTED_INDEX", "IP", 0)
    ix.add_sparse(base)
    bits = _bitset(9 * TILE + 123, 0.3, 2)
    post = sm.Postings(base)
    for ratio in (0.0, 0.3):
        _same_bits(ix.search_sparse(queries, 1008, {"drop_ratio_search": ratio}, bitset=bits),
                   sm.search(base, queries, 1008, "IP", ratio, None, bits, post=post), f"k=1008 over 10 tiles, ratio {ratio}")
    base = datagen.sparse_splade(2 * TILE + 300, 24, 33)
    queries = datagen.sparse_splade(4100, 6, 34)
    cfg = _build_cfg("BM25", base)
    ix = kb.Index("SPARSE_WAND", "BM25", 0, cfg)
    ix.add_sparse(base)
    got = ix.search_sparse(queries, 1009, cfg)
    assert ix.last_stage_info()["engine"] == "large_k"
    _same_bits(got, sm.search(base, queries, 1009, "BM25", bm25=(K1, B, cfg["bm25_avgdl"])), "k=1009, one-tile chunks")


@pytest.mark.parametrize("metric", ["IP", "BM25"])
def test_size_bytes_is_what_the_index_holds(kb, metric):
    base = datagen.sparse_splade(TILE + 99, 24, 41)
    ip, ix_, _ = base
    ix = kb.Index("SPARSE_INVERTED_INDEX", metric, 0, _build_cfg(metric, base))
    ix.add_sparse(base)
    n, nnz, nterms = ip.size - 1, int(ip[-1]), np.unique(ix_).size
    device = 4 * nterms + 8 * (nterms + 1) + 8 * nnz + (4 * n if metric == "BM25" else 0)
    host = 8 * (n + 1) + 8 * nnz
    assert ix.size() == device + host


def test_bruteforce_slot_reuse_and_search_keys(kb):
    base, queries = _data("splade", 3 * TILE + 10, 42)
    small, small_q = _data("hashed", 900, 43)
    bm = _build_cfg("BM25", base)
    post = sm.Postings(base)
    # build-only keys are not checked on a BruteForce call; each call sees only its own rows and metric
    for metric, cfg in (("IP", {"quant_type": "u16", "inverted_index_algo": "nope"}), ("BM25", bm), ("IP", {})):
        got = kb.brute_force_search_sparse(base, queries, 20, metric, cfg)
        want = sm.search(base, queries, 20, metric, bm25=(K1, B, bm["bm25_avgdl"]) if metric == "BM25" else None, post=post)
        _same_bits(got, want, f"BruteForce {metric}")
        ids, _ = kb.brute_force_search_sparse(small, small_q, 20, "IP")
        assert ids.max() < 900
    with pytest.raises(kb.KnowhereError) as e:
        kb.brute_force_search_sparse(base, queries, 20, "BM25", dict(bm, bm25_b=1.5))
    assert e.value.status == 3


def test_range_search_reports_its_engine_and_blob_keys_are_checked(kb):
    import struct
    base, queries = _data("splade", 2000, 44)
    cfg = _build_cfg("BM25", base)
    ix = kb.Index("SPARSE_INVERTED_INDEX", "BM25", 0, cfg)
    ix.add_sparse(base)
    ix.search_sparse(queries, 1009, cfg)
    assert ix.last_stage_info()["engine"] == "large_k"
    ix.range_search_sparse(queries, 0.5, None, cfg)
    assert ix.last_stage_info()["engine"] == "sparse"
    blob = ix.serialize()
    at = blob.find(struct.pack("<f", K1))
    assert at > 0
    bad = blob[:at] + struct.pack("<f", 5.0) + blob[at + 4:]
    with pytest.raises(kb.KnowhereError) as e:
        kb.Index.deserialize(bad)
    assert e.value.status == 19
