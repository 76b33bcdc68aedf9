"""IVF_FLAT / IVF_PQ parity against the compiled reference (GPU).

Parity protocol (SURVEY §8c): the index is trained and populated by the reference
(faiss IndexIVFFlat / IndexIVFPQ == what Knowhere's IvfIndexNode wraps), exported, and imported
into the GPU index, so both sides search the SAME centroids / codebooks / codes.  Then
ids must match (up to boundary ties) and distances agree to 1e-4 relative."""
import numpy as np
import pytest

from knowhere_b200 import datagen
from tests.util import assert_topk_parity, recall_at_k

pytestmark = pytest.mark.gpu


def _mk_ref(ref, kind, xb, metric, nlist, m=0, refine=False):
    r = ref.RefIvf(kind, xb.shape[1], metric, nlist, m, 8, refine=refine)
    r.train(xb)
    r.add(xb)
    return r


def _import(kb, r, kind, metric, xb, refine=False):
    cfg = {"nlist": r.nlist}
    if kind == "IVF_PQ":
        cfg.update(m=r.m, nbits=8, refine=refine, refine_type="flat")
    ix = kb.Index(kind, "L2" if metric == 0 else "IP", xb.shape[1], cfg)
    ix.ivf_import(r.centroids(), r.pq_centroids() if kind == "IVF_PQ" else None, list(r.lists()),
                  raw=xb if refine else None)
    assert ix.count() == xb.shape[0]
    return ix


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("nb,d,nlist,nprobe,nq,k", [(20000, 128, 64, 8, 100, 10), (5000, 32, 16, 16, 33, 5)])
def test_ivfflat_imported_index_parity(kb, ref, metric, nb, d, nlist, nprobe, nq, k):
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(nq, d, 43)
    r = _mk_ref(ref, "IVF_FLAT", xb, metric, nlist)
    ix = _import(kb, r, "IVF_FLAT", metric, xb)
    I0, D0 = r.search(xq, k, nprobe)
    ids, dist = ix.search(xq, k, {"nprobe": nprobe})
    assert_topk_parity(ids, dist, I0, D0, what="IVF_FLAT")


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("m,d", [(16, 128), (8, 64), (32, 128), (48, 96)])
def test_ivfpq_imported_index_parity(kb, ref, metric, m, d):
    nb, nlist, nprobe, nq, k = 30000, 64, 8, 100, 10
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(nq, d, 43)
    r = _mk_ref(ref, "IVF_PQ", xb, metric, nlist, m)
    ix = _import(kb, r, "IVF_PQ", metric, xb)
    I0, D0 = r.search(xq, k, nprobe)
    ids, dist = ix.search(xq, k, {"nprobe": nprobe})
    # PQ codes collide (identical codes => identical ADC distance): allow tie rows, compare sets
    # (every differing id is still verified to sit exactly at the k-th distance)
    assert_topk_parity(ids, dist, I0, D0, rtol=1e-4, atol=1e-3, what=f"IVF_PQ m={m}", max_tie_rows=nq)
    # coarse stage must agree exactly with the reference quantizer
    CI, CD = r.coarse(xq, nprobe)
    # (indirectly checked by the result parity above; direct check through nprobe=1 results)
    ids1, _ = ix.search(xq, 1, {"nprobe": 1})
    I1, _ = r.search(xq, 1, 1)
    assert (ids1 == I1).mean() > 0.97


@pytest.mark.parametrize("refine_k", [1, 4])
def test_ivfpq_refine_parity(kb, ref, refine_k):
    nb, d, nlist, m, nprobe, nq, k = 30000, 128, 64, 16, 16, 100, 10
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(nq, d, 43)
    r = _mk_ref(ref, "IVF_PQ", xb, 0, nlist, m, refine=True)
    ix = _import(kb, r, "IVF_PQ", 0, xb, refine=True)
    I0, D0 = r.search(xq, k, nprobe, refine_k=float(refine_k))
    ids, dist = ix.search(xq, k, {"nprobe": nprobe, "refine_k": refine_k})
    assert_topk_parity(ids, dist, I0, D0, what="IVF_PQ+refine")
    gt, _ = ref.flat_search(xb, xq, k, 0)
    assert recall_at_k(gt, ids) >= recall_at_k(gt, I0) - 1e-9


def test_ivfpq_export_roundtrip(kb, ref):
    nb, d, nlist, m = 8000, 64, 32, 16
    xb = datagen.clustered(nb, d, 1)
    r = _mk_ref(ref, "IVF_PQ", xb, 0, nlist, m)
    ix = _import(kb, r, "IVF_PQ", 0, xb)
    for l in (0, 5, 31):
        ids0, codes0 = r.get_list(l)
        ids1, codes1 = ix.ivf_export_list(l, m)
        assert np.array_equal(ids0, ids1) and np.array_equal(codes0, codes1)


@pytest.mark.parametrize("kind,m", [("IVF_FLAT", 0), ("IVF_PQ", 16)])
def test_ivf_gpu_build_recall_vs_reference(kb, ref, kind, m):
    """Index built entirely on the GPU (own k-means / PQ / encoding): recall@10 must reach the
    reference-built index's recall at identical parameters (north_star parity bar for IVF)."""
    nb, d, nlist, nprobe, nq, k = 40000, 128, 128, 16, 1000, 10
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(nq, d, 43)
    gt, _ = ref.flat_search(xb, xq, k, 0)
    r = _mk_ref(ref, kind, xb, 0, nlist, m)
    I0, _ = r.search(xq, k, nprobe)
    cfg = {"nlist": nlist}
    if m:
        cfg.update(m=m, nbits=8)
    ix = kb.Index(kind, "L2", d, cfg)
    ix.build(xb)
    ids, dist = ix.search(xq, k, {"nprobe": nprobe})
    rec_ref, rec_gpu = recall_at_k(gt, I0), recall_at_k(gt, ids)
    print(f"{kind}: recall ref={rec_ref:.4f} gpu={rec_gpu:.4f}")
    # the GPU k-means uses float atomics (run-to-run variation of ~0.01 at this size); without refine the GPU-built
    # codebooks land 0.01-0.03 below the reference-built ones here, with refine both reach the same recall
    assert rec_gpu >= rec_ref - 0.035
    # and the GPU-built index exported to the reference gives the same answers on the CPU
    r2 = ref.RefIvf(kind, d, 0, nlist, m, 8)
    c, pq = ix.ivf_export_centroids(m)
    cs = m if m else d * 4
    r2.import_state(c, pq, [(l,) + ix.ivf_export_list(l, cs) for l in range(nlist)])
    I2, D2 = r2.search(xq, k, nprobe)
    assert_topk_parity(ids, dist, I2, D2, rtol=1e-4, atol=1e-3, what=f"{kind} gpu-built vs cpu search",
                       max_tie_rows=nq // 4)


def test_ivf_small_batch_splits_probes(kb, ref):
    # nq < 2*SMs => several CTAs per query; results must not depend on the split
    nb, d, nlist, m = 20000, 64, 64, 16
    xb = datagen.clustered(nb, d, 3)
    xq = datagen.clustered(300, d, 4)
    r = _mk_ref(ref, "IVF_PQ", xb, 0, nlist, m)
    ix = _import(kb, r, "IVF_PQ", 0, xb)
    a = ix.search(xq, 10, {"nprobe": 32})
    b = ix.search(xq[:3].copy(), 10, {"nprobe": 32})
    assert np.array_equal(a[0][:3], b[0]) and np.array_equal(a[1][:3], b[1])


def test_ivf_bitset_and_serialize(kb, ref):
    nb, d, nlist, m = 10000, 64, 32, 16
    xb = datagen.clustered(nb, d, 5)
    xq = datagen.clustered(20, d, 6)
    ix = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m})
    ix.build(xb)
    mask = np.zeros(nb, bool)
    mask[1::2] = True
    ids, _ = ix.search(xq, 10, {"nprobe": 32}, bitset=np.packbits(mask, bitorder="little"))
    assert not mask[ids[ids >= 0]].any()
    a = ix.search(xq, 10, {"nprobe": 8})
    ix2 = kb.Index.deserialize(ix.serialize())
    b = ix2.search(xq, 10, {"nprobe": 8})
    assert np.array_equal(a[0], b[0]) and np.allclose(a[1], b[1])


def test_ivf_errors(kb):
    ix = kb.Index("IVF_FLAT", "L2", 16, {"nlist": 4})
    with pytest.raises(kb.KnowhereError) as e:
        ix.add(np.zeros((10, 16), np.float32))
    assert e.value.status == 8          # index_not_trained
    with pytest.raises(kb.KnowhereError) as e:
        kb.Index("IVF_PQ", "L2", 30, {"nlist": 4, "m": 16})
    assert e.value.status == 1          # invalid_args (dim % m)
    with pytest.raises(kb.KnowhereError):
        kb.Index("NOPE", "L2", 16)


def test_ivf_range_search(kb, ref):
    """IVF RangeSearch (ivf.cc:1229-1500): with every list probed and the empty-bucket heuristic off,
    IVF_FLAT must return exactly the FLAT range result; IVF_PQ must return exactly the ids whose ADC
    distance (as reported by Search) is inside the radius."""
    nb, d, nlist, m = 6000, 32, 16, 8
    xb = datagen.clustered(nb, d, 11)
    xq = datagen.clustered(15, d, 12)
    I, D = ref.flat_search(xb, xq, 30, 0)
    radius = float(np.median(D[:, 20]))
    lims0, ids0, dis0 = ref.flat_range_search(xb, xq, radius, 0)
    ix = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
    ix.build(xb)
    lims, ids, dis = ix.range_search(xq, radius, config={"nprobe": nlist, "max_empty_result_buckets": 0})
    assert np.array_equal(lims, lims0)
    for i in range(len(xq)):
        assert set(ids[lims[i]:lims[i + 1]].tolist()) == set(ids0[lims0[i]:lims0[i + 1]].tolist())
        assert (np.diff(dis[lims[i]:lims[i + 1]]) >= 0).all()
    # range_filter: keep range_filter <= d < radius (range_util.h:23-26)
    rf = float(np.median(D[:, 5]))
    lims2, ids2, dis2 = ix.range_search(xq, radius, range_filter=rf, config={"nprobe": nlist, "max_empty_result_buckets": 0})
    assert (dis2 >= rf).all() and (dis2 < radius).all()
    # IVF_PQ: consistency with Search on the same ADC distances
    pq = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m})
    pq.build(xb)
    sI, sD = pq.search(xq, 200, {"nprobe": nlist})
    lims3, ids3, dis3 = pq.range_search(xq, radius, config={"nprobe": nlist, "max_empty_result_buckets": 0})
    for i in range(len(xq)):
        want = set(sI[i][sD[i] < radius].tolist())
        got = set(ids3[lims3[i]:lims3[i + 1]].tolist())
        if (sD[i] < radius).sum() < 200:          # top-200 covers the whole ball
            assert got == want
    # IP metric: radius < d
    xbn = xb / np.linalg.norm(xb, axis=1, keepdims=True)
    xqn = xq / np.linalg.norm(xq, axis=1, keepdims=True)
    fi = kb.Index("IVF_FLAT", "IP", d, {"nlist": nlist})
    fi.build(xbn)
    l4, i4, d4 = fi.range_search(xqn, 0.9, config={"nprobe": nlist, "max_empty_result_buckets": 0})
    # float64 inner products of the fp32 rows; only a row within the fp32 summation bound of 0.9 may go either way
    ip = xqn.astype(np.float64) @ xbn.astype(np.float64).T
    bound = (d + 2) * 2.0 ** -24 * (np.abs(xqn).astype(np.float64) @ np.abs(xbn).astype(np.float64).T)
    for i in range(len(xq)):
        got = set(i4[l4[i]:l4[i + 1]].tolist())
        assert set(np.nonzero(ip[i] - bound[i] > 0.9)[0].tolist()) <= got
        assert got <= set(np.nonzero(ip[i] + bound[i] > 0.9)[0].tolist())
        assert (d4[l4[i]:l4[i + 1]] > np.float32(0.9)).all()
        assert (np.diff(d4[l4[i]:l4[i + 1]]) <= 0).all()


@pytest.mark.parametrize("world", [2, 4])
def test_ivf_list_sharding_single_gpu(kb, world):
    """kb2_index_set_shard + kb2_merge_topk on ONE GPU: `world` shard handles (size-balanced list packing) built
    from the same quantizers; the merge of their local top-k must equal the unsharded search."""
    nb, d, nlist, m, nq, k = 30000, 64, 64, 16, 400, 10
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(nq, d, 43)
    cfgb = {"nlist": nlist, "m": m, "refine": True, "refine_type": "flat"}
    full = kb.Index("IVF_PQ", "L2", d, cfgb)
    full.build(xb)
    cent, pq = full.ivf_export_centroids(m)
    # (a) pure ADC search: local top-k by ADC merged == global top-k by ADC, exactly
    # (b) with refine each shard refines its own k*refine_k candidates, so the merged result considers a
    #     superset of the unsharded candidates: it can only be better (pointwise smaller-or-equal distances)
    cfg_adc, cfg_ref = {"nprobe": 16, "refine_k": 1}, {"nprobe": 16, "refine_k": 4}
    full_adc = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m})
    kb._check(kb.lib().kb2_ivf_import_begin(full_adc.h, nlist, cent.ctypes.data, pq.ctypes.data))
    full_adc.add(xb)
    I0, D0 = full_adc.search(xq, k, cfg_adc)
    I1, D1 = full.search(xq, k, cfg_ref)
    adc_ids, adc_dis, ref_ids, ref_dis, sizes = [], [], [], [], 0
    per_rank_rows = [0] * world
    for rank in range(world):
        sh = kb.Index("IVF_PQ", "L2", d, cfgb)
        sh.set_shard(rank, world)
        kb._check(kb.lib().kb2_ivf_import_begin(sh.h, nlist, cent.ctypes.data, pq.ctypes.data))
        sh.add(xb)
        for l in range(nlist):
            n_l = kb.lib().kb2_ivf_list_size(sh.h, l)
            assert n_l in (0, kb.lib().kb2_ivf_list_size(full.h, l))      # a list lives on exactly one shard
            sizes += n_l
            per_rank_rows[rank] += n_l
        a = sh.search(xq, k, cfg_ref)
        ref_ids.append(a[0]); ref_dis.append(a[1])
        sh2 = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m})
        sh2.set_shard(rank, world)
        kb._check(kb.lib().kb2_ivf_import_begin(sh2.h, nlist, cent.ctypes.data, pq.ctypes.data))
        sh2.add(xb)
        b = sh2.search(xq, k, cfg_adc)
        adc_ids.append(b[0]); adc_dis.append(b[1])
    assert sizes == nb
    # size-balanced packing (longest list first onto the lightest shard): shards within a few percent of each other
    assert max(per_rank_rows) - min(per_rank_rows) <= 0.05 * nb / world + 2000
    mi, md = kb.merge_topk(np.stack(adc_ids), np.stack(adc_dis), "L2")
    assert_topk_parity(mi, md, I0, D0, rtol=1e-6, atol=1e-6, what="sharded ADC merge", max_tie_rows=nq // 10)
    mi, md = kb.merge_topk(np.stack(ref_ids), np.stack(ref_dis), "L2")
    assert (md <= D1 * (1 + 1e-6)).all()


@pytest.mark.parametrize("kind,m", [("IVF_FLAT", 0), ("IVF_PQ", 16)])
def test_ivf_bitset_after_import_and_deserialize(kb, ref, kind, m):
    """A BitsetView addresses vectors by id (bitsetview.h:131-175).  After import / Deserialize the rows used to be
    numbered in list order, so the filter hit the wrong vectors; now rows are renumbered by label.  Checked against the
    reference's own filtered search (ids identical) and through GetVectorByIds."""
    nb, d, nlist, nq, k = 12000, 64, 32, 50, 10
    xb = datagen.clustered(nb, d, 21)
    xq = datagen.clustered(nq, d, 22)
    r = _mk_ref(ref, kind, xb, 0, nlist, m, refine=False)
    ix = _import(kb, r, kind, 0, xb)
    mask = np.random.default_rng(5).random(nb) < 0.4
    bits = np.packbits(mask, bitorder="little")
    a_ids, a_dis = ix.search(xq, k, {"nprobe": nlist}, bitset=bits)
    assert not mask[a_ids[a_ids >= 0]].any()
    # exact expectation for IVF_FLAT with every list probed: brute force over the kept rows
    if kind == "IVF_FLAT":
        gt, gd = ref.flat_search(xb[~mask], xq, k, 0)
        gt = np.nonzero(~mask)[0][gt]
        assert_topk_parity(a_ids, a_dis, gt, gd, what="IVF_FLAT bitset after import")
        v = ix.get_vector_by_ids(np.array([0, 17, nb - 1]))
        assert np.array_equal(v, xb[[0, 17, nb - 1]])
    ix2 = kb.Index.deserialize(ix.serialize())
    b_ids, b_dis = ix2.search(xq, k, {"nprobe": nlist}, bitset=bits)
    assert np.array_equal(a_ids, b_ids) and np.allclose(a_dis, b_dis)
    # an index built here, serialised and loaded: same filtered answer as before the round trip
    ix3 = kb.Index(kind, "L2", d, dict({"nlist": nlist}, **({"m": m} if m else {})))
    ix3.build(xb)
    c_ids, _ = ix3.search(xq, k, {"nprobe": 8}, bitset=bits)
    ix4 = kb.Index.deserialize(ix3.serialize())
    d_ids, _ = ix4.search(xq, k, {"nprobe": 8}, bitset=bits)
    assert np.array_equal(c_ids, d_ids) and not mask[d_ids[d_ids >= 0]].any()
    with pytest.raises(kb.KnowhereError) as e:
        ix.search(xq, k, {"nprobe": 4}, bitset=bits[: nb // 16])      # too short a bitmap
    assert e.value.status == 1


def test_ivfpq_add_after_search(kb):
    """Add() after the first Search() (the sealed list layout is unpacked and rebuilt): same result as one big add."""
    nb, d, nlist, m = 20000, 64, 32, 16
    xb = datagen.clustered(nb, d, 31)
    xq = datagen.clustered(40, d, 32)
    one = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m})
    one.train(xb)
    cent, pq = one.ivf_export_centroids(m)
    one.add(xb)
    two = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m})
    kb._check(kb.lib().kb2_ivf_import_begin(two.h, nlist, cent.ctypes.data, pq.ctypes.data))
    two.add(xb[:12000].copy())
    two.search(xq, 10, {"nprobe": 8})
    two.add(xb[12000:].copy())
    a = one.search(xq, 10, {"nprobe": 8})
    b = two.search(xq, 10, {"nprobe": 8})
    assert two.count() == nb and np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_ivf_build_is_deterministic(kb):
    """two GPU builds of the same data give bit-identical quantizers (no float atomics in k-means)"""
    nb, d, nlist, m = 30000, 64, 64, 16
    xb = datagen.clustered(nb, d, 9)
    outs = []
    for _ in range(2):
        ix = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m})
        ix.train(xb)
        outs.append(ix.ivf_export_centroids(m))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


def _with_env(name, value, fn):
    import os
    old = os.environ.get(name)
    os.environ[name] = value
    try:
        return fn()
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


@pytest.mark.parametrize("metric", [0, 1])
@pytest.mark.parametrize("d", [128, 96])
def test_ivfflat_tc_engine_matches_scan_and_reference(kb, ref, metric, d):
    """IVF_FLAT list-major tensor-core engine (kb2_ivfflat_tc.cuh: 3xTF32 filter + exact fp32 re-rank) against the query-major
    exact scan of the same index and against the reference's IndexIVFFlat: identical ids, distances to fp32 rounding."""
    nb, nlist, nprobe, nq, k = 60000, 64, 16, 2000, 10
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(nq, d, 43)
    r = _mk_ref(ref, "IVF_FLAT", xb, metric, nlist)
    ix = _import(kb, r, "IVF_FLAT", metric, xb)
    ix.enable_kernel_timing(True)
    a_ids, a_dis = _with_env("KB2_FLAT_ENGINE", "tc", lambda: ix.search(xq, k, {"nprobe": nprobe}))
    assert ix.last_stage_info()["engine"] == "tc"
    b_ids, b_dis = _with_env("KB2_FLAT_ENGINE", "scan", lambda: ix.search(xq, k, {"nprobe": nprobe}))
    assert ix.last_stage_info()["engine"] == "scan"
    assert_topk_parity(a_ids, a_dis, b_ids, b_dis, rtol=2e-6, atol=1e-5, what="IVF_FLAT tc vs scan", max_tie_rows=2)
    I0, D0 = r.search(xq, k, nprobe)
    assert_topk_parity(a_ids, a_dis, I0, D0, what="IVF_FLAT tc vs reference")
    # with a bitset
    mask = np.random.default_rng(1).random(nb) < 0.5
    bits = np.packbits(mask, bitorder="little")
    c_ids, c_dis = _with_env("KB2_FLAT_ENGINE", "tc", lambda: ix.search(xq, k, {"nprobe": nprobe}, bitset=bits))
    d_ids, d_dis = _with_env("KB2_FLAT_ENGINE", "scan", lambda: ix.search(xq, k, {"nprobe": nprobe}, bitset=bits))
    assert not mask[c_ids[c_ids >= 0]].any()
    assert_topk_parity(c_ids, c_dis, d_ids, d_dis, rtol=2e-6, atol=1e-5, what="IVF_FLAT tc vs scan (bitset)", max_tie_rows=2)


def test_ivfflat_tc_engine_small_lists_and_fallback(kb):
    """lists shorter than k (no phase-A bound => every row survives => candidate rows overflow) must fall back to the exact
    scan transparently; ragged tails (list length not a multiple of 128) are masked."""
    nb, d, nlist, nq, k = 3000, 32, 256, 600, 10      # ~12 rows per list
    xb = datagen.clustered(nb, d, 7)
    xq = datagen.clustered(nq, d, 8)
    ix = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
    ix.build(xb)
    a = _with_env("KB2_FLAT_ENGINE", "tc", lambda: ix.search(xq, k, {"nprobe": 64}))
    b = _with_env("KB2_FLAT_ENGINE", "scan", lambda: ix.search(xq, k, {"nprobe": 64}))
    assert_topk_parity(a[0], a[1], b[0], b[1], rtol=2e-6, atol=1e-5, what="IVF_FLAT tc small lists", max_tie_rows=2)


@pytest.mark.parametrize("np_dtype", [np.int8, np.float16])
def test_typed_ingest_matches_widened_fp32(kb, np_dtype):
    """int8 / fp16 data and queries (kb2_index_*_typed: widened to fp32 on the device like the reference's
    index_node_data_mock_wrapper.cc:24-60) give exactly the answer of the same values passed as fp32."""
    nb, d, nlist, m = 20000, 96, 32, 48
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(64, d, 43)
    if np_dtype == np.int8:
        s = 127.0 / np.abs(xb).max()
        xb_t, xq_t = np.clip(np.round(xb * s), -127, 127).astype(np.int8), np.clip(np.round(xq * s), -127, 127).astype(np.int8)
    else:
        xb_t, xq_t = xb.astype(np.float16), xq.astype(np.float16)
    a = kb.Index("IVF_PQ", "IP", d, {"nlist": nlist, "m": m})
    a.build(xb_t)
    b = kb.Index("IVF_PQ", "IP", d, {"nlist": nlist, "m": m})
    b.build(xb_t.astype(np.float32))
    ra = a.search(xq_t, 10, {"nprobe": 8})
    rb = b.search(xq_t.astype(np.float32), 10, {"nprobe": 8})
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
    f = kb.Index("FLAT", "L2", d)
    f.add(xb_t)
    ids, dist = f.search(xq_t, 5)
    gi, gd = kb.brute_force_search(xb_t.astype(np.float32), xq_t.astype(np.float32), 5, "L2")
    assert np.array_equal(ids, gi)


@pytest.mark.parametrize("rtype", ["fp16", "bf16"])
def test_ivfpq_low_precision_refine_store(kb, rtype):
    """refine_type fp16 / bf16 (ivf_config.h:97-128, refine_utils.cc:99-160): the refine store keeps 16-bit rows and the
    re-rank computes fp32 distances on the decoded values — exactly what a flat store holding the rounded rows gives."""
    import torch
    nb, d, nlist, m, nq, k = 30000, 64, 32, 16, 200, 10
    xb = datagen.clustered(nb, d, 42)
    xq = datagen.clustered(nq, d, 43)
    a = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m, "refine": True, "refine_type": rtype})
    a.build(xb)
    assert not a.has_raw_data()
    cent, pq = a.ivf_export_centroids(m)
    lists = [(l,) + a.ivf_export_list(l, m) for l in range(nlist)]
    t = torch.from_numpy(xb).to(torch.float16 if rtype == "fp16" else torch.bfloat16).to(torch.float32).numpy()
    b = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m, "refine": True, "refine_type": "flat"})
    b.ivf_import(cent, pq, lists, raw=t)
    cfg = {"nprobe": 8, "refine_k": 4}
    ra, rb = a.search(xq, k, cfg), b.search(xq, k, cfg)
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1].view(np.uint32), rb[1].view(np.uint32))
    # container round trip keeps the store type and the answers; the store is half the size of the fp32 one
    c = kb.Index.deserialize(a.serialize())
    rc = c.search(xq, k, cfg)
    assert np.array_equal(ra[0], rc[0]) and np.array_equal(ra[1], rc[1])
    assert a.size() < b.size() - nb * d * 1.5

