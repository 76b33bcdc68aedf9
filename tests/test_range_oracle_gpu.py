"""RangeSearch of FLAT, BruteForce, IVF_FLAT, IVF_PQ and HNSW's exact scan against a float64 oracle (GPU).

The oracle distances and per-row bounds are those of the k-NN oracle test (`flat_oracle`, and `pq_oracle`'s ADC
distances for IVF_PQ).  `check_range` is the one acceptance rule used by every case; for each query:

1. lims starts at 0, does not decrease and ends at len(ids);
2. ids are distinct, belong to the index and are not filtered out by the bitset;
3. each returned distance is within the bound of the oracle;
4. each returned fp32 distance lies in the window by the library's rule: L2 keeps range_filter <= d < radius,
   IP / COSINE keep radius < d <= range_filter;
5. hits are ordered best first, equal distances by id;
6. nothing is missed: every valid row whose oracle distance lies inside the window by more than its bound is returned;
7. nothing is extra: no row whose oracle distance lies outside the window by more than its bound is returned.

Rows within their bound of an edge may go either way.  Case ids name the path they reach: the FLAT row split across
`nsplit` CTAs (range_scan_rows: min(2 * SMs / nq, n / 1024), 132 SMs), the IVF split of each query's probes (nsplit > 1
when nq < 2 * SMs), IVF_PQ code layout kind 1 (rotated 16-groups, m % 16 == 0 and m / 16 <= 3) or kind 2 (plain bytes),
the hit-buffer retry (range_scan: 2^20 hits or 256 per query before it), and HNSW's graph path or exact-scan fallback.
"""
import functools

import numpy as np
import pytest

from knowhere_b200 import datagen
from tests.test_exact_oracle_gpu import U, flat_oracle, pq_oracle

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

INVALID_ARGS, NOT_IMPLEMENTED = 1, 7
HIT_CAP = 1 << 20                         # range_scan's first hit buffer for nq <= 4096


# ------------------------------------------------------------------------------------------------ acceptance rule
def in_window(dist, metric, radius, range_filter=None):
    """the library's range rule on fp32 distances (in_range_host)"""
    d = np.asarray(dist, np.float32)
    if metric == "L2":
        ok = d < np.float32(radius)
        if range_filter is not None:
            ok &= d >= np.float32(range_filter)
    else:
        ok = d > np.float32(radius)
        if range_filter is not None:
            ok &= d <= np.float32(range_filter)
    return ok


def check_range(lims, ids, dist, D, B, labels, metric, radius, range_filter=None, valid=None, what=""):
    """The acceptance rule (module docstring).  D, B: [nq, n] oracle distance / bound per row (row = position in
    `labels`); metric "L2" or "IP" (COSINE is IP on normalised rows); valid: [n] bool, False for rows the bitset filters
    out.  Returns the number of hits."""
    lims, ids, dist = np.asarray(lims), np.asarray(ids), np.asarray(dist)
    labels = np.asarray(labels, np.int64)
    nq, n = D.shape
    valid = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    # 1. lims
    assert lims.shape == (nq + 1,), f"{what}: lims shape {lims.shape}"
    assert lims[0] == 0 and (np.diff(lims) >= 0).all(), f"{what}: lims {lims[:8]}"
    assert lims[-1] == ids.size == dist.size, f"{what}: lims end {lims[-1]}, {ids.size} ids, {dist.size} distances"
    r = float(np.float32(radius))
    f = None if range_filter is None else float(np.float32(range_filter))
    sgn = 1.0 if metric == "L2" else -1.0
    order = np.argsort(labels, kind="stable")
    sl = labels[order]
    for i in range(nq):
        msg = f"{what} q{i}"
        g, dd = ids[lims[i]:lims[i + 1]], dist[lims[i]:lims[i + 1]]
        # 2. ids
        assert np.unique(g).size == g.size, f"{msg}: duplicate ids"
        p = np.searchsorted(sl, g)
        assert (p < n).all() and (sl[np.minimum(p, n - 1)] == g).all(), f"{msg}: ids not in the index"
        rows = order[p]
        assert valid[rows].all(), f"{msg}: filtered rows returned {g[~valid[rows]][:8]}"
        # 3. distances
        od, ob = D[i, rows], B[i, rows]
        bad = np.nonzero(np.abs(dd.astype(np.float64) - od) > ob)[0]
        assert bad.size == 0, (f"{msg}: distance of id {g[bad[0]]} is {dd[bad[0]]!r}, oracle {od[bad[0]]!r}, "
                               f"bound {ob[bad[0]]:.3g}")
        # 4. window, exactly on the fp32 distances
        win = in_window(dd, metric, radius, range_filter)
        assert win.all(), f"{msg}: id {g[~win][0]} at {dd[~win][0]!r} outside radius {radius!r} / filter {range_filter!r}"
        # 5. order
        key = sgn * dd.astype(np.float64)
        ok = (key[1:] > key[:-1]) | ((key[1:] == key[:-1]) & (g[1:] > g[:-1]))
        assert ok.all(), f"{msg}: not in (distance, id) order at rank {int(np.argmin(ok))}"
        # 6. / 7. against the oracle
        Di, Bi = D[i], B[i]
        if metric == "L2":
            inside = Di + Bi < r
            outside = Di - Bi >= r
            if f is not None:
                inside &= Di - Bi >= f
                outside |= Di + Bi < f
        else:
            inside = Di - Bi > r
            outside = Di + Bi <= r
            if f is not None:
                inside &= Di + Bi <= f
                outside |= Di - Bi > f
        got = np.zeros(n, bool)
        got[rows] = True
        missing = np.nonzero(valid & inside & ~got)[0]
        assert missing.size == 0, (f"{msg}: {missing.size} rows inside the window missing, e.g. id {labels[missing[0]]} "
                                   f"at oracle {Di[missing[0]]!r}")
        extra = np.nonzero(outside & got)[0]
        assert extra.size == 0, f"{msg}: id {labels[extra[0]]} at oracle {Di[extra[0]]!r} is outside the window"
    return int(lims[-1])


def window_of(D, metric, lo, hi, skip_last=False):
    """(radius, range_filter) at the hi and lo quantiles of all (query, row) distances, best first"""
    S = D[:-1] if skip_last else D
    key = S if metric == "L2" else -S
    sgn = 1.0 if metric == "L2" else -1.0
    r, f = np.quantile(key, [hi, lo])
    return float(sgn * r), float(sgn * f)


def per_query(lims, ids, dist):
    return [(ids[lims[i]:lims[i + 1]], dist[lims[i]:lims[i + 1]]) for i in range(len(lims) - 1)]


def same_result(a, b, what=""):
    """two range results equal: lims, ids and distance bits"""
    assert np.array_equal(a[0], b[0]), f"{what}: lims differ"
    assert np.array_equal(a[1], b[1]), f"{what}: ids differ"
    assert np.array_equal(np.asarray(a[2]).view(np.uint32), np.asarray(b[2]).view(np.uint32)), f"{what}: distances differ"


def bits_of(mask):
    return np.packbits(mask, bitorder="little")


def custom_ids(n, seed):
    return np.random.default_rng(seed).permutation(n).astype(np.int64) * 3 + 11


def oracle_metric(metric):
    return "L2" if metric == "L2" else "IP"


def status_of(kb, fn):
    with pytest.raises(kb.KnowhereError) as e:
        fn()
    return e.value.status, str(e.value)


# ------------------------------------------------------------------------------------------------ FLAT / BruteForce
FLAT_SHAPES = [
    # nq, n, d
    pytest.param(20, 1000, 32, id="n1000-nsplit1"),
    pytest.param(1, 50000, 128, id="nq1-n50000-nsplit48"),
    pytest.param(10, 4001, 17, id="d17-nsplit3-tail1"),           # splits of 1344 rows, the last 1313 rows: a 1-row chunk
    pytest.param(50, 3000, 1, id="d1-nsplit2-tail24"),            # splits of 1504 and 1496 rows
    pytest.param(100, 20000, 128, id="d128-nsplit3"),
    pytest.param(8, 2000, 16384, id="d16384-smem64k"),            # 65 664 bytes of shared memory per CTA
]


@pytest.mark.parametrize("filtered", [False, True], ids=["radius", "range_filter"])
@pytest.mark.parametrize("custom", [False, True], ids=["rowids", "customids"])
@pytest.mark.parametrize("metric", ["L2", "IP", "COSINE"])
@pytest.mark.parametrize("nq,n,d", FLAT_SHAPES)
def test_flat_range_matches_oracle(kb, nq, n, d, metric, custom, filtered):
    """FLAT and BruteForce (range_scan_rows).  The last query of a batch points away from the data, so it has no hit."""
    if metric == "COSINE" and d == 1:
        pytest.skip("every COSINE distance is 1 at d = 1")
    xb = datagen.uniform(n, d, 300 + d)
    xq = datagen.uniform(nq, d, 400 + d)
    far = nq > 1
    if far:
        xq[-1] = xq[-1] + 1000.0 if metric == "L2" else -xq[-1]
    labels = custom_ids(n, 6) if custom else np.arange(n, dtype=np.int64)
    D, B = flat_oracle(xb, xq, metric)
    radius, rf = window_of(D, metric, 0.002, 0.02, skip_last=far)
    rf = rf if filtered else None
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb, labels if custom else None)
    om = oracle_metric(metric)
    res = ix.range_search(xq, radius, rf)
    hits = check_range(*res, D, B, labels, om, radius, rf, what=f"FLAT {metric}")
    assert hits > 0
    if far:
        assert res[0][-1] == res[0][-2], "the far query has no hit"
    if not custom:
        bf = kb.brute_force_range_search(xb, xq, radius, rf, metric)
        check_range(*bf, D, B, labels, om, radius, rf, what=f"BruteForce {metric}")


def test_bruteforce_range_device_tensors(kb):
    """brute_force_range_search with base and queries in device memory: the same result as from host memory."""
    n, nq, d = 20000, 40, 64
    xb = datagen.uniform(n, d, 51)
    xq = datagen.uniform(nq, d, 52)
    D, B = flat_oracle(xb, xq, "L2")
    radius, rf = window_of(D, "L2", 0.001, 0.01)
    dev = kb.brute_force_range_search(torch.from_numpy(xb).cuda(), torch.from_numpy(xq).cuda(), radius, rf, "L2")
    assert check_range(*dev, D, B, np.arange(n), "L2", radius, rf, what="BruteForce device") > 0
    same_result(dev, kb.brute_force_range_search(xb, xq, radius, rf, "L2"), "device vs host")


@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_flat_range_translated_data(kb, metric):
    """Rows 1000 + N(0, 1), where the norm-expanded k-NN keys cancel: the range scan takes direct differences, so its L2
    distances stay within the bound of the oracle."""
    n, nq, d = 20000, 50, 128
    rng = np.random.default_rng(7)
    xb = (1000.0 + rng.standard_normal((n, d))).astype(np.float32)
    xq = (1000.0 + rng.standard_normal((nq, d))).astype(np.float32)
    D, B = flat_oracle(xb, xq, metric)
    radius, rf = window_of(D, metric, 0.001, 0.01)
    ix = kb.Index("FLAT", metric, d)
    ix.add(xb)
    assert check_range(*ix.range_search(xq, radius), D, B, np.arange(n), metric, radius, what="FLAT translated") > 0
    check_range(*ix.range_search(xq, radius, rf), D, B, np.arange(n), metric, radius, rf, what="FLAT translated rf")


# ------------------------------------------------------------------------------------------------ boundary semantics
@functools.lru_cache(maxsize=1)
def _int_data():
    rng = np.random.default_rng(5)
    return rng.integers(0, 4, (3000, 8)).astype(np.float32), rng.integers(0, 4, (20, 8)).astype(np.float32)


@pytest.mark.parametrize("kind", ["FLAT", "BruteForce", "IVF_FLAT"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_range_boundaries_bit_exact(kb, kind, metric):
    """Small-integer vectors: every distance is exact in fp32.  radius and range_filter are distances rows attain; L2
    excludes radius and includes range_filter, IP includes range_filter and excludes radius."""
    xb, xq = _int_data()
    n = xb.shape[0]
    Dx = ((xq[:, None, :] - xb[None]) ** 2).sum(-1) if metric == "L2" else xq @ xb.T
    vals = np.unique(Dx)
    lo, hi = vals[len(vals) // 4], vals[len(vals) // 2]
    radius, rf = (float(hi), float(lo)) if metric == "L2" else (float(lo), float(hi))
    assert (Dx == radius).any() and (Dx == rf).any()
    if kind == "IVF_FLAT":
        ix = kb.Index("IVF_FLAT", metric, 8, {"nlist": 16})
        ix.build(xb)
        run = lambda f: ix.range_search(xq, radius, f, {"nprobe": 16, "max_empty_result_buckets": 0})
    elif kind == "FLAT":
        ix = kb.Index("FLAT", metric, 8)
        ix.add(xb)
        run = lambda f: ix.range_search(xq, radius, f)
    else:
        run = lambda f: kb.brute_force_range_search(xb, xq, radius, f, metric)
    for f in (None, rf):
        lims, ids, dist = run(f)
        for i in range(xq.shape[0]):
            want = np.nonzero(in_window(Dx[i], metric, radius, f))[0]
            g, dd = ids[lims[i]:lims[i + 1]], dist[lims[i]:lims[i + 1]]
            assert np.array_equal(np.sort(g), want), f"{kind} {metric} q{i} filter={f}: wrong hit set"
            assert not np.isin(np.nonzero(Dx[i] == radius)[0], g).any(), f"{kind} {metric} q{i}: a row at the radius"
            assert np.isin(np.nonzero(Dx[i] == rf)[0], g).all(), f"{kind} {metric} q{i}: a row at range_filter missing"
            assert np.array_equal(dd, Dx[i, g]), f"{kind} {metric} q{i}: distances not exact"
            key = dd if metric == "L2" else -dd
            assert np.array_equal(g, g[np.lexsort((g, key))]), f"{kind} {metric} q{i}: not in (distance, id) order"
        assert lims[-1] > 0 and lims[-1] < xq.shape[0] * n


# ------------------------------------------------------------------------------------------------ bitsets
@functools.lru_cache(maxsize=1)
def _bitset_data():
    return datagen.clustered(20000, 64, 81), datagen.clustered(100, 64, 82)


@pytest.mark.parametrize("frac", [0.0, 0.5, 0.99, 1.0])
@pytest.mark.parametrize("kind", ["FLAT", "IVF_FLAT", "IVF_PQ-kind1", "IVF_PQ-kind2"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_range_bitset(kb, kind, metric, frac):
    """Bitsets that filter no row, half, 99 % and every row."""
    xb, xq = _bitset_data()
    n, d = xb.shape
    mask = np.random.default_rng(int(frac * 100)).random(n) < frac if frac < 1.0 else np.ones(n, bool)
    bits = bits_of(mask)
    cfg = {"nprobe": 32, "max_empty_result_buckets": 0}
    if kind == "FLAT":
        ix = kb.Index("FLAT", metric, d)
        ix.add(xb)
    elif kind == "IVF_FLAT":
        ix = kb.Index("IVF_FLAT", metric, d, {"nlist": 32})
        ix.build(xb)
    else:
        m = 16 if kind.endswith("kind1") else 8
        ix = kb.Index("IVF_PQ", metric, d, {"nlist": 32, "m": m})
        ix.build(xb)
    if kind.startswith("IVF_PQ"):
        D, B, labels = pq_oracle(ix, xq, m, metric)
    else:
        (D, B), labels = flat_oracle(xb, xq, metric), np.arange(n)
    radius, rf = window_of(D, metric, 0.002, 0.02)
    res = ix.range_search(xq, radius, rf, cfg, bitset=bits)
    hits = check_range(*res, D, B, labels, metric, radius, rf, valid=~mask[labels], what=f"{kind} bitset {frac}")
    assert (hits == 0) == (frac == 1.0)


# ------------------------------------------------------------------------------------------------ hit-buffer overflow
@pytest.mark.parametrize("kind", ["FLAT", "IVF_FLAT"])
def test_range_hit_buffer_overflow_retry(kb, kind):
    """More than 2^20 hits: range_scan's first launch overflows its buffer and a second launch runs into a buffer of
    the reported count.  The launch counter shows the retry; the result still passes the acceptance rule."""
    n, nq, d = 200000, 8, 16
    xb = datagen.uniform(n, d, 61)
    xq = datagen.uniform(nq, d, 62)
    D, B = flat_oracle(xb, xq, "L2")
    cfg = {}
    if kind == "FLAT":
        ix = kb.Index("FLAT", "L2", d)
        ix.add(xb)
    else:
        ix = kb.Index("IVF_FLAT", "L2", d, {"nlist": 64})
        ix.build(xb)
        cfg = {"nprobe": 64, "max_empty_result_buckets": 0}
    small = float(np.quantile(D, 0.01))
    check_range(*ix.range_search(xq, small, None, cfg), D, B, np.arange(n), "L2", small, what=f"{kind} small")
    base = ix.last_counters()["launches"]
    radius = float(np.quantile(D, 0.9))
    res = ix.range_search(xq, radius, None, cfg)
    assert ix.last_counters()["launches"] == base + 1, "the overflowing scan runs a second time"
    hits = check_range(*res, D, B, np.arange(n), "L2", radius, what=f"{kind} overflow")
    assert hits > HIT_CAP


def test_hnsw_graph_range_overflow_matches_reference(kb, ref):
    """HNSW graph path (ef < n / 2) on a 20 000-row integer base with a radius that covers about 95 % of the rows.  Each
    query's BFS queue (16 384 entries) overflows, so every query is rerun with a queue of n entries, and both passes
    overflow the hit buffer and run again: four launches.  Each query's hits are the reference's, bit for bit."""
    n, nq, d, ef = 20000, 100, 32, 32
    rng = np.random.default_rng(29)
    xb = rng.integers(0, 16, (n, d)).astype(np.float32)
    xq = rng.integers(0, 16, (nq, d)).astype(np.float32)
    h = ref.RefHnsw(d, 16, 0, 100)
    h.add(xb)
    g = h.export()
    ix = kb.Index("HNSW", "L2", d, {"M": 16, "efConstruction": 100})
    ix.hnsw_import(xb, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    D = (xq.astype(np.float64) ** 2).sum(1)[:, None] + (xb.astype(np.float64) ** 2).sum(1)[None] - 2.0 * (xq.astype(np.float64) @ xb.T)
    radius = float(np.quantile(D, 0.95)) + 0.5
    lims0, ids0, dis0 = h.range_search(xq, radius, ef, None, 0)
    lims, ids, dis = ix.range_search(xq, radius, config={"ef": ef})
    assert ix.last_counters()["launches"] == 4, ix.last_counters()
    assert lims[-1] > HIT_CAP
    for i in range(nq):
        a = set(zip(ids0[lims0[i]:lims0[i + 1]].tolist(), dis0[lims0[i]:lims0[i + 1]].view(np.uint32).tolist()))
        b = set(zip(ids[lims[i]:lims[i + 1]].tolist(), dis[lims[i]:lims[i + 1]].view(np.uint32).tolist()))
        assert a == b, f"query {i}: {len(a - b)} hits only in the reference, {len(b - a)} only here"


# ------------------------------------------------------------------------------------------------ IVF, every list probed
@functools.lru_cache(maxsize=1)
def _ivf_data():
    n, d = 20000, 64
    rng = np.random.default_rng(83)
    return {"clustered": (datagen.clustered(n, d, 81), datagen.clustered(400, d, 82)),
            "translated": ((1000.0 + rng.standard_normal((n, d))).astype(np.float32),
                           (1000.0 + rng.standard_normal((400, d))).astype(np.float32))}


@pytest.mark.parametrize("nq", [20, 400], ids=["nq20-nsplit14", "nq400-nsplit1"])
@pytest.mark.parametrize("data", ["clustered", "translated"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_ivf_flat_all_lists_range_matches_oracle(kb, metric, data, nq):
    """nprobe = nlist with the empty-probe heuristic off: IVF_FLAT scans every row with direct differences, so its range
    result passes the FLAT oracle, with and without range_filter."""
    xb, xq = _ivf_data()[data]
    xq = xq[:nq]
    n, d = xb.shape
    ix = kb.Index("IVF_FLAT", metric, d, {"nlist": 32})
    ix.build(xb)
    D, B = flat_oracle(xb, xq, metric)
    radius, rf = window_of(D, metric, 0.002, 0.02)
    cfg = {"nprobe": 32, "max_empty_result_buckets": 0}
    assert check_range(*ix.range_search(xq, radius, None, cfg), D, B, np.arange(n), metric, radius,
                       what=f"IVF_FLAT {data}") > 0
    check_range(*ix.range_search(xq, radius, rf, cfg), D, B, np.arange(n), metric, radius, rf, what=f"IVF_FLAT {data} rf")


PQ_KINDS = [pytest.param(16, 128, id="m16-kind1"), pytest.param(48, 96, id="m48-kind1"),
            pytest.param(8, 64, id="m8-kind2"), pytest.param(64, 128, id="m64-kind2")]


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("m,d", PQ_KINDS)
def test_ivfpq_all_lists_range_matches_adc_oracle(kb, m, d, metric):
    """nprobe = nlist with the heuristic off: IVF_PQ's range result passes the ADC oracle, nq below and above 2 * SMs."""
    xb = datagen.clustered(10000, d, 91)
    xq = datagen.clustered(300, d, 92)
    ix = kb.Index("IVF_PQ", metric, d, {"nlist": 32, "m": m, "nbits": 8})
    ix.build(xb)
    D, B, labels = pq_oracle(ix, xq, m, metric)
    radius, rf = window_of(D, metric, 0.002, 0.02)
    cfg = {"nprobe": 32, "max_empty_result_buckets": 0}
    for q in (slice(0, 10), slice(0, 300)):
        assert check_range(*ix.range_search(xq[q].copy(), radius, None, cfg), D[q], B[q], labels, metric, radius,
                           what=f"IVF_PQ m{m} nq={q.stop}") > 0
        check_range(*ix.range_search(xq[q].copy(), radius, rf, cfg), D[q], B[q], labels, metric, radius, rf,
                    what=f"IVF_PQ m{m} nq={q.stop} rf")


# ------------------------------------------------------------------------------------------------ max_empty_result_buckets
def probe_order(cent, xq, metric):
    """every query's lists in coarse order (float64), and whether two consecutive ones lie within a bound of a tie"""
    C, Q = cent.astype(np.float64), xq.astype(np.float64)
    d = C.shape[1]
    if metric == "L2":
        key = ((Q[:, None, :] - C[None]) ** 2).sum(-1)
        S = ((np.abs(Q)[:, None, :] + np.abs(C)[None]) ** 2).sum(-1)
    else:
        key = -(Q @ C.T)
        S = np.abs(Q) @ np.abs(C).T
    bound = 4.0 * (d + 2) * U * S
    order = np.argsort(key, axis=1, kind="stable")
    k, b = np.take_along_axis(key, order, 1), np.take_along_axis(bound, order, 1)
    tie = np.diff(k, axis=1) <= b[:, 1:] + b[:, :-1]
    return order, tie


def heuristic_model(hits, list_of, order, metric, radius, range_filter, max_empty):
    """faiss's rule: walk the probes in coarse order, a probe is empty when it adds no (valid) hit inside the radius,
    stop after the probe that makes max_empty consecutive empty ones; range_filter applies afterwards.  hits: the
    index's own (ids, dist) with the heuristic off and no range_filter.  Returns (kept ids, their distances, the number
    of probes walked, the number of radius hits the cut drops)."""
    ids, dist = hits
    lists = list_of[ids]
    cut, run = len(order), 0
    for j, l in enumerate(order):
        run = run + 1 if not (lists == l).any() else 0
        if run == max_empty:
            cut = j + 1
            break
    walked = np.isin(lists, order[:cut])
    keep = walked & in_window(dist, metric, radius, range_filter)
    return ids[keep], dist[keep], cut, int((~walked).sum())


def _ids_to_list(ix, code_size, nlist, n):
    out = np.full(n, -1, np.int64)
    for l in range(nlist):
        ids, _ = ix.ivf_export_list(l, code_size)
        out[ids] = l
    return out


@functools.lru_cache(maxsize=None)
def _heuristic_index(kb, kind, metric):
    n, d, nlist = 20000, 64, 64
    xb = datagen.clustered(n, d, 121)
    xq = datagen.clustered(100, d, 122)
    m = 16 if kind == "IVF_PQ" else 0
    cfg = {"nlist": nlist, "m": m} if m else {"nlist": nlist}
    ix = kb.Index(kind, metric, d, cfg)
    ix.build(xb)
    cent = ix.ivf_export_centroids(m)[0]
    return ix, xq, cent, _ids_to_list(ix, m if m else 4 * d, nlist, n)


def hits_off(ix, xq, radius):
    """each query's hits with every list probed, the heuristic off and no range_filter"""
    return per_query(*ix.range_search(xq, radius, None, {"nprobe": ix.ivf_nlist(), "max_empty_result_buckets": 0}))


def filter_hiding_nearest_two(off, list_of, order, metric):
    """a range_filter that removes every hit of the two nearest lists for about half the queries"""
    edge = []
    for (ids, dist), o in zip(off, order):
        near = np.isin(list_of[ids], o[:2])
        if near.any():
            edge.append(dist[near].max() if metric == "L2" else dist[near].min())
    e = np.float32(np.median(edge))
    return float(np.nextafter(e, np.float32(np.inf if metric == "L2" else -np.inf)))


def check_heuristic(ix, xq, off, order, tie, list_of, metric, radius, rf, max_empty, what):
    """the heuristic's result against heuristic_model, query by query, exactly; returns (queries checked, queries
    whose cut dropped radius hits)"""
    on = per_query(*ix.range_search(xq, radius, rf, {"nprobe": ix.ivf_nlist(), "max_empty_result_buckets": max_empty}))
    checked = cut_short = 0
    for i in range(xq.shape[0]):
        ids, dist, cut, dropped = heuristic_model(off[i], list_of, order[i], metric, radius, rf, max_empty)
        if tie[i, :cut].any():
            continue
        checked += 1
        cut_short += dropped > 0
        key = dist if metric == "L2" else -dist
        o = np.lexsort((ids, key))
        assert np.array_equal(on[i][0], ids[o]) and np.array_equal(on[i][1], dist[o]), \
            f"{what} q{i}: {on[i][0].size} hits, the model keeps {ids.size} (cut after probe {cut})"
    return checked, cut_short


@pytest.mark.parametrize("filtered", [False, True], ids=["radius", "range_filter"])
@pytest.mark.parametrize("max_empty", [1, 2, 5])
@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("kind", ["IVF_FLAT", "IVF_PQ"])
def test_max_empty_result_buckets_matches_model(kb, kind, metric, max_empty, filtered):
    """The empty-probe heuristic against a numpy model fed with the index's own hits (heuristic off): each row's fp32
    distance does not depend on the probe split, so the comparison is exact.  Queries with a near tie between two
    consecutive probes up to the cut are skipped.  The range_filter removes every hit of the two nearest lists for about
    half the queries: those probes still count as non-empty."""
    ix, xq, cent, list_of = _heuristic_index(kb, kind, metric)
    D = flat_oracle(cent, xq, metric)[0]          # query-to-centroid distances: radii that leave far lists empty
    radius = window_of(D, metric, 0.01, 0.06)[0]
    off = hits_off(ix, xq, radius)
    order, tie = probe_order(cent, xq, metric)
    rf = filter_hiding_nearest_two(off, list_of, order, metric) if filtered else None
    checked, cut_short = check_heuristic(ix, xq, off, order, tie, list_of, metric, radius, rf, max_empty,
                                         f"{kind} {metric} max_empty={max_empty}")
    assert checked >= 0.8 * xq.shape[0]
    assert cut_short > 0, "the heuristic drops hits of some query"


@pytest.mark.parametrize("max_empty", [1, 2])
def test_max_empty_counts_hits_before_range_filter(kb, max_empty):
    """Lists on a line: list j's rows lie about (10 j)^2 from the query.  range_filter removes every hit of the two
    nearest lists; those probes still hold hits inside the radius, so they are not empty and the search goes on to lists
    2 to 4, stopping at the empty lists beyond the radius."""
    d, nlist, per = 8, 8, 40
    rng = np.random.default_rng(3)
    cent = np.zeros((nlist, d), np.float32)
    cent[:, 0] = 10.0 * np.arange(nlist)
    rows = np.concatenate([cent[l] + 0.1 * rng.standard_normal((per, d)).astype(np.float32) for l in range(nlist)])
    lists = [(l, np.arange(l * per, (l + 1) * per, dtype=np.int64), rows[l * per:(l + 1) * per]) for l in range(nlist)]
    ix = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
    ix.ivf_import(cent, None, lists)
    xq = np.zeros((3, d), np.float32)
    radius, rf = 2000.0, 150.0
    lims, ids, dist = ix.range_search(xq, radius, rf, {"nprobe": nlist, "max_empty_result_buckets": max_empty})
    want = np.arange(2 * per, 5 * per)
    for i in range(xq.shape[0]):
        assert np.array_equal(np.sort(ids[lims[i]:lims[i + 1]]), want), f"q{i}: lists 2 to 4 expected"
    list_of = np.repeat(np.arange(nlist), per)
    order, tie = probe_order(cent, xq, "L2")
    checked, _ = check_heuristic(ix, xq, hits_off(ix, xq, radius), order, tie, list_of, "L2", radius, rf, max_empty,
                                 "lists on a line")
    assert checked == xq.shape[0]


# ------------------------------------------------------------------------------------------------ shards on one GPU
def merged(parts, metric):
    """the union of the shards' per-query hits, best first and by id"""
    out = []
    for hits in zip(*[per_query(*p) for p in parts]):
        ids = np.concatenate([h[0] for h in hits])
        dist = np.concatenate([h[1] for h in hits])
        o = np.lexsort((ids, dist if metric == "L2" else -dist))
        out.append((ids[o], dist[o]))
    return out


def assert_union_equal(parts, full, metric, what):
    for i, ((a, ad), (b, bd)) in enumerate(zip(merged(parts, metric), per_query(*full))):
        assert np.array_equal(a, b) and np.array_equal(ad.view(np.uint32), bd.view(np.uint32)), \
            f"{what} q{i}: {a.size} hits over the shards, {b.size} unsharded"


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("kind", ["FLAT", "HNSW-fallback"])
@pytest.mark.parametrize("metric", ["L2", "IP"])
def test_shard_range_with_bitset(kb, kind, metric, world):
    """Row-sliced shards (FLAT, and HNSW with ef >= n / 2, which takes the exact scan): a shard's local row r is global
    row shard_lo + r, in the bitset too.  The union of the shards' hits equals the unsharded result."""
    n, nq, d = 6000, 30, 32
    xb = datagen.uniform(n, d, 71)
    xq = datagen.uniform(nq, d, 72)
    mask = np.random.default_rng(73).random(n) < 0.5
    mask[: n // 2] |= np.arange(n // 2) % 3 == 0          # uneven across the shards
    bits = bits_of(mask)
    D, B = flat_oracle(xb, xq, metric)
    radius, rf = window_of(D, metric, 0.005, 0.05)
    cfg = {"ef": n // 2} if kind.startswith("HNSW") else None

    def make(rank=None):
        ix = kb.Index("HNSW", metric, d, {"M": 8, "efConstruction": 40}) if cfg else kb.Index("FLAT", metric, d)
        if rank is not None:
            ix.set_shard(rank, world)
        ix.build(xb)
        return ix
    full = make().range_search(xq, radius, rf, cfg, bitset=bits)
    assert check_range(*full, D, B, np.arange(n), metric, radius, rf, valid=~mask, what=f"{kind} unsharded") > 0
    parts = [make(r).range_search(xq, radius, rf, cfg, bitset=bits) for r in range(world)]
    assert_union_equal(parts, full, metric, f"{kind} world {world}")


@pytest.mark.parametrize("world", [2, 3])
def test_ivf_flat_shard_range_with_bitset(kb, world):
    """List-sharded IVF_FLAT (one quantizer, each list on one shard) with the heuristic off: the union of the shards' hits
    equals the unsharded result.  (With the heuristic on, lists held by other shards look empty to a shard.)"""
    n, nq, d, nlist = 20000, 50, 64, 32
    xb = datagen.clustered(n, d, 42)
    xq = datagen.clustered(nq, d, 43)
    mask = np.random.default_rng(44).random(n) < 0.3
    bits = bits_of(mask)
    src = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
    src.build(xb)
    cent = src.ivf_export_centroids(0)[0]
    cfg = {"nprobe": nlist, "max_empty_result_buckets": 0}
    D, B = flat_oracle(xb, xq, "L2")
    radius, rf = window_of(D, "L2", 0.002, 0.02)

    def make(rank=None):
        ix = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
        if rank is not None:
            ix.set_shard(rank, world)
        kb._check(kb.lib().kb2_ivf_import_begin(ix.h, nlist, cent.ctypes.data, None))
        ix.add(xb)
        return ix
    full = make().range_search(xq, radius, rf, cfg, bitset=bits)
    assert check_range(*full, D, B, np.arange(n), "L2", radius, rf, valid=~mask, what="IVF_FLAT unsharded") > 0
    parts = [make(r).range_search(xq, radius, rf, cfg, bitset=bits) for r in range(world)]
    assert_union_equal(parts, full, "L2", f"IVF_FLAT world {world}")


def test_flat_shard_several_adds_refuses_bitset(kb):
    """A FLAT shard built by several add() calls does not hold one contiguous slice of global rows, so a bitset cannot be
    mapped: range search refuses it as search does, and still answers without a bitset."""
    n, d = 4000, 16
    xb = datagen.uniform(n, d, 91)
    xq = datagen.uniform(4, d, 92)
    sh = kb.Index("FLAT", "L2", d)
    sh.set_shard(0, 2)
    sh.add(xb[:2000])
    sh.add(xb[2000:])
    bits = bits_of(np.zeros(n, bool))
    want = status_of(kb, lambda: sh.search(xq, 5, bitset=bits))
    assert want[0] == NOT_IMPLEMENTED
    assert status_of(kb, lambda: sh.range_search(xq, 1e9, bitset=bits)) == want
    lims, ids, dist = sh.range_search(xq, 3.0e38)
    assert lims[-1] == 4 * sh.count()


# ------------------------------------------------------------------------------------------------ edges
@functools.lru_cache(maxsize=None)
def _edge_index(kb, kind, metric):
    xb = datagen.clustered(5000, 32, 131)
    ix = kb.Index(kind, metric, 32, {"nlist": 16} if kind == "IVF_FLAT" else None)
    ix.build(xb)
    return ix, xb


@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("kind", ["FLAT", "IVF_FLAT"])
def test_range_edges(kb, kind, metric):
    """nq = 0, a radius with no hit, a radius that includes every row, and queries repeated within one batch."""
    ix, xb = _edge_index(kb, kind, metric)
    n = xb.shape[0]
    xq = datagen.clustered(6, 32, 132)
    cfg = {"nprobe": 16, "max_empty_result_buckets": 0} if kind == "IVF_FLAT" else None
    lims, ids, dist = ix.range_search(xq[:0].copy(), 1.0, None, cfg)
    assert lims.tolist() == [0] and ids.size == 0 and dist.size == 0
    lims, ids, _ = ix.range_search(xq, 0.0 if metric == "L2" else 3.0e38, None, cfg)
    assert (lims == 0).all() and ids.size == 0
    every = 3.0e38 if metric == "L2" else -3.0e38
    D, B = flat_oracle(xb, xq, metric)
    res = ix.range_search(xq, every, None, cfg)
    assert np.array_equal(res[0], np.arange(7) * n)
    check_range(*res, D, B, np.arange(n), metric, every, what=f"{kind} every row")
    rep = np.repeat(xq, 3, axis=0)
    radius = window_of(D, metric, 0.0, 0.05)[0]
    for c in (cfg, {"nprobe": 4} if kind == "IVF_FLAT" else None):
        got = per_query(*ix.range_search(rep, radius, None, c))
        assert sum(g[0].size for g in got) > 0
        for i in range(0, len(got), 3):
            for j in (i + 1, i + 2):
                assert np.array_equal(got[i][0], got[j][0]) and np.array_equal(got[i][1], got[j][1]), f"copy {j} of {i}"


def test_range_dimension_too_large_for_exact_scan(kb):
    """The exact range scan keeps the query in shared memory (4 * dim + 128 bytes, at most 227 KB): one dimension past
    that is refused with a status, and the index and the device keep working."""
    d = (227 * 1024 - 128) // 4 + 1
    n = 64
    xb = datagen.uniform(n, d, 141)
    xq = datagen.uniform(2, d, 142)
    ix = kb.Index("FLAT", "L2", d)
    ix.add(xb)
    st, msg = status_of(kb, lambda: ix.range_search(xq, 1e12))
    assert st == NOT_IMPLEMENTED and "dimension" in msg, msg
    st, msg = status_of(kb, lambda: kb.brute_force_range_search(xb, xq, 1e12, None, "L2"))
    assert st == NOT_IMPLEMENTED, msg
    # k-NN search re-ranks its candidates with the query in shared memory too
    st, msg = status_of(kb, lambda: ix.search(xq, 5))
    assert st == INVALID_ARGS and "dimension" in msg, msg
    more = datagen.uniform(8, d, 143)
    ix.add(more)
    assert ix.count() == n + 8
    assert np.array_equal(ix.get_vector_by_ids(np.array([3, n + 5], np.int64)), np.stack([xb[3], more[5]]))
    small = kb.Index("FLAT", "L2", 16)
    xs = datagen.uniform(1000, 16, 144)
    small.add(xs)
    Ds, Bs = flat_oracle(xs, xs[:4], "L2")
    r = window_of(Ds, "L2", 0.0, 0.05)[0]
    assert check_range(*small.range_search(xs[:4].copy(), r), Ds, Bs, np.arange(1000), "L2", r, what="after refusal") > 0
