"""Item widths of the IVF_PQ filter kernel (kb2_ivfpq_tc.cuh) against the query-major LUT engine.

The consumer warpgroups run one unrolled wgmma pipeline per item width in 16-column units (1 to 16): each 64-code half of
a tile is contracted in blocks of near-equal width, at most MAXW columns each.  With nprobe == nlist every list is probed
by every query of the batch, so the batch size sets the width of every item: nq = 16 c - 5 lands in width class c, nq = 1
in the narrowest, and 300 is cut into two items.  Each width must return the LUT engine's rows bit
for bit, for both metrics and both geometries of the engine."""
import os

import numpy as np
import pytest

from knowhere_b200 import datagen

pytestmark = pytest.mark.gpu

BATCHES = [1] + [16 * c - 5 for c in range(1, 17)] + [300]


def _search(ix, xq, k, cfg, engine):
    old = os.environ.get("KB2_PQ_ENGINE")
    os.environ["KB2_PQ_ENGINE"] = engine
    try:
        return ix.search(xq, k, cfg)
    finally:
        if old is None:
            os.environ.pop("KB2_PQ_ENGINE", None)
        else:
            os.environ["KB2_PQ_ENGINE"] = old


@pytest.fixture(scope="module")
def indexes(kb):
    nb, nlist, out = 20000, 16, {}
    for metric in ("L2", "IP"):
        for d, m in ((128, 16), (96, 48)):
            ix = kb.Index("IVF_PQ", metric, d, {"nlist": nlist, "m": m, "nbits": 8})
            xb = datagen.clustered(nb, d, 11)
            ix.train(xb)
            ix.add(xb)
            out[metric, d] = ix
    return out


@pytest.mark.parametrize("nq", BATCHES)
@pytest.mark.parametrize("metric", ["L2", "IP"])
@pytest.mark.parametrize("d", [128, 96])
def test_ivfpq_tc_engine_every_width(indexes, metric, d, nq):
    nb, nlist, k = 20000, 16, 10
    ix = indexes[metric, d]
    cfg = {"nprobe": nlist}
    xq = datagen.clustered(nq, d, 12)
    i0, d0 = _search(ix, xq, k, cfg, "lut")
    i1, d1 = _search(ix, xq, k, cfg, "tc")
    assert ix.last_stage_info()["engine"] == "tc", f"nq={nq}: tensor-core engine was not selected"
    assert ix.last_counters()["codes"] >= nq * nb, f"nq={nq}: the filter pass did not scan every (query, code) pair"
    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32)), f"nq={nq}: distances differ in {(d0 != d1).any(axis=1).sum()} rows"
    assert np.array_equal(i0, i1), f"nq={nq}: ids differ in {(i0 != i1).any(axis=1).sum()} rows"
