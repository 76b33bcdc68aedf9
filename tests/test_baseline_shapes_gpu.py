"""Id-level parity at the BASELINE shapes (VERDICT r1 "parity holes"): the index is built on the GPU, exported, and the
SAME index is searched by the compiled reference (faiss IndexIVFFlat / IndexIVFPQ + IndexRefine from oracle/_ref); ids
must be identical up to exact-distance boundary ties, distances within 1e-4 relative (tests/ut/test_search.cc:185-268 is
the reference's own, much weaker, recall > 0.6 check for these index types)."""
import numpy as np
import pytest

from knowhere_b200 import datagen
from tests.util import assert_topk_parity, recall_at_k

pytestmark = pytest.mark.gpu


def _export(ref, ix, kind, d, nlist, m, xb, refine):
    r = ref.RefIvf(kind, d, 0, nlist, m, 8, refine=refine)
    cent, pq = ix.ivf_export_centroids(m)
    cs = m if m else d * 4
    r.import_state(cent, pq, ((l,) + ix.ivf_export_list(l, cs) for l in range(nlist)), raw=xb if refine else None)
    return r


def test_c2_shape_ivfflat_1m(kb, ref):
    """C2: IVF_FLAT L2 1M x 128, nlist 1024, nprobe 32, batch 1000, k 10"""
    n, d, nlist, nprobe, nq, k = 1_000_000, 128, 1024, 32, 1000, 10
    xb = datagen.clustered(n, d, 42)
    xq = datagen.clustered(nq, d, 43)
    ix = kb.Index("IVF_FLAT", "L2", d, {"nlist": nlist})
    ix.build(xb)
    ix.enable_kernel_timing(True)
    ids, dist = ix.search(xq, k, {"nprobe": nprobe})
    assert ix.last_stage_info()["engine"] == "tc"      # the list-major tensor-core engine serves this shape
    r = _export(ref, ix, "IVF_FLAT", d, nlist, 0, xb, False)
    I0, D0 = r.search(xq, k, nprobe)
    assert_topk_parity(ids, dist, I0, D0, rtol=1e-4, atol=1e-4, what="C2 IVF_FLAT 1M", max_tie_rows=nq // 100)
    print("C2 shape: identical rows", (ids == I0).all(1).mean())
    assert (ids == I0).all(1).mean() > 0.99


@pytest.mark.parametrize("refine_k", [1, 4])
def test_c3_params_ivfpq_1m(kb, ref, refine_k):
    """C3 parameters (m 16, nbits 8, nlist 4096, nprobe 64, batch 10000, k 10) on a 1M x 128 index: the batch goes
    through the list-major tensor-core engine; compared with the reference's IndexIVFPQ(+IndexRefine) on the same index."""
    n, d, nlist, m, nprobe, nq, k = 1_000_000, 128, 4096, 16, 64, 10000, 10
    xb = datagen.clustered(n, d, 42)
    xq = datagen.clustered(nq, d, 43)
    ix = kb.Index("IVF_PQ", "L2", d, {"nlist": nlist, "m": m, "nbits": 8, "refine": True, "refine_type": "flat"})
    ix.build(xb)
    ix.enable_kernel_timing(True)
    ids, dist = ix.search(xq, k, {"nprobe": nprobe, "refine_k": refine_k})
    assert ix.last_stage_info()["engine"] == "tc"
    r = _export(ref, ix, "IVF_PQ", d, nlist, m, xb, True)
    I0, D0 = r.search(xq, k, nprobe, refine_k=float(refine_k))
    same = (ids == I0).all(1).mean()
    print(f"C3 params refine_k={refine_k}: identical rows {same:.4f}")
    # refine_k=1: ADC distances tie for identical codes => boundary ties; with refine the exact distances separate them
    assert_topk_parity(ids, dist, I0, D0, rtol=1e-4, atol=1e-3, what="C3-params IVF_PQ 1M",
                       max_tie_rows=nq // (10 if refine_k == 1 else 200))
    gt, _ = ref.flat_search(xb, xq[:500], k, 0)
    assert recall_at_k(gt, ids[:500]) >= recall_at_k(gt, I0[:500]) - 1e-9
