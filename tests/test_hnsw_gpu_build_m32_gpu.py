"""HNSW built on the GPU with M = 32: level 0 rows of 2M = 64 links, the widest the link kernel keeps.  A full row re-selected
with the new node is 65 candidates (hnsw_link_kernel's kLinkSlots)."""
import numpy as np
import pytest

from knowhere_b200 import datagen
from tests.util import recall_at_k

pytestmark = pytest.mark.gpu


def test_gpu_build_m32(kb):
    X = datagen.clustered(30000, 32, 3)
    Q = datagen.clustered(200, 32, 4)
    ix = kb.Index("HNSW", "L2", 32, {"M": 32, "efConstruction": 64})
    ix.build(X)
    g = ix.hnsw_export()
    assert g["cum"][1] == 64 and (g["neighbors"] < 30000).all()
    flat = kb.Index("FLAT", "L2", 32)
    flat.build(X)
    gt, _ = flat.search(Q, 10)
    ids, _ = ix.search(Q, 10, {"ef": 64})
    assert recall_at_k(gt, ids) >= 0.9
