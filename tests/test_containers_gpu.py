"""Both stream formats, meta() and a search of the loaded index, byte for byte and bit for bit against
tests/golden/containers.npz (written by tests/golden/make_container_golden.py): every index type's KB2I section, faiss
conversion, meta fields and build keys stay exactly as they were."""
import json
import os

import numpy as np
import pytest

from tests.golden import make_container_golden as g

pytestmark = pytest.mark.gpu
Z = np.load(os.path.join(os.path.dirname(__file__), "golden", "containers.npz"))


def _case(name, what, default=None):
    key = f"{name}/{what}"
    return Z[key] if key in Z.files else default


@pytest.mark.parametrize("name", sorted(g.CASES))
def test_container_round_trip(kb, name):
    b0 = _case(name, "B0").tobytes()
    dx = kb.Index.deserialize(b0)
    assert dx.serialize() == _case(name, "B1", _case(name, "B0")).tobytes()
    assert dx.meta() == json.loads(str(_case(name, "meta")))
    ids, dist = g.search(dx, json.loads(str(_case(name, "search_cfg"))), g.CASES[name][2])
    np.testing.assert_array_equal(ids, _case(name, "ids"))
    np.testing.assert_array_equal(dist.view(np.uint32), _case(name, "dist_bits"))
    f0 = _case(name, "F0")
    if f0 is not None:
        assert kb.Index.deserialize_faiss(f0.tobytes()).serialize_faiss() == _case(name, "F1", f0).tobytes()
    recipe = _case(name, "recipe")
    if recipe is not None:
        assert g.built(json.loads(str(recipe))).serialize() == b0


def test_cagra_refusals(kb):
    ix = g.built(g.recipe("GPU_CAGRA", "L2", {"intermediate_graph_degree": 32, "graph_degree": 16}))
    hn = g.built(g.recipe("HNSW", "L2", {"M": 8, "efConstruction": 40})).hnsw_export()
    with pytest.raises(kb.KnowhereError) as e:
        ix.hnsw_import(g.X, hn["levels"], hn["offsets"], hn["neighbors"], hn["cum"], hn["entry_point"], hn["max_level"])
    assert e.value.status == 7
    with pytest.raises(kb.KnowhereError) as e:
        ix.range_search(g.Q[:0], 100.0)
    assert e.value.status == 7
