"""Generates tests/golden/containers.npz: the bytes of both stream formats, meta() and one search answer for every index
type, so tests/test_containers_gpu.py can hold later code to exactly what this code writes and answers.
Run on an H100:  python tests/golden/make_container_golden.py [out.npz]

For each case the file holds
- B0 = serialize() of the index and B1 = serialize(deserialize(B0)) (B1 only where it differs from B0),
- F0 = serialize_faiss() and F1 = serialize_faiss(deserialize_faiss(F0)) where the type has a faiss stream (F1 only
  where it differs from F0),
- meta() of deserialize(B0) and the ids and distance bits of one search of it,
- the build recipe (type, metric, create config, custom ids or not) when two builds from it gave the same B0, so the test
  can rebuild the index from its JSON and compare."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import knowhere_b200 as kb  # noqa: E402
from knowhere_b200 import datagen  # noqa: E402

N, D, NQ, K = 400, 16, 8, 10
X = datagen.clustered(N, D, 42)
Q = datagen.clustered(NQ, D, 43)
IDS = (1000 + 7 * np.arange(N)).astype(np.int64)
DOC_LIMS = np.arange(0, N + 1, 5, dtype=np.int64)          # 80 documents of 5 rows
Q_LIMS = np.array([0, 3, 5, 8], dtype=np.int64)            # 3 query lists over the NQ query rows


def built(recipe):
    ix = kb.Index(recipe["type"], recipe["metric"], D, recipe["config"])
    ix.build(X, IDS if recipe["ids"] else None)
    return ix


def hnsw_imported():
    g = built(dict(type="HNSW", metric="L2", config={"M": 8, "efConstruction": 40}, ids=False)).hnsw_export()
    ix = kb.Index("HNSW", "L2", D, {"M": 8, "efConstruction": 40})
    ix.hnsw_import(X, g["levels"], g["offsets"], g["neighbors"], g["cum"], g["entry_point"], g["max_level"])
    return ix


def hnsw_emb_list():
    ix = hnsw_imported()
    ix.set_emb_list(DOC_LIMS, "MAX_SIM_L2")
    return ix


def recipe(type_, metric, config, ids=False):
    return dict(type=type_, metric=metric, config=config, ids=ids)


PQ = {"nlist": 8, "m": 4, "nbits": 8}
# name: (recipe or maker, search config, emb-list search)
CASES = {
    "flat_l2": (recipe("FLAT", "L2", {}), {}, False),
    "flat_ip_ids": (recipe("FLAT", "IP", {}, ids=True), {}, False),
    "flat_cosine": (recipe("FLAT", "COSINE", {}), {}, False),
    "ivf_flat": (recipe("IVF_FLAT", "L2", {"nlist": 8}), {"nprobe": 4}, False),
    "ivf_pq": (recipe("IVF_PQ", "L2", PQ), {"nprobe": 4}, False),
    "ivf_pq_refine_fp32": (recipe("IVF_PQ", "L2", dict(PQ, refine=True, refine_type="flat")), {"nprobe": 4, "refine_k": 2}, False),
    "ivf_pq_refine_fp16": (recipe("IVF_PQ", "IP", dict(PQ, refine=True, refine_type="fp16")), {"nprobe": 4, "refine_k": 2}, False),
    "hnsw_imported": (hnsw_imported, {"ef": 32}, False),
    "hnsw_ids": (recipe("HNSW", "IP", {"M": 8, "efConstruction": 40}, ids=True), {"ef": 32}, False),
    "cagra": (recipe("GPU_CAGRA", "L2", {"intermediate_graph_degree": 32, "graph_degree": 16}), {}, False),
    "hnsw_emb_list": (hnsw_emb_list, {"ef": 32}, True),
}


def search(ix, cfg, emb):
    if emb:
        return ix.search_emb_list(Q, Q_LIMS, 5, cfg)
    return ix.search(Q, K, cfg)


def blob(b):
    return np.frombuffer(b, np.uint8)


def main(out_path):
    out = {}
    for name, (how, cfg, emb) in CASES.items():
        make = how if callable(how) else (lambda r=how: built(r))
        ix = make()
        b0 = ix.serialize()
        again = make().serialize()
        dx = kb.Index.deserialize(b0)
        out[f"{name}/B0"] = blob(b0)
        b1 = dx.serialize()
        if b1 != b0:
            out[f"{name}/B1"] = blob(b1)
        out[f"{name}/meta"] = np.array(json.dumps(dx.meta()))
        out[f"{name}/search_cfg"] = np.array(json.dumps(cfg))
        ids, dist = search(dx, cfg, emb)
        out[f"{name}/ids"], out[f"{name}/dist_bits"] = ids, dist.view(np.uint32)
        try:
            f0 = ix.serialize_faiss()
        except kb.KnowhereError as e:
            print(f"{name}: no faiss stream ({e})")
        else:
            out[f"{name}/F0"] = blob(f0)
            f1 = kb.Index.deserialize_faiss(f0).serialize_faiss()
            if f1 != f0:
                out[f"{name}/F1"] = blob(f1)
        if not callable(how) and b0 == again:
            out[f"{name}/recipe"] = np.array(json.dumps(how))
        print(f"{name}: B0 {len(b0)} bytes, rebuild {'deterministic' if b0 == again else 'not deterministic'}")
    np.savez_compressed(out_path, **out)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "containers.npz"))
