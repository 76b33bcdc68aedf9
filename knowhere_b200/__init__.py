"""knowhere_b200 — host-side Python binding of the H100-native ANN search core.

This is only the ctypes stub over the C ABI in include/knowhere_b200.h (the product is the
CUDA library).  There is NO CPU fallback: if the shared library is missing the import fails
loudly, and every call fails with status 22 (cuda_runtime_error) when no sm_90 GPU is present.
"""
import ctypes
import json
import os

import numpy as np

from ._build import LIB, build  # noqa: F401

METRIC_L2, METRIC_IP = 0, 1
_METRICS = {"L2": 0, "IP": 1, "COSINE": 2, "BM25": 6, 0: 0, 1: 1, 2: 2, 6: 6}

_lib = None


class KnowhereError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"knowhere status {status}: {msg}")
        self.status = status


def lib():
    global _lib
    if _lib is None:
        path = os.environ.get("KB2_LIB", LIB)   # development aid: A/B two builds on the same box
        if not os.path.exists(path):
            raise ImportError(
                f"{LIB} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        _lib = ctypes.CDLL(path)
        _declare(_lib)
    return _lib


def _declare(L):
    c = ctypes
    vp, i64, i32, f32 = c.c_void_p, c.c_int64, c.c_int, c.c_float
    L.kb2_version.restype = c.c_char_p
    L.kb2_last_error.restype = c.c_char_p
    L.kb2_device_count.restype = i32
    L.kb2_index_create.argtypes = [c.c_char_p, i32, i32, c.c_char_p, i32, c.POINTER(vp)]
    L.kb2_index_destroy.argtypes = [vp]
    L.kb2_index_destroy.restype = None
    L.kb2_index_set_stream.argtypes = [vp, vp]
    L.kb2_index_set_shard.argtypes = [vp, i32, i32]
    L.kb2_index_train.argtypes = [vp, vp, i64]
    L.kb2_index_train_typed.argtypes = [vp, vp, i32, i64]
    L.kb2_index_add_typed.argtypes = [vp, vp, i32, i64, vp]
    L.kb2_index_search_typed.argtypes = [vp, vp, i32, i64, i32, c.c_char_p, vp, i64, vp, vp]
    L.kb2_index_add.argtypes = [vp, vp, i64, vp]
    L.kb2_index_search.argtypes = [vp, vp, i64, i32, c.c_char_p, vp, i64, vp, vp]
    L.kb2_index_range_search.argtypes = [vp, vp, i64, f32, f32, i32, c.c_char_p, vp, i64,
                                         c.POINTER(vp), c.POINTER(vp), c.POINTER(vp)]
    L.kb2_free.argtypes = [vp]
    L.kb2_free.restype = None
    L.kb2_index_count.argtypes = [vp]
    L.kb2_index_count.restype = i64
    L.kb2_index_dim.argtypes = [vp]
    L.kb2_index_size_bytes.argtypes = [vp]
    L.kb2_index_size_bytes.restype = i64
    L.kb2_index_is_trained.argtypes = [vp]
    L.kb2_index_has_raw_data.argtypes = [vp]
    L.kb2_index_get_vector_by_ids.argtypes = [vp, vp, i64, vp]
    L.kb2_ivf_import_begin.argtypes = [vp, i64, vp, vp]
    L.kb2_ivf_import_list.argtypes = [vp, i64, i64, vp, vp]
    L.kb2_ivf_import_finish.argtypes = [vp, vp, i64]
    L.kb2_ivf_nlist.argtypes = [vp]
    L.kb2_ivf_nlist.restype = i64
    L.kb2_ivf_list_size.argtypes = [vp, i64]
    L.kb2_ivf_list_size.restype = i64
    L.kb2_ivf_export_centroids.argtypes = [vp, vp, vp]
    L.kb2_ivf_export_list.argtypes = [vp, i64, vp, vp]
    L.kb2_hnsw_import.argtypes = [vp, i64, vp, vp, vp, vp, vp, i32, c.c_int32, c.c_int32]
    L.kb2_hnsw_export_meta.argtypes = [vp, vp]
    L.kb2_hnsw_export.argtypes = [vp, vp, vp, vp, vp]
    L.kb2_hnsw_last_stats.argtypes = [vp, vp]
    L.kb2_index_serialize.argtypes = [vp, c.POINTER(vp), c.POINTER(c.c_size_t)]
    L.kb2_index_deserialize.argtypes = [vp, c.c_size_t, i32, c.POINTER(vp)]
    L.kb2_bruteforce_search.argtypes = [vp, i64, i32, i32, vp, i64, i32, vp, i64, vp, vp, i32, vp]
    L.kb2_bruteforce_range_search.argtypes = [vp, i64, i32, i32, vp, i64, f32, f32, i32, vp, i64,
                                              c.POINTER(vp), c.POINTER(vp), c.POINTER(vp), i32, vp]
    L.kb2_bruteforce_search_emb_list.argtypes = [vp, vp, i64, i32, i32, vp, vp, i64, i32, vp, i64, vp, vp, vp, i32, vp]
    L.kb2_merge_topk.argtypes = [i32, i32, i64, i32, vp, vp, vp, vp, i32, vp]
    L.kb2_index_set_emb_list.argtypes = [vp, vp, i64, i32]
    L.kb2_index_emb_list_offsets.argtypes = [vp, vp, vp]
    L.kb2_index_search_emb_list.argtypes = [vp, vp, vp, i64, i32, c.c_char_p, vp, i64, vp, vp, vp]
    L.kb2_index_emb_list_stage_ms.argtypes = [vp, vp]
    L.kb2_index_add_sparse.argtypes = [vp, vp, vp, vp, i64]
    L.kb2_index_search_sparse.argtypes = [vp, vp, vp, vp, i64, i32, c.c_char_p, vp, i64, vp, vp]
    L.kb2_index_range_search_sparse.argtypes = [vp, vp, vp, vp, i64, f32, f32, i32, c.c_char_p, vp, i64,
                                                c.POINTER(vp), c.POINTER(vp), c.POINTER(vp)]
    L.kb2_bruteforce_search_sparse.argtypes = [vp, vp, vp, i64, vp, vp, vp, i64, i32, i32, c.c_char_p, vp, i64, vp, vp, i32]
    L.kb2_debug_cagra_knn_graph.argtypes = [vp, i64, i32, i32, c.c_char_p, vp, vp, vp, vp, i32, vp, i32]
    L.kb2_debug_muvera_encode.argtypes = [vp, vp, i64, i32, i32, i32, i32, i32, vp, vp, i32]
    if hasattr(L, "kb2_faiss_describe"):
        L.kb2_faiss_describe.argtypes = [vp, c.c_size_t, i32, vp, c.c_size_t]
        L.kb2_faiss_rewrite.argtypes = [vp, c.c_size_t, i32, c.POINTER(vp), c.POINTER(c.c_size_t)]
        L.kb2_index_deserialize_faiss.argtypes = [vp, c.c_size_t, i32, i32, c.POINTER(vp)]
        L.kb2_index_serialize_faiss.argtypes = [vp, c.POINTER(vp), c.POINTER(c.c_size_t)]
        L.kb2_index_deserialize_from_file.argtypes = [c.c_char_p, i32, c.POINTER(vp)]
        L.kb2_index_get_meta.argtypes = [vp, vp, c.c_size_t]
    if hasattr(L, "kb2_comm_unique_id"):   # (a stale build without the communicator API fails at Comm(), not at import)
        L.kb2_comm_unique_id.argtypes = [vp]
        L.kb2_comm_create.argtypes = [vp, i32, i32, i32, c.POINTER(vp)]
        L.kb2_comm_destroy.argtypes = [vp]
        L.kb2_comm_destroy.restype = None
        L.kb2_comm_all_gather.argtypes = [vp, vp, vp, c.c_size_t, vp]
        L.kb2_index_set_comm.argtypes = [vp, vp]
    L.kb2_index_last_search_counters.argtypes = [vp, vp]
    L.kb2_index_enable_kernel_timing.argtypes = [vp, i32]
    L.kb2_index_last_kernel_ms.argtypes = [vp, c.POINTER(f32)]
    L.kb2_index_last_stage_info.argtypes = [vp, vp]


def _check(status):
    if status != 0:
        raise KnowhereError(status, lib().kb2_last_error().decode())


def _ptr(a):
    """numpy array / torch tensor / None -> raw address."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data
    if hasattr(a, "data_ptr"):  # torch tensor (plumbing for device memory)
        assert a.is_contiguous()
        return a.data_ptr()
    raise TypeError(type(a))


def _is_torch(a):
    return hasattr(a, "data_ptr")


def _dtype_code(a):
    """KB2_DTYPE_* of a numpy array / torch tensor (fp32 0, fp16 1, bf16 2, int8 3)"""
    name = str(a.dtype).replace("torch.", "")
    code = {"float32": 0, "float16": 1, "bfloat16": 2, "int8": 3}.get(name)
    if code is None:
        raise TypeError(f"unsupported element type {a.dtype}")
    return code


def _cfg(cfg):
    return json.dumps(cfg or {}).encode()


def device_count():
    return lib().kb2_device_count()


def version():
    return lib().kb2_version().decode()


class Index:
    """Mirror of knowhere::Index<IndexNode> (reference include/knowhere/index/index.h:160-235) over the C ABI."""

    def __init__(self, index_type, metric="L2", dim=0, config=None, device=0, _handle=None):
        self.L = lib()
        self.h = ctypes.c_void_p()
        self.type = index_type
        if _handle is not None:
            self.h = _handle
            self.dim = self.L.kb2_index_dim(self.h)
            return
        self.dim = dim
        _check(self.L.kb2_index_create(index_type.encode(), _METRICS[metric], dim, _cfg(config), device,
                                       ctypes.byref(self.h)))

    def __del__(self):
        try:
            if self.h:
                self.L.kb2_index_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # -- Build = Train + Add (index_node.h:100-104)
    def train(self, x):
        _check(self.L.kb2_index_train_typed(self.h, _ptr(x), _dtype_code(x), x.shape[0]))

    def add(self, x, ids=None):
        _check(self.L.kb2_index_add_typed(self.h, _ptr(x), _dtype_code(x), x.shape[0], _ptr(ids)))

    def build(self, x, ids=None):
        self.train(x)
        self.add(x, ids)

    def set_stream(self, cuda_stream):
        _check(self.L.kb2_index_set_stream(self.h, ctypes.c_void_p(cuda_stream)))

    def set_shard(self, rank, world):
        _check(self.L.kb2_index_set_shard(self.h, rank, world))

    def set_comm(self, comm):
        """attach a Comm: search() on this sharded index becomes a collective returning the merged global top-k"""
        self._comm = comm   # keep it alive
        _check(self.L.kb2_index_set_comm(self.h, comm.h if comm is not None else None))

    def search(self, q, k, config=None, bitset=None, out=None):
        """q: [nq, dim] float32 numpy (host) or torch cuda tensor (device).  Returns (ids, dist)."""
        nq = q.shape[0]
        if out is not None:
            ids, dist = out
        elif _is_torch(q) and q.is_cuda:
            import torch
            ids = torch.empty((nq, k), dtype=torch.int64, device=q.device)
            dist = torch.empty((nq, k), dtype=torch.float32, device=q.device)
        else:
            ids = np.empty((nq, k), np.int64)
            dist = np.empty((nq, k), np.float32)
        nbits = 0 if bitset is None else (bitset.numel() if _is_torch(bitset) else bitset.size) * 8
        _check(self.L.kb2_index_search_typed(self.h, _ptr(q), _dtype_code(q), nq, k, _cfg(config), _ptr(bitset), nbits,
                                             _ptr(ids), _ptr(dist)))
        return ids, dist

    def range_search(self, q, radius, range_filter=None, config=None, bitset=None):
        nq = q.shape[0]
        pl, pi, pd = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        nbits = 0 if bitset is None else bitset.size * 8
        _check(self.L.kb2_index_range_search(self.h, _ptr(q), nq, radius,
                                             0.0 if range_filter is None else range_filter,
                                             0 if range_filter is None else 1, _cfg(config), _ptr(bitset), nbits,
                                             ctypes.byref(pl), ctypes.byref(pi), ctypes.byref(pd)))
        return _take_range(self.L, nq, pl, pi, pd)

    def count(self):
        return self.L.kb2_index_count(self.h)

    def size(self):
        return self.L.kb2_index_size_bytes(self.h)

    def is_trained(self):
        return bool(self.L.kb2_index_is_trained(self.h))

    def has_raw_data(self):
        return bool(self.L.kb2_index_has_raw_data(self.h))

    def get_vector_by_ids(self, ids):
        ids = np.ascontiguousarray(ids, np.int64)
        out = np.empty((ids.size, self.dim), np.float32)
        _check(self.L.kb2_index_get_vector_by_ids(self.h, _ptr(ids), ids.size, _ptr(out)))
        return out

    # -- import / export of trained state
    def ivf_import(self, centroids, pq_centroids, lists, raw=None):
        """lists: iterable of (list_no, ids int64[n], codes uint8[n*code_size])."""
        nlist = centroids.shape[0]
        _check(self.L.kb2_ivf_import_begin(self.h, nlist, _ptr(centroids), _ptr(pq_centroids)))
        for l, ids, codes in lists:
            if len(ids):
                _check(self.L.kb2_ivf_import_list(self.h, l, len(ids), _ptr(np.ascontiguousarray(ids, np.int64)),
                                                  _ptr(np.ascontiguousarray(codes).view(np.uint8).reshape(-1))))
        _check(self.L.kb2_ivf_import_finish(self.h, _ptr(raw), 0 if raw is None else raw.shape[0]))

    def ivf_nlist(self):
        return self.L.kb2_ivf_nlist(self.h)

    def ivf_export_centroids(self, m=0):
        nlist = self.ivf_nlist()
        c = np.empty((nlist, self.dim), np.float32)
        pq = np.empty((m, 256, self.dim // m), np.float32) if m else None
        _check(self.L.kb2_ivf_export_centroids(self.h, _ptr(c), _ptr(pq)))
        return c, pq

    def ivf_export_list(self, l, code_size):
        n = self.L.kb2_ivf_list_size(self.h, l)
        ids = np.empty(n, np.int64)
        codes = np.empty((n, code_size), np.uint8)
        if n:
            _check(self.L.kb2_ivf_export_list(self.h, l, _ptr(ids), _ptr(codes)))
        return ids, codes

    def hnsw_import(self, vectors, levels, offsets, neighbors, cum, entry_point, max_level):
        _check(self.L.kb2_hnsw_import(self.h, vectors.shape[0], _ptr(vectors), _ptr(levels), _ptr(offsets),
                                      _ptr(neighbors), _ptr(cum), len(cum), entry_point, max_level))

    def hnsw_export(self):
        meta = np.zeros(5, np.int64)
        _check(self.L.kb2_hnsw_export_meta(self.h, _ptr(meta)))
        n, ep, ml, nl, nc = [int(v) for v in meta]
        levels = np.empty(n, np.int32)
        offsets = np.empty(n + 1, np.int64)
        neighbors = np.empty(nl, np.int32)
        cum = np.empty(nc, np.int32)
        _check(self.L.kb2_hnsw_export(self.h, _ptr(levels), _ptr(offsets), _ptr(neighbors), _ptr(cum)))
        return dict(levels=levels, offsets=offsets, neighbors=neighbors, cum=cum, entry_point=ep, max_level=ml)

    def hnsw_last_stats(self):
        s = np.zeros(2, np.int64)
        _check(self.L.kb2_hnsw_last_stats(self.h, _ptr(s)))
        return int(s[0]), int(s[1])

    def serialize(self):
        p, n = ctypes.c_void_p(), ctypes.c_size_t()
        _check(self.L.kb2_index_serialize(self.h, ctypes.byref(p), ctypes.byref(n)))
        try:
            return ctypes.string_at(p, n.value)
        finally:
            self.L.kb2_free(p)

    @staticmethod
    def deserialize(blob, device=0):
        L = lib()
        h = ctypes.c_void_p()
        buf = ctypes.create_string_buffer(blob, len(blob))
        _check(L.kb2_index_deserialize(ctypes.cast(buf, ctypes.c_void_p), len(blob), device, ctypes.byref(h)))
        return Index("?", _handle=h)

    # -- the reference's wire format (faiss fourcc stream = the BinarySet payload)
    def serialize_faiss(self):
        p, n = ctypes.c_void_p(), ctypes.c_size_t()
        _check(self.L.kb2_index_serialize_faiss(self.h, ctypes.byref(p), ctypes.byref(n)))
        try:
            return ctypes.string_at(p, n.value)
        finally:
            self.L.kb2_free(p)

    @staticmethod
    def deserialize_faiss(blob, device=0, with_norm=False):
        L = lib()
        h = ctypes.c_void_p()
        buf = ctypes.create_string_buffer(blob, len(blob))
        _check(L.kb2_index_deserialize_faiss(ctypes.cast(buf, ctypes.c_void_p), len(blob), 1 if with_norm else 0, device,
                                             ctypes.byref(h)))
        return Index("?", _handle=h)

    @staticmethod
    def deserialize_from_file(path, device=0):
        L = lib()
        h = ctypes.c_void_p()
        _check(L.kb2_index_deserialize_from_file(path.encode(), device, ctypes.byref(h)))
        return Index("?", _handle=h)

    def meta(self):
        buf = ctypes.create_string_buffer(1024)
        _check(self.L.kb2_index_get_meta(self.h, ctypes.cast(buf, ctypes.c_void_p), 1024))
        return json.loads(buf.value.decode())

    # -- emb-lists (multi-vector documents) on HNSW / IVF_FLAT: the reference's TokenANN strategy, or MUVERA with the create
    #    keys {"emb_list_strategy": "muvera", "muvera_num_projections": P, "muvera_num_repeats": R, "muvera_seed": S}
    #    (DESIGN §4.11)
    def set_emb_list(self, lims, metric):
        """attach document offsets (int64 [n_docs + 1], ending at count()) and the MAX_SIM metric that pairs with the
        index metric (MAX_SIM_L2 - L2, MAX_SIM_IP - IP, MAX_SIM / MAX_SIM_COSINE - COSINE); on a MUVERA index this
        encodes the documents and builds the base index over them"""
        lims = lims if _is_torch(lims) else np.ascontiguousarray(lims, np.int64)
        _check(self.L.kb2_index_set_emb_list(self.h, _ptr(lims), int(lims.shape[0]) - 1,
                                             _EMB_METRICS.get(str(metric).upper(), -1)))

    def emb_list_offsets(self):
        n = ctypes.c_int64()
        _check(self.L.kb2_index_emb_list_offsets(self.h, ctypes.byref(n), None))
        lims = np.empty(n.value + 1, np.int64)
        _check(self.L.kb2_index_emb_list_offsets(self.h, ctypes.byref(n), _ptr(lims)))
        return lims

    def search_emb_list(self, q, q_lims, k, config=None, bitset=None, stats=False):
        """q: [rows, dim] float32 query tokens, q_lims: int64 [n_lists + 1] (numpy or CUDA tensors).  Returns (ids, dist)
        [n_lists, k] (CUDA tensors when q is), documents best first; with stats=True also int64 [query lists,
        candidates re-ranked, token x row distances].  config: retrieval_ann_ratio (default 3), emb_list_rerank (MUVERA,
        default true) and the base search keys; bitset: one bit per document."""
        if not _is_torch(q_lims):
            q_lims = np.ascontiguousarray(q_lims, np.int64)
        n_lists = int(q_lims.shape[0]) - 1
        if _is_torch(q) and q.is_cuda:
            import torch
            ids = torch.empty((n_lists, k), dtype=torch.int64, device=q.device)
            dist = torch.empty((n_lists, k), dtype=torch.float32, device=q.device)
        else:
            ids = np.empty((n_lists, k), np.int64)
            dist = np.empty((n_lists, k), np.float32)
        st = np.zeros(3, np.int64)
        nbits = 0 if bitset is None else (bitset.numel() if _is_torch(bitset) else bitset.size) * 8
        _check(self.L.kb2_index_search_emb_list(self.h, _ptr(q), _ptr(q_lims), n_lists, k, _cfg(config), _ptr(bitset),
                                                nbits, _ptr(ids), _ptr(dist), _ptr(st)))
        return (ids, dist, st) if stats else (ids, dist)

    def emb_list_stage_ms(self):
        """device ms of the last search_emb_list's stages (with enable_kernel_timing): stage 1, candidates, re-rank,
        select"""
        v = np.zeros(4, np.float32)
        _check(self.L.kb2_index_emb_list_stage_ms(self.h, _ptr(v)))
        return dict(stage1=float(v[0]), candidates=float(v[1]), rerank=float(v[2]), select=float(v[3]))

    # -- sparse float vectors: SPARSE_INVERTED_INDEX / SPARSE_WAND (DESIGN §4.13).  Row sets are CSR: an (indptr, indices,
    #    values) tuple of numpy arrays or CUDA tensors, or any object with .indptr / .indices / .data.
    def add_sparse(self, rows):
        ip, ix, val, n = _csr(rows)
        _check(self.L.kb2_index_add_sparse(self.h, _ptr(ip), _ptr(ix), _ptr(val), n))

    def search_sparse(self, q, k, config=None, bitset=None):
        """Exact top-k of the query rows: (ids, dist) [nq, k], CUDA tensors when the query arrays are; dist is the score."""
        ip, ix, val, nq = _csr(q)
        ids, dist = _out(ip, nq, k)
        _check(self.L.kb2_index_search_sparse(self.h, _ptr(ip), _ptr(ix), _ptr(val), nq, k, _cfg(config), _ptr(bitset),
                                              _nbits(bitset), _ptr(ids), _ptr(dist)))
        return ids, dist

    def range_search_sparse(self, q, radius, range_filter=None, config=None, bitset=None):
        """(lims, ids, dist): the rows with radius < score <= range_filter, each query's best first."""
        ip, ix, val, nq = _csr(q)
        pl, pi, pd = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        _check(self.L.kb2_index_range_search_sparse(self.h, _ptr(ip), _ptr(ix), _ptr(val), nq, radius,
                                                    0.0 if range_filter is None else range_filter,
                                                    0 if range_filter is None else 1, _cfg(config), _ptr(bitset),
                                                    _nbits(bitset), ctypes.byref(pl), ctypes.byref(pi), ctypes.byref(pd)))
        return _take_range(self.L, nq, pl, pi, pd)

    # -- introspection for bench.py
    def last_counters(self):
        c = np.zeros(8, np.int64)
        _check(self.L.kb2_index_last_search_counters(self.h, _ptr(c)))
        return dict(launches=int(c[0]), codes=int(c[1]), code_bytes=int(c[2]), pairs=int(c[3]), h2d=int(c[4]),
                    d2h=int(c[5]), survivors=int(c[6]), flagged=int(c[7]))

    def enable_kernel_timing(self, on=True):
        _check(self.L.kb2_index_enable_kernel_timing(self.h, 1 if on else 0))

    def last_stage_info(self):
        v = np.zeros(4, np.float32)
        _check(self.L.kb2_index_last_stage_info(self.h, _ptr(v)))
        return dict(stage_ms=float(v[0]), kernel_ms=float(v[1]), engine=("scan", "tc", "large_k", "hnsw_wide", "cagra", "sparse")[int(round(v[2]))], comm_ms=float(v[3]))

    def last_kernel_ms(self):
        v = ctypes.c_float()
        _check(self.L.kb2_index_last_kernel_ms(self.h, ctypes.byref(v)))
        return v.value


def faiss_describe(blob, with_norm=False):
    """host-only parse of a faiss fourcc stream -> dict (no GPU needed)"""
    L = lib()
    src = ctypes.create_string_buffer(blob, len(blob))
    out = ctypes.create_string_buffer(1024)
    _check(L.kb2_faiss_describe(ctypes.cast(src, ctypes.c_void_p), len(blob), 1 if with_norm else 0,
                                ctypes.cast(out, ctypes.c_void_p), 1024))
    return json.loads(out.value.decode())


def faiss_rewrite(blob, with_norm=False):
    """host-only: parse and re-emit with this library's writer"""
    L = lib()
    src = ctypes.create_string_buffer(blob, len(blob))
    p, n = ctypes.c_void_p(), ctypes.c_size_t()
    _check(L.kb2_faiss_rewrite(ctypes.cast(src, ctypes.c_void_p), len(blob), 1 if with_norm else 0, ctypes.byref(p), ctypes.byref(n)))
    try:
        return ctypes.string_at(p, n.value)
    finally:
        L.kb2_free(p)


class Comm:
    """NCCL communicator owned by the library (kb2_comm_*).  `bcast_bytes(bytes_or_None) -> bytes` is the host
    application's way to ship rank 0's 128-byte id to every rank (tests / bench: torch.distributed.broadcast_object_list)."""

    def __init__(self, rank, world, device, bcast_bytes):
        self.L = lib()
        self.rank, self.world = rank, world
        uid = None
        if rank == 0:
            buf = (ctypes.c_uint8 * 128)()
            _check(self.L.kb2_comm_unique_id(ctypes.cast(buf, ctypes.c_void_p)))
            uid = bytes(buf)
        uid = bcast_bytes(uid)
        assert len(uid) == 128
        self.h = ctypes.c_void_p()
        src = ctypes.create_string_buffer(uid, 128)
        _check(self.L.kb2_comm_create(ctypes.cast(src, ctypes.c_void_p), rank, world, device, ctypes.byref(self.h)))

    def all_gather(self, send, recv, stream=0):
        nbytes = send.numel() * send.element_size()
        _check(self.L.kb2_comm_all_gather(self.h, _ptr(send), _ptr(recv), nbytes, ctypes.c_void_p(stream)))

    def close(self):
        if self.h:
            self.L.kb2_comm_destroy(self.h)
            self.h = None


def _take_range(L, nq, pl, pi, pd):
    lims = np.ctypeslib.as_array(ctypes.cast(pl, ctypes.POINTER(ctypes.c_int64)), (nq + 1,)).copy()
    tot = int(lims[-1])
    if tot:
        ids = np.ctypeslib.as_array(ctypes.cast(pi, ctypes.POINTER(ctypes.c_int64)), (tot,)).copy()
        dist = np.ctypeslib.as_array(ctypes.cast(pd, ctypes.POINTER(ctypes.c_float)), (tot,)).copy()
    else:
        ids, dist = np.empty(0, np.int64), np.empty(0, np.float32)
    L.kb2_free(pl)
    L.kb2_free(pi)
    L.kb2_free(pd)
    return lims, ids, dist


def _nbits(bitset):
    return 0 if bitset is None else (bitset.numel() if _is_torch(bitset) else bitset.size) * 8


def _csr(rows):
    """(indptr int64, indices uint32, values float32, n) of a CSR row set, without scipy: an (indptr, indices, values)
    tuple of numpy arrays or torch tensors, or any object with .indptr / .indices / .data.  Torch tensors stay where
    they are (int32 indices pass as their uint32 bits); numpy arrays are converted."""
    ip, ix, val = rows if isinstance(rows, tuple) else (rows.indptr, rows.indices, rows.data)
    if _is_torch(ip):
        import torch
        ip = ip.to(torch.int64).contiguous()
        if ix.dtype != torch.int32:
            if ix.numel() and (int(ix.min()) < 0 or int(ix.max()) > 0xFFFFFFFF):
                raise KnowhereError(1, "sparse indices must lie in [0, 2^32)")
            ix = ix.to(torch.int64).to(torch.int32)   # the same 32 bits as uint32
        ix = ix.contiguous()
        val = val.to(torch.float32).contiguous()
        return ip, ix, val, int(ip.numel()) - 1
    ip = np.ascontiguousarray(ip, np.int64)
    ix = np.asarray(ix)
    if ix.dtype != np.uint32:
        if ix.size and (ix.min() < 0 or ix.max() > 0xFFFFFFFF):
            raise KnowhereError(1, "sparse indices must lie in [0, 2^32)")
        ix = ix.astype(np.uint32)
    return ip, np.ascontiguousarray(ix), np.ascontiguousarray(val, np.float32), ip.size - 1


def _out(like, nq, k):
    if _is_torch(like) and like.is_cuda:
        import torch
        return (torch.empty((nq, k), dtype=torch.int64, device=like.device),
                torch.empty((nq, k), dtype=torch.float32, device=like.device))
    return np.empty((nq, k), np.int64), np.empty((nq, k), np.float32)


def brute_force_search_sparse(base, queries, k, metric="IP", config=None, bitset=None, device=0):
    """knowhere::BruteForce::SearchSparse (reference src/common/comp/brute_force.cc:1227-1340): the exact top-k of the
    query rows over the base rows, both CSR as Index.add_sparse takes them.  BM25 takes bm25_k1, bm25_b and bm25_avgdl
    from config."""
    L = lib()
    bp, bi, bv, nb = _csr(base)
    qp, qi, qv, nq = _csr(queries)
    ids, dist = _out(qp, nq, k)
    _check(L.kb2_bruteforce_search_sparse(_ptr(bp), _ptr(bi), _ptr(bv), nb, _ptr(qp), _ptr(qi), _ptr(qv), nq,
                                          _METRICS[metric], k, _cfg(config), _ptr(bitset), _nbits(bitset), _ptr(ids),
                                          _ptr(dist), device))
    return ids, dist


def brute_force_search(base, queries, k, metric="L2", bitset=None, device=0, stream=0):
    """knowhere::BruteForce::Search (reference include/knowhere/comp/brute_force.h:26-69)."""
    L = lib()
    nq = queries.shape[0]
    if _is_torch(queries) and queries.is_cuda:
        import torch
        ids = torch.empty((nq, k), dtype=torch.int64, device=queries.device)
        dist = torch.empty((nq, k), dtype=torch.float32, device=queries.device)
    else:
        ids = np.empty((nq, k), np.int64)
        dist = np.empty((nq, k), np.float32)
    nbits = 0 if bitset is None else bitset.size * 8
    _check(L.kb2_bruteforce_search(_ptr(base), base.shape[0], base.shape[1], _METRICS[metric], _ptr(queries), nq, k,
                                   _ptr(bitset), nbits, _ptr(ids), _ptr(dist), device, ctypes.c_void_p(stream)))
    return ids, dist


# emb-list metrics (reference index_param.h:280-285; names are case-insensitive, "MAX_SIM" is MAX_SIM_COSINE).  Names the
# library has no metric for (MAX_SIM_HAMMING, MAX_SIM_JACCARD) go through as -1, which it rejects as an invalid metric.
_EMB_METRICS = {"MAX_SIM": 5, "MAX_SIM_COSINE": 5, "MAX_SIM_IP": 4, "MAX_SIM_L2": 3}


def debug_muvera_encode(x, lims, num_projections=4, num_repeats=7, seed=42, mean=True, device=0):
    """The MUVERA encoder on the device (validation hook): (projections [R, P, dim], encodings [n_items, R * 2^P * dim])
    of the items lims[i] .. lims[i + 1] of the float32 rows x; mean=True encodes documents, False query lists."""
    L = lib()
    x = np.ascontiguousarray(x, np.float32)
    lims = np.ascontiguousarray(lims, np.int64)
    n_items, dim = lims.shape[0] - 1, x.shape[1]
    proj = np.empty((num_repeats, num_projections, dim), np.float32)
    fde = np.empty((n_items, num_repeats * (1 << num_projections) * dim), np.float32)
    _check(L.kb2_debug_muvera_encode(_ptr(x), _ptr(lims), n_items, dim, num_projections, num_repeats, seed, 1 if mean else 0,
                                     _ptr(proj), _ptr(fde), device))
    return proj, fde


def brute_force_search_emb_list(base, base_lims, queries, query_lims, k, metric="MAX_SIM", bitset=None, device=0,
                                stream=0, stats=False):
    """knowhere::BruteForce::Search over emb-lists with a MAX_SIM metric (reference src/common/comp/brute_force.cc:424-665).

    base: [rows, dim] float32; base_lims: int64 [n_docs + 1], document i = base rows [lims[i], lims[i+1]).  queries /
    query_lims likewise for the query lists.  Each may be a numpy array or a CUDA tensor.  Returns (ids, dist) of shape
    [n_lists, k] (CUDA tensors when queries are), ids = document indices best first and dist = the MaxSim score; with
    stats=True also an int64 array [query lists, candidate slots re-ranked, lists scored exactly over every document]."""
    L = lib()
    for lims in (base_lims, query_lims):
        if _is_torch(lims) and str(lims.dtype) != "torch.int64":
            raise TypeError("list offsets must be int64")
    if not _is_torch(base_lims):
        base_lims = np.ascontiguousarray(base_lims, np.int64)
    if not _is_torch(query_lims):
        query_lims = np.ascontiguousarray(query_lims, np.int64)
    n_docs, n_lists = int(base_lims.shape[0]) - 1, int(query_lims.shape[0]) - 1
    if base.ndim != 2 or queries.ndim != 2 or queries.shape[1] != base.shape[1]:
        raise KnowhereError(1, "base and queries must be [rows, dim] with the same dim")
    if n_docs < 1 or n_lists < 0 or int(base_lims[-1]) != base.shape[0] or int(query_lims[-1]) != queries.shape[0]:
        raise KnowhereError(1, "list offsets must end at the row count of their dataset")
    if _is_torch(queries) and queries.is_cuda:
        import torch
        ids = torch.empty((n_lists, k), dtype=torch.int64, device=queries.device)
        dist = torch.empty((n_lists, k), dtype=torch.float32, device=queries.device)
    else:
        ids = np.empty((n_lists, k), np.int64)
        dist = np.empty((n_lists, k), np.float32)
    st = np.zeros(3, np.int64)
    nbits = 0 if bitset is None else (bitset.numel() if _is_torch(bitset) else bitset.size) * 8
    _check(L.kb2_bruteforce_search_emb_list(_ptr(base), _ptr(base_lims), n_docs, base.shape[1],
                                            _EMB_METRICS.get(str(metric).upper(), -1), _ptr(queries), _ptr(query_lims),
                                            n_lists, k, _ptr(bitset), nbits, _ptr(ids), _ptr(dist), _ptr(st), device,
                                            ctypes.c_void_p(stream)))
    return (ids, dist, st) if stats else (ids, dist)


def debug_cagra_knn_graph(x, metric="L2", config=None, device=0):
    """validation hook (kb2_debug_cagra_knn_graph): step 1 of the GPU_CAGRA build alone, exact or NN-descent as the build
    keys in config say.  x: CUDA tensor [n, d] fp32.  Returns (G0 int32 CUDA tensor [n, m], keys fp32 CUDA tensor [n, m],
    NN-descent iterations run, updates(t) numpy int64, device ms), m = min(intermediate_graph_degree, n - 1)."""
    import torch
    L = lib()
    n, d = x.shape
    m = min(int((config or {}).get("intermediate_graph_degree", 128)), n - 1)
    ids = torch.empty((n, m), dtype=torch.int32, device=x.device)
    keys = torch.empty((n, m), dtype=torch.float32, device=x.device)
    iters = ctypes.c_int()
    upd = np.zeros(1000, np.int64)
    ms = ctypes.c_float()
    _check(L.kb2_debug_cagra_knn_graph(_ptr(x), n, d, _METRICS[metric], _cfg(config), _ptr(ids), _ptr(keys),
                                       ctypes.byref(iters), _ptr(upd), len(upd), ctypes.byref(ms), device))
    return ids, keys, iters.value, upd[:iters.value].copy(), ms.value


def brute_force_range_search(base, queries, radius, range_filter=None, metric="L2", bitset=None, device=0):
    L = lib()
    nq = queries.shape[0]
    pl, pi, pd = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    nbits = 0 if bitset is None else bitset.size * 8
    _check(L.kb2_bruteforce_range_search(_ptr(base), base.shape[0], base.shape[1], _METRICS[metric], _ptr(queries),
                                         nq, radius, 0.0 if range_filter is None else range_filter,
                                         0 if range_filter is None else 1, _ptr(bitset), nbits, ctypes.byref(pl),
                                         ctypes.byref(pi), ctypes.byref(pd), device, None))
    return _take_range(L, nq, pl, pi, pd)


def merge_topk(ids, dist, metric="L2", device=0, stream=0):
    """ids/dist: [world, nq, k] gathered per-shard results -> global [nq, k]."""
    L = lib()
    world, nq, k = ids.shape
    if _is_torch(ids) and ids.is_cuda:
        import torch
        oi = torch.empty((nq, k), dtype=torch.int64, device=ids.device)
        od = torch.empty((nq, k), dtype=torch.float32, device=ids.device)
    else:
        oi = np.empty((nq, k), np.int64)
        od = np.empty((nq, k), np.float32)
    _check(L.kb2_merge_topk(_METRICS[metric], world, nq, k, _ptr(ids), _ptr(dist), _ptr(oi), _ptr(od), device,
                            ctypes.c_void_p(stream)))
    return oi, od
