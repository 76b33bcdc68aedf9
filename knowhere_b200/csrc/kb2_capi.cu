// kb2_capi.cu — the extern "C" boundary declared in include/knowhere_b200.h.
// Everything behind it is CUDA; there is no CPU fallback: without a usable sm_90 device every
// entry point fails with KB2_CUDA_RUNTIME_ERROR.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <atomic>
#include <cstring>
#include <memory>

#include "kb2_fourcc.h"
#include "kb2_hnsw.cuh"
#include "kb2_index.cuh"
#include "kb2_maxsim.cuh"
#include "kb2_range.cuh"

using namespace kb2;

namespace {
thread_local std::string g_last_error;

template <typename F>
int
guarded(F&& f) {
    try {
        f();
        return KB2_SUCCESS;
    } catch (const Error& e) {
        g_last_error = e.what();
        cudaGetLastError();
        return e.status;
    } catch (const std::bad_alloc&) {
        g_last_error = "host allocation failed";
        return KB2_MALLOC_ERROR;
    } catch (const std::exception& e) {
        g_last_error = e.what();
        return KB2_INTERNAL_ERROR;
    } catch (...) {
        g_last_error = "unknown error";
        return KB2_INTERNAL_ERROR;
    }
}

int
usable_devices() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int ok = 0;
    for (int i = 0; i < n; i++) {
        cudaDeviceProp p;
        if (cudaGetDeviceProperties(&p, i) == cudaSuccess && p.major == 9 && p.minor == 0) ok++;
    }
    return ok;
}

void
require_device(int device) {
    // validated devices are cached: cudaGetDeviceProperties costs milliseconds and this sits on per-call paths
    static std::atomic<uint64_t> ok_mask{0};
    if (device >= 0 && device < 64 && (ok_mask.load(std::memory_order_relaxed) >> device) & 1) {
        KB2_CUDA_CHECK(cudaSetDevice(device));
        return;
    }
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        cudaGetLastError();
        throw Error(KB2_CUDA_RUNTIME_ERROR, "no CUDA device available (this library has no CPU fallback)");
    }
    KB2_REQUIRE(device >= 0 && device < n, KB2_INVALID_ARGS, "bad device ordinal");
    cudaDeviceProp p;
    KB2_CUDA_CHECK(cudaGetDeviceProperties(&p, device));
    KB2_REQUIRE(p.major == 9 && p.minor == 0, KB2_CUDA_RUNTIME_ERROR,
                "device is not sm_90 (this library ships sm_90a SASS only)");
    KB2_CUDA_CHECK(cudaSetDevice(device));
    if (device < 64) ok_mask.fetch_or(1ull << device, std::memory_order_relaxed);
}

struct Handle {
    std::unique_ptr<IndexBase> ix;
};
inline IndexBase*
ix_of(kb2_index_t h) {
    KB2_REQUIRE(h != nullptr, KB2_INVALID_ARGS, "null index handle");
    return reinterpret_cast<Handle*>(h)->ix.get();
}
template <typename T>
inline T*
ix_as(kb2_index_t h, const char* what) {
    T* p = dynamic_cast<T*>(ix_of(h));
    KB2_REQUIRE(p != nullptr || !dynamic_cast<MuveraIndex*>(ix_of(h)), KB2_NOT_IMPLEMENTED,
                std::string(what) + " calls on a MUVERA emb-list index (its base holds the documents' encodings)");
    KB2_REQUIRE(p != nullptr, KB2_INVALID_ARGS, std::string("handle is not an ") + what + " index");
    return p;
}
// guarded() call of f(ix) on the handle's index (checked to be a T), under the index's lock and on its device
template <typename T, typename F>
int
on_index(kb2_index_t h, const char* what, F&& f) {
    return guarded([&] {
        T* ix = ix_as<T>(h, what);
        std::lock_guard<std::mutex> lk(ix->mu);
        KB2_CUDA_CHECK(cudaSetDevice(ix->device));
        f(ix);
    });
}
template <typename F>
int
on_index(kb2_index_t h, F&& f) {
    return on_index<IndexBase>(h, "", std::forward<F>(f));
}
// guarded call of f(sparse index), under its lock and on its device; a dense handle names its own entry points
template <typename F>
int
on_sparse(kb2_index_t h, F&& f) {
    return on_index(h, [&](IndexBase* ix) {
        auto* sx = dynamic_cast<SparseIndex*>(ix);
        KB2_REQUIRE(sx != nullptr, KB2_INVALID_ARGS,
                    ix->type + " holds dense rows: use kb2_index_add / kb2_index_search / kb2_index_range_search");
        sx->last = Counters{};
        sx->wait_caller_work();
        f(sx);
    });
}
kb2_index_t
to_handle(std::unique_ptr<IndexBase> ix) {
    auto* h = new Handle();
    h->ix = std::move(ix);
    return reinterpret_cast<kb2_index_t>(h);
}
// a byte vector handed to the caller as a malloc'ed blob (released with kb2_free)
void
blob_out(const std::vector<uint8_t>& b, uint8_t** out, size_t* out_size) {
    *out = (uint8_t*)malloc(b.size() ? b.size() : 1);
    KB2_REQUIRE(*out != nullptr, KB2_MALLOC_ERROR, "malloc failed");
    memcpy(*out, b.data(), b.size());
    *out_size = b.size();
}

int
parse_metric(int metric, const JsonObj& cfg) {
    if (cfg.has("metric_type")) {
        const std::string m = cfg.get_str("metric_type", "L2");
        if (m == "L2") return KB2_METRIC_L2;
        if (m == "IP") return KB2_METRIC_IP;
        if (m == "COSINE") return KB2_METRIC_COSINE;
        if (m == "BM25") return KB2_METRIC_BM25;
        throw Error(KB2_INVALID_METRIC_TYPE, "unsupported metric_type " + m);
    }
    return metric;
}
}  // namespace

extern "C" {

const char*
kb2_version(void) {
    return "knowhere_b200 0.1 (sm_90a)";
}
const char*
kb2_last_error(void) {
    return g_last_error.c_str();
}
int
kb2_device_count(void) {
    return usable_devices();
}

int
kb2_index_create(const char* index_type, int metric, int dim, const char* json_cfg, int device, kb2_index_t* out) {
    return guarded([&] {
        KB2_REQUIRE(out != nullptr && index_type != nullptr, KB2_INVALID_ARGS, "null argument");
        *out = nullptr;
        JsonObj cfg = JsonObj::parse(json_cfg);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        metric = parse_metric(metric, cfg);
        const std::string t = index_type;
        if (is_sparse_type(t)) {
            // sparse_index_node.cc:114-119; sparse rows have no fixed dimension
            KB2_REQUIRE(metric == KB2_METRIC_IP || metric == KB2_METRIC_BM25, KB2_INVALID_METRIC_TYPE,
                        t + " only supports metric_type IP or BM25");
            dim = 0;
        } else {
            KB2_REQUIRE(metric == KB2_METRIC_L2 || metric == KB2_METRIC_IP || metric == KB2_METRIC_COSINE,
                        KB2_INVALID_METRIC_TYPE, "metric must be L2, IP or COSINE");
            if (dim <= 0) dim = (int)cfg.get_int("dim", 0);
            KB2_REQUIRE(dim > 0, KB2_INVALID_ARGS, "dim must be positive");
        }
        require_device(device);
        std::unique_ptr<IndexBase> ix = make_index(t);
        KB2_REQUIRE(ix, KB2_INVALID_ARGS, "unknown index type " + t);
        // emb_list_strategy muvera: the handle keeps the token rows and builds its base at kb2_index_set_emb_list.  The
        // strategy is read on the types that take emb-lists only; the others refuse kb2_index_set_emb_list, as for TokenANN
        MuveraParams mp;
        if (ix->takes_emb_list() && muvera_params_of(cfg, mp)) ix = std::make_unique<MuveraIndex>();
        // COSINE = inner product of L2-normalised vectors: data is normalised when it enters the index and
        // queries when they are searched (what the reference does for IVF_PQ, ivf.cc:557-565,1067-1071; for FLAT
        // the reference keeps inverse norms instead, flat.cc:57-62 — same similarities)
        ix->init(t, metric, dim, device);
        ix->configure(cfg);
        *out = to_handle(std::move(ix));
    });
}

void
kb2_index_destroy(kb2_index_t h) {
    if (!h) return;
    Handle* hh = reinterpret_cast<Handle*>(h);
    if (hh->ix) cudaSetDevice(hh->ix->device);
    delete hh;
}

int
kb2_index_set_stream(kb2_index_t h, void* cuda_stream) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        std::lock_guard<std::mutex> lk(ix->mu);
        ix->set_stream((cudaStream_t)cuda_stream);
    });
}

int
kb2_index_set_shard(kb2_index_t h, int rank, int world) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        KB2_REQUIRE(world >= 1 && rank >= 0 && rank < world, KB2_INVALID_ARGS, "bad shard rank/world");
        KB2_REQUIRE(ix->count() == 0, KB2_INVALID_ARGS, "set_shard must precede add/import");
        if (world > 1) ix->refuse(IndexBase::kShard);
        ix->shard_rank = rank;
        ix->shard_world = world;
    });
}

namespace {
// element types of the reference's data-type registrations: fp16 / bf16 / int8 indexes are "mock" wrappers that convert the
// whole dataset and every query batch to fp32 (include/knowhere/index/index_factory.h:95-103,
// src/index/index_node_data_mock_wrapper.cc:24-60); here the widening runs on the device
__global__ void
widen_kernel(const void* __restrict__ src, int dtype, int64_t n, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v;
    if (dtype == KB2_DTYPE_F16) v = __half2float(((const __half*)src)[i]);
    else if (dtype == KB2_DTYPE_BF16) v = __bfloat162float(((const __nv_bfloat16*)src)[i]);
    else v = (float)((const int8_t*)src)[i];
    out[i] = v;
}
// device fp32 view of `count` elements of type dtype (host or device source); valid until the next typed call on the handle
const float*
widen_to_f32(IndexBase* ix, const void* x, int dtype, int64_t count) {
    if (dtype == KB2_DTYPE_F32) return (const float*)x;
    KB2_REQUIRE(dtype == KB2_DTYPE_F16 || dtype == KB2_DTYPE_BF16 || dtype == KB2_DTYPE_INT8, KB2_INVALID_ARGS, "unknown data type");
    if (count <= 0 || !x) return nullptr;
    const size_t esz = dtype == KB2_DTYPE_INT8 ? 1 : 2;
    const void* dsrc = x;
    if (!is_device_ptr(x)) {
        ix->s_typed_raw.ensure((size_t)count * esz);
        KB2_CUDA_CHECK(cudaMemcpyAsync(ix->s_typed_raw.p, x, (size_t)count * esz, cudaMemcpyHostToDevice, ix->stream));
        ix->last.h2d += (int64_t)count * (int64_t)esz;
        dsrc = ix->s_typed_raw.p;
    }
    ix->s_typed_f32.ensure((size_t)count);
    widen_kernel<<<grid1d(count, 256), 256, 0, ix->stream>>>(dsrc, dtype, count, ix->s_typed_f32.p);
    KB2_CUDA_CHECK(cudaGetLastError());
    return ix->s_typed_f32.p;
}
}  // namespace

int
kb2_index_train_typed(kb2_index_t h, const void* x, int dtype, int64_t n) {
    return on_index(h, [&](IndexBase* ix) {
        KB2_REQUIRE(x != nullptr || n == 0, KB2_INVALID_ARGS, "null training data");
        KB2_REQUIRE(!ix->emb_list, KB2_NOT_IMPLEMENTED, "Train on an emb-list index");
        ix->wait_caller_work();
        const float* xf = widen_to_f32(ix, x, dtype, n * ix->dim);
        ix->train(ix->cosine && !ix->raw_rows_on_entry() ? ix->normalized(xf, n) : xf, n);
    });
}
int
kb2_index_train(kb2_index_t h, const float* x, int64_t n) {
    return kb2_index_train_typed(h, x, KB2_DTYPE_F32, n);
}

int
kb2_index_add_typed(kb2_index_t h, const void* x, int dtype, int64_t n, const int64_t* ids) {
    return on_index(h, [&](IndexBase* ix) {
        KB2_REQUIRE(x != nullptr || n == 0, KB2_INVALID_ARGS, "null data");
        KB2_REQUIRE(!ix->emb_list, KB2_NOT_IMPLEMENTED, "AddEmbList is not implemented: rows cannot be added to an emb-list index");
        ix->wait_caller_work();
        const float* xf = widen_to_f32(ix, x, dtype, n * ix->dim);
        ix->add(ix->cosine && !ix->raw_rows_on_entry() ? ix->normalized(xf, n) : xf, n, ids);
    });
}
int
kb2_index_add(kb2_index_t h, const float* x, int64_t n, const int64_t* ids) {
    return kb2_index_add_typed(h, x, KB2_DTYPE_F32, n, ids);
}

int
kb2_index_search_typed(kb2_index_t h, const void* queries, int dtype, int64_t nq, int k, const char* json, const uint8_t* bitset,
                       int64_t bitset_nbits, int64_t* out_ids, float* out_dist) {
    return on_index(h, [&](IndexBase* ix) {
        KB2_REQUIRE(nq >= 0 && k > 0, KB2_INVALID_ARGS, "bad nq / k");
        KB2_REQUIRE(!ix->emb_list, KB2_EMB_LIST_INNER_ERROR, "emb-list index: search with query list offsets (kb2_index_search_emb_list)");
        if (nq == 0) return;
        KB2_REQUIRE(queries && out_ids && out_dist, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(is_device_ptr(out_ids) == is_device_ptr(out_dist), KB2_INVALID_ARGS,
                    "out_ids and out_dist must both be host or both be device buffers");
        JsonObj cfg = JsonObj::parse(json);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        ix->last = Counters{};
        ix->wait_caller_work();
        const float* qf = widen_to_f32(ix, queries, dtype, nq * ix->dim);
        ix->search(ix->cosine ? ix->normalized(qf, nq) : qf, nq, k, cfg, bitset, bitset_nbits, out_ids, out_dist);
    });
}
int
kb2_index_search(kb2_index_t h, const float* queries, int64_t nq, int k, const char* json, const uint8_t* bitset,
                 int64_t bitset_nbits, int64_t* out_ids, float* out_dist) {
    return kb2_index_search_typed(h, queries, KB2_DTYPE_F32, nq, k, json, bitset, bitset_nbits, out_ids, out_dist);
}

int
kb2_index_range_search(kb2_index_t h, const float* queries, int64_t nq, float radius, float range_filter,
                       int has_range_filter, const char* json, const uint8_t* bitset, int64_t bitset_nbits,
                       int64_t** out_lims, int64_t** out_ids, float** out_dist) {
    return on_index(h, [&](IndexBase* ix) {
        KB2_REQUIRE(out_lims && out_ids && out_dist, KB2_INVALID_ARGS, "null output");
        KB2_REQUIRE(!ix->emb_list, KB2_EMB_LIST_INNER_ERROR, "RangeSearch is not supported on an emb-list index");
        JsonObj cfg = JsonObj::parse(json);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        ix->last = Counters{};
        ix->wait_caller_work();
        range_search_index(*ix, ix->cosine ? ix->normalized(queries, nq) : queries, nq, radius, range_filter,
                           has_range_filter != 0, cfg, bitset, bitset_nbits, out_lims, out_ids, out_dist);
    });
}

void
kb2_free(void* p) {
    free(p);
}

int64_t
kb2_index_count(kb2_index_t h) {
    return h ? reinterpret_cast<Handle*>(h)->ix->count() : 0;
}
int
kb2_index_dim(kb2_index_t h) {
    return h ? reinterpret_cast<Handle*>(h)->ix->dim : 0;
}
int64_t
kb2_index_size_bytes(kb2_index_t h) {
    return h ? reinterpret_cast<Handle*>(h)->ix->size_bytes() : 0;
}
int
kb2_index_is_trained(kb2_index_t h) {
    return h ? (int)reinterpret_cast<Handle*>(h)->ix->is_trained() : 0;
}
int
kb2_index_has_raw_data(kb2_index_t h) {
    // COSINE stores the normalised vectors, not the caller's raw data
    return h ? (int)(reinterpret_cast<Handle*>(h)->ix->has_raw() && !reinterpret_cast<Handle*>(h)->ix->cosine) : 0;
}
int
kb2_index_get_vector_by_ids(kb2_index_t h, const int64_t* ids, int64_t n, float* out) {
    return on_index(h, [&](IndexBase* ix) {
        KB2_REQUIRE(!ix->cosine, KB2_NOT_IMPLEMENTED, "GetVectorByIds: a COSINE index keeps normalised vectors only");
        ix->get_vectors(ids, n, out);
    });
}

// ---------------------------------------------------------------- IVF import / export
int
kb2_ivf_import_begin(kb2_index_t h, int64_t nlist, const float* centroids, const float* pq_centroids) {
    return on_index<IvfIndex>(h, "IVF", [&](IvfIndex* iv) {
        KB2_REQUIRE(!iv->emb_list, KB2_NOT_IMPLEMENTED, "import into an emb-list index");
        iv->import_begin(nlist, centroids, pq_centroids);
    });
}
int
kb2_ivf_import_list(kb2_index_t h, int64_t list_no, int64_t list_size, const int64_t* ids, const uint8_t* codes) {
    return guarded([&] {
        auto* iv = ix_as<IvfIndex>(h, "IVF");
        std::lock_guard<std::mutex> lk(iv->mu);
        KB2_REQUIRE(!iv->emb_list, KB2_NOT_IMPLEMENTED, "import into an emb-list index");
        if (list_size > 0) iv->import_list(list_no, list_size, ids, codes);
    });
}
int
kb2_ivf_import_finish(kb2_index_t h, const float* raw, int64_t n_raw) {
    return on_index<IvfIndex>(h, "IVF", [&](IvfIndex* iv) {
        KB2_REQUIRE(!iv->emb_list, KB2_NOT_IMPLEMENTED, "import into an emb-list index");
        iv->import_finish(raw, n_raw);
    });
}
int64_t
kb2_ivf_nlist(kb2_index_t h) {
    auto* iv = dynamic_cast<IvfIndex*>(reinterpret_cast<Handle*>(h)->ix.get());
    return iv ? iv->nlist : -1;
}
int64_t
kb2_ivf_list_size(kb2_index_t h, int64_t list_no) {
    int64_t r = -1;
    on_index<IvfIndex>(h, "IVF", [&](IvfIndex* iv) {
        iv->seal();
        KB2_REQUIRE(list_no >= 0 && list_no < iv->nlist, KB2_INVALID_ARGS, "list number out of range");
        r = iv->h_list_len[list_no];
    });
    return r;
}
int
kb2_ivf_export_centroids(kb2_index_t h, float* centroids, float* pq_centroids) {
    return on_index<IvfIndex>(h, "IVF", [&](IvfIndex* iv) {
        KB2_REQUIRE(iv->trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        if (centroids)
            KB2_CUDA_CHECK(cudaMemcpy(centroids, iv->centroids.p, (size_t)iv->nlist * iv->dim * 4, cudaMemcpyDefault));
        if (pq_centroids && iv->is_pq)
            KB2_CUDA_CHECK(cudaMemcpy(pq_centroids, iv->pqc.p, (size_t)iv->M * 256 * iv->dsub * 4, cudaMemcpyDefault));
    });
}
int
kb2_ivf_export_list(kb2_index_t h, int64_t list_no, int64_t* ids, uint8_t* codes) {
    return on_index<IvfIndex>(h, "IVF", [&](IvfIndex* iv) {
        iv->export_list(list_no, ids, codes);
    });
}

// ---------------------------------------------------------------- HNSW import / export
int
kb2_hnsw_import(kb2_index_t h, int64_t n, const float* vectors, const int32_t* levels, const int64_t* offsets,
                const int32_t* neighbors, const int32_t* cum_nneighbor, int n_cum, int32_t entry_point,
                int32_t max_level) {
    return on_index<HnswIndex>(h, "HNSW", [&](HnswIndex* hn) {
        hn->refuse(IndexBase::kHnswImport);
        // the attached document offsets and doc_of_row describe the current rows
        KB2_REQUIRE(!hn->emb_list, KB2_NOT_IMPLEMENTED, "import into an emb-list index");
        hn->import_graph(n, vectors, levels, offsets, neighbors, cum_nneighbor, n_cum, entry_point, max_level);
    });
}
int
kb2_hnsw_export_meta(kb2_index_t h, int64_t* out5) {
    return guarded([&] {
        auto* hn = ix_as<HnswIndex>(h, "HNSW");
        out5[0] = hn->n;
        out5[1] = hn->entry_point;
        out5[2] = hn->max_level;
        out5[3] = (int64_t)hn->h_neighbors.size();
        out5[4] = (int64_t)hn->h_cum.size();
    });
}
int
kb2_hnsw_export(kb2_index_t h, int32_t* levels, int64_t* offsets, int32_t* neighbors, int32_t* cum) {
    return guarded([&] {
        auto* hn = ix_as<HnswIndex>(h, "HNSW");
        memcpy(levels, hn->h_levels.data(), hn->h_levels.size() * 4);
        memcpy(offsets, hn->h_offsets.data(), hn->h_offsets.size() * 8);
        memcpy(neighbors, hn->h_neighbors.data(), hn->h_neighbors.size() * 4);
        memcpy(cum, hn->h_cum.data(), hn->h_cum.size() * 4);
    });
}
int
kb2_hnsw_last_stats(kb2_index_t h, int64_t* out2) {
    return guarded([&] {
        auto* hn = ix_as<HnswIndex>(h, "HNSW");
        out2[0] = hn->last_ndis;
        out2[1] = hn->last_nhops;
    });
}

// ---------------------------------------------------------------- serialisation ("KB2I" container)
int
kb2_index_serialize(kb2_index_t h, uint8_t** out, size_t* out_size) {
    return on_index(h, [&](IndexBase* ix) {
        std::vector<uint8_t> blob;
        serialize_index(*ix, blob);
        blob_out(blob, out, out_size);
    });
}
int
kb2_index_deserialize(const uint8_t* blob, size_t size, int device, kb2_index_t* out) {
    return guarded([&] {
        KB2_REQUIRE(blob && out, KB2_INVALID_ARGS, "null argument");
        require_device(device);
        *out = to_handle(deserialize_index(blob, size, device));
    });
}

// ---------------------------------------------------------------- faiss fourcc streams (the reference's BinarySet payload)
namespace {
std::unique_ptr<IndexBase>
index_from_faiss(const FaissIndexData& o, int device) {
    std::unique_ptr<IndexBase> ix = make_index(o.kind);
    KB2_REQUIRE(ix, KB2_NOT_IMPLEMENTED, "faiss stream: unsupported index kind");
    ix->init(o.kind, o.cosine ? KB2_METRIC_COSINE : o.metric, o.d, device);
    ix->from_faiss(o);
    return ix;
}

void
index_to_faiss(IndexBase& ix, FaissIndexData& o) {
    o.kind = ix.type;
    o.d = ix.dim;
    o.metric = ix.metric;
    KB2_REQUIRE(!ix.cosine, KB2_NOT_IMPLEMENTED, "faiss stream: a COSINE index keeps normalised vectors only (the reference stores raw rows + norms)");
    KB2_REQUIRE(ix.shard_world == 1, KB2_NOT_IMPLEMENTED, "serialising a shard");
    o.ntotal = ix.count();
    ix.to_faiss(o);
}
}  // namespace

int
kb2_faiss_describe(const uint8_t* blob, size_t size, int with_norm, char* json_out, size_t cap) {
    return guarded([&] {
        KB2_REQUIRE(blob && json_out && cap > 0, KB2_INVALID_ARGS, "null argument");
        FaissReader rd{BlobReader{blob, size}, with_norm != 0};
        const FaissIndexData o = rd.read_index();
        const std::string s = faiss_describe(o);
        KB2_REQUIRE(s.size() + 1 <= cap, KB2_INVALID_ARGS, "output buffer too small");
        memcpy(json_out, s.c_str(), s.size() + 1);
    });
}
// parse + re-emit on the host (no device): the writer's output for exactly what the reader understood
int
kb2_faiss_rewrite(const uint8_t* blob, size_t size, int with_norm, uint8_t** out, size_t* out_size) {
    return guarded([&] {
        KB2_REQUIRE(blob && out && out_size, KB2_INVALID_ARGS, "null argument");
        FaissReader rd{BlobReader{blob, size}, with_norm != 0};
        const FaissIndexData o = rd.read_index();
        std::vector<uint8_t> b;
        FaissWriter wr{BlobWriter{b}};
        wr.write_index(o);
        blob_out(b, out, out_size);
    });
}
int
kb2_index_deserialize_faiss(const uint8_t* blob, size_t size, int with_norm, int device, kb2_index_t* out) {
    return guarded([&] {
        KB2_REQUIRE(blob && out, KB2_INVALID_ARGS, "null argument");
        *out = nullptr;
        FaissReader rd{BlobReader{blob, size}, with_norm != 0};
        const FaissIndexData o = rd.read_index();   // parse (and reject) before touching the device
        require_device(device);
        *out = to_handle(index_from_faiss(o, device));
    });
}
int
kb2_index_serialize_faiss(kb2_index_t h, uint8_t** out, size_t* out_size) {
    return on_index(h, [&](IndexBase* ix) {
        KB2_REQUIRE(out && out_size, KB2_INVALID_ARGS, "null argument");
        FaissIndexData o;
        index_to_faiss(*ix, o);
        std::vector<uint8_t> blob;
        FaissWriter wr{BlobWriter{blob}};
        wr.write_index(o);
        blob_out(blob, out, out_size);
    });
}
// IndexNode::DeserializeFromFile (index_node.h:329-395): a file holding either container
int
kb2_index_deserialize_from_file(const char* path, int device, kb2_index_t* out) {
    std::vector<uint8_t> buf;
    int st = guarded([&] {
        KB2_REQUIRE(path && out, KB2_INVALID_ARGS, "null argument");
        FILE* f = fopen(path, "rb");
        KB2_REQUIRE(f != nullptr, KB2_INVALID_ARGS, std::string("cannot open ") + path);
        fseek(f, 0, SEEK_END);
        const long n = ftell(f);
        fseek(f, 0, SEEK_SET);
        buf.resize(n > 0 ? (size_t)n : 0);
        const size_t got = buf.empty() ? 0 : fread(buf.data(), 1, buf.size(), f);
        fclose(f);
        KB2_REQUIRE(got == buf.size() && got >= 4, KB2_INVALID_BINARY_SET, "short read");
    });
    if (st != KB2_SUCCESS) return st;
    uint32_t magic;
    memcpy(&magic, buf.data(), 4);
    if (magic == 0x4932424b) return kb2_index_deserialize(buf.data(), buf.size(), device, out);
    return kb2_index_deserialize_faiss(buf.data(), buf.size(), 0, device, out);
}
// IndexNode::GetIndexMeta (index_node.h:329-395): JSON description of the loaded index
int
kb2_index_get_meta(kb2_index_t h, char* json_out, size_t cap) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        KB2_REQUIRE(json_out && cap > 0, KB2_INVALID_ARGS, "null argument");
        const char* m = ix->cosine ? "COSINE" : ix->metric == KB2_METRIC_IP ? "IP" : ix->metric == KB2_METRIC_BM25 ? "BM25" : "L2";
        std::string s = "{\"type\": \"" + ix->type + "\", \"dim\": " + std::to_string(ix->dim) + ", \"rows\": " + std::to_string(ix->count()) +
                        ", \"metric_type\": \"" + m + "\"" +
                        ", \"size_bytes\": " + std::to_string(ix->size_bytes()) + ", \"device\": " + std::to_string(ix->device) +
                        ", \"shard_rank\": " + std::to_string(ix->shard_rank) + ", \"shard_world\": " + std::to_string(ix->shard_world);
        ix->append_meta(s);
        s += "}";
        KB2_REQUIRE(s.size() + 1 <= cap, KB2_INVALID_ARGS, "output buffer too small");
        memcpy(json_out, s.c_str(), s.size() + 1);
    });
}

// ---------------------------------------------------------------- BruteForce
// One scratch FLAT object per device, reused across calls (stream, events, selection scratch); a device-resident base is
// viewed in place (no copy), a host base is staged into the scratch buffer.
namespace {
struct BfSlot {
    std::mutex mu;
    std::unique_ptr<FlatIndex> fi;
    msim::Scratch el;   // emb-list search (kb2_bruteforce_search_emb_list)
};
BfSlot g_bf[64];

FlatIndex&
bf_prepare(BfSlot& slot, int device, int metric, int dim, void* cuda_stream, const float* base, int64_t nb) {
    if (!slot.fi) {
        slot.fi.reset(new FlatIndex());
        slot.fi->type = "FLAT";
        slot.fi->device = device;
        slot.fi->init_common();
    }
    FlatIndex& fi = *slot.fi;
    fi.cosine = (metric == KB2_METRIC_COSINE);
    fi.metric = fi.cosine ? KB2_METRIC_IP : metric;
    fi.dim = dim;
    if (cuda_stream) fi.set_stream((cudaStream_t)cuda_stream); else fi.use_own_stream();
    fi.wait_caller_work();
    fi.last = Counters{};
    const size_t cnt = (size_t)nb * dim;
    if (fi.cosine) {
        const float* dx = fi.to_device(base, cnt, fi.s_cos_in);
        fi.base.ensure(cnt);
        normalize_rows_kernel<<<grid1d(nb * 32, 256), 256, 0, fi.stream>>>(dx, nb, dim, fi.base.p);
    } else if (is_device_ptr(base)) {
        fi.base.borrow(base, cnt);
    } else {
        fi.base.ensure(cnt);
        KB2_CUDA_CHECK(cudaMemcpyAsync(fi.base.p, base, cnt * 4, cudaMemcpyHostToDevice, fi.stream));
        fi.last.h2d += (int64_t)cnt * 4;
    }
    fi.n_used = cnt;
    fi.norms.ensure(nb);
    row_norms_kernel<<<grid1d(nb * 32, 256), 256, 0, fi.stream>>>(fi.base.p, nb, dim, fi.norms.p);
    fi.norms_used = (size_t)nb;
    KB2_CUDA_CHECK(cudaGetLastError());
    return fi;
}

// checks of the dense BruteForce calls; the device becomes current
void
bf_check(int metric, int device) {
    KB2_REQUIRE(metric == KB2_METRIC_L2 || metric == KB2_METRIC_IP || metric == KB2_METRIC_COSINE, KB2_INVALID_METRIC_TYPE,
                "metric must be L2, IP or COSINE");
    require_device(device);
    KB2_REQUIRE(device < 64, KB2_INVALID_ARGS, "bad device ordinal");
}
// f(fi, queries) on the device's scratch FLAT over `base`, under the slot lock (COSINE queries arrive normalised)
void
bf_run(int device, int metric, int dim, void* cuda_stream, const float* base, int64_t nb, const float* queries, int64_t nq,
       const std::function<void(FlatIndex&, const float*)>& f) {
    BfSlot& slot = g_bf[device];
    std::lock_guard<std::mutex> lk(slot.mu);
    FlatIndex& fi = bf_prepare(slot, device, metric, dim, cuda_stream, base, nb);
    f(fi, fi.cosine ? fi.normalized(queries, nq) : queries);
    fi.base.release();   // never keep a view of caller memory (or a stale copy) between calls
    fi.n_used = 0;
}
}  // namespace

int
kb2_bruteforce_search(const float* base, int64_t nb, int dim, int metric, const float* queries, int64_t nq, int k,
                      const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist, int device,
                      void* cuda_stream) {
    return guarded([&] {
        KB2_REQUIRE(base && queries && out_ids && out_dist, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(nb > 0 && dim > 0 && nq >= 0 && k > 0, KB2_INVALID_ARGS, "bad sizes");
        bf_check(metric, device);
        if (nq == 0) return;
        bf_run(device, metric, dim, cuda_stream, base, nb, queries, nq, [&](FlatIndex& fi, const float* q) {
            fi.search(q, nq, k, JsonObj{}, bitset, bitset_nbits, out_ids, out_dist);
        });
    });
}
int
kb2_bruteforce_range_search(const float* base, int64_t nb, int dim, int metric, const float* queries, int64_t nq,
                            float radius, float range_filter, int has_range_filter, const uint8_t* bitset,
                            int64_t bitset_nbits, int64_t** out_lims, int64_t** out_ids, float** out_dist, int device,
                            void* cuda_stream) {
    return guarded([&] {
        KB2_REQUIRE(base && queries, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(nb > 0 && dim > 0 && nq >= 0, KB2_INVALID_ARGS, "bad sizes");
        bf_check(metric, device);
        bf_run(device, metric, dim, cuda_stream, base, nb, queries, nq, [&](FlatIndex& fi, const float* q) {
            range_search_index(fi, q, nq, radius, range_filter, has_range_filter != 0, JsonObj{}, bitset, bitset_nbits, out_lims,
                               out_ids, out_dist);
        });
    });
}

namespace {
// host copy of n + 1 list offsets (host or device), checked: they start at 0 and do not decrease
std::vector<int64_t>
read_lims(const int64_t* lims, int64_t n, const char* what) {
    std::vector<int64_t> h((size_t)n + 1);
    if (is_device_ptr(lims)) KB2_CUDA_CHECK(cudaMemcpy(h.data(), lims, h.size() * 8, cudaMemcpyDeviceToHost));
    else memcpy(h.data(), lims, h.size() * 8);
    KB2_REQUIRE(h[0] == 0, KB2_INVALID_ARGS, std::string(what) + " offsets must start at 0");
    for (int64_t i = 0; i < n; i++)
        KB2_REQUIRE(h[i + 1] >= h[i], KB2_INVALID_ARGS, std::string(what) + " offsets must not decrease");
    return h;
}
}  // namespace

int
kb2_bruteforce_search_emb_list(const float* base, const int64_t* base_lims, int64_t n_docs, int dim, int metric,
                               const float* queries, const int64_t* query_lims, int64_t n_lists, int k,
                               const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist,
                               int64_t* out_stats, int device, void* cuda_stream) {
    return guarded([&] {
        KB2_REQUIRE(base && base_lims && queries && query_lims && out_ids && out_dist, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(n_docs > 0 && dim > 0 && n_lists >= 0, KB2_INVALID_ARGS, "bad sizes");
        KB2_REQUIRE(k > 0 && k <= kMaxLargeK, KB2_INVALID_ARGS, "k out of range (1..16384)");
        KB2_REQUIRE(metric == KB2_METRIC_MAX_SIM_L2 || metric == KB2_METRIC_MAX_SIM_IP || metric == KB2_METRIC_MAX_SIM_COSINE,
                    KB2_INVALID_METRIC_TYPE, "metric must be MAX_SIM_L2, MAX_SIM_IP or MAX_SIM_COSINE");
        require_device(device);
        KB2_REQUIRE(device < 64, KB2_INVALID_ARGS, "bad device ordinal");
        if (out_stats) out_stats[0] = out_stats[1] = out_stats[2] = 0;
        const std::vector<int64_t> xl = read_lims(base_lims, n_docs, "base");
        const std::vector<int64_t> ql = read_lims(query_lims, n_lists, "query");
        const int64_t nb = xl.back();
        // positions of the selection entries and TMA row coordinates are 32-bit
        KB2_REQUIRE(nb > 0 && nb < (1ll << 31) && n_docs < (1ll << 31) && ql.back() < (1ll << 31), KB2_INVALID_ARGS,
                    "emb-list sizes out of range (base rows 1 .. 2^31 - 1)");
        KB2_REQUIRE(!bitset || bitset_nbits <= 0 || bitset_nbits >= n_docs, KB2_INVALID_ARGS,
                    "bitset has fewer bits than the base has documents");
        if (n_lists == 0) return;
        const int inner = metric == KB2_METRIC_MAX_SIM_L2 ? KB2_METRIC_L2 : metric == KB2_METRIC_MAX_SIM_IP ? KB2_METRIC_IP
                                                                                                            : KB2_METRIC_COSINE;
        BfSlot& slot = g_bf[device];
        std::lock_guard<std::mutex> lk(slot.mu);
        FlatIndex& fi = bf_prepare(slot, device, inner, dim, cuda_stream, base, nb);
        const int64_t nq_rows = ql.back();
        const float* dq = fi.cosine ? fi.normalized(queries, nq_rows) : fi.to_device(queries, (size_t)nq_rows * dim, fi.s_q);
        const uint8_t* dbits = msim::doc_bits_to_device(bitset, bitset_nbits, n_docs, slot.el.bits, fi.stream);
        int64_t* d_ids;
        float* d_dist;
        fi.device_out(n_lists, k, out_ids, out_dist, d_ids, d_dist);
        int64_t stats[3] = {0, 0, 0};
        msim::search(fi, slot.el, dq, xl, ql, dim, fi.metric, k, dbits, d_ids, d_dist, stats);
        fi.results_out(n_lists, k, out_ids, out_dist, d_ids, d_dist);
        fi.base.release();
        fi.n_used = 0;
        if (out_stats) memcpy(out_stats, stats, sizeof(stats));
    });
}

// ---------------------------------------------------------------- sparse float vectors (kb2_sparse.cuh)
int
kb2_index_add_sparse(kb2_index_t h, const int64_t* indptr, const uint32_t* indices, const float* values, int64_t n) {
    return on_sparse(h, [&](SparseIndex* sx) { sx->add_rows(indptr, indices, values, n); });
}
int
kb2_index_search_sparse(kb2_index_t h, const int64_t* q_indptr, const uint32_t* q_indices, const float* q_values, int64_t nq, int k,
                        const char* json, const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist) {
    return on_sparse(h, [&](SparseIndex* sx) {
        JsonObj cfg = JsonObj::parse(json);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        sx->search_sparse(q_indptr, q_indices, q_values, nq, k, cfg, bitset, bitset_nbits, out_ids, out_dist, false);
    });
}
int
kb2_index_range_search_sparse(kb2_index_t h, const int64_t* q_indptr, const uint32_t* q_indices, const float* q_values, int64_t nq,
                              float radius, float range_filter, int has_range_filter, const char* json, const uint8_t* bitset,
                              int64_t bitset_nbits, int64_t** out_lims, int64_t** out_ids, float** out_dist) {
    return on_sparse(h, [&](SparseIndex* sx) {
        KB2_REQUIRE(out_lims && out_ids && out_dist, KB2_INVALID_ARGS, "null output");
        JsonObj cfg = JsonObj::parse(json);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        sx->range_search_sparse(q_indptr, q_indices, q_values, nq, radius, range_filter, has_range_filter != 0, cfg, bitset,
                                bitset_nbits, out_lims, out_ids, out_dist);
    });
}
// The base rows become the rows of a per-device scratch sparse index (same build, same kernels), searched without
// drop_ratio_search.  Its stream, events and search scratch are reused across calls; its rows and postings are not kept.
namespace {
struct SparseBfSlot {
    std::mutex mu;
    std::unique_ptr<SparseIndex> sx;
};
SparseBfSlot g_sparse_bf[64];
}  // namespace

int
kb2_bruteforce_search_sparse(const int64_t* base_indptr, const uint32_t* base_indices, const float* base_values, int64_t nb,
                             const int64_t* q_indptr, const uint32_t* q_indices, const float* q_values, int64_t nq, int metric, int k,
                             const char* json, const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist,
                             int device) {
    return guarded([&] {
        KB2_REQUIRE(nb > 0 && nq >= 0, KB2_INVALID_ARGS, "bad sizes");
        KB2_REQUIRE(k > 0 && k <= kMaxLargeK, KB2_INVALID_ARGS, "k out of range (1..16384)");
        KB2_REQUIRE(metric == KB2_METRIC_IP || metric == KB2_METRIC_BM25, KB2_INVALID_METRIC_TYPE, "metric must be IP or BM25");
        JsonObj cfg = JsonObj::parse(json);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        require_device(device);
        KB2_REQUIRE(device < 64, KB2_INVALID_ARGS, "bad device ordinal");
        SparseBfSlot& slot = g_sparse_bf[device];
        std::lock_guard<std::mutex> lk(slot.mu);
        if (!slot.sx) {
            slot.sx.reset(new SparseIndex());
            slot.sx->init("SPARSE_INVERTED_INDEX", metric, 0, device);
        }
        SparseIndex& sx = *slot.sx;
        sx.metric = metric;
        sx.last = Counters{};
        sx.clear_rows();
        try {
            sx.set_bm25(cfg);   // the search config's BM25 parameters; no build-only key is checked here
            sx.wait_caller_work();
            sx.add_rows(base_indptr, base_indices, base_values, nb);
            sx.search_sparse(q_indptr, q_indices, q_values, nq, k, cfg, bitset, bitset_nbits, out_ids, out_dist, true);
        } catch (...) {
            sx.clear_rows();
            throw;
        }
        sx.clear_rows();
    });
}

// ---------------------------------------------------------------- emb-list search on an index (TokenANN)
int
kb2_index_set_emb_list(kb2_index_t h, const int64_t* lims, int64_t n_docs, int metric) {
    return on_index(h, [&](IndexBase* ix) {
        ix->refuse(IndexBase::kEmbList);
        KB2_REQUIRE(lims != nullptr && n_docs >= 1, KB2_INVALID_ARGS, "emb-list offsets: null, or no document");
        set_emb_list(*ix, read_lims(lims, n_docs, "document"), metric);
    });
}
int
kb2_index_emb_list_offsets(kb2_index_t h, int64_t* n_docs, int64_t* lims) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        std::lock_guard<std::mutex> lk(ix->mu);
        KB2_REQUIRE(n_docs != nullptr, KB2_INVALID_ARGS, "null argument");
        KB2_REQUIRE(ix->emb_list != nullptr, KB2_INVALID_ARGS, "the index has no emb-list offsets");
        *n_docs = ix->emb_list->n_docs();
        if (lims) memcpy(lims, ix->emb_list->lims.data(), ix->emb_list->lims.size() * 8);
    });
}
int
kb2_index_search_emb_list(kb2_index_t h, const float* queries, const int64_t* query_lims, int64_t n_lists, int k,
                          const char* json, const uint8_t* bitset, int64_t bitset_nbits, int64_t* out_ids, float* out_dist,
                          int64_t* out_stats) {
    return on_index(h, [&](IndexBase* ix) {
        // index_node.cc:275-297: a query with list offsets needs an emb-list index
        KB2_REQUIRE(ix->emb_list != nullptr, KB2_EMB_LIST_INNER_ERROR, "the index has no emb-list offsets (kb2_index_set_emb_list)");
        KB2_REQUIRE(query_lims && out_ids && out_dist && n_lists >= 0, KB2_INVALID_ARGS, "null buffer or bad list count");
        KB2_REQUIRE(k > 0 && k <= kMaxLargeK, KB2_INVALID_ARGS, "k out of range (1..16384)");
        KB2_REQUIRE(is_device_ptr(out_ids) == is_device_ptr(out_dist), KB2_INVALID_ARGS,
                    "out_ids and out_dist must both be host or both be device buffers");
        JsonObj cfg = JsonObj::parse(json);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        if (out_stats) out_stats[0] = out_stats[1] = out_stats[2] = 0;
        const std::vector<int64_t> ql = read_lims(query_lims, n_lists, "query");
        KB2_REQUIRE(ql.back() < (1ll << 31), KB2_INVALID_ARGS, "emb-list sizes out of range (query rows < 2^31)");
        KB2_REQUIRE(queries || ql.back() == 0, KB2_INVALID_ARGS, "null queries");
        ix->last = Counters{};
        ix->wait_caller_work();
        int64_t stats[3] = {0, 0, 0};
        search_emb_list(*ix, queries, ql, k, cfg, bitset, bitset_nbits, out_ids, out_dist, stats);
        if (out_stats) memcpy(out_stats, stats, sizeof(stats));
    });
}
int
kb2_index_emb_list_stage_ms(kb2_index_t h, float* out4) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        std::lock_guard<std::mutex> lk(ix->mu);
        KB2_REQUIRE(out4 != nullptr && ix->emb_list != nullptr, KB2_INVALID_ARGS, "null argument or no emb-list offsets");
        memcpy(out4, ix->emb_list->stage_ms, sizeof(ix->emb_list->stage_ms));
    });
}

// ---------------------------------------------------------------- multi-GPU: NCCL communicator behind the ABI
int
kb2_comm_unique_id(uint8_t* out128) {
    return guarded([&] {
        KB2_REQUIRE(out128 != nullptr, KB2_INVALID_ARGS, "null buffer");
        static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
        ncclUniqueId id;
        KB2_NCCL_CHECK(Comm::api().GetUniqueId(&id));
        memcpy(out128, &id, 128);
    });
}
int
kb2_comm_create(const uint8_t* id128, int rank, int world, int device, kb2_comm_t* out) {
    return guarded([&] {
        KB2_REQUIRE(id128 && out, KB2_INVALID_ARGS, "null argument");
        KB2_REQUIRE(world >= 1 && rank >= 0 && rank < world, KB2_INVALID_ARGS, "bad rank/world");
        *out = nullptr;
        require_device(device);
        ncclUniqueId id;
        memcpy(&id, id128, 128);
        std::unique_ptr<Comm> c(new Comm());
        c->rank = rank;
        c->world = world;
        c->device = device;
        KB2_NCCL_CHECK(Comm::api().CommInitRank(&c->comm, world, id, rank));
        *out = reinterpret_cast<kb2_comm_t>(c.release());
    });
}
void
kb2_comm_destroy(kb2_comm_t c) {
    delete reinterpret_cast<Comm*>(c);
}
int
kb2_comm_all_gather(kb2_comm_t c, const void* send, void* recv, size_t bytes, void* cuda_stream) {
    return guarded([&] {
        KB2_REQUIRE(c && send && recv, KB2_INVALID_ARGS, "null argument");
        Comm* cc = reinterpret_cast<Comm*>(c);
        KB2_CUDA_CHECK(cudaSetDevice(cc->device));
        cc->all_gather(send, recv, bytes, (cudaStream_t)cuda_stream);
    });
}
int
kb2_index_set_comm(kb2_index_t h, kb2_comm_t c) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        std::lock_guard<std::mutex> lk(ix->mu);
        Comm* cc = reinterpret_cast<Comm*>(c);
        if (cc) {
            KB2_REQUIRE(cc->rank == ix->shard_rank && cc->world == ix->shard_world, KB2_INVALID_ARGS,
                        "communicator rank/world differ from kb2_index_set_shard");
            KB2_REQUIRE(cc->device == ix->device, KB2_INVALID_ARGS, "communicator lives on another device");
        }
        ix->set_comm(cc);
    });
}

// ---------------------------------------------------------------- multi-GPU merge
int
kb2_merge_topk(int metric, int world, int64_t nq, int k, const int64_t* in_ids, const float* in_dist, int64_t* out_ids,
               float* out_dist, int device, void* cuda_stream) {
    return guarded([&] {
        KB2_REQUIRE(in_ids && in_dist && out_ids && out_dist, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(world >= 1 && k >= 1 && (int64_t)world * k <= kMaxSortEntries, KB2_INVALID_ARGS, "world*k too large");
        require_device(device);
        merge_topk_device(metric, world, nq, k, in_ids, in_dist, out_ids, out_dist, (cudaStream_t)cuda_stream);
    });
}

// ---------------------------------------------------------------- validation hook for the two contractions
int
kb2_debug_gemm_keys(const float* q, int64_t nq, const float* x, int64_t nb, int dim, int metric, int use_tc, float* out_keys,
                    int device) {
    return guarded([&] {
        require_device(device);
        KB2_REQUIRE(is_device_ptr(q) && is_device_ptr(x) && is_device_ptr(out_keys), KB2_INVALID_ARGS,
                    "debug_gemm_keys takes device pointers");
        const int64_t ldk = (nb + 3) & ~(int64_t)3;
        DevBuf<float> qn, xn;
        qn.ensure(nq);
        xn.ensure(nb);
        row_norms_kernel<<<grid1d(nq * 32, 256), 256>>>(q, nq, dim, qn.p);
        row_norms_kernel<<<grid1d(nb * 32, 256), 256>>>(x, nb, dim, xn.p);
        const bool ran_tc = launch_gemm_keys(nullptr, use_tc ? 1 : 0, metric, q, x, qn.p, xn.p, (int)nq, (int)nb, dim, out_keys,
                                             ldk, nullptr, nullptr, 0);
        KB2_CUDA_CHECK(cudaGetLastError());
        KB2_CUDA_CHECK(cudaDeviceSynchronize());
        KB2_REQUIRE(!use_tc || ran_tc, KB2_INTERNAL_ERROR, "tensor-core contraction unavailable (tensor map / alignment)");
    });
}

// ---------------------------------------------------------------- validation hook for the IVF build's k-means
int
kb2_debug_kmeans(const float* x, int64_t n, int dim, int k, int metric, int niter, uint64_t seed, float* out_centroids,
                 int device) {
    return guarded([&] {
        require_device(device);
        KB2_REQUIRE(x && out_centroids, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(is_device_ptr(x) && is_device_ptr(out_centroids), KB2_INVALID_ARGS, "debug_kmeans takes device pointers");
        KB2_REQUIRE(metric == KB2_METRIC_L2 || metric == KB2_METRIC_IP, KB2_INVALID_METRIC_TYPE, "metric must be L2 or IP");
        KB2_REQUIRE(dim > 0 && k > 0 && niter >= 0 && n < (1ll << 31), KB2_INVALID_ARGS, "bad sizes");
        KB2_CUDA_CHECK(cudaDeviceSynchronize());   // the caller's rows are ready before the default stream reads them
        kmeans_train(x, n, dim, k, metric, niter, seed, out_centroids, nullptr);
        KB2_CUDA_CHECK(cudaDeviceSynchronize());
        KB2_CUDA_CHECK(cudaGetLastError());
    });
}

// ---------------------------------------------------------------- validation hook for the MUVERA encoder
int
kb2_debug_muvera_encode(const float* x, const int64_t* lims, int64_t n_items, int dim, int num_projections, int num_repeats,
                        int seed, int mean, float* out_projections, float* out_fde, int device) {
    return guarded([&] {
        require_device(device);
        KB2_REQUIRE(lims && n_items >= 0 && dim > 0, KB2_INVALID_ARGS, "bad sizes");
        KB2_REQUIRE(num_projections >= 1 && num_projections <= 7 && num_repeats >= 1 && num_repeats <= 32, KB2_OUT_OF_RANGE_IN_JSON,
                    "muvera_num_projections (1..7) or muvera_num_repeats (1..32) out of range");
        const MuveraParams mp{num_projections, num_repeats, seed};
        const std::vector<int64_t> hl = read_lims(lims, n_items, "item");
        const int64_t ntok = hl.back(), E = (int64_t)num_repeats * (1ll << num_projections) * dim;
        KB2_REQUIRE(x || ntok == 0, KB2_INVALID_ARGS, "null rows");
        const std::vector<float> hp = muvera_projections(mp, dim);
        if (out_projections) KB2_CUDA_CHECK(cudaMemcpy(out_projections, hp.data(), hp.size() * 4, cudaMemcpyDefault));
        if (!out_fde || n_items == 0) return;
        DevBuf<float> dp, dx, dout;
        DevBuf<int64_t> dl;
        DevBuf<uint8_t> bucket;
        dp.ensure(hp.size());
        dl.ensure(hl.size());
        dx.ensure((size_t)std::max<int64_t>(ntok, 1) * dim);
        dout.ensure((size_t)n_items * E);
        KB2_CUDA_CHECK(cudaMemcpy(dp.p, hp.data(), hp.size() * 4, cudaMemcpyHostToDevice));
        KB2_CUDA_CHECK(cudaMemcpy(dl.p, hl.data(), hl.size() * 8, cudaMemcpyHostToDevice));
        if (ntok) KB2_CUDA_CHECK(cudaMemcpy(dx.p, x, (size_t)ntok * dim * 4, cudaMemcpyDefault));
        muvera_encode(mp, dim, dp.p, dx.p, ntok, dl.p, 0, n_items, mean != 0, bucket, dout.p, nullptr);
        KB2_CUDA_CHECK(cudaDeviceSynchronize());
        KB2_CUDA_CHECK(cudaMemcpy(out_fde, dout.p, (size_t)n_items * E * 4, cudaMemcpyDefault));
    });
}

// ---------------------------------------------------------------- validation hook for GPU_CAGRA's intermediate graph
int
kb2_debug_cagra_knn_graph(const float* x, int64_t n, int dim, int metric, const char* json, int32_t* out_ids, float* out_keys,
                          int* out_iters, int64_t* out_updates, int updates_cap, float* out_ms, int device) {
    return guarded([&] {
        require_device(device);
        KB2_REQUIRE(x && out_ids && out_keys, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(is_device_ptr(x) && is_device_ptr(out_ids) && is_device_ptr(out_keys), KB2_INVALID_ARGS,
                    "debug_cagra_knn_graph takes device rows, ids and keys");
        KB2_REQUIRE(metric == KB2_METRIC_L2 || metric == KB2_METRIC_IP, KB2_INVALID_METRIC_TYPE, "metric must be L2 or IP");
        KB2_REQUIRE(n >= 2 && n < (1ll << 31) && dim > 0, KB2_INVALID_ARGS, "bad sizes");
        JsonObj cfg = JsonObj::parse(json);
        KB2_REQUIRE(cfg.ok, KB2_INVALID_PARAM_IN_JSON, "malformed json");
        CagraIndex ix;
        ix.init("GPU_CAGRA", metric, dim, device);
        ix.configure(cfg);
        ix.n = n;
        ix.d_vecs.borrow(x, (size_t)n * dim);
        ix.d_norms.alloc_exact((size_t)n);
        KB2_CUDA_CHECK(cudaDeviceSynchronize());   // the caller's rows are ready before the index's stream reads them
        row_norms_kernel<<<grid1d(n * 32, 256), 256, 0, ix.stream>>>(x, n, dim, ix.d_norms.p);
        const int m = (int)std::min<int64_t>(ix.igd, n - 1);
        KB2_CUDA_CHECK(cudaEventRecord(ix.ev0, ix.stream));
        ix.knn_graph(m, out_ids, out_keys);
        KB2_CUDA_CHECK(cudaEventRecord(ix.ev1, ix.stream));
        KB2_CUDA_CHECK(cudaStreamSynchronize(ix.stream));
        KB2_CUDA_CHECK(cudaGetLastError());
        if (out_iters) *out_iters = (int)ix.nnd_updates.size();
        for (int t = 0; out_updates && t < (int)ix.nnd_updates.size() && t < updates_cap; t++) out_updates[t] = ix.nnd_updates[t];
        float ms = 0.f;
        KB2_CUDA_CHECK(cudaEventElapsedTime(&ms, ix.ev0, ix.ev1));
        if (out_ms) *out_ms = ms;
    });
}

// ---------------------------------------------------------------- introspection
int
kb2_index_last_search_counters(kb2_index_t h, int64_t* out8) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        const Counters& c = ix->last;
        out8[0] = c.launches;
        out8[1] = c.codes;
        out8[2] = c.code_bytes;
        out8[3] = c.pairs;
        out8[4] = c.h2d;
        out8[5] = c.d2h;
        out8[6] = c.survivors;
        out8[7] = c.flagged;
    });
}
int
kb2_index_enable_kernel_timing(kb2_index_t h, int on) {
    return guarded([&] { ix_of(h)->timing = (on != 0); });
}
int
kb2_index_last_kernel_ms(kb2_index_t h, float* out_ms) {
    return guarded([&] { *out_ms = ix_of(h)->last_kernel_ms; });
}
int
kb2_index_last_stage_info(kb2_index_t h, float* out4) {
    return guarded([&] {
        IndexBase* ix = ix_of(h);
        out4[0] = ix->last_stage_ms;
        out4[1] = ix->last_kernel_ms;
        out4[2] = (float)ix->last_engine;
        out4[3] = ix->last_comm_ms;
    });
}

}  // extern "C"
