// kb2_range.cuh — RangeSearch, multi-GPU candidate merge, and the "KB2I" serialisation container.
//
// RangeSearch (reference: flat.cc:154-234, ivf.cc:1229-1500, include/knowhere/range_util.h:23-26):
// the scan kernels emit every in-range hit into a global append buffer; the host orders each query's
// hits best-first, applies max_empty_result_buckets (ivf_config.h:51-58) and builds lims.
#pragma once
#include <algorithm>
#include <cstring>
#include <memory>

#include "kb2_blob.h"
#include "kb2_cagra.cuh"
#include "kb2_emb_list_index.cuh"
#include "kb2_hnsw.cuh"
#include "kb2_index.cuh"
#include "kb2_sparse.cuh"

namespace kb2 {

inline void
range_search_index(IndexBase& ix, const float* queries, int64_t nq, float radius, float range_filter, bool has_filter,
                   const JsonObj& cfg, const uint8_t* bitset, int64_t nbits, int64_t** out_lims, int64_t** out_ids,
                   float** out_dist) {
    ix.refuse(IndexBase::kRangeSearch);
    KB2_REQUIRE(ix.count() > 0, KB2_EMPTY_INDEX, "index is empty");
    if (nq == 0) {
        *out_lims = (int64_t*)calloc(1, sizeof(int64_t));
        *out_ids = (int64_t*)malloc(8);
        *out_dist = (float*)malloc(4);
        return;
    }
    RangeParams rp{};
    rp.sp.queries = ix.to_device(queries, (size_t)nq * ix.dim, ix.s_q);
    rp.sp.nq = (int)nq;
    rp.sp.d = ix.dim;
    rp.sp.metric = ix.metric;
    rp.sp.bitset = ix.bitset_to_device(bitset, nbits);
    rp.radius = radius;
    rp.range_filter = range_filter;
    rp.has_filter = has_filter ? 1 : 0;
    rp.single_len = -1;
    int nprobe = 0;
    const std::vector<RangeHit> h = ix.range_hits(rp, cfg, nprobe);
    const std::vector<int64_t> hlabels = ix.labels.host(ix.count());
    struct Out { int64_t q; int probe; float dist; int64_t label; };
    std::vector<Out> o;
    o.reserve(h.size());
    for (const RangeHit& e : h) o.push_back(Out{e.q, e.probe, e.dist, hlabels.empty() ? (int64_t)e.pos : hlabels[e.pos]});
    const size_t found = o.size();
    const bool is_ip = ix.metric == KB2_METRIC_IP;
    std::sort(o.begin(), o.end(), [&](const Out& a, const Out& b) {
        if (a.q != b.q) return a.q < b.q;
        if (a.dist != b.dist) return is_ip ? a.dist > b.dist : a.dist < b.dist;
        return a.label < b.label;
    });
    // max_empty_result_buckets: drop hits of probes after `max_empty` consecutive empty probes.  A probe's hits are then
    // every hit inside the radius (IvfIndex::range_hits), so range_filter applies here, after the cut.
    std::vector<char> keep(found, 1);
    const int max_empty = nprobe > 0 ? range_max_empty(cfg) : 0;
    if (max_empty > 0) {
        size_t i = 0;
        std::vector<int> per_probe(nprobe);
        while (i < found) {
            size_t j = i;
            std::fill(per_probe.begin(), per_probe.end(), 0);
            while (j < found && o[j].q == o[i].q) per_probe[o[j++].probe]++;
            int cut = nprobe, run = 0;
            for (int pj = 0; pj < nprobe; pj++) {
                run = per_probe[pj] == 0 ? run + 1 : 0;
                if (run == max_empty) { cut = pj + 1; break; }
            }
            for (size_t t = i; t < j; t++)
                keep[t] = o[t].probe < cut && in_range_host(o[t].dist, radius, range_filter, has_filter, ix.metric);
            i = j;
        }
    }
    int64_t* lims = (int64_t*)calloc(nq + 1, sizeof(int64_t));
    size_t total = 0;
    for (size_t i = 0; i < found; i++) total += keep[i];
    int64_t* ids = (int64_t*)malloc(std::max<size_t>(total, 1) * 8);
    float* dist = (float*)malloc(std::max<size_t>(total, 1) * 4);
    KB2_REQUIRE(lims && ids && dist, KB2_MALLOC_ERROR, "malloc failed");
    size_t w = 0;
    for (size_t i = 0; i < found; i++) {
        if (!keep[i]) continue;
        ids[w] = o[i].label;
        dist[w] = o[i].dist;
        lims[o[i].q + 1]++;
        w++;
    }
    for (int64_t i = 0; i < nq; i++) lims[i + 1] += lims[i];
    *out_lims = lims;
    *out_ids = ids;
    *out_dist = dist;
}

inline void
merge_topk_device(int metric, int world, int64_t nq, int k, const int64_t* in_ids, const float* in_dist,
                  int64_t* out_ids, float* out_dist, cudaStream_t st) {
    const size_t cnt = (size_t)world * nq * k;
    DevBuf<int64_t> b_ids, b_oids;
    DevBuf<float> b_dist, b_odist;
    const int64_t* d_in_ids = in_ids;
    const float* d_in_dist = in_dist;
    if (!is_device_ptr(in_ids)) {
        b_ids.ensure(cnt);
        b_dist.ensure(cnt);
        KB2_CUDA_CHECK(cudaMemcpyAsync(b_ids.p, in_ids, cnt * 8, cudaMemcpyHostToDevice, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(b_dist.p, in_dist, cnt * 4, cudaMemcpyHostToDevice, st));
        d_in_ids = b_ids.p;
        d_in_dist = b_dist.p;
    }
    int64_t* d_oids = out_ids;
    float* d_odist = out_dist;
    const bool dev_out = is_device_ptr(out_ids);
    if (!dev_out) {
        b_oids.ensure((size_t)nq * k);
        b_odist.ensure((size_t)nq * k);
        d_oids = b_oids.p;
        d_odist = b_odist.p;
    }
    launch_merge_topk(metric, world, nq, k, d_in_ids, d_in_dist, d_oids, d_odist, st);
    KB2_CUDA_CHECK(cudaGetLastError());
    if (!dev_out) {
        KB2_CUDA_CHECK(cudaMemcpyAsync(out_ids, d_oids, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(out_dist, d_odist, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, st));
    }
    KB2_CUDA_CHECK(cudaStreamSynchronize(st));
}

// ------------------------------------------------------------------------------------------
// "KB2I" container: little-endian, self-describing.  (Reference persistence is the faiss fourcc
// stream inside a BinarySet — K/impl/index_write.cpp:716-745; wire compatibility is SURVEY §8f
// rank 2 and not claimed here.)
// ------------------------------------------------------------------------------------------
// a fresh index of the named type (before IndexBase::init), or null when the type is unknown
inline std::unique_ptr<IndexBase>
make_index(const std::string& type) {
    if (type == "FLAT") return std::make_unique<FlatIndex>();
    if (type == "IVF_FLAT" || type == "IVF_PQ") {
        auto iv = std::make_unique<IvfIndex>();
        iv->is_pq = (type == "IVF_PQ");
        return iv;
    }
    if (type == "HNSW") return std::make_unique<HnswIndex>();
    if (type == "GPU_CAGRA" || type == "GPU_CUVS_CAGRA") return std::make_unique<CagraIndex>();
    if (is_sparse_type(type)) return std::make_unique<SparseIndex>();
    return nullptr;
}

inline void
serialize_index(IndexBase& ix, std::vector<uint8_t>& blob) {
    // a MUVERA index is stored as its base (the documents' FDE rows) followed by its emb-list section
    auto* mv = dynamic_cast<MuveraIndex*>(&ix);
    KB2_REQUIRE(!mv || ix.emb_list, KB2_INVALID_ARGS, "a MUVERA index is serialised once its documents are attached (kb2_index_set_emb_list)");
    IndexBase& body = mv ? mv->base_index() : ix;
    BlobWriter w{blob};
    w.put<uint32_t>(0x4932424b);  // "KB2I"
    w.put<uint32_t>(1);
    w.put_str(body.type);
    w.put<int32_t>(body.cosine ? KB2_METRIC_COSINE : body.metric);
    w.put<int32_t>(body.dim);
    body.save(w);
    // MUVERA: "ELMV", the strategy (1: MUVERA), the MAX_SIM metric, P, R, S, the token dimension, n_docs,
    // offsets[n_docs + 1] and the token rows [offsets[n_docs]][d] as added; the projections are drawn again on load
    if (mv) {
        w.put<uint32_t>(kEmbListMuveraTag);
        w.put<int32_t>(1);
        w.put<int32_t>(ix.emb_list->metric);
        w.put<int32_t>(mv->mp.P);
        w.put<int32_t>(mv->mp.R);
        w.put<int32_t>(mv->mp.S);
        w.put<int32_t>(ix.dim);
        w.put<int64_t>(ix.emb_list->n_docs());
        w.put_bytes(ix.emb_list->lims.data(), ix.emb_list->lims.size() * 8);
        std::vector<float> t((size_t)ix.count() * ix.dim);
        if (!t.empty()) KB2_CUDA_CHECK(cudaMemcpy(t.data(), mv->tokens.p, t.size() * 4, cudaMemcpyDeviceToHost));
        w.put_bytes(t.data(), t.size() * 4);
        return;
    }
    // optional trailing section of an emb-list index: "ELST", the MAX_SIM metric, n_docs, offsets[n_docs + 1]
    if (ix.emb_list) {
        w.put<uint32_t>(kEmbListTag);
        w.put<int32_t>(ix.emb_list->metric);
        w.put<int64_t>(ix.emb_list->n_docs());
        w.put_bytes(ix.emb_list->lims.data(), ix.emb_list->lims.size() * 8);
    }
}

inline std::unique_ptr<IndexBase>
deserialize_index(const uint8_t* blob, size_t size, int device) {
    BlobReader r{blob, size};
    KB2_REQUIRE(r.get<uint32_t>() == 0x4932424b, KB2_INVALID_BINARY_SET, "bad magic");
    KB2_REQUIRE(r.get<uint32_t>() == 1, KB2_INVALID_BINARY_SET, "unsupported version");
    const std::string type = r.get_str();
    const int metric = r.get<int32_t>();
    const int dim = r.get<int32_t>();
    if (is_sparse_type(type)) {
        KB2_REQUIRE(dim == 0, KB2_INVALID_BINARY_SET, "bad dim in blob");
        KB2_REQUIRE(metric == KB2_METRIC_IP || metric == KB2_METRIC_BM25, KB2_INVALID_BINARY_SET, "bad metric in blob");
    } else {
        KB2_REQUIRE(dim > 0 && dim <= (1 << 20), KB2_INVALID_BINARY_SET, "bad dim in blob");
        KB2_REQUIRE(metric == KB2_METRIC_L2 || metric == KB2_METRIC_IP || metric == KB2_METRIC_COSINE, KB2_INVALID_BINARY_SET,
                    "bad metric in blob");
    }
    std::unique_ptr<IndexBase> ix = make_index(type);
    KB2_REQUIRE(ix, KB2_INVALID_BINARY_SET, "unknown index type in blob");
    ix->init(type, metric, dim, device);   // COSINE: the stored vectors are already normalised; queries will be
    ix->load(r);
    if (r.o < r.n) {
        const uint32_t tag = r.get<uint32_t>();
        KB2_REQUIRE(tag == kEmbListTag || tag == kEmbListMuveraTag, KB2_INVALID_BINARY_SET, "unknown section after the index in blob");
        MuveraParams mp;
        int d = 0;
        if (tag == kEmbListMuveraTag) {
            KB2_REQUIRE(r.get<int32_t>() == 1, KB2_INVALID_BINARY_SET, "unknown emb-list strategy in blob");
        }
        const int el_metric = r.get<int32_t>();
        if (tag == kEmbListMuveraTag) {
            mp.P = r.get<int32_t>();
            mp.R = r.get<int32_t>();
            mp.S = r.get<int32_t>();
            d = r.get<int32_t>();
            KB2_REQUIRE(ix->takes_emb_list() && mp.P >= 1 && mp.P <= 7 && mp.R >= 1 && mp.R <= 32 && d > 0 && (int64_t)mp.R * (1 << mp.P) * d == dim,
                        KB2_INVALID_BINARY_SET, "bad MUVERA parameters in blob");
        }
        const int64_t nd = r.get<int64_t>();
        KB2_REQUIRE(nd >= 1 && (uint64_t)nd < (r.n - r.o) / 8, KB2_INVALID_BINARY_SET, "bad emb-list document count in blob");
        std::vector<int64_t> lims((size_t)nd + 1);
        memcpy(lims.data(), r.get_bytes(lims.size() * 8), lims.size() * 8);
        KB2_REQUIRE(lims[0] == 0, KB2_INVALID_BINARY_SET, "bad emb-list offsets in blob");
        for (int64_t i = 0; i < nd; i++) KB2_REQUIRE(lims[i + 1] >= lims[i], KB2_INVALID_BINARY_SET, "bad emb-list offsets in blob");
        if (tag == kEmbListTag) {
            set_emb_list(*ix, std::move(lims), el_metric);
            return ix;
        }
        KB2_REQUIRE(lims[nd] >= 1 && (uint64_t)lims[nd] <= (r.n - r.o) / ((size_t)d * 4), KB2_INVALID_BINARY_SET,
                    "bad MUVERA token count in blob");
        auto mv = std::make_unique<MuveraIndex>();
        mv->init(type, metric, d, device);
        mv->mp = mp;
        mv->add((const float*)r.get_bytes((size_t)lims[nd] * d * 4), lims[nd], nullptr);
        set_emb_list(*mv, std::move(lims), el_metric, std::move(ix));
        return mv;
    }
    return ix;
}

}  // namespace kb2
