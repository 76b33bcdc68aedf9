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

namespace kb2 {

inline void
range_search_index(IndexBase& ix, const float* queries, int64_t nq, float radius, float range_filter, bool has_filter,
                   const JsonObj& cfg, const uint8_t* bitset, int64_t nbits, int64_t** out_lims, int64_t** out_ids,
                   float** out_dist) {
    cudaStream_t st = ix.stream;
    FlatIndex* fi = dynamic_cast<FlatIndex*>(&ix);
    IvfIndex* iv = dynamic_cast<IvfIndex*>(&ix);
    HnswIndex* hn = dynamic_cast<HnswIndex*>(&ix);
    KB2_REQUIRE(fi || iv || hn, KB2_NOT_IMPLEMENTED, "RangeSearch: unknown index class");
    KB2_REQUIRE(!dynamic_cast<CagraIndex*>(&ix), KB2_NOT_IMPLEMENTED, "RangeSearch is not implemented on GPU_CAGRA");
    KB2_REQUIRE(ix.count() > 0, KB2_EMPTY_INDEX, "index is empty");
    if (nq == 0) {
        *out_lims = (int64_t*)calloc(1, sizeof(int64_t));
        *out_ids = (int64_t*)malloc(8);
        *out_dist = (float*)malloc(4);
        return;
    }
    const float* dq = ix.to_device(queries, (size_t)nq * ix.dim, ix.s_q);
    const uint8_t* dbits = ix.bitset_to_device(bitset, nbits);
    RangeParams rp{};
    IvfScanParams& sp = rp.sp;
    sp.queries = dq;
    sp.nq = (int)nq;
    sp.d = ix.dim;
    sp.metric = ix.metric;
    sp.bitset = dbits;
    rp.radius = radius;
    rp.range_filter = range_filter;
    rp.has_filter = has_filter ? 1 : 0;
    rp.single_len = -1;
    int nprobe = 1;
    int max_empty = 0;
    size_t smem = (size_t)ix.dim * 4 + 64;
    DevBuf<RangeHit> hits;
    unsigned long long found = 0;
    bool graph_hits = false;   // hits came from the HNSW traversal (range_filter still to be applied)
    if (hn) {
        bool bf = false;
        found = hn->range_hits(dq, nq, radius, cfg, dbits, hits, bf);
        graph_hits = !bf;
    }
    if (fi || (hn && !graph_hits)) {
        // exact scan of the stored vectors (FLAT; HNSW when the reference falls back to brute force)
        rp.kind = 0;
        sp.vecs = fi ? fi->base.p : hn->d_vecs.p;
        sp.rows = nullptr;
        rp.single_len = ix.count();
        sp.nsplit = (int)std::min<int64_t>(std::max<int64_t>(1, (2 * num_sms() + nq - 1) / nq),
                                           std::max<int64_t>(1, ix.count() / 1024));
        smem += 64;
    } else if (iv) {
        KB2_REQUIRE(iv->trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        iv->seal();
        nprobe = (int)std::min<int64_t>(std::max<int64_t>(cfg.get_int("nprobe", 8), 1), iv->nlist);
        max_empty = (int)cfg.get_int("max_empty_result_buckets", 2);
        ix.s_probe_ids.ensure((size_t)nq * nprobe);
        ix.s_probe_dis.ensure((size_t)nq * nprobe);
        iv->coarse_probes(dq, 0, nq, nprobe);
        sp.probe_ids = ix.s_probe_ids.p;
        sp.probe_dis = ix.s_probe_dis.p;
        sp.nprobe = nprobe;
        sp.list_off = iv->list_off.p;
        sp.list_len = iv->list_len.p;
        sp.rows = iv->rows.p;
        sp.vecs = iv->vecs.p;
        sp.pq_centroids = iv->pqc.p;
        sp.M = iv->M;
        sp.dsub = iv->dsub;
        sp.codes = (const uint4*)iv->codes.p;
        sp.npad = iv->npad;
        sp.t1 = iv->t1.p;
        rp.kind = iv->is_pq ? (iv->G > 0 ? 1 : 2) : 0;
        rp.G = iv->G;
        rp.codes_b = iv->codes.p;
        sp.nsplit = (nq < 2 * num_sms()) ? (int)std::min<int64_t>(nprobe, (2 * num_sms() + nq - 1) / nq) : 1;
        const int np_max = (nprobe + sp.nsplit - 1) / sp.nsplit;
        smem += (size_t)(np_max + 1) * 4 + (size_t)np_max * 12;
        if (iv->is_pq) smem += (size_t)iv->M * 1024;
        KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_NOT_IMPLEMENTED, "range search: m too large");
    }
    DevBuf<unsigned long long> cnt;
    cnt.ensure(1);
    unsigned long long cap = (unsigned long long)std::max<int64_t>(1 << 20, nq * 256);
    for (int attempt = 0; attempt < 2 && !graph_hits; attempt++) {
        hits.ensure(cap);
        KB2_CUDA_CHECK(cudaMemsetAsync(cnt.p, 0, 8, st));
        rp.hits = hits.p;
        rp.count = cnt.p;
        rp.cap = cap;
        launch<range_scan_kernel>((unsigned)(nq * sp.nsplit), kScanThreads, smem, st, rp);
        ix.last.launches++;
        KB2_CUDA_CHECK(cudaGetLastError());
        KB2_CUDA_CHECK(cudaMemcpyAsync(&found, cnt.p, 8, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        if (found <= cap) break;
        cap = found;
    }
    std::vector<RangeHit> h(found);
    if (found) KB2_CUDA_CHECK(cudaMemcpy(h.data(), hits.p, found * sizeof(RangeHit), cudaMemcpyDeviceToHost));
    ix.last.d2h += (int64_t)(found * sizeof(RangeHit));
    // labels
    std::vector<int32_t> hrows;
    std::vector<int64_t> hlabels;
    const bool custom = fi ? fi->custom_labels : (iv ? iv->custom_labels : hn->custom_labels);
    if (iv) {
        hrows.resize(iv->npad);
        KB2_CUDA_CHECK(cudaMemcpy(hrows.data(), iv->rows.p, iv->npad * 4, cudaMemcpyDeviceToHost));
    }
    if (custom) {
        const int64_t n = ix.count();
        hlabels.resize(n);
        if (hn) hlabels = hn->h_labels;
        else KB2_CUDA_CHECK(cudaMemcpy(hlabels.data(), fi ? fi->labels.p : iv->labels.p, n * 8, cudaMemcpyDeviceToHost));
    }
    struct Out { int64_t q; int probe; float dist; int64_t label; };
    std::vector<Out> o;
    o.reserve(found);
    for (size_t i = 0; i < found; i++) {
        if (graph_hits) {
            // pass-0 hits of a query whose BFS queue overflowed are incomplete: the rerun (later entries) has them all
            if (i < hn->range_pass0_hits && hn->range_overflowed[h[i].q]) continue;
            if (!in_range_host(h[i].dist, radius, range_filter, has_filter, ix.metric)) continue;
        }
        int64_t row = iv ? (int64_t)hrows[h[i].pos] : (int64_t)h[i].pos;
        o.push_back(Out{h[i].q, h[i].probe, h[i].dist, custom ? hlabels[row] : row});
    }
    found = o.size();
    const bool is_ip = ix.metric == KB2_METRIC_IP;
    std::sort(o.begin(), o.end(), [&](const Out& a, const Out& b) {
        if (a.q != b.q) return a.q < b.q;
        if (a.dist != b.dist) return is_ip ? a.dist > b.dist : a.dist < b.dist;
        return a.label < b.label;
    });
    // max_empty_result_buckets: drop hits of probes after `max_empty` consecutive empty probes
    std::vector<char> keep(found, 1);
    if (iv && max_empty > 0) {
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
            for (size_t t = i; t < j; t++) keep[t] = o[t].probe < cut;
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
inline void
serialize_index(IndexBase& ix, std::vector<uint8_t>& blob) {
    BlobWriter w{blob};
    w.put<uint32_t>(0x4932424b);  // "KB2I"
    w.put<uint32_t>(1);
    w.put_str(ix.type);
    w.put<int32_t>(ix.cosine ? KB2_METRIC_COSINE : ix.metric);
    w.put<int32_t>(ix.dim);
    if (auto* fi = dynamic_cast<FlatIndex*>(&ix)) {
        const int64_t n = fi->count();
        w.put<int64_t>(n);
        w.put<int32_t>(fi->custom_labels ? 1 : 0);
        std::vector<float> h((size_t)n * ix.dim);
        if (n) KB2_CUDA_CHECK(cudaMemcpy(h.data(), fi->base.p, h.size() * 4, cudaMemcpyDeviceToHost));
        w.put_bytes(h.data(), h.size() * 4);
        if (fi->custom_labels) {
            std::vector<int64_t> l(n);
            if (n) KB2_CUDA_CHECK(cudaMemcpy(l.data(), fi->labels.p, n * 8, cudaMemcpyDeviceToHost));
            w.put_bytes(l.data(), n * 8);
        }
    } else if (auto* iv = dynamic_cast<IvfIndex*>(&ix)) {
        KB2_REQUIRE(iv->trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        KB2_REQUIRE(iv->shard_world == 1, KB2_NOT_IMPLEMENTED, "serialising a shard");
        iv->seal();
        w.put<int64_t>(iv->nlist);
        w.put<int32_t>(iv->M);
        w.put<int32_t>(iv->nbits);
        w.put<int32_t>(iv->refine ? 1 + iv->refine_kind : 0);   // 0 none, 1 fp32, 2 fp16, 3 bf16 refine store
        DevBuf<float> dec;
        const float* v32 = (iv->is_pq && iv->refine) ? iv->vecs_f32(dec) : nullptr;
        if (v32) KB2_CUDA_CHECK(cudaStreamSynchronize(iv->stream));
        std::vector<float> c((size_t)iv->nlist * ix.dim);
        KB2_CUDA_CHECK(cudaMemcpy(c.data(), iv->centroids.p, c.size() * 4, cudaMemcpyDeviceToHost));
        w.put_bytes(c.data(), c.size() * 4);
        if (iv->is_pq) {
            std::vector<float> pc((size_t)iv->M * 256 * iv->dsub);
            KB2_CUDA_CHECK(cudaMemcpy(pc.data(), iv->pqc.p, pc.size() * 4, cudaMemcpyDeviceToHost));
            w.put_bytes(pc.data(), pc.size() * 4);
        }
        const size_t cs = iv->is_pq ? (size_t)iv->M : (size_t)ix.dim * 4;
        for (int64_t l = 0; l < iv->nlist; l++) {
            const int64_t len = iv->h_list_len[l];
            w.put<int64_t>(len);
            if (!len) continue;
            std::vector<int64_t> ids(len);
            std::vector<uint8_t> cd((size_t)len * cs);
            iv->export_list(l, ids.data(), cd.data());
            w.put_bytes(ids.data(), len * 8);
            w.put_bytes(cd.data(), cd.size());
            if (iv->is_pq && iv->refine) {
                std::vector<float> rv((size_t)len * ix.dim);
                KB2_CUDA_CHECK(cudaMemcpy(rv.data(), v32 + iv->h_list_off[l] * ix.dim, rv.size() * 4, cudaMemcpyDeviceToHost));
                w.put_bytes(rv.data(), rv.size() * 4);
            }
        }
    } else if (auto* cg = dynamic_cast<CagraIndex*>(&ix)) {
        cg->serialize(w);
    } else if (auto* hn = dynamic_cast<HnswIndex*>(&ix)) {
        hn->serialize(w);
    } else {
        throw Error(KB2_NOT_IMPLEMENTED, "serialize: unknown index class");
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
    const int metric_raw = r.get<int32_t>();
    const bool cosine = metric_raw == KB2_METRIC_COSINE;
    const int metric = cosine ? KB2_METRIC_IP : metric_raw;
    const int dim = r.get<int32_t>();
    KB2_REQUIRE(dim > 0 && dim <= (1 << 20), KB2_INVALID_BINARY_SET, "bad dim in blob");
    KB2_REQUIRE(metric == KB2_METRIC_L2 || metric == KB2_METRIC_IP, KB2_INVALID_BINARY_SET, "bad metric in blob");
    std::unique_ptr<IndexBase> ix;
    if (type == "FLAT") {
        auto* fi = new FlatIndex();
        ix.reset(fi);
        fi->type = type; fi->metric = metric; fi->dim = dim; fi->device = device;
        fi->init_common();
        const int64_t n = r.get<int64_t>();
        KB2_REQUIRE(n >= 0 && (uint64_t)n <= size / ((size_t)dim * 4), KB2_INVALID_BINARY_SET, "bad row count in blob");
        const int custom = r.get<int32_t>();
        const float* data = (const float*)r.get_bytes((size_t)n * dim * 4);
        const int64_t* labels = custom ? (const int64_t*)r.get_bytes((size_t)n * 8) : nullptr;
        // blob memory may be unaligned: stage through vectors
        std::vector<float> hd((size_t)n * dim);
        memcpy(hd.data(), data, hd.size() * 4);
        std::vector<int64_t> hl;
        if (custom) { hl.resize(n); memcpy(hl.data(), labels, n * 8); }
        fi->add(hd.data(), n, custom ? hl.data() : nullptr);
    } else if (type == "IVF_FLAT" || type == "IVF_PQ") {
        auto* iv = new IvfIndex();
        ix.reset(iv);
        iv->type = type; iv->metric = metric; iv->dim = dim; iv->device = device;
        iv->is_pq = (type == "IVF_PQ");
        iv->init_common();
        const int64_t nlist = r.get<int64_t>();
        iv->M = r.get<int32_t>();
        iv->nbits = r.get<int32_t>();
        {
            const int rf = r.get<int32_t>();
            KB2_REQUIRE(rf >= 0 && rf <= 3, KB2_INVALID_BINARY_SET, "bad refine field in blob");
            iv->refine = rf != 0;
            iv->refine_kind = rf ? rf - 1 : 0;
        }
        KB2_REQUIRE(nlist >= 1 && (uint64_t)nlist <= size / ((size_t)dim * 4), KB2_INVALID_BINARY_SET, "bad nlist in blob");
        if (iv->is_pq)
            KB2_REQUIRE(iv->M > 0 && dim % iv->M == 0 && iv->nbits == 8, KB2_INVALID_BINARY_SET, "bad m / nbits in blob");
        std::vector<float> c((size_t)nlist * dim);
        memcpy(c.data(), r.get_bytes(c.size() * 4), c.size() * 4);
        std::vector<float> pc;
        if (iv->is_pq) {
            pc.resize((size_t)iv->M * 256 * (dim / iv->M));
            memcpy(pc.data(), r.get_bytes(pc.size() * 4), pc.size() * 4);
        }
        iv->import_begin(nlist, c.data(), iv->is_pq ? pc.data() : nullptr);
        const size_t cs = iv->is_pq ? (size_t)iv->M : (size_t)dim * 4;
        std::vector<float> raw_rows;  // import order
        for (int64_t l = 0; l < nlist; l++) {
            const int64_t len = r.get<int64_t>();
            KB2_REQUIRE(len >= 0 && (uint64_t)len <= size / 8, KB2_INVALID_BINARY_SET, "bad list length in blob");
            if (!len) continue;
            std::vector<int64_t> ids(len);
            memcpy(ids.data(), r.get_bytes(len * 8), len * 8);
            const uint8_t* cd = r.get_bytes((size_t)len * cs);
            iv->import_list(l, len, ids.data(), cd);
            if (iv->is_pq && iv->refine) {
                const uint8_t* rv = r.get_bytes((size_t)len * dim * 4);
                const size_t o = raw_rows.size();
                raw_rows.resize(o + (size_t)len * dim);
                memcpy(raw_rows.data() + o, rv, (size_t)len * dim * 4);
            }
        }
        const bool with_raw = iv->is_pq && iv->refine;
        iv->import_finish(with_raw ? raw_rows.data() : nullptr, with_raw ? (int64_t)(raw_rows.size() / dim) : 0, true);
    } else if (type == "GPU_CAGRA" || type == "GPU_CUVS_CAGRA") {
        auto* cg = new CagraIndex();
        ix.reset(cg);
        cg->type = type; cg->metric = metric; cg->dim = dim; cg->device = device;
        cg->init_common();
        cg->deserialize(r);
    } else if (type == "HNSW") {
        auto* hn = new HnswIndex();
        ix.reset(hn);
        hn->type = type; hn->metric = metric; hn->dim = dim; hn->device = device;
        hn->init_common();
        hn->deserialize(r);
    } else {
        throw Error(KB2_INVALID_BINARY_SET, "unknown index type in blob");
    }
    ix->cosine = cosine;   // stored vectors are already normalised; queries will be
    if (r.o < r.n) {
        KB2_REQUIRE(r.get<uint32_t>() == kEmbListTag, KB2_INVALID_BINARY_SET, "unknown section after the index in blob");
        const int el_metric = r.get<int32_t>();
        const int64_t nd = r.get<int64_t>();
        KB2_REQUIRE(nd >= 1 && (uint64_t)nd < (r.n - r.o) / 8, KB2_INVALID_BINARY_SET, "bad emb-list document count in blob");
        std::vector<int64_t> lims((size_t)nd + 1);
        memcpy(lims.data(), r.get_bytes(lims.size() * 8), lims.size() * 8);
        KB2_REQUIRE(lims[0] == 0, KB2_INVALID_BINARY_SET, "bad emb-list offsets in blob");
        for (int64_t i = 0; i < nd; i++) KB2_REQUIRE(lims[i + 1] >= lims[i], KB2_INVALID_BINARY_SET, "bad emb-list offsets in blob");
        set_emb_list(*ix, std::move(lims), el_metric);
    }
    return ix;
}

}  // namespace kb2
