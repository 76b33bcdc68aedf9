// kb2_index.cuh — host-side index objects behind the C ABI (the IndexBase interface, FLAT, IVF_FLAT, IVF_PQ).
// They play the role of the reference's IndexNode implementations
//   FlatIndexNode  src/index/flat/flat.cc:33-427
//   IvfIndexNode   src/index/ivf/ivf.cc:68-1972   (IVF_FLAT + IVF_PQ branches)
// but hand the WHOLE query batch to the device in one call (like the in-tree GPU precedent,
// src/common/cuvs/integration/cuvs_knowhere_index.cuh:508-632) instead of nq thread-pool tasks.
#pragma once
#include <algorithm>
#include <functional>
#include <memory>
#include <mutex>
#include <vector>

#include "kb2_build.cuh"
#include "kb2_comm.h"
#include "kb2_fourcc.h"
#include "kb2_gemm_tc.cuh"
#include "kb2_ivf.cuh"
#include "kb2_ivfpq_tc.cuh"
#include "kb2_ivfflat_tc.cuh"
#include "kb2_json.h"
#include "kb2_large_k.cuh"

namespace kb2 {

constexpr int kMaxK = 1024;            // largest k' any selection kernel keeps
constexpr int kMaxSortEntries = 8192;  // finalize sorts at most this many candidates per query
constexpr int kMaxLargeK = 16384;      // largest candidate window of the large-k path (DESIGN §4.9)
// scratch of the large-k path beyond the buffers every search uses: queries are processed in groups that fit it, whatever nq
constexpr int64_t kLargeKScratch = 1ll << 30;
// IVF probes (DESIGN §4.9.1).  Up to kMaxWindowProbes the coarse stage selects them in one kMaxK window and one scan CTA holds
// a query's share of them in shared memory; above, up to kMaxNprobe (the reference's range), the coarse stage takes the
// large-k selection, no scan CTA holds more than kScanSliceProbes probes, and the queries run in groups whose probe arrays
// and scan scratch fit kProbeScratch.
constexpr int kMaxWindowProbes = kMaxK - 16;   // 1008
constexpr int kMaxNprobe = 65536;
constexpr int kScanSliceProbes = 1024;
constexpr int64_t kProbeScratch = 1ll << 30;

struct Counters {
    int64_t launches = 0, codes = 0, code_bytes = 0, pairs = 0, h2d = 0, d2h = 0;
    // tensor-core PQ engine: codes re-evaluated exactly / queries redone by the LUT kernel.  FLAT: flagged = queries whose
    // re-ranked window was not certified and which were redone by flat_exact_scan_kernel
    int64_t survivors = 0, flagged = 0;
};

// grow-by-doubling append of `count` elements (device->device or host->device)
template <typename T>
inline void
dev_append(DevBuf<T>& buf, size_t& used, const T* src, size_t count, cudaStream_t st) {
    if (used + count > buf.n) {
        size_t cap = std::max(used + count, buf.n * 2);
        DevBuf<T> nb;
        nb.ensure(cap);
        if (used) KB2_CUDA_CHECK(cudaMemcpyAsync(nb.p, buf.p, used * sizeof(T), cudaMemcpyDeviceToDevice, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        buf = std::move(nb);
    }
    if (count) KB2_CUDA_CHECK(cudaMemcpyAsync(buf.p + used, src, count * sizeof(T), cudaMemcpyDefault, st));
    used += count;
}

// Row -> external id of a dense index.  While every id is its row no array exists and device() is null, which every kernel
// reads as "the id is the row"; the first custom id, or ids that are not the rows (a shard's slice), turn it into an array.
struct RowLabels {
    DevBuf<int64_t> d;
    size_t used = 0;
    bool custom = false;
    const int64_t* device() const { return custom ? d.p : nullptr; }
    // ids of the m rows stored after the `have` ones: ids[0, m) (host or device), else first_id + i.  `force` keeps an
    // array even without ids.
    void
    append(int64_t have, const int64_t* ids, int64_t m, int64_t first_id, bool force, cudaStream_t st) {
        if (!custom && (ids || force)) {
            std::vector<int64_t> h(have);
            for (int64_t i = 0; i < have; i++) h[i] = i;
            used = 0;
            if (have) dev_append(d, used, h.data(), (size_t)have, st);
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
            custom = true;
        }
        if (!custom || m <= 0) return;
        std::vector<int64_t> h;
        if (!ids) {
            h.resize(m);
            for (int64_t i = 0; i < m; i++) h[i] = first_id + i;
        }
        dev_append(d, used, ids ? ids : h.data(), (size_t)m, st);
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    // the first n ids on the host, or nothing while they are the rows
    std::vector<int64_t>
    host(int64_t n) const {
        std::vector<int64_t> h(custom ? n : 0);
        if (!h.empty()) KB2_CUDA_CHECK(cudaMemcpy(h.data(), d.p, h.size() * 8, cudaMemcpyDeviceToHost));
        return h;
    }
};

struct EmbListState;   // kb2_emb_list_index.cuh

// ============================================================================================
struct IndexBase {
    std::string type;
    std::shared_ptr<EmbListState> emb_list;   // document offsets of an emb-list index (kb2_index_set_emb_list), or null
    int metric = KB2_METRIC_L2, dim = 0, device = 0;
    bool cosine = false;   // COSINE: metric == IP over vectors normalised on entry (see kb2_index_create)
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int shard_rank = 0, shard_world = 1;
    // FLAT and HNSW shards keep a row slice of each add(): rows offered over all calls, first global row of the first slice
    int64_t n_global = 0, shard_lo = 0;
    // rows [lo, hi) of an n-row add() that this shard keeps (all of them without sharding)
    std::pair<int64_t, int64_t>
    shard_slice(int64_t n) const {
        return {n * shard_rank / shard_world, n * (shard_rank + 1) / shard_world};
    }
    RowLabels labels;
    std::mutex mu;
    Counters last;
    bool timing = false;
    float last_kernel_ms = 0.f;      // dominant kernel of the last search (IVF_PQ tensor-core engine: the filter kernel)
    float last_stage_ms = 0.f;       // whole list-scan stage of the last search (all engines)
    int last_engine = 0;             // 0: query-major scan kernels, 1: list-major tensor-core engine, 2: large-k path,
                                     // 3: HNSW beam with one query per CTA (hnsw_wide_kernel), 4: GPU_CAGRA,
                                     // 5: sparse tile scoring (kb2_sparse.cuh)
    float last_comm_ms = 0.f;        // collectives (+ merge) of the last sharded search
    Comm* comm = nullptr;            // not owned (kb2_index_set_comm)
    virtual void set_comm(Comm* c) { comm = c; }
    bool distributed() const { return comm != nullptr && shard_world > 1; }
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr, ev_in = nullptr;
    cudaEvent_t ev_c0 = nullptr, ev_c1 = nullptr, ev_c2 = nullptr, ev_c3 = nullptr;   // collectives of a sharded search
    DevBuf<unsigned long long> d_counter;
    PinnedBuf h_counter;   // pinned landing zone of the per-search device counters (no pageable async copy)

    // per-search scratch (grow-only, reused across calls)
    DevBuf<float> s_q, s_keys, s_qn, s_out_dist, s_probe_dis;
    DevBuf<uint64_t> s_partial, s_partial2;
    DevBuf<int64_t> s_out_ids, s_probe_ids;
    DevBuf<uint8_t> s_bitset;
    DevBuf<float> s_cos_in, s_cos_out, s_typed_f32;
    // multi-GPU (kb2_index_set_comm): staging of the local top-k and of the gathered per-shard candidates
    DevBuf<int64_t> s_loc_ids, s_g_ids;
    DevBuf<float> s_loc_dist, s_g_dist;
    void
    ensure_gather_buffers(int64_t nq, int k) {
        s_loc_ids.ensure((size_t)nq * k);
        s_loc_dist.ensure((size_t)nq * k);
        s_g_ids.ensure((size_t)shard_world * nq * k);
        s_g_dist.ensure((size_t)shard_world * nq * k);
    }
    DevBuf<uint8_t> s_typed_raw;
    DevBuf<uint32_t> s_cert;   // dense_knn: [0] max |x|^2 (float bits), [1] uncertified count, [2..] uncertified queries
    // large-k path (kb2_large_k.cuh): key rows / running best sets, selected candidates, and the finalize's sort buffers
    DevBuf<uint64_t> s_lk_rows, s_lk_cand;
    DevBuf<float> s_lk_key;
    DevBuf<int64_t> s_lk_label, s_lk_label2;
    DevBuf<int32_t> s_lk_slot, s_lk_slot2, s_lk_order, s_lk_off;
    DevBuf<uint32_t> s_lk_okey, s_lk_okey2, s_lk_info;
    DevBuf<uint8_t> s_lk_tmp;

    // device buffers a search writes its [nq][k] result to: the caller's, or s_out_* when the caller's are on the host
    void
    device_out(int64_t nq, int k, int64_t* out_ids, float* out_dist, int64_t*& d_ids, float*& d_dist) {
        d_ids = out_ids;
        d_dist = out_dist;
        if (is_device_ptr(out_ids)) return;
        s_out_ids.ensure((size_t)nq * k);
        s_out_dist.ensure((size_t)nq * k);
        d_ids = s_out_ids.p;
        d_dist = s_out_dist.p;
    }
    // sharded search: one fused all-gather ships every shard's local top-k (s_loc_*), and the merge kernel writes the result
    void
    gather_merge(int64_t nq, int k, int64_t* d_ids, float* d_dist) {
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev_c2, stream));
        comm->all_gather2(s_loc_ids.p, s_g_ids.p, (size_t)nq * k * 8, s_loc_dist.p, s_g_dist.p, (size_t)nq * k * 4, stream);
        launch_merge_topk(metric, shard_world, nq, k, s_g_ids.p, s_g_dist.p, d_ids, d_dist, stream);
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev_c3, stream));
        last.launches += 3;
    }

    // L2-normalised device copy of n rows (COSINE)
    const float*
    normalized(const float* x, int64_t n) {
        if (n <= 0 || !x) return x;
        const float* dx = to_device(x, (size_t)n * dim, s_cos_in);
        s_cos_out.ensure((size_t)n * dim);
        normalize_rows_kernel<<<grid1d(n * 32, 256), 256, 0, stream>>>(dx, n, dim, s_cos_out.p);
        KB2_CUDA_CHECK(cudaGetLastError());
        return s_cos_out.p;
    }

    virtual ~IndexBase() {
        for (cudaEvent_t e : {ev0, ev1, ev2, ev3, ev_in, ev_c0, ev_c1, ev_c2, ev_c3})
            if (e) cudaEventDestroy(e);
        if (own_stream && stream) cudaStreamDestroy(stream);
    }
    // Stream contract: work runs on the handle's stream.  With the library-owned (non-blocking) stream, device buffers
    // handed in by the caller may still be in flight on the caller's side: order our stream after everything already
    // queued on the legacy default stream (which itself waits for all blocking streams, e.g. torch's default stream).
    // Callers that produce inputs on their own NON-blocking stream pass it through kb2_index_set_stream instead.
    void
    wait_caller_work() {
        if (!own_stream || !ev_in) return;
        KB2_CUDA_CHECK(cudaEventRecord(ev_in, cudaStreamLegacy));
        KB2_CUDA_CHECK(cudaStreamWaitEvent(stream, ev_in, 0));
    }
    // a new index: type, metric (COSINE: IP over rows normalised on entry), dim and device, then its stream and events
    void
    init(const std::string& t, int m, int d, int dev) {
        type = t;
        cosine = (m == KB2_METRIC_COSINE);
        metric = cosine ? KB2_METRIC_IP : m;
        dim = d;
        device = dev;
        init_common();
    }
    void
    init_common() {
        KB2_CUDA_CHECK(cudaSetDevice(device));
        KB2_CUDA_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        own_stream = true;
        KB2_CUDA_CHECK(cudaEventCreate(&ev0));
        KB2_CUDA_CHECK(cudaEventCreate(&ev1));
        KB2_CUDA_CHECK(cudaEventCreate(&ev2));
        KB2_CUDA_CHECK(cudaEventCreate(&ev3));
        KB2_CUDA_CHECK(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
        for (cudaEvent_t* e : {&ev_c0, &ev_c1, &ev_c2, &ev_c3}) KB2_CUDA_CHECK(cudaEventCreate(e));
        d_counter.ensure(16);
        h_counter.ensure(128);
    }
    void
    set_stream(cudaStream_t s) {
        if (own_stream && stream) cudaStreamDestroy(stream);
        stream = s;
        own_stream = false;
    }
    void
    use_own_stream() {
        if (own_stream) return;
        KB2_CUDA_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
        own_stream = true;
    }

    // returns a device pointer to `count` floats of `src` (copying H2D on the stream if needed)
    const float*
    to_device(const float* src, size_t count, DevBuf<float>& buf, bool count_io = true) {
        if (is_device_ptr(src)) return src;
        buf.ensure(count);
        KB2_CUDA_CHECK(cudaMemcpyAsync(buf.p, src, count * sizeof(float), cudaMemcpyHostToDevice, stream));
        if (count_io) last.h2d += (int64_t)(count * sizeof(float));
        return buf.p;
    }
    const uint8_t*
    bitset_to_device(const uint8_t* bits, int64_t nbits) {
        if (!bits || nbits <= 0) return nullptr;
        // the kernels index the bitmap by any stored row: a shorter bitmap would be read out of bounds
        KB2_REQUIRE(nbits >= bitset_rows(), KB2_INVALID_ARGS, "bitset has fewer bits than the index has rows");
        if (is_device_ptr(bits)) return bits;
        const size_t nbytes = (size_t)((nbits + 7) / 8);
        s_bitset.ensure(nbytes);
        KB2_CUDA_CHECK(cudaMemcpyAsync(s_bitset.p, bits, nbytes, cudaMemcpyHostToDevice, stream));
        last.h2d += (int64_t)nbytes;
        return s_bitset.p;
    }
    // write [nq*k] results to the caller (device: results were produced in place)
    void
    results_out(int64_t nq, int k, int64_t* out_ids, float* out_dist, const int64_t* d_ids, const float* d_dist) {
        if (d_ids != out_ids) {
            KB2_CUDA_CHECK(cudaMemcpyAsync(out_ids, d_ids, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, stream));
            KB2_CUDA_CHECK(cudaMemcpyAsync(out_dist, d_dist, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, stream));
            last.d2h += nq * k * 12;
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    virtual void train(const float* x, int64_t n) = 0;
    virtual void add(const float* x, int64_t n, const int64_t* ids) = 0;
    virtual void search(const float* q, int64_t nq, int k, const JsonObj& cfg, const uint8_t* bitset, int64_t nbits,
                        int64_t* out_ids, float* out_dist) = 0;
    virtual int64_t count() const = 0;
    // rows a BitsetView must cover (whole index, also on a shard)
    virtual int64_t bitset_rows() const { return shard_world > 1 ? n_global : count(); }
    virtual int64_t size_bytes() const = 0;
    virtual bool is_trained() const = 0;
    virtual bool has_raw() const = 0;
    virtual void get_vectors(const int64_t* ids, int64_t n, float* out) {
        throw Error(KB2_NOT_IMPLEMENTED, "GetVectorByIds not supported by this index");
    }

    // build keys of kb2_index_create
    virtual void configure(const JsonObj&) {}
    // the type's section of the KB2I container (kb2_range.cuh writes the framing around it)
    virtual void save(BlobWriter& w) = 0;
    virtual void load(BlobReader& r) = 0;
    // the faiss fourcc stream (the reference's BinarySet payload): fields beyond the common header
    virtual void to_faiss(FaissIndexData&) { throw Error(KB2_NOT_IMPLEMENTED, "faiss stream: unknown index class"); }
    virtual void from_faiss(const FaissIndexData&) { throw Error(KB2_NOT_IMPLEMENTED, "faiss stream: unsupported index kind"); }
    // the type's fields of GetIndexMeta, appended to the common JSON prefix
    virtual void append_meta(std::string&) const {}
    // operations a type may leave out: refuse() throws the type's status and message where the operation starts
    enum Op { kShard, kHnswImport, kRangeSearch, kEmbList };
    virtual void refuse(Op) const {}
    // RangeSearch (kb2_range.cuh): every hit of the rp.sp.nq queries described by rp (queries, bitset, radius, filter), on
    // the host, its pos the index's row.  A type whose hits carry the rank of their probed list sets nprobe, and
    // max_empty_result_buckets applies.
    virtual std::vector<RangeHit>
    range_hits(const RangeParams&, const JsonObj&, int&) {
        throw Error(KB2_NOT_IMPLEMENTED, "RangeSearch: unknown index class");
    }
    virtual bool takes_emb_list() const { return false; }   // kb2_index_set_emb_list
    // rows reach add() / train() as the caller gave them, also under COSINE (a MUVERA emb-list index encodes raw tokens)
    virtual bool raw_rows_on_entry() const { return false; }
    // emb-lists (kb2_emb_list_index.cuh): the fp32 rows the MaxSim re-rank reads, and each row's position among them (null:
    // row order)
    virtual std::pair<const float*, const int32_t*>
    emb_list_rows() {
        throw Error(KB2_NOT_IMPLEMENTED, "emb-lists are not implemented on " + type);
    }
    // emb-lists: the config of the stage-1 search, which returns vec_topk rows per token for k documents per query list
    virtual void emb_list_base_config(JsonObj&, int k, int vec_topk) const {}
};

// ============================================================================================
// Dense candidate generation shared by FLAT and the IVF coarse quantizer:
//   partial[nq][S][Kout] <- per (query, base-slice) best Ksel approximate keys
// ============================================================================================
struct DensePlan {
    int Ksel = 32;
    int S = 1;        // slot capacity per query
    int used = 0;     // slots filled
    int64_t stride() const { return (int64_t)S * Ksel; }
};

inline DensePlan
dense_candidates(IndexBase& ix, const float* Q, int64_t nq, const float* X, const float* xn, int64_t n, int d,
                 int metric, int k_need, const uint8_t* bitset, int64_t bit_offset) {
    cudaStream_t st = ix.stream;
    DensePlan pl;
    pl.Ksel = next_pow2(std::max(32, k_need));
    KB2_REQUIRE(pl.Ksel <= kMaxK, KB2_INVALID_ARGS, "k too large for the GPU selection kernels (max 1008)");
    pl.S = std::max(2, kMaxSortEntries / pl.Ksel);
    ix.s_partial.ensure((size_t)nq * pl.stride());
    ix.s_qn.ensure(nq);
    if (metric == KB2_METRIC_L2) {
        row_norms_kernel<<<grid1d(nq * 32, 256), 256, 0, st>>>(Q, nq, d, ix.s_qn.p);
        ix.last.launches++;
    }
    const int64_t max_key_elems = 64ll << 20;  // 256 MB of keys
    int64_t chunk = std::min<int64_t>(n, std::max<int64_t>(1024, max_key_elems / std::max<int64_t>(nq, 1)));
    if (chunk < n) chunk = std::max<int64_t>(128, chunk / 128 * 128);
    const int64_t ldk = (chunk + 3) & ~(int64_t)3;   // 16-byte aligned key rows (vector stores in the epilogues)
    ix.s_keys.ensure((size_t)nq * ldk);
    int nsplit = (int)std::min<int64_t>(std::max<int64_t>(1, (2 * num_sms() + nq - 1) / nq),
                                        std::max<int64_t>(1, chunk / 512));
    nsplit = std::min(nsplit, pl.S - 1);
    {
        // empty-entry fill of the slots this call can touch only.  (The whole [nq][S][Ksel] scratch used to be filled: 655 MB
        // per search at C3's coarse stage, where ONE 1 KB slot per query is used -- ~0.1 ms of a 2.4 ms step.)
        const int64_t n_chunks = (n + chunk - 1) / chunk;
        const int64_t slots = std::min<int64_t>(pl.S, n_chunks * nsplit);
        KB2_CUDA_CHECK(cudaMemset2DAsync(ix.s_partial.p, (size_t)pl.stride() * 8, 0xFF, (size_t)slots * pl.Ksel * 8, (size_t)nq, st));
    }
    const size_t sel_smem = (size_t)kScanWarps * 2 * pl.Ksel * 8;
    for (int64_t c0 = 0; c0 < n; c0 += chunk) {
        const int64_t cols = std::min(chunk, n - c0);
        if (pl.used + nsplit > pl.S) {
            const int n_in = pl.used * pl.Ksel;
            const int n_sort = next_pow2(n_in);
            launch<reduce_partials_kernel>((unsigned)nq, 256, (size_t)n_sort * 8, st, ix.s_partial.p, (int)pl.stride(), n_in,
                                           n_sort, pl.Ksel);
            ix.last.launches++;
            pl.used = 1;
        }
        launch_gemm_keys(st, 1, metric, Q, X + c0 * d, ix.s_qn.p, xn + c0, (int)nq, (int)cols, d, ix.s_keys.p, ldk,
                         bitset, nullptr, c0 + bit_offset);
        const int per_slice = (int)(((cols + nsplit - 1) / nsplit + 31) / 32 * 32);
        const size_t hist_smem = (size_t)per_slice * 4 + 4160;
        if (pl.Ksel >= 64 && hist_smem <= (size_t)kMaxDynSmem) {
            launch<select_keys_hist_kernel>(dim3((unsigned)nq, nsplit), 256, hist_smem, st,
                ix.s_keys.p, ldk, (int)cols, std::min(k_need, pl.Ksel), pl.Ksel, ix.s_partial.p, pl.S, pl.used, (uint32_t)c0);
        } else {
            launch<select_keys_kernel>(dim3((unsigned)nq, nsplit), kScanThreads, sel_smem, st,
                ix.s_keys.p, ldk, (int)cols, pl.Ksel, pl.Ksel, ix.s_partial.p, pl.S, pl.used, (uint32_t)c0);
        }
        ix.last.launches += 2;
        pl.used += nsplit;
    }
    KB2_CUDA_CHECK(cudaGetLastError());
    return pl;
}

inline void
launch_finalize(IndexBase& ix, FinalizeParams fp, int64_t nq) {
    fp.n_sort = next_pow2(std::max(fp.n_partial, 2));
    KB2_REQUIRE(fp.n_sort <= kMaxSortEntries, KB2_INTERNAL_ERROR, "finalize: too many partial candidates");
    KB2_REQUIRE(fp.k_sel <= kMaxK && fp.k_out <= fp.k_sel, KB2_INVALID_ARGS, "k too large");
    if (fp.k_sel <= 128 && fp.d <= 1024 && (fp.n_partial <= 256 || fp.counts)) {
        // one warp per query (see finalize_warp_kernel); variable-length rows longer than 256 entries fall through to the
        // CTA kernel below, which then skips the short ones (measured at C3: a 512-entry register sort for the tail costs
        // more than that second launch)
        const size_t smem_w = (size_t)kFinWarps * ((size_t)((fp.d + 3) & ~3) * 4 + 128 * 24);
        const unsigned g = (unsigned)((nq + kFinWarps - 1) / kFinWarps);
        if (fp.n_partial <= 128)
            launch<finalize_warp_kernel<4>>(g, kFinWarps * 32, smem_w, ix.stream, fp, nq);
        else
            launch<finalize_warp_kernel<8>>(g, kFinWarps * 32, smem_w, ix.stream, fp, nq);
        ix.last.launches++;
        KB2_CUDA_CHECK(cudaGetLastError());
        if (fp.n_partial <= 256) return;
        fp.split_small = 256;
    }
    const size_t smem = (size_t)fp.n_sort * 8 + (size_t)fp.k_sel * 16 + (size_t)fp.d * 4 + 16;
    KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_INVALID_ARGS, "dimension too large for the exact re-rank");
    unsigned grid = (unsigned)nq;
    if (fp.split_small > 0 && nq > 8 * num_sms()) {   // tail pass: a few CTAs per SM walk the rows, most of which they skip
        grid = 8u * num_sms();
        fp.row_loop_nq = nq;
    }
    launch<finalize_kernel>(grid, 256, smem, ix.stream, fp);
    ix.last.launches++;
    KB2_CUDA_CHECK(cudaGetLastError());
}

// ============================================================================================
// Large-k path (DESIGN §4.9): windows of K > kMaxK candidates per query.  Key rows -> select_rows_kernel -> large finalize.
// ============================================================================================
// large-k scratch per launch row besides the rows its keys come from: K candidates and the finalize's sort buffers
inline int64_t
large_k_row_bytes(int K) {
    return (int64_t)K * 48 + 16;
}
// launch rows per group so that `per_row` bytes each stay within kLargeKScratch
inline int64_t
large_k_group(int64_t nrows, int64_t per_row) {
    return std::max<int64_t>(1, std::min<int64_t>(nrows, kLargeKScratch / std::max<int64_t>(per_row, 1)));
}

// out row b <- the min(K, valid) best entries of input row b (b < rows), unsorted, kEmpty padded
template <typename T>
inline void
large_k_select(IndexBase& ix, const T* in, int64_t ld, int64_t len, uint32_t pos_base, int K, uint64_t* out, int64_t out_ld,
               int64_t rows) {
    launch<select_rows_kernel<T>>((unsigned)rows, kSelThreads, 0, ix.stream, in, ld, len, pos_base, K, out, out_ld);
    ix.last.launches++;
    KB2_CUDA_CHECK(cudaGetLastError());
}

// Finalize of `rows` launch rows of K selected candidates each (row b: query fp.qlist[b], or q0 + b): keys (exact from
// fp.raw / fp.raw16 when fp.rerank), labels, (key, label) order by two stable segmented radix sorts (label, then key),
// the fp.k_out best written to fp.out_*, and with fp.cert the certification finalize_row applies.
inline void
large_k_finalize(IndexBase& ix, const FinalizeParams& fp, const uint64_t* cand, int64_t cand_ld, int K, int64_t rows, int64_t q0) {
    cudaStream_t st = ix.stream;
    const int64_t n = rows * K;
    KB2_REQUIRE(n < (1ll << 31), KB2_INTERNAL_ERROR, "large-k finalize: group too large");
    ix.s_lk_key.ensure(n);
    ix.s_lk_label.ensure(n);
    ix.s_lk_label2.ensure(n);
    ix.s_lk_slot.ensure(n);
    ix.s_lk_slot2.ensure(n);
    ix.s_lk_order.ensure(n);
    ix.s_lk_okey.ensure(n);
    ix.s_lk_okey2.ensure(n);
    ix.s_lk_info.ensure((size_t)rows * 4);
    ix.s_lk_off.ensure((size_t)rows + 1);
    LargeFin lf{cand, cand_ld, K, q0, ix.s_lk_key.p, ix.s_lk_label.p, ix.s_lk_slot.p, ix.s_lk_okey.p, ix.s_lk_order.p,
                ix.s_lk_info.p};
    KB2_CUDA_CHECK(cudaMemsetAsync(ix.s_lk_info.p, 0, (size_t)rows * 16, st));
    launch<large_rerank_kernel>(dim3((unsigned)rows, (unsigned)((K + 255) / 256)), 256, (size_t)fp.d * 4 + 16, st, fp, lf);
    segment_offsets_kernel<<<grid1d(rows + 1, 256), 256, 0, st>>>(ix.s_lk_off.p, rows, K);
    const int32_t* off = ix.s_lk_off.p;
    size_t b1 = 0, b2 = 0;
    cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b1, ix.s_lk_label.p, ix.s_lk_label2.p, ix.s_lk_slot.p, ix.s_lk_slot2.p,
                                             (int)n, (int)rows, off, off + 1, 0, 64, st);
    cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b2, ix.s_lk_okey.p, ix.s_lk_okey2.p, ix.s_lk_slot2.p, ix.s_lk_order.p,
                                             (int)n, (int)rows, off, off + 1, 0, 32, st);
    ix.s_lk_tmp.ensure(std::max(b1, b2));
    // stable radix sorts: by label, then by key => (key, label) order, equal pairs in slot order
    cub::DeviceSegmentedRadixSort::SortPairs(ix.s_lk_tmp.p, b1, ix.s_lk_label.p, ix.s_lk_label2.p, ix.s_lk_slot.p,
                                             ix.s_lk_slot2.p, (int)n, (int)rows, off, off + 1, 0, 64, st);
    large_gather_keys_kernel<<<grid1d(n, 256), 256, 0, st>>>(lf, ix.s_lk_slot2.p, n);
    cub::DeviceSegmentedRadixSort::SortPairs(ix.s_lk_tmp.p, b2, ix.s_lk_okey.p, ix.s_lk_okey2.p, ix.s_lk_slot2.p,
                                             ix.s_lk_order.p, (int)n, (int)rows, off, off + 1, 0, 32, st);
    large_emit_kernel<<<grid1d(rows * fp.k_out, 256), 256, 0, st>>>(fp, lf, rows);
    ix.last.launches += 7;
    KB2_CUDA_CHECK(cudaGetLastError());
}

// dense_knn for windows k_out + 16 > kMaxK.  The key chunks of the contraction are those of dense_candidates; each query
// keeps its K = k_out + 16 best in a running set (best of the first chunk, then best of set + next chunk), which the large
// finalize re-ranks exactly and certifies.  Uncertified queries are redone from directly accumulated distances: the dense
// mode of range_scan_kernel writes each one's full key row, and the same selection and finalize run on it.
inline int64_t
dense_knn_large(IndexBase& ix, const float* Q, int64_t nq, const float* X, const float* xn, int64_t n, int d, int metric,
                int k_out, const uint8_t* bitset, int64_t bit_base, const int64_t* labels, int64_t* out_ids, float* out_dist,
                bool certify, cudaEvent_t ev_cand) {
    cudaStream_t st = ix.stream;
    const int K = k_out + 16;
    FinalizeParams fp{};
    fp.k_sel = K;
    fp.k_out = k_out;
    fp.labels = labels;
    fp.rerank = 1;
    fp.raw = X;
    fp.raw_by_pos = 1;
    fp.queries = Q;
    fp.d = d;
    fp.metric = metric;
    fp.out_ids = out_ids;
    fp.out_dist = out_dist;
    if (certify) {
        ix.s_cert.ensure((size_t)nq + 2);
        KB2_CUDA_CHECK(cudaMemsetAsync(ix.s_cert.p, 0, 8, st));
        pqtc::max_abs_kernel<<<2 * num_sms(), 256, 0, st>>>(xn, n, ix.s_cert.p);
        fp.cert = ix.s_cert.p;
    }
    ix.s_qn.ensure(nq);
    if (metric == KB2_METRIC_L2) {
        row_norms_kernel<<<grid1d(nq * 32, 256), 256, 0, st>>>(Q, nq, d, ix.s_qn.p);
        ix.last.launches++;
    }
    // per query: two running sets of 2K entries, then the finalize's scratch
    const int64_t g = large_k_group(nq, (int64_t)K * 32 + large_k_row_bytes(K));
    const int64_t max_key_elems = 64ll << 20;  // 256 MB of keys, as in dense_candidates
    int64_t chunk = std::min<int64_t>(n, std::max<int64_t>(1024, max_key_elems / g));
    if (chunk < n) chunk = std::max<int64_t>(128, chunk / 128 * 128);
    const int64_t ldk = (chunk + 3) & ~(int64_t)3;
    ix.s_keys.ensure((size_t)g * ldk);
    ix.s_lk_rows.ensure((size_t)g * 4 * K);
    for (int64_t q0 = 0; q0 < nq; q0 += g) {
        const int64_t rows = std::min(g, nq - q0);
        uint64_t* A = ix.s_lk_rows.p;
        uint64_t* B = A + (size_t)g * 2 * K;
        for (int64_t c0 = 0; c0 < n; c0 += chunk) {
            const int64_t cols = std::min(chunk, n - c0);
            launch_gemm_keys(st, 1, metric, Q + q0 * d, X + c0 * d, ix.s_qn.p + q0, xn + c0, (int)rows, (int)cols, d, ix.s_keys.p,
                             ldk, bitset, nullptr, c0 + bit_base);
            ix.last.launches++;
            if (c0 == 0) {
                large_k_select<float>(ix, ix.s_keys.p, ldk, cols, 0u, K, A, 2 * K, rows);
            } else {
                large_k_select<float>(ix, ix.s_keys.p, ldk, cols, (uint32_t)c0, K, A + K, 2 * K, rows);
                large_k_select<uint64_t>(ix, A, 2 * K, 2 * K, 0u, K, B, 2 * K, rows);
                std::swap(A, B);
            }
        }
        if (ev_cand && q0 + rows == nq) KB2_CUDA_CHECK(cudaEventRecord(ev_cand, st));
        large_k_finalize(ix, fp, A, 2 * K, K, rows, q0);
    }
    if (!certify) return 0;
    uint32_t* hc = (uint32_t*)ix.h_counter.p;
    KB2_CUDA_CHECK(cudaMemcpyAsync(hc, ix.s_cert.p + 1, 4, cudaMemcpyDeviceToHost, st));
    KB2_CUDA_CHECK(cudaStreamSynchronize(st));
    const int64_t nredo = hc[0];
    if (nredo == 0) return 0;
    const int64_t ldr = round_up(n, 32);
    const int64_t g2 = large_k_group(nredo, ldr * 8 + large_k_row_bytes(K));
    ix.s_lk_rows.ensure((size_t)g2 * ldr);
    ix.s_lk_cand.ensure((size_t)g2 * K);
    RangeParams rp{};
    rp.sp.queries = Q;
    rp.sp.nq = (int)nq;
    rp.sp.d = d;
    rp.sp.metric = metric;
    rp.sp.bitset = bitset;
    rp.sp.vecs = X;
    rp.kind = 0;
    rp.single_len = n;
    rp.bit_base = bit_base;
    rp.dense = ix.s_lk_rows.p;
    rp.dense_ld = ldr;
    const size_t smem = (size_t)d * 4 + 128;
    KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_INVALID_ARGS, "dimension too large for the exact redo scan");
    const uint32_t* qlist = ix.s_cert.p + 2;
    fp.cert = nullptr;
    for (int64_t r0 = 0; r0 < nredo; r0 += g2) {
        const int64_t rows = std::min(g2, nredo - r0);
        rp.sp.nsplit = (int)std::min<int64_t>(std::max<int64_t>(1, (2 * num_sms() + rows - 1) / rows), std::max<int64_t>(1, n / 1024));
        rp.qlist = qlist + r0;
        KB2_CUDA_CHECK(cudaMemsetAsync(ix.s_lk_rows.p, 0xFF, (size_t)rows * ldr * 8, st));
        launch<range_scan_kernel>((unsigned)(rows * rp.sp.nsplit), kScanThreads, smem, st, rp);
        ix.last.launches++;
        KB2_CUDA_CHECK(cudaGetLastError());
        large_k_select<uint64_t>(ix, ix.s_lk_rows.p, ldr, n, 0u, K, ix.s_lk_cand.p, K, rows);
        fp.qlist = (const int32_t*)(qlist + r0);
        large_k_finalize(ix, fp, ix.s_lk_cand.p, K, K, rows, 0);
    }
    return nredo;
}

// Exact dense k-NN of the nq queries Q against the n rows X with norms xn (FLAT, BruteForce, HNSW's exact fallback, the IVF
// coarse quantizer): candidates from the norm-expanded keys, then finalize re-ranks the k_sel best of each query exactly
// and writes the k_out best.  `bit_base` is the bitset position of row 0; `labels` (or nullptr: the row) is the reported id.
// With `certify`, queries whose re-ranked window finalize could not certify (data whose norms are large against the
// distances: the norm-expanded keys cancel) are searched again with directly accumulated distances, and their rows of the
// result are finalized again from those candidates.  On ordinary data there are none and this costs one 4-byte copy.
// `ev_cand`, if given, is recorded once the candidates are queued.  Returns the number of queries redone.  Windows
// k_out + 16 above kMaxK take the large-k path (dense_knn_large); k_sel is then k_out + 16.
inline int64_t
dense_knn(IndexBase& ix, const float* Q, int64_t nq, const float* X, const float* xn, int64_t n, int d, int metric, int k_out,
          int k_sel, const uint8_t* bitset, int64_t bit_base, const int64_t* labels, int64_t* out_ids, float* out_dist,
          bool certify, cudaEvent_t ev_cand = nullptr) {
    if (k_out + 16 > kMaxK)
        return dense_knn_large(ix, Q, nq, X, xn, n, d, metric, k_out, bitset, bit_base, labels, out_ids, out_dist, certify, ev_cand);
    cudaStream_t st = ix.stream;
    const DensePlan pl = dense_candidates(ix, Q, nq, X, xn, n, d, metric, k_out + 16, bitset, bit_base);
    if (ev_cand) KB2_CUDA_CHECK(cudaEventRecord(ev_cand, st));
    FinalizeParams fp{};
    fp.partial = ix.s_partial.p;
    fp.partial_stride = pl.stride();
    fp.n_partial = pl.used * pl.Ksel;
    fp.k_sel = std::min(pl.Ksel, k_sel);
    fp.k_out = k_out;
    fp.labels = labels;
    fp.rerank = 1;
    fp.raw = X;
    fp.raw_by_pos = 1;
    fp.queries = Q;
    fp.d = d;
    fp.metric = metric;
    fp.out_ids = out_ids;
    fp.out_dist = out_dist;
    if (certify) {
        // certification of the re-ranked window (fin_certify) needs max |x|^2 over the rows
        ix.s_cert.ensure((size_t)nq + 2);
        KB2_CUDA_CHECK(cudaMemsetAsync(ix.s_cert.p, 0, 8, st));
        pqtc::max_abs_kernel<<<2 * num_sms(), 256, 0, st>>>(xn, n, ix.s_cert.p);
        fp.cert = ix.s_cert.p;
    }
    launch_finalize(ix, fp, nq);
    if (!certify) return 0;
    uint32_t* hc = (uint32_t*)ix.h_counter.p;
    KB2_CUDA_CHECK(cudaMemcpyAsync(hc, ix.s_cert.p + 1, 4, cudaMemcpyDeviceToHost, st));
    KB2_CUDA_CHECK(cudaStreamSynchronize(st));
    const int64_t nredo = hc[0];
    if (nredo == 0) return 0;
    const int K = pl.Ksel;
    int nsplit = (int)std::min<int64_t>(std::max<int64_t>(1, (2 * num_sms() + nredo - 1) / nredo), std::max<int64_t>(1, n / 1024));
    nsplit = std::min(nsplit, kMaxSortEntries / K);
    ix.s_partial2.ensure((size_t)nq * nsplit * K);
    const size_t smem = (size_t)kScanWarps * 2 * K * 8 + (size_t)d * 4;
    KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_INVALID_ARGS, "dimension too large for the exact redo scan");
    const dim3 g((unsigned)nredo, (unsigned)nsplit);
    const uint32_t* qlist = ix.s_cert.p + 2;
    with_metric(metric, [&](auto m) {
        launch<flat_exact_scan_kernel<decltype(m)::value>>(g, kScanThreads, smem, st, Q, X, n, d, bitset, bit_base, qlist, K,
                                                           ix.s_partial2.p);
    });
    ix.last.launches++;
    KB2_CUDA_CHECK(cudaGetLastError());
    fp.partial = ix.s_partial2.p;
    fp.partial_stride = (int64_t)nsplit * K;
    fp.n_partial = nsplit * K;
    fp.cert = nullptr;
    fp.qlist = (const int32_t*)qlist;
    launch_finalize(ix, fp, nredo);
    return nredo;
}

// ============================================================================================
// RangeSearch scans (range_scan_kernel); kb2_range.cuh orders the hits and builds lims
// ============================================================================================
inline std::vector<RangeHit>
hits_to_host(IndexBase& ix, const RangeHit* hits, size_t n) {
    std::vector<RangeHit> h(n);
    if (n) KB2_CUDA_CHECK(cudaMemcpy(h.data(), hits, n * sizeof(RangeHit), cudaMemcpyDeviceToHost));
    ix.last.d2h += (int64_t)(n * sizeof(RangeHit));
    return h;
}

// the hits of range_scan_kernel over rp (rp.sp.nq x rp.sp.nsplit CTAs of smem bytes), row positions as the scan emits them.
// A scan whose hits overflow the buffer runs once more into a buffer of the count it reported.
inline std::vector<RangeHit>
range_scan(IndexBase& ix, RangeParams rp, size_t smem) {
    cudaStream_t st = ix.stream;
    DevBuf<RangeHit> hits;
    DevBuf<unsigned long long> cnt;
    cnt.ensure(1);
    unsigned long long cap = (unsigned long long)std::max<int64_t>(1 << 20, (int64_t)rp.sp.nq * 256), found = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
        hits.ensure(cap);
        KB2_CUDA_CHECK(cudaMemsetAsync(cnt.p, 0, 8, st));
        rp.hits = hits.p;
        rp.count = cnt.p;
        rp.cap = cap;
        launch<range_scan_kernel>((unsigned)((int64_t)rp.sp.nq * rp.sp.nsplit), kScanThreads, smem, st, rp);
        ix.last.launches++;
        KB2_CUDA_CHECK(cudaGetLastError());
        KB2_CUDA_CHECK(cudaMemcpyAsync(&found, cnt.p, 8, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        if (found <= cap) break;
        cap = found;
    }
    return hits_to_host(ix, hits.p, found);
}

// range_scan of the n rows X, stored in row order (FLAT, HNSW's brute-force case).  A shard's local row r is bitset
// position shard_lo + r.
inline std::vector<RangeHit>
range_scan_rows(IndexBase& ix, RangeParams rp, const float* X, int64_t n) {
    const int64_t nq = rp.sp.nq;
    const size_t smem = (size_t)ix.dim * 4 + 128;
    KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_NOT_IMPLEMENTED, "range search: dimension too large for the exact scan");
    rp.kind = 0;
    rp.sp.vecs = X;
    rp.sp.rows = nullptr;
    rp.single_len = n;
    rp.bit_base = ix.shard_world > 1 ? ix.shard_lo : 0;
    rp.sp.nsplit = (int)std::min<int64_t>(std::max<int64_t>(1, (2 * num_sms() + nq - 1) / nq), std::max<int64_t>(1, n / 1024));
    return range_scan(ix, rp, smem);
}

// max_empty_result_buckets (ivf_config.h:51-58): an IVF range search stops after this many consecutive probes that add
// no hit inside the radius; 0 or less scans every probe
inline int
range_max_empty(const JsonObj& cfg) {
    return (int)cfg.get_int("max_empty_result_buckets", 2);
}

// ============================================================================================
// FLAT
// ============================================================================================
struct FlatIndex : IndexBase {
    DevBuf<float> base, norms;
    size_t n_used = 0, norms_used = 0;
    int n_add_calls = 0;

    void train(const float*, int64_t) override {}
    bool is_trained() const override { return true; }
    bool has_raw() const override { return true; }
    int64_t count() const override { return (int64_t)(n_used / std::max(dim, 1)); }
    int64_t size_bytes() const override { return (int64_t)(n_used * 4 + norms_used * 4 + labels.used * 8); }

    void
    add(const float* x, int64_t n, const int64_t* ids) override {
        if (n <= 0) return;
        const auto [lo, hi] = shard_slice(n);
        const int64_t m = hi - lo;
        if (n_add_calls++ == 0) shard_lo = lo;
        if (m > 0) {
            dev_append(base, n_used, x + lo * dim, (size_t)m * dim, stream);
            DevBuf<float> tmp;
            tmp.ensure(m);
            row_norms_kernel<<<grid1d(m * 32, 256), 256, 0, stream>>>(base.p + n_used - (size_t)m * dim, m, dim, tmp.p);
            dev_append(norms, norms_used, tmp.p, (size_t)m, stream);
            KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        }
        // a shard's ids are global rows: an id array from its first add() on
        labels.append(count() - m, ids ? ids + lo : nullptr, m, n_global + lo, shard_world > 1, stream);
        n_global += n;
    }

    void
    search(const float* q, int64_t nq, int k, const JsonObj&, const uint8_t* bitset, int64_t nbits, int64_t* out_ids,
           float* out_dist) override {
        const int64_t n = count();
        KB2_REQUIRE(n > 0, KB2_EMPTY_INDEX, "index is empty");
        KB2_REQUIRE(k > 0 && k <= kMaxLargeK, KB2_INVALID_ARGS, "k out of range (1..16384)");
        const float* dq = to_device(q, (size_t)nq * dim, s_q);
        const uint8_t* dbits = bitset_to_device(bitset, nbits);
        int64_t* d_ids;
        float* d_dist;
        device_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev0, stream));
        // bitset indexes internal rows == labels when labels are the identity (like BitsetView over segment offsets);
        // a shard holds the contiguous slice [shard_lo, shard_lo + n) of ONE add() call, so bit = shard_lo + local row
        KB2_REQUIRE(!(dbits && shard_world > 1 && n_add_calls > 1), KB2_NOT_IMPLEMENTED,
                    "FLAT shard: bitset after several add() calls");
        last.flagged = dense_knn(*this, dq, nq, base.p, norms.p, n, dim, metric, k, k + 16, dbits, shard_world > 1 ? shard_lo : 0,
                                 labels.device(), d_ids, d_dist, true, timing ? ev1 : nullptr);
        last.codes = nq * n;
        last.code_bytes = n * (int64_t)dim * 4;  // list-major contraction reads the base once per batch
        last.pairs = nq;
        results_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        last_engine = (k + 16 > kMaxK) ? 2 : 0;
        if (timing) {
            KB2_CUDA_CHECK(cudaEventElapsedTime(&last_stage_ms, ev0, ev1));
            last_kernel_ms = last_stage_ms;
        }
    }

    void
    get_vectors(const int64_t* ids, int64_t n, float* out) override {
        KB2_REQUIRE(!labels.custom, KB2_NOT_IMPLEMENTED, "GetVectorByIds with custom ids");
        std::vector<int64_t> h(n);
        if (is_device_ptr(ids)) {
            KB2_CUDA_CHECK(cudaMemcpy(h.data(), ids, n * 8, cudaMemcpyDeviceToHost));
        } else {
            memcpy(h.data(), ids, n * 8);
        }
        for (int64_t i = 0; i < n; i++) {
            KB2_REQUIRE(h[i] >= 0 && h[i] < count(), KB2_INVALID_ARGS, "id out of range");
            KB2_CUDA_CHECK(cudaMemcpyAsync(out + i * dim, base.p + h[i] * dim, (size_t)dim * 4, cudaMemcpyDefault, stream));
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    void
    save(BlobWriter& w) override {
        const int64_t n = count();
        w.put<int64_t>(n);
        w.put<int32_t>(labels.custom ? 1 : 0);
        std::vector<float> h((size_t)n * dim);
        if (n) KB2_CUDA_CHECK(cudaMemcpy(h.data(), base.p, h.size() * 4, cudaMemcpyDeviceToHost));
        w.put_bytes(h.data(), h.size() * 4);
        const std::vector<int64_t> l = labels.host(n);
        w.put_bytes(l.data(), l.size() * 8);
    }
    void
    load(BlobReader& r) override {
        const int64_t n = r.get<int64_t>();
        KB2_REQUIRE(n >= 0 && (uint64_t)n <= r.n / ((size_t)dim * 4), KB2_INVALID_BINARY_SET, "bad row count in blob");
        const int custom = r.get<int32_t>();
        const float* data = (const float*)r.get_bytes((size_t)n * dim * 4);
        const int64_t* l = custom ? (const int64_t*)r.get_bytes((size_t)n * 8) : nullptr;
        // blob memory may be unaligned: stage through vectors
        std::vector<float> hd((size_t)n * dim);
        memcpy(hd.data(), data, hd.size() * 4);
        std::vector<int64_t> hl;
        if (custom) { hl.resize(n); memcpy(hl.data(), l, n * 8); }
        add(hd.data(), n, custom ? hl.data() : nullptr);
    }
    void
    to_faiss(FaissIndexData& o) override {
        KB2_REQUIRE(!labels.custom, KB2_NOT_IMPLEMENTED, "faiss stream: FLAT with custom ids");
        o.xb.resize((size_t)o.ntotal * o.d);
        if (o.ntotal) KB2_CUDA_CHECK(cudaMemcpy(o.xb.data(), base.p, o.xb.size() * 4, cudaMemcpyDeviceToHost));
    }
    void
    from_faiss(const FaissIndexData& o) override {
        if (o.ntotal) add(o.cosine ? normalized(o.xb.data(), o.ntotal) : o.xb.data(), o.ntotal, nullptr);
    }
    std::vector<RangeHit>
    range_hits(const RangeParams& rp, const JsonObj&, int&) override {
        KB2_REQUIRE(!(rp.sp.bitset && shard_world > 1 && n_add_calls > 1), KB2_NOT_IMPLEMENTED,
                    "FLAT shard: bitset after several add() calls");
        return range_scan_rows(*this, rp, base.p, count());
    }
};

// ============================================================================================
// IVF_FLAT / IVF_PQ
// ============================================================================================
struct IvfIndex : IndexBase {
    bool is_pq = false;
    int64_t nlist = 128;
    int M = 0, nbits = 8, dsub = 0;
    bool refine = false;
    int refine_kind = 0;       // refine store element type: 0 fp32 ("flat"), 1 fp16, 2 bf16 (ivf_config.h:97-128)
    bool trained = false;
    // trained state
    DevBuf<float> centroids, cnorms, pqc;
    // flat (insertion-order) staging, valid while !sealed
    DevBuf<int32_t> f_assign;
    DevBuf<uint8_t> f_codes;
    DevBuf<float> f_vecs;
    size_t f_assign_used = 0, f_codes_used = 0, f_vecs_used = 0;
    int64_t n_total = 0;
    // sealed (list-order) layout
    bool sealed = false;
    int64_t npad = 0;
    int G = 0;                 // 16-sub-quantizer groups when the skewed kernel applies, else 0
    std::vector<int64_t> h_list_off;
    std::vector<int32_t> h_list_len, h_list_cnt_all, h_list_owner;
    DevBuf<int32_t> list_owner;   // [nlist] rank that holds each list (size-balanced packing, identical on every rank)
    DevBuf<int64_t> list_off;
    DevBuf<int32_t> list_len, rows, pos_of_row;
    DevBuf<uint8_t> codes;     // [G][npad][16] or [npad][M]
    DevBuf<uint16_t> vecs16;          // refine store when refine_kind != 0 (vecs is released after seal)
    DevBuf<float> t1, vecs, vnorm2;   // vnorm2[pos] = |x|^2 (IVF_FLAT: row term of the list-major tensor-core engine)
    DevBuf<int32_t> s_qkey, s_qkey2, s_qidx, s_qperm;
    DevBuf<uint8_t> s_sort_tmp;

    bool keeps_vecs() const { return !is_pq || refine; }
    bool is_trained() const override { return trained; }
    bool has_raw() const override { return keeps_vecs() && refine_kind == 0; }
    // fp32 view of the list-order vector store (decoded into tmp when it is kept in 16 bits)
    const float*
    vecs_f32(DevBuf<float>& tmp) {
        if (!refine_kind || !is_pq) return vecs.p;
        tmp.ensure((size_t)npad * dim);
        widen16_kernel<<<grid1d(npad * dim, 256), 256, 0, stream>>>(vecs16.p, npad * dim, refine_kind, tmp.p);
        return tmp.p;
    }
    int64_t count() const override { return n_total; }
    int64_t bitset_rows() const override { return n_total; }   // a shard holds every row (it owns whole lists)
    int64_t
    size_bytes() const override {
        return (int64_t)(centroids.bytes() + pqc.bytes() + codes.bytes() + t1.bytes() + vecs.bytes() + vecs16.bytes() + rows.bytes() +
                         pos_of_row.bytes() + f_codes.bytes() + f_vecs.bytes() + f_assign.bytes());
    }

    void
    set_centroids_common() {
        cnorms.ensure(nlist);
        row_norms_kernel<<<grid1d(nlist * 32, 256), 256, 0, stream>>>(centroids.p, nlist, dim, cnorms.p);
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    // ---------------------------------------------------------------- Train (ivf.cc:545-807)
    void
    train(const float* x, int64_t n) override {
        KB2_REQUIRE(!trained, KB2_INDEX_ALREADY_TRAINED, "index already trained");
        KB2_REQUIRE(n > 0, KB2_INVALID_ARGS, "empty training set");
        // refused before anything changes, so that a refused train() leaves the configured nlist for the next one
        if (is_pq) {
            KB2_REQUIRE(nbits == 8, KB2_NOT_IMPLEMENTED, "IVF_PQ: only nbits=8 is implemented on the GPU path");
            KB2_REQUIRE(M > 0 && dim % M == 0, KB2_INVALID_ARGS, "IVF_PQ: dim must be a multiple of m");
            KB2_REQUIRE(n >= 256, KB2_INVALID_ARGS, "IVF_PQ: need at least 256 training rows for nbits=8");
        }
        // MatchNlist (ivf.cc:479-489)
        if (nlist * 39 > n) nlist = std::max<int64_t>(1, n / 39);
        DevBuf<float> xbuf;
        const float* dx = to_device(x, (size_t)n * dim, xbuf, false);
        centroids.alloc_exact((size_t)nlist * dim);
        kmeans_train(dx, n, dim, (int)nlist, metric, 25, 1234, centroids.p, stream);
        set_centroids_common();
        if (is_pq) {
            dsub = dim / M;
            // residuals of (a subsample of) the training set: F/IndexIVF.cpp:1307-1329, IndexIVFPQ.cpp:76-95
            const int64_t nt = std::min<int64_t>(n, 256 * 256);
            DevBuf<float> sample;
            const float* xt = dx;
            if (nt < n) {
                std::mt19937_64 rng(1234 + 7);
                std::vector<int32_t> perm(n);
                for (int64_t i = 0; i < n; i++) perm[i] = (int32_t)i;
                for (int64_t i = 0; i < nt; i++) std::swap(perm[i], perm[i + (int64_t)(rng() % (uint64_t)(n - i))]);
                DevBuf<int32_t> didx;
                didx.ensure(nt);
                KB2_CUDA_CHECK(cudaMemcpyAsync(didx.p, perm.data(), nt * 4, cudaMemcpyHostToDevice, stream));
                sample.ensure((size_t)nt * dim);
                gather_rows_kernel<<<grid1d(nt * 32, 256), 256, 0, stream>>>(dx, didx.p, nt, dim, dim, sample.p);
                KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
                xt = sample.p;
            }
            DevBuf<int32_t> asg;
            asg.ensure(nt);
            AssignScratch sc;
            assign_nearest(xt, nt, dim, centroids.p, (int)nlist, metric, asg.p, nullptr, sc, stream);
            pqc.alloc_exact((size_t)M * 256 * dsub);
            tc_ready = false;
            DevBuf<float> sub;
            sub.ensure((size_t)nt * dsub);
            for (int m = 0; m < M; m++) {
                slice_residual_kernel<<<grid1d(nt * dsub, 256), 256, 0, stream>>>(xt, centroids.p, asg.p, nt, dim, m, dsub,
                                                                                sub.p);
                // every sub-quantizer is seeded identically, like the reference (one ClusteringParameters, seed 1234, for all
                // M Clustering objects: F/impl/ProductQuantizer.cpp:130-180) => the M codebooks start from the same 256 rows
                kmeans_train(sub.p, nt, dsub, 256, KB2_METRIC_L2, 25, 1234, pqc.p + (size_t)m * 256 * dsub, stream);
            }
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        trained = true;
    }

    // ---------------------------------------------------------------- Add (ivf.cc:809-844; F/IndexIVF.cpp:212-287)
    void
    add(const float* x, int64_t n, const int64_t* ids) override {
        KB2_REQUIRE(trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        if (n <= 0) return;
        if (sealed) unseal();
        DevBuf<float> xbuf;
        const float* dx = to_device(x, (size_t)n * dim, xbuf, false);
        DevBuf<int32_t> asg;
        asg.ensure(n);
        AssignScratch sc;
        assign_nearest(dx, n, dim, centroids.p, (int)nlist, metric, asg.p, nullptr, sc, stream);
        dev_append(f_assign, f_assign_used, asg.p, (size_t)n, stream);
        if (is_pq) {
            DevBuf<uint8_t> cb;
            cb.ensure((size_t)n * M);
            pq_encode_kernel<<<grid1d(n * 32, 256), 256, 0, stream>>>(dx, centroids.p, asg.p, pqc.p, n, dim, M, dsub, cb.p);
            dev_append(f_codes, f_codes_used, cb.p, (size_t)n * M, stream);
        }
        if (keeps_vecs()) dev_append(f_vecs, f_vecs_used, dx, (size_t)n * dim, stream);
        labels.append(n_total, ids, n, n_total, false, stream);
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        KB2_CUDA_CHECK(cudaGetLastError());
        n_total += n;
    }

    // ---------------------------------------------------------------- list-order layout
    void
    seal() {
        if (sealed) return;
        const int64_t n = n_total;
        cudaStream_t st = stream;
        // list sizes
        DevBuf<int32_t> dcnt;
        dcnt.ensure(nlist);
        KB2_CUDA_CHECK(cudaMemsetAsync(dcnt.p, 0, nlist * 4, st));
        if (n) histogram_kernel<<<grid1d(n, 256), 256, 0, st>>>(f_assign.p, n, dcnt.p);
        h_list_cnt_all.assign(nlist, 0);
        KB2_CUDA_CHECK(cudaMemcpyAsync(h_list_cnt_all.data(), dcnt.p, nlist * 4, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        h_list_off.assign(nlist, 0);
        h_list_len.assign(nlist, 0);
        std::vector<int64_t> first_rank(nlist, 0);
        int64_t cur = 0, rank = 0;
        // list -> shard: greedy size-balanced packing (longest list first onto the lightest shard; SURVEY 8e), computed from
        // the global list sizes, which every rank holds, so all ranks derive the same table.
        h_list_owner.assign(nlist, 0);
        if (shard_world > 1) {
            std::vector<int64_t> order(nlist), load(shard_world, 0);
            for (int64_t l = 0; l < nlist; l++) order[l] = l;
            std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return h_list_cnt_all[a] > h_list_cnt_all[b]; });
            for (int64_t l : order) {
                int best = 0;
                for (int r = 1; r < shard_world; r++)
                    if (load[r] < load[best]) best = r;
                h_list_owner[l] = best;
                load[best] += h_list_cnt_all[l];
            }
        }
        list_owner.alloc_exact(nlist);
        KB2_CUDA_CHECK(cudaMemcpyAsync(list_owner.p, h_list_owner.data(), nlist * 4, cudaMemcpyHostToDevice, st));
        for (int64_t l = 0; l < nlist; l++) {
            first_rank[l] = rank;
            rank += h_list_cnt_all[l];
            const bool owned = h_list_owner[l] == shard_rank;
            h_list_len[l] = owned ? h_list_cnt_all[l] : 0;
            h_list_off[l] = cur;
            cur += round_up(h_list_len[l], 32);
        }
        npad = cur + 32;
        KB2_REQUIRE(npad < (int64_t)0xfffffff0ll, KB2_INVALID_ARGS, "index too large for 32-bit positions");
        list_off.alloc_exact(nlist);
        list_len.alloc_exact(nlist);
        DevBuf<int64_t> d_first;
        d_first.ensure(nlist);
        KB2_CUDA_CHECK(cudaMemcpyAsync(list_off.p, h_list_off.data(), nlist * 8, cudaMemcpyHostToDevice, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(list_len.p, h_list_len.data(), nlist * 4, cudaMemcpyHostToDevice, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_first.p, first_rank.data(), nlist * 8, cudaMemcpyHostToDevice, st));
        // stable sort rows by list id
        rows.alloc_exact(npad);
        pos_of_row.alloc_exact(std::max<int64_t>(n, 1));
        fill_i32_kernel<<<grid1d(npad, 256), 256, 0, st>>>(rows.p, npad, -1);
        if (n) {
            DevBuf<int32_t> idx_in, idx_out, key_out;
            idx_in.ensure(n);
            idx_out.ensure(n);
            key_out.ensure(n);
            iota_kernel<<<grid1d(n, 256), 256, 0, st>>>(idx_in.p, n);
            size_t tmp_bytes = 0;
            int end_bit = 1;
            while ((1ll << end_bit) < nlist) end_bit++;
            cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, f_assign.p, key_out.p, idx_in.p, idx_out.p, (int)n, 0,
                                            end_bit, st);
            DevBuf<uint8_t> tmp;
            tmp.ensure(tmp_bytes);
            cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, f_assign.p, key_out.p, idx_in.p, idx_out.p, (int)n, 0,
                                            end_bit, st);
            place_rows_kernel<<<grid1d(n, 256), 256, 0, st>>>(key_out.p, idx_out.p, n, d_first.p, list_off.p, list_len.p,
                                                            rows.p, pos_of_row.p);
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        }
        // payload in list order
        if (is_pq) {
            G = (M % 16 == 0 && M / 16 <= 3) ? M / 16 : 0;
            DevBuf<float> t1_flat;
            if (metric == KB2_METRIC_L2) {
                t1_flat.ensure(std::max<int64_t>(n, 1));
                if (n) pq_t1_kernel<<<grid1d(n * 32, 256), 256, 0, st>>>(f_codes.p, centroids.p, f_assign.p, pqc.p, n, dim, M,
                                                                         dsub, t1_flat.p);
                t1.alloc_exact(npad);
                gather_f32_kernel<<<grid1d(npad, 256), 256, 0, st>>>(t1_flat.p, rows.p, npad, t1.p, 0.f);
            }
            if (G > 0) {
                codes.alloc_exact((size_t)G * npad * 16);
                layout_codes_kernel<<<grid1d((int64_t)G * npad * 16, 256), 256, 0, st>>>(f_codes.p, rows.p, npad, M, G, codes.p);
            } else {
                codes.alloc_exact((size_t)npad * M);
                layout_codes_plain_kernel<<<grid1d(npad * M, 256), 256, 0, st>>>(f_codes.p, rows.p, npad, M, codes.p);
            }
        }
        if (keeps_vecs()) {
            vecs.alloc_exact((size_t)npad * dim);
            gather_rows_kernel<<<grid1d(npad * 32, 256), 256, 0, st>>>(f_vecs.p, rows.p, npad, dim, dim, vecs.p);
            if (!is_pq) {
                vnorm2.alloc_exact(npad);
                row_norms_kernel<<<grid1d(npad * 32, 256), 256, 0, st>>>(vecs.p, npad, dim, vnorm2.p);
            } else if (refine_kind) {
                vecs16.alloc_exact((size_t)npad * dim);
                narrow_kernel<<<grid1d(npad * dim, 256), 256, 0, st>>>(vecs.p, npad * dim, refine_kind, vecs16.p);
                KB2_CUDA_CHECK(cudaStreamSynchronize(st));
                vecs.release();
            }
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        KB2_CUDA_CHECK(cudaGetLastError());
        // the insertion-order payload is no longer needed (assign stays: small)
        f_codes.release();
        f_vecs.release();
        sealed = true;
    }

    // rebuild the insertion-order payload from the list-order one so that add() can append
    void
    unseal() {
        KB2_REQUIRE(shard_world == 1, KB2_NOT_IMPLEMENTED, "add() after search on a sharded index");
        const int64_t n = n_total;
        cudaStream_t st = stream;
        if (is_pq) {
            // gather the codes back into insertion order: one thread per (row, m)
            f_codes.alloc_exact((size_t)std::max<int64_t>(n, 1) * M);
            if (n) unlayout_codes_kernel<<<grid1d(n * M, 256), 256, 0, st>>>(codes.p, pos_of_row.p, n, npad, M, G, f_codes.p);
            f_codes_used = (size_t)n * M;
        }
        if (keeps_vecs()) {
            DevBuf<float> dec;
            const float* v32 = vecs_f32(dec);
            f_vecs.alloc_exact((size_t)std::max<int64_t>(n, 1) * dim);
            gather_rows_kernel<<<grid1d(n * 32, 256), 256, 0, st>>>(v32, pos_of_row.p, n, dim, dim, f_vecs.p);
            f_vecs_used = (size_t)n * dim;
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        sealed = false;
    }

    // the scan parameters every IVF scan starts from: the queries, the bitset, the probes in s_probe_* and the list store.
    // rp.sp for the query-major scan kernels, rp whole for range_scan_kernel (RangeSearch, the large-k path).
    RangeParams
    list_params(const float* dq, int64_t nq, int nprobe, const uint8_t* dbits) const {
        RangeParams rp{};
        IvfScanParams& sp = rp.sp;
        sp.queries = dq;
        sp.nq = (int)nq;
        sp.d = dim;
        sp.metric = metric;
        sp.bitset = dbits;
        sp.probe_ids = s_probe_ids.p;
        sp.probe_dis = s_probe_dis.p;
        sp.nprobe = nprobe;
        sp.list_off = list_off.p;
        sp.list_len = list_len.p;
        sp.rows = rows.p;
        sp.vecs = vecs.p;
        sp.pq_centroids = pqc.p;
        sp.M = M;
        sp.dsub = dsub;
        sp.codes = (const uint4*)codes.p;
        sp.npad = npad;
        sp.t1 = t1.p;
        rp.kind = is_pq ? (G > 0 ? 1 : 2) : 0;
        rp.G = G;
        rp.codes_b = codes.p;
        rp.single_len = -1;
        return rp;
    }

    // ---------------------------------------------------------------- query-major scan launch (all IVF kinds)
    void
    launch_scan(IvfScanParams sp, unsigned grid, int Ksel, int np_max, bool has_bits) {
        cudaStream_t st = stream;
        const uint8_t* dbits = has_bits ? sp.bitset : nullptr;
        const size_t common_smem = (size_t)kScanWarps * 2 * Ksel * 8 + (size_t)(np_max + 1) * 4 + (size_t)np_max * 12 +
                                   (size_t)dim * 4 + 64 + 8 * (2 * kScanWarps + 4) + (size_t)4 * Ksel * 8;   // + CTA bound block + merge buffer
        if (is_pq) {
            const size_t smem_skewed = (size_t)G * 65536 + common_smem;
            if (G > 0 && smem_skewed <= (size_t)kMaxDynSmem) {
                const size_t smem = smem_skewed;
                with_metric(metric, [&](auto m) {
                    constexpr int MM = decltype(m)::value;
                    if (G == 1) {
                        if (dbits) launch<ivfpq_scan_kernel<1, MM, true>>(grid, kScanThreads, smem, st, sp);
                        else launch<ivfpq_scan_kernel<1, MM, false>>(grid, kScanThreads, smem, st, sp);
                    } else if (G == 2) {
                        if (dbits) launch<ivfpq_scan_kernel<2, MM, true>>(grid, kScanThreads, smem, st, sp);
                        else launch<ivfpq_scan_kernel<2, MM, false>>(grid, kScanThreads, smem, st, sp);
                    } else {
                        if (dbits) launch<ivfpq_scan_kernel<3, MM, true>>(grid, kScanThreads, smem, st, sp);
                        else launch<ivfpq_scan_kernel<3, MM, false>>(grid, kScanThreads, smem, st, sp);
                    }
                });
            } else {
                // one M KB table instead of 64 KB per 16 sub-quantizers: any m, and the skewed kernel's fallback at large k
                // (its 2K-entry candidate buffers) or many probes per CTA, where the replicated tables do not fit beside them
                const size_t smem = (size_t)M * 1024 + (size_t)kScanWarps * 2 * Ksel * 8 + (size_t)(np_max + 1) * 4 +
                                    (size_t)np_max * 12 + (size_t)dim * 4;
                KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_NOT_IMPLEMENTED, "IVF_PQ: m too large for the generic kernel");
                with_metric(metric, [&](auto m) {
                    launch<ivfpq_scan_generic_kernel<decltype(m)::value>>(grid, kScanThreads, smem, st, sp, codes.p, G);
                });
            }
        } else {
            KB2_REQUIRE(dim % 4 == 0, KB2_NOT_IMPLEMENTED, "IVF_FLAT: dim must be a multiple of 4 on the GPU path");
            with_metric(metric, [&](auto m) {
                launch<ivfflat_scan_kernel<decltype(m)::value>>(grid, kScanThreads, common_smem, st, sp);
            });
        }
        last.launches++;
        KB2_CUDA_CHECK(cudaGetLastError());
    }

    // ---------------------------------------------------------------- list-major tensor-core engine (kb2_ivfpq_tc.cuh)
    static constexpr int kTcCandCap = 2048;     // survivor slots per query (overflow -> LUT kernel redoes the query)
    static constexpr double kTcMinQpl = 8.0;    // queries per list from which the list-major engine is taken (use_tc_engine)
    static constexpr int kTcACodes = 3000;      // phase A: codes per query its bound is taken from
    DevBuf<uint16_t> tc_pqc16, s_qb16;
    DevBuf<float> tc_pqc_t;   // codebook transposed for the in-kernel tables of bound_kernel<..., 3, 2>
    DevBuf<float> tc_maxn2, s_qnorm, s_pair_base, s_lut, s_bound;
    DevBuf<int32_t> s_lcount, s_lstart, s_items, s_pair_q, s_plan_out, s_flaglist, s_resp;
    DevBuf<uint64_t> s_cand;
    DevBuf<uint32_t> s_cand_cnt, s_logcnt;
    DevBuf<uint4> s_log;
    float tc_rmax = 0.f, tc_rowmax = 0.f;
    bool tc_ready = false;

    DevBuf<uint8_t> tc_codes_plain;   // un-rotated code bytes for the geometries whose decode assembles 16-byte chunks from several sub-quantizers
    // engine instances: <G=1, dsub=8> (m16 d128: C3) and <G=3, dsub=2> (m48 d96: C5)
    bool tc_geom_18() const { return G == 1 && M == 16 && dsub == 8; }
    bool tc_geom_32() const { return G == 3 && M == 48 && dsub == 2; }
    DevBuf<int32_t> s_items2, s_bal_idx, s_bal_idx2;
    DevBuf<uint32_t> s_bal_key, s_bal_key2;
    // Side stream of the list-major engine: the plan (pairs grouped by list, item table, cost sort: seven small, latency-bound
    // launches that depend on the coarse result only) runs beside phase A (which fills the SMs with 3 x 128 threads each) and
    // joins before the filter kernel.  With KB2_TC_VERBOSE set everything stays on the handle's stream, so that the stage
    // timings do not overlap.
    cudaStream_t side_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    bool side_pending = false;   // forked, not yet joined (only ever observed true after an exception)
    bool
    plan_overlap() {
        if (getenv("KB2_TC_VERBOSE")) return false;
        if (!side_stream) {
            KB2_CUDA_CHECK(cudaStreamCreateWithFlags(&side_stream, cudaStreamNonBlocking));
            KB2_CUDA_CHECK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
            KB2_CUDA_CHECK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
        }
        return true;
    }
    ~IvfIndex() override {
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_join) cudaEventDestroy(ev_join);
        if (side_stream) cudaStreamDestroy(side_stream);
    }
    // ---- the list-major pipeline (kb2_listmajor.cuh) of both tensor-core engines
    struct ItemTable {
        const int32_t *list, *q0, *nq;   // [*n_items] in descending estimated cost
        const int32_t* n_items;
        int32_t* ticket;                 // zeroed: the persistent kernel draws the items through it
    };
    // Plan on stream ps: the (query, probe) pairs grouped by list (-> s_pair_q, s_pair_base), cut into items of <= item_cap
    // queries (a multiple of 16) and sorted by the estimated cost tiles x (tile_cost + col_cost x columns).
    ItemTable
    plan_items(const int64_t* probe_ids, const float* probe_dis, int64_t nq, int nprobe, int item_cap, int tile_cost, int col_cost,
               cudaStream_t ps) {
        const int64_t npairs = nq * nprobe;
        const int64_t max_items = nlist + npairs / item_cap + 2;
        s_lcount.ensure((size_t)2 * nlist);
        s_lstart.ensure((size_t)nlist);
        s_items.ensure((size_t)3 * max_items);
        s_items2.ensure((size_t)3 * max_items);
        s_bal_key.ensure((size_t)max_items); s_bal_key2.ensure((size_t)max_items);
        s_bal_idx.ensure((size_t)max_items); s_bal_idx2.ensure((size_t)max_items);
        s_plan_out.ensure(8);
        s_pair_q.ensure((size_t)npairs);
        s_pair_base.ensure((size_t)npairs);
        KB2_CUDA_CHECK(cudaMemsetAsync(s_lcount.p, 0, (size_t)2 * nlist * 4, ps));
        KB2_CUDA_CHECK(cudaMemsetAsync(s_plan_out.p + 4, 0, 4, ps));
        // pairs on empty lists (or on other shards' lists) get no slot, so the tail of the pair array stays unwritten: mark it
        // as no query (-1) for gather_split_queries_kernel, which reads every entry below npairs
        KB2_CUDA_CHECK(cudaMemsetAsync(s_pair_q.p, 0xFF, (size_t)npairs * 4, ps));
        lm::count_pairs_kernel<<<grid1d(npairs, 256), 256, 0, ps>>>(probe_ids, npairs, list_len.p, s_lcount.p);
        int32_t* items = s_items.p;   // list | q0 | nq
        lm::plan_kernel<<<1, 1024, 0, ps>>>(s_lcount.p, (int)nlist, item_cap, s_lstart.p, items, items + max_items,
                                            items + 2 * max_items, s_plan_out.p);
        lm::item_cost_kernel<<<grid1d(max_items, 256), 256, 0, ps>>>(s_plan_out.p, items, items + 2 * max_items, list_len.p, max_items,
                                                                     tile_cost, col_cost, s_bal_key.p, s_bal_idx.p);
        size_t tmp_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, s_bal_key.p, s_bal_key2.p, s_bal_idx.p, s_bal_idx2.p, (int)max_items, 0, 16, ps);
        s_sort_tmp.ensure(tmp_bytes);
        cub::DeviceRadixSort::SortPairs(s_sort_tmp.p, tmp_bytes, s_bal_key.p, s_bal_key2.p, s_bal_idx.p, s_bal_idx2.p, (int)max_items, 0, 16, ps);
        lm::deal_items_kernel<<<grid1d(max_items, 256), 256, 0, ps>>>(s_plan_out.p, s_bal_idx2.p, items, items + max_items,
                                                                      items + 2 * max_items, s_items2.p, s_items2.p + max_items,
                                                                      s_items2.p + 2 * max_items);
        lm::fill_pairs_kernel<<<grid1d(npairs, 256), 256, 0, ps>>>(probe_ids, probe_dis, npairs, nprobe, metric, list_len.p, s_lstart.p,
                                                                   s_lcount.p + nlist, s_pair_q.p, s_pair_base.p);
        last.launches += 7;
        return {s_items2.p, s_items2.p + max_items, s_items2.p + 2 * max_items, s_plan_out.p, s_plan_out.p + 4};
    }
    // n_logs survivor logs of cap entries each; the counts and the overflow word cnt[n_logs] are zeroed on the handle's stream
    struct SurvivorLogs {
        uint4* log;
        uint32_t* cnt;
        uint32_t cap;
    };
    SurvivorLogs
    alloc_logs(int n_logs, uint32_t cap) {
        s_log.ensure((size_t)n_logs * cap);
        s_logcnt.ensure((size_t)n_logs + 1);
        KB2_CUDA_CHECK(cudaMemsetAsync(s_logcnt.p, 0, ((size_t)n_logs + 1) * 4, stream));
        return {s_log.p, s_logcnt.p, cap};
    }

    // probe slices of the redo of a flagged query: their Ksel-entry outputs fill its kTcCandCap-entry candidate row
    static int
    tc_redo_split(int nprobe, int Ksel) {
        return std::max(1, std::min(kTcCandCap / Ksel, nprobe));
    }

    bool
    use_tc_engine(int64_t nq, int nprobe, int Ksel) const {
        if (!is_pq || !(tc_geom_18() || tc_geom_32())) return false;
        const char* e = getenv("KB2_PQ_ENGINE");
        if (e && !strcmp(e, "lut")) return false;
        if (nprobe < 8 || Ksel > kTcCandCap / 2) return false;
        // the redo of a flagged query splits its probes over the kTcCandCap / Ksel slices of its candidate row: above
        // kScanSliceProbes per slice the scan kernels' probe arrays would not fit, so those searches stay query-major
        if ((nprobe + tc_redo_split(nprobe, Ksel) - 1) / tc_redo_split(nprobe, Ksel) > kScanSliceProbes) return false;
        if (e && !strcmp(e, "tc")) return true;
        // the decode of a list is amortised over the queries that probe it.  Measured at C5 (100M x 96, nlist 65536, 19.5
        // queries per list on average): the query-major LUT engine needs 34.5 ms per 10000-query batch on two GPUs, so the
        // list-major engine is taken from kTcMinQpl queries per list on
        return (double)nq * nprobe >= kTcMinQpl * (double)nlist;
    }

    void
    search_tc(IvfScanParams sp, int64_t nq, int nprobe, int Ksel, int k_base, bool has_bits) {
        cudaStream_t st = stream;
        const bool dist = distributed();
        if (!tc_ready) {
            tc_pqc16.alloc_exact((size_t)M * 256 * dsub);
            tc_maxn2.alloc_exact(M + 4);
            KB2_CUDA_CHECK(cudaMemsetAsync(tc_maxn2.p + M, 0, 16, st));
            pqtc::prepare_tables_kernel<<<M, 256, 0, st>>>(pqc.p, dsub, (__nv_bfloat16*)tc_pqc16.p, tc_maxn2.p);
            if (tc_geom_32()) {
                tc_pqc_t.alloc_exact((size_t)M * 256 * dsub);
                pqtc::transpose_codebook_kernel<<<grid1d((int64_t)M * 256 * dsub, 256), 256, 0, st>>>(pqc.p, M, dsub, tc_pqc_t.p);
            }
            if (metric == KB2_METRIC_L2 && npad > 0)
                pqtc::max_abs_kernel<<<num_sms() * 2, 256, 0, st>>>(t1.p, npad, (uint32_t*)(tc_maxn2.p + M));
            if (dsub < 8) {
                tc_codes_plain.alloc_exact((size_t)G * npad * 16);
                pqtc::unrotate_codes_kernel<<<grid1d((int64_t)G * npad * 16, 256), 256, 0, st>>>(codes.p, (int64_t)G * npad, npad,
                                                                                            tc_codes_plain.p);
            }
            std::vector<float> h(M + 4);
            KB2_CUDA_CHECK(cudaMemcpyAsync(h.data(), tc_maxn2.p, (M + 4) * 4, cudaMemcpyDeviceToHost, st));
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
            double acc = 0;
            for (int i = 0; i < M; i++) acc += h[i];
            tc_rmax = (float)std::sqrt(acc) * 1.0001f;
            tc_rowmax = 0.5f * h[M] * 1.0001f;   // max |t1| / 2: the largest row term of the admission test
            tc_ready = true;
        }
        // development aid: KB2_TC_VERBOSE=1 prints the device time of every stage of this engine
        const bool verbose = getenv("KB2_TC_VERBOSE") != nullptr;
        std::vector<std::pair<const char*, cudaEvent_t>> marks;
        auto mark = [&](const char* name) {
            if (!verbose) return;
            cudaEvent_t e;
            cudaEventCreate(&e);
            cudaEventRecord(e, st);
            marks.emplace_back(name, e);
        };
        mark("start");
        // the plan below depends on the coarse result only: with the side stream it runs beside phase A
        const bool ov = plan_overlap();
        cudaStream_t ps = ov ? side_stream : st;
        if (ov) {
            if (side_pending) {
                // a previous call left between fork and join (an error was thrown): drain its side-stream work before the
                // scratch buffers are reused
                KB2_CUDA_CHECK(cudaStreamSynchronize(side_stream));
                side_pending = false;
            }
            KB2_CUDA_CHECK(cudaEventRecord(ev_fork, st));
            KB2_CUDA_CHECK(cudaStreamWaitEvent(side_stream, ev_fork, 0));
            side_pending = true;
        }
        // ---- phase A: exact scan of each query's nearest lists -> upper bound of its k_base-th best key.  A bound taken from ANY
        //      subset of the codes is valid on every rank, so with a communicator the query is handled by the rank that owns
        //      its nearest list (1/world of the batch each; tables only for those) and the bounds are min-reduced.
        const char* e_p0 = getenv("KB2_TC_P0");
        const int p0 = std::max(1, std::min((e_p0 ? atoi(e_p0) : 8) * std::max(1, shard_world), nprobe));   // at most this many lists
        s_bound.ensure((size_t)nq);
        if (tc_geom_18()) s_lut.ensure((size_t)nq * 4096);
        const int32_t* qlist = nullptr;
        const uint32_t* qcount = nullptr;
        unsigned bound_grid = (unsigned)nq;
        if (dist) {
            s_resp.ensure((size_t)nq + 1);
            pqtc::compact_resp_kernel<<<1, 1024, 0, st>>>(sp.probe_ids, nprobe, nq, list_owner.p, shard_rank, s_resp.p + 1,
                                                          (uint32_t*)s_resp.p);
            pqtc::fill_f32_kernel<<<grid1d(nq, 256), 256, 0, st>>>(s_bound.p, nq, INFINITY);
            qlist = s_resp.p + 1;
            qcount = (const uint32_t*)s_resp.p;
            bound_grid = (unsigned)std::min<int64_t>(nq, std::max<int64_t>(4 * num_sms(), 2 * nq / shard_world));
            last.launches += 2;
        }
        {
            const size_t smem = pqtc::bound_smem(pqtc::bound_kmax(kTcACodes, k_base));
            with_metric(metric, [&](auto m) {
                constexpr int MM = decltype(m)::value;
                if (tc_geom_32()) {
                    // m48 x dsub2: three groups through one in-kernel table each (no [nq][m][256] table in global memory)
                    launch<pqtc::bound_kernel<MM, 3, 2, 128>>(bound_grid, 128, smem, st, nullptr, qlist, qcount, nq, sp.probe_ids,
                                                              sp.probe_dis, nprobe, p0, kTcACodes, k_base, list_off.p, list_len.p,
                                                              (const uint4*)codes.p, t1.p, sp.bitset, rows.p, s_bound.p,
                                                              d_counter.p + 4, npad, sp.queries, tc_pqc_t.p);
                } else {
                    // m16 x dsub8: the batch's tables from lut_build_kernel, 8 warps per CTA over them
                    pqtc::lut_build_kernel<MM><<<num_sms(), 256, 0, st>>>(sp.queries, nq, qlist, qcount, pqc.p, s_lut.p);
                    mark("lut");
                    launch<pqtc::bound_kernel<MM, 1, 8, 256>>(bound_grid, 256, smem, st, s_lut.p, qlist, qcount, nq, sp.probe_ids,
                                                              sp.probe_dis, nprobe, p0, kTcACodes, k_base, list_off.p, list_len.p,
                                                              (const uint4*)codes.p, t1.p, sp.bitset, rows.p, s_bound.p,
                                                              d_counter.p + 4, 0, nullptr, nullptr);
                }
            });
            KB2_CUDA_CHECK(cudaGetLastError());
            last.launches += 2;
        }
        if (dist) comm->all_reduce_min_f32(s_bound.p, s_bound.p, (size_t)nq, st);
        mark("phaseA");
        // ---- plan: pairs grouped by list, work items of <= 256 queries.  Per tile: decode ~ constant, contraction ~ columns
        //      (+ the test K-step)
        const ItemTable items = plan_items(sp.probe_ids, sp.probe_dis, nq, nprobe, pqtc::NQT, 600, 5, ps);
        s_qb16.ensure((size_t)nq * dim);
        s_qnorm.ensure((size_t)nq);
        s_cand.ensure((size_t)nq * kTcCandCap);
        s_cand_cnt.ensure((size_t)2 * nq);
        KB2_CUDA_CHECK(cudaMemsetAsync(s_cand_cnt.p, 0, (size_t)2 * nq * 4, ps));
        pqtc::prepare_queries_kernel<<<grid1d(nq * 32, 256), 256, 0, ps>>>(sp.queries, nq, dim, (__nv_bfloat16*)s_qb16.p, s_qnorm.p);
        if (ov) {
            KB2_CUDA_CHECK(cudaGetLastError());
            KB2_CUDA_CHECK(cudaEventRecord(ev_join, side_stream));
            KB2_CUDA_CHECK(cudaStreamWaitEvent(st, ev_join, 0));
            side_pending = false;
        }
        mark("plan");
        // ---- tensor-core filter + exact re-evaluation of the survivors
        pqtc::Params tp{};
        tp.metric = metric;
        tp.nq = (int)nq;
        tp.nprobe = nprobe;
        tp.queries = sp.queries;
        tp.qb16 = (const __nv_bfloat16*)s_qb16.p;
        tp.qnorm = s_qnorm.p;
        tp.n_items = items.n_items;
        tp.ticket = items.ticket;
        tp.item_list = items.list;
        tp.item_q0 = items.q0;
        tp.item_nq = items.nq;
        tp.pair_q = s_pair_q.p;
        tp.pair_base = s_pair_base.p;
        tp.bound = s_bound.p;
        tp.k_need = k_base;
        tp.margin_coef = (metric == KB2_METRIC_L2 ? 2.f : 1.f) * pqtc::kErrCoef * tc_rmax;
        tp.rmax = (metric == KB2_METRIC_L2) ? tc_rowmax : 0.f;
        tp.list_off = list_off.p;
        tp.list_len = list_len.p;
        tp.codes = (const uint4*)codes.p;
        tp.codes_plain = (const uint4*)tc_codes_plain.p;
        tp.npad = npad;
        tp.t1 = t1.p;
        tp.pqc = pqc.p;
        tp.pqc16 = (const uint4*)tc_pqc16.p;
        tp.bitset = sp.bitset;
        tp.rows = rows.p;
        const int n_logs = 2 * num_sms();   // one per epilogue group
        const SurvivorLogs logs = alloc_logs(n_logs, (uint32_t)std::clamp<int64_t>(nq * 1024 / n_logs, 16384, 1 << 19));
        tp.log = logs.log;
        tp.log_cnt = logs.cnt;
        tp.log_cap = logs.cap;
        tp.qflag = s_cand_cnt.p + nq;
        tp.counters = d_counter.p;
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev2, st));
        with_metric(metric, [&](auto m) {
            constexpr int MM = decltype(m)::value;
            if (tc_geom_18())
                launch<pqtc::ivfpq_tc_filter_kernel<MM, 1, 8>>(num_sms(), pqtc::THREADS, pqtc::TcCfg<1, 8>::SMEM_BYTES, st, tp);
            else
                launch<pqtc::ivfpq_tc_filter_kernel<MM, 3, 2>>(num_sms(), pqtc::THREADS, pqtc::TcCfg<3, 2>::SMEM_BYTES, st, tp);
        });
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev3, st));
        KB2_CUDA_CHECK(cudaGetLastError());
#ifdef KB2_FILTER_STALLS
        pqtc::filter_stalls_print_kernel<<<1, 1, 0, st>>>(num_sms());
#endif
        mark("tc_filter");
        // ---- survivors: group by query, exact fp32 keys (bit-identical to the LUT engine's)
        lm::scatter_survivors_kernel<<<dim3(16, n_logs), 256, 0, st>>>(logs.log, logs.cnt, logs.cap, s_cand.p, s_cand_cnt.p, kTcCandCap,
                                                                       tp.qflag, d_counter.p);
        // exact_eval trims every survivor row to its k_base best.  Measured at C3: step 1.977 -> 1.957 ms
        const float* eval_lut = (tc_geom_18() && !dist) ? s_lut.p : nullptr;   // tables of the whole batch exist only without a communicator
        with_metric(metric, [&](auto m) {
            constexpr int MM = decltype(m)::value;
            if (tc_geom_18())
                pqtc::exact_eval_kernel<MM, 1, 8><<<(unsigned)nq, 128, 0, st>>>(sp.queries, pqc.p, eval_lut, s_bound.p, (const uint4*)codes.p,
                                                                               npad, t1.p, sp.bitset, rows.p, s_cand.p, s_cand_cnt.p,
                                                                               kTcCandCap, tp.qflag, logs.cnt + n_logs, k_base);
            else
                pqtc::exact_eval_kernel<MM, 3, 2><<<(unsigned)nq, 128, 0, st>>>(sp.queries, pqc.p, eval_lut, s_bound.p, (const uint4*)codes.p,
                                                                               npad, t1.p, sp.bitset, rows.p, s_cand.p, s_cand_cnt.p,
                                                                               kTcCandCap, tp.qflag, logs.cnt + n_logs, k_base);
        });
        KB2_CUDA_CHECK(cudaGetLastError());
        last.launches += 4;
        mark("scatter+eval");
        // ---- flagged queries (no bound / buffer overflow): complete LUT scan into their candidate rows
        {
            IvfScanParams f = sp;
            f.nsplit = tc_redo_split(nprobe, Ksel);   // probe slices per flagged query: their lists fill the row
            f.partial = s_cand.p;
            f.partial_stride = kTcCandCap;
            f.clear_to = kTcCandCap - (f.nsplit - 1) * Ksel;   // == Ksel (nothing to clear) when the slices fill the row
            s_flaglist.ensure((size_t)nq + 1);
            pqtc::compact_flags_kernel<<<1, 1024, 0, st>>>(tp.qflag, nq, s_flaglist.p + 1, (uint32_t*)s_flaglist.p);
            last.launches++;
            f.only_flagged = tp.qflag;
            f.flag_list = s_flaglist.p + 1;
            f.flag_count = (const uint32_t*)s_flaglist.p;
            f.qperm = nullptr;
            f.lut_global = nullptr;   // the redo pass builds its own tables (a handful of queries)
            f.counters = d_counter.p + 4;
            launch_scan(f, (unsigned)std::min<int64_t>(nq * f.nsplit, 3 * num_sms()), Ksel, (nprobe + f.nsplit - 1) / f.nsplit, has_bits);
        }
        mark("fallback");
        if (verbose) {
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
            fprintf(stderr, "[kb2 tc]");
            for (size_t i = 1; i < marks.size(); i++) {
                float ms = 0.f;
                cudaEventElapsedTime(&ms, marks[i - 1].second, marks[i].second);
                fprintf(stderr, " %s %.3f ms |", marks[i].first, ms);
            }
            uint32_t hn = 0;
            cudaMemcpy(&hn, s_plan_out.p, 4, cudaMemcpyDeviceToHost);
            unsigned long long hc2[8];
            cudaMemcpy(hc2, d_counter.p, 64, cudaMemcpyDeviceToHost);
            fprintf(stderr, " items %u survivors %llu flagged %llu (row overflows %llu, no bound %llu)\n", hn, hc2[2], hc2[7],
                    hc2[6] & 0xffffffffull, hc2[6] >> 32);
            for (auto& m : marks) cudaEventDestroy(m.second);
        }
    }

    // ---------------------------------------------------------------- IVF_FLAT list-major tensor-core engine (kb2_ivfflat_tc.cuh)
    DevBuf<float> s_qhi, s_qlo;
    bool
    use_flat_tc_engine(int64_t nq, int nprobe, int k) const {
        if (is_pq || dim % fltc::BK != 0 || dim < fltc::BK || npad >= (1ll << 31)) return false;
        const char* e = getenv("KB2_FLAT_ENGINE");
        if (e && !strcmp(e, "scan")) return false;
        if (k + 16 > kTcCandCap / 2) return false;
        // every (query, probe) pair gets its own split copy of the query (8 bytes per dimension): above kMaxWindowProbes
        // probes the engine is taken only where those copies fit the group's scratch
        if (nprobe > kMaxWindowProbes && ((double)nq * nprobe + fltc::NQ_ITEM) * dim * 8 > (double)kProbeScratch) return false;
        if (e && !strcmp(e, "tc")) return true;
        // a list tile is amortised over the queries probing it
        return (double)nq * nprobe >= 8.0 * (double)nlist && nq >= 64;
    }

    // returns false when some query overflowed its candidate row (caller falls back to the query-major scan)
    bool
    search_flat_tc(IvfScanParams sp, int64_t nq, int nprobe, int Ksel, int k, bool has_bits) {
        cudaStream_t st = stream;
        const int64_t npairs = nq * nprobe;
        const int64_t npairs_pad = npairs + fltc::NQ_ITEM;
        // items of <= 32 queries (small B tiles, 5 stages in flight) while a list is probed by few queries, else <= 128
        const int item_cap = ((double)npairs / (double)std::max<int64_t>(1, nlist) <= 40.0) ? 32 : 128;
        // ---- phase A: exact k-th best key over the query's nearest probed lists (query-major kernel) = admission bound
        const int pA = std::min(nprobe, std::max(1, 2 * shard_world));
        s_bound.ensure((size_t)nq);
        {
            IvfScanParams a = sp;
            a.nprobe = pA;
            a.probe_stride = nprobe;
            a.nsplit = 1;
            a.partial = s_partial2.p;
            a.partial_stride = 0;
            a.counters = nullptr;
            a.qperm = nullptr;
            launch_scan(a, (unsigned)nq, Ksel, pA, has_bits);
            fltc::extract_bound_kernel<<<grid1d(nq, 256), 256, 0, st>>>(s_partial2.p, Ksel, k, nq, s_bound.p);
            if (distributed()) comm->all_reduce_min_f32(s_bound.p, s_bound.p, (size_t)nq, st);
            last.launches += 1;
        }
        // ---- plan: pairs grouped by list, items of <= item_cap queries (a tile is bound by its HBM stream)
        const ItemTable items = plan_items(sp.probe_ids, sp.probe_dis, nq, nprobe, item_cap, 1000, 2, st);
        s_qnorm.ensure((size_t)nq);
        s_cand.ensure((size_t)nq * kTcCandCap);
        s_cand_cnt.ensure((size_t)2 * nq + 4);
        s_qhi.ensure((size_t)npairs_pad * dim);
        s_qlo.ensure((size_t)npairs_pad * dim);
        KB2_CUDA_CHECK(cudaMemsetAsync(s_cand_cnt.p, 0, ((size_t)2 * nq + 4) * 4, st));
        // pairs of lists owned by other shards leave holes at the end of the pair array: point them at no query
        fltc::gather_split_queries_kernel<<<grid1d(npairs_pad * 32, 256), 256, 0, st>>>(sp.queries, s_pair_q.p, npairs, npairs_pad, dim,
                                                                                     s_qhi.p, s_qlo.p);
        row_norms_kernel<<<grid1d(nq * 32, 256), 256, 0, st>>>(sp.queries, nq, dim, s_qnorm.p);
        CUtensorMap tx, thi, tlo;
        KB2_REQUIRE(tc::make_tmap(&tx, vecs.p, npad, dim) && tc::make_tmap(&thi, s_qhi.p, npairs_pad, dim, item_cap) &&
                        tc::make_tmap(&tlo, s_qlo.p, npairs_pad, dim, item_cap),
                    KB2_INTERNAL_ERROR, "IVF_FLAT tensor-core engine: tensor map encoding failed");
        fltc::Params fpar{};
        fpar.metric = metric;
        fpar.d = dim;
        fpar.n_items = items.n_items;
        fpar.ticket = items.ticket;
        fpar.item_list = items.list;
        fpar.item_q0 = items.q0;
        fpar.item_nq = items.nq;
        fpar.pair_q = s_pair_q.p;
        fpar.qnorm2 = s_qnorm.p;
        fpar.bound = s_bound.p;
        fpar.list_off = list_off.p;
        fpar.list_len = list_len.p;
        fpar.xnorm2 = vnorm2.p;
        fpar.bitset = sp.bitset;
        fpar.rows = rows.p;
        const int n_logs = num_sms();   // one per CTA
        const SurvivorLogs logs = alloc_logs(n_logs, (uint32_t)std::clamp<int64_t>(nq * 1024 / n_logs, 32768, 1 << 20));
        fpar.log = logs.log;
        fpar.log_cnt = logs.cnt;
        fpar.log_cap = logs.cap;
        fpar.counters = d_counter.p;
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev2, st));
        with_metric(metric, [&](auto m) {
            constexpr int MM = decltype(m)::value;
            if (item_cap == 32)
                launch<fltc::ivfflat_tc_kernel<MM, 32>>(num_sms(), fltc::THREADS, fltc::FlCfg<32>::SMEM_BYTES, st, tx, thi, tlo, fpar);
            else
                launch<fltc::ivfflat_tc_kernel<MM, 128>>(num_sms(), fltc::THREADS, fltc::FlCfg<128>::SMEM_BYTES, st, tx, thi, tlo, fpar);
        });
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev3, st));
        KB2_CUDA_CHECK(cudaGetLastError());
        uint32_t* qflag = s_cand_cnt.p + nq;
        lm::scatter_survivors_kernel<<<dim3(16, n_logs), 256, 0, st>>>(logs.log, logs.cnt, logs.cap, s_cand.p, s_cand_cnt.p, kTcCandCap,
                                                                       qflag, nullptr);
        fltc::count_flags_kernel<<<grid1d(nq, 256), 256, 0, st>>>(qflag, nq, logs.cnt + n_logs, s_cand_cnt.p + 2 * nq);
        last.launches += 6;
        uint32_t* hflag = (uint32_t*)h_counter.p + 12;
        KB2_CUDA_CHECK(cudaMemcpyAsync(hflag, s_cand_cnt.p + 2 * nq, 4, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        last.flagged = hflag[0];
        return hflag[0] == 0;
    }

    // coarse quantizer for queries [q_lo, q_hi): top-nprobe centroids with exact dis0 (F/IndexIVF.cpp:336-342) into rows
    // [q_lo, q_hi) of s_probe_ids / s_probe_dis
    void
    coarse_probes(const float* dq, int64_t q_lo, int64_t q_hi, int nprobe) {
        const int64_t m = q_hi - q_lo;
        if (m <= 0) return;
        dense_knn(*this, dq + q_lo * dim, m, centroids.p, cnorms.p, nlist, dim, metric, nprobe,
                  (int)std::min<int64_t>(nprobe + 16, nlist), nullptr, 0, nullptr, s_probe_ids.p + q_lo * nprobe,
                  s_probe_dis.p + q_lo * nprobe, false);
    }

    // ---------------------------------------------------------------- large-k path (DESIGN §4.9)
    // Candidate windows k_base > kMaxK: the dense mode of range_scan_kernel writes every probed row's key to its query's
    // row (slot = rank of the row among the query's probed rows, lists padded to 32), select_rows_kernel keeps the k_base
    // best, and the large finalize refines them (IVF_PQ with refine), maps labels and orders them.  Queries run in groups
    // whose rows fit kLargeKScratch.
    void
    search_large(const float* dq, int64_t nq, int nprobe, int k, int k_base, bool use_refine, const uint8_t* dbits,
                 int64_t* d_ids, float* d_dist) {
        cudaStream_t st = stream;
        // row length: the nprobe longest lists, each padded to 32 rows
        std::vector<int64_t> padded(nlist);
        for (int64_t l = 0; l < nlist; l++) padded[l] = round_up(h_list_len[l], 32);
        std::partial_sort(padded.begin(), padded.begin() + nprobe, padded.end(), std::greater<int64_t>());
        int64_t L = 32;
        for (int j = 0; j < nprobe; j++) L += padded[j];
        const int K = k_base;
        const int64_t g = large_k_group(nq, L * 8 + large_k_row_bytes(K));
        s_lk_rows.ensure((size_t)g * L);
        s_lk_cand.ensure((size_t)g * K);
        RangeParams rp = list_params(dq, nq, nprobe, dbits);
        IvfScanParams& sp = rp.sp;
        rp.dense = s_lk_rows.p;
        rp.dense_ld = L;
        rp.scanned = d_counter.p;
        sp.nsplit = (g < 2 * num_sms()) ? (int)std::min<int64_t>(nprobe, (2 * num_sms() + g - 1) / g) : 1;
        sp.nsplit = std::max(sp.nsplit, (nprobe + kScanSliceProbes - 1) / kScanSliceProbes);
        const int np_max = (nprobe + sp.nsplit - 1) / sp.nsplit;
        const size_t smem = (size_t)dim * 4 + 64 + (size_t)(np_max + 1) * 4 + (size_t)np_max * 12 + (is_pq ? (size_t)M * 1024 : 0);
        KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_NOT_IMPLEMENTED, "large-k search: m too large");
        FinalizeParams fp{};
        fp.k_sel = K;
        fp.k_out = k;
        fp.rows = rows.p;
        fp.labels = labels.device();
        fp.rerank = use_refine ? 1 : 0;
        fp.raw = vecs.p;
        fp.raw16 = (is_pq && refine_kind) ? vecs16.p : nullptr;
        fp.raw16_kind = refine_kind;
        fp.raw_by_pos = 1;
        fp.queries = dq;
        fp.d = dim;
        fp.metric = metric;
        fp.out_ids = d_ids;
        fp.out_dist = d_dist;
        KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p, 0, 8, st));
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev0, st));
        for (int64_t q0 = 0; q0 < nq; q0 += g) {
            const int64_t rws = std::min(g, nq - q0);
            rp.q0 = q0;
            KB2_CUDA_CHECK(cudaMemsetAsync(s_lk_rows.p, 0xFF, (size_t)rws * L * 8, st));
            launch<range_scan_kernel>((unsigned)(rws * sp.nsplit), kScanThreads, smem, st, rp);
            last.launches++;
            KB2_CUDA_CHECK(cudaGetLastError());
            large_k_select<uint64_t>(*this, s_lk_rows.p, L, L, 0u, K, s_lk_cand.p, K, rws);
            large_k_finalize(*this, fp, s_lk_cand.p, K, K, rws, q0);
        }
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev1, st));
        unsigned long long* hc = (unsigned long long*)h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(hc, d_counter.p, 8, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        last.codes = (int64_t)hc[0];
        last.code_bytes = last.codes * (is_pq ? (int64_t)M : (int64_t)dim * 4);
        last.pairs = nq * nprobe;
        last.survivors = 0;
        last.flagged = 0;
    }

    // ---------------------------------------------------------------- Search (ivf.cc:887-1168)
    void
    search(const float* q, int64_t nq, int k, const JsonObj& cfg, const uint8_t* bitset, int64_t nbits, int64_t* out_ids,
           float* out_dist) override {
        KB2_REQUIRE(trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        KB2_REQUIRE(n_total > 0, KB2_EMPTY_INDEX, "index is empty");
        seal();
        const int nprobe = search_nprobe(cfg);
        // a sharded search all-gathers the probes of one kMaxK window per query
        KB2_REQUIRE(nprobe <= kMaxWindowProbes || shard_world == 1, KB2_OUT_OF_RANGE_IN_JSON,
                    "nprobe too large for the GPU path (max 1008)");
        const bool use_refine = is_pq && refine;
        const double refine_k = cfg.get_num("refine_k", 1.0);
        KB2_REQUIRE(refine_k >= 1.0, KB2_OUT_OF_RANGE_IN_JSON, "refine_k must be >= 1");
        KB2_REQUIRE(k > 0 && (use_refine ? (double)k * refine_k : (double)k) <= (double)kMaxLargeK, KB2_INVALID_ARGS,
                    "k (x refine_k) out of range (max 16384)");
        const int k_base = use_refine ? (int)((double)k * refine_k) : k;  // K/IndexRefine.cpp:80-83
        const bool dist = distributed();
        KB2_REQUIRE(!dist || (int64_t)shard_world * k <= kMaxSortEntries, KB2_INVALID_ARGS, "world * k too large for the merge");

        cudaStream_t st = stream;
        // (Uploading host queries in four pieces on a side stream with the coarse stage started per piece was measured at C3:
        //  e2e 2.10 / 2.03 ms without vs 2.12 / 2.09 ms with -- four quarter-size coarse passes cost what the copy hides.)
        const float* dq = to_device(q, (size_t)nq * dim, s_q);
        const uint8_t* dbits = bitset_to_device(bitset, nbits);
        int64_t* d_ids;
        float* d_dist;
        device_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        if (nprobe > kMaxWindowProbes) {
            search_many_probes(dq, nq, nprobe, k, k_base, use_refine, dbits, d_ids, d_dist);
            results_out(nq, k, out_ids, out_dist, d_ids, d_dist);
            return;
        }

        // ---- coarse quantizer.  With a communicator every rank ranks the centroids for its slice of the batch only and the
        //      probe lists are all-gathered (in place; slices padded to the same length).
        const int64_t per = dist ? (nq + shard_world - 1) / shard_world : nq;
        const int64_t nq_pad = dist ? per * shard_world : nq;
        s_probe_ids.ensure((size_t)nq_pad * nprobe);
        s_probe_dis.ensure((size_t)nq_pad * nprobe);
        if (dist) {
            const int64_t q_lo = std::min<int64_t>(nq, per * shard_rank), q_hi = std::min<int64_t>(nq, q_lo + per);
            coarse_probes(dq, q_lo, q_hi, nprobe);
            if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev_c0, st));
            comm->all_gather2(s_probe_ids.p + per * shard_rank * nprobe, s_probe_ids.p, (size_t)per * nprobe * 8,
                              s_probe_dis.p + per * shard_rank * nprobe, s_probe_dis.p, (size_t)per * nprobe * 4, st);
            if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev_c1, st));
        } else {
            coarse_probes(dq, 0, nq, nprobe);
        }
        scan_probes(dq, nq, nprobe, k, k_base, use_refine, dbits, d_ids, d_dist, out_ids, out_dist);
    }

    // nprobe of a search config: the reference's range check (1..kMaxNprobe), then clamped to [1, nlist]
    int
    search_nprobe(const JsonObj& cfg) const {
        const long long v = cfg.get_int("nprobe", 8);
        KB2_REQUIRE(v <= kMaxNprobe, KB2_OUT_OF_RANGE_IN_JSON, "nprobe out of range (1..65536)");
        return (int)std::min<int64_t>(std::max<long long>(v, 1), nlist);
    }

    // Search above kMaxWindowProbes probes: the queries run in groups, one host iteration each, whose probe arrays
    // (12 bytes a probe), list-major pairs (8 bytes a probe), scan slices and candidate rows fit kProbeScratch.  Each group
    // ranks its probes (coarse_probes: the large-k selection) and runs scan_probes on them, which picks the engine as it
    // does for any batch; the results land in the group's rows of d_ids / d_dist.
    void
    search_many_probes(const float* dq, int64_t nq, int nprobe, int k, int k_base, bool use_refine, const uint8_t* dbits,
                       int64_t* d_ids, float* d_dist) {
        const int Ksel = next_pow2(std::max(32, k_base));
        const int64_t slices = (nprobe + kScanSliceProbes - 1) / kScanSliceProbes;
        const int64_t per_query = (int64_t)nprobe * 20 + (slices + 1) * Ksel * 8 + (int64_t)kTcCandCap * 8 + 4096 * 4 + dim * 2;
        const int64_t g = std::max<int64_t>(1, std::min<int64_t>(nq, kProbeScratch / per_query));
        s_probe_ids.ensure((size_t)g * nprobe);
        s_probe_dis.ensure((size_t)g * nprobe);
        Counters sum{};
        float stage_ms = 0.f, kernel_ms = 0.f;
        int engine = 0;
        for (int64_t q0 = 0; q0 < nq; q0 += g) {
            const int64_t rows = std::min(g, nq - q0);
            const float* gq = dq + q0 * dim;
            coarse_probes(gq, 0, rows, nprobe);
            int64_t* gi = d_ids + q0 * k;
            float* gd = d_dist + q0 * k;
            scan_probes(gq, rows, nprobe, k, k_base, use_refine, dbits, gi, gd, gi, gd);
            sum.codes += last.codes;
            sum.code_bytes += last.code_bytes;
            sum.pairs += last.pairs;
            sum.survivors += last.survivors;
            sum.flagged += last.flagged;
            stage_ms += last_stage_ms;
            kernel_ms += last_kernel_ms;
            engine = std::max(engine, last_engine);   // a batch some of whose groups went list-major reports the list-major engine
        }
        last.codes = sum.codes;
        last.code_bytes = sum.code_bytes;
        last.pairs = sum.pairs;
        last.survivors = sum.survivors;
        last.flagged = sum.flagged;
        last_engine = engine;
        if (timing) {
            last_stage_ms = stage_ms;
            last_kernel_ms = kernel_ms;
            last_comm_ms = 0.f;
        }
    }

    // Scan of the nq queries' probes in s_probe_ids / s_probe_dis (rows [0, nq)) and the finalize into d_ids / d_dist, which
    // results_out copies to out_ids / out_dist.  The engine: the large-k path for windows k_base > kMaxK, else the list-major
    // tensor-core engines where use_tc_engine / use_flat_tc_engine take them, else the query-major scan kernels.
    void
    scan_probes(const float* dq, int64_t nq, int nprobe, int k, int k_base, bool use_refine, const uint8_t* dbits, int64_t* d_ids,
                float* d_dist, int64_t* out_ids, float* out_dist) {
        cudaStream_t st = stream;
        const bool dist = distributed();
        if (k_base > kMaxK) {
            KB2_REQUIRE(!dist, KB2_NOT_IMPLEMENTED, "sharded search with k (x refine_k) above 1024");
            search_large(dq, nq, nprobe, k, k_base, use_refine, dbits, d_ids, d_dist);
            results_out(nq, k, out_ids, out_dist, d_ids, d_dist);
            last_engine = 2;
            if (timing) {
                KB2_CUDA_CHECK(cudaEventElapsedTime(&last_stage_ms, ev0, ev1));
                last_kernel_ms = last_stage_ms;
                last_comm_ms = 0.f;
            }
            return;
        }

        // ---- visiting order of the queries: sorted by nearest list, so that CTAs resident at the same
        //      time probe the same lists (L2 reuse of codes; results are order-independent)
        const int32_t* qperm = nullptr;
        const bool tc_engine = use_tc_engine(nq, nprobe, next_pow2(std::max(32, k_base)));
        if (nq >= 2 * num_sms() && !tc_engine) {
            s_qkey.ensure(nq); s_qkey2.ensure(nq); s_qidx.ensure(nq); s_qperm.ensure(nq);
            first_probe_kernel<<<grid1d(nq, 256), 256, 0, st>>>(s_probe_ids.p, nprobe, nq, s_qkey.p, s_qidx.p);
            size_t tmp_bytes = 0;
            int end_bit = 1;
            while ((1ll << end_bit) < nlist) end_bit++;
            cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, s_qkey.p, s_qkey2.p, s_qidx.p, s_qperm.p, (int)nq, 0, end_bit, st);
            s_sort_tmp.ensure(tmp_bytes);
            cub::DeviceRadixSort::SortPairs(s_sort_tmp.p, tmp_bytes, s_qkey.p, s_qkey2.p, s_qidx.p, s_qperm.p, (int)nq, 0,
                                            end_bit, st);
            qperm = s_qperm.p;
            last.launches += 3;
        }

        // ---- list scan
        int nsplit = 1;
        if (nq < 2 * num_sms()) nsplit = (int)std::min<int64_t>(nprobe, (2 * num_sms() + nq - 1) / nq);
        const int Ksel = next_pow2(std::max(32, k_base));
        while ((int64_t)nsplit * Ksel > kMaxSortEntries) nsplit--;
        // no CTA holds more than kScanSliceProbes probes; slices whose outputs exceed what finalize sorts are cut to the
        // Ksel best of each query first (select_rows_kernel)
        nsplit = std::max(nsplit, (nprobe + kScanSliceProbes - 1) / kScanSliceProbes);
        const bool cut_slices = (int64_t)nsplit * Ksel > kMaxSortEntries;
        const int np_max = (nprobe + nsplit - 1) / nsplit;
        s_partial2.ensure((size_t)nq * nsplit * Ksel);
        KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p, 0, 64, st));
        IvfScanParams sp = list_params(dq, nq, nprobe, dbits).sp;
        sp.nsplit = nsplit;
        sp.K = Ksel;
        sp.kout = Ksel;
        sp.partial = s_partial2.p;
        sp.counters = d_counter.p;
        sp.qperm = qperm;
        const unsigned grid = (unsigned)(nq * nsplit);
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev0, st));
        const uint64_t* fin_partial = s_partial2.p;
        int64_t fin_stride = (int64_t)nsplit * Ksel;
        int fin_n = nsplit * Ksel;
        const uint32_t *fin_counts = nullptr, *fin_flags = nullptr;
        bool flat_tc = false;
        if (tc_engine) {
            search_tc(sp, nq, nprobe, Ksel, k_base, dbits != nullptr);
            fin_partial = s_cand.p;
            fin_stride = kTcCandCap;
            fin_n = kTcCandCap;
            fin_counts = s_cand_cnt.p;
            fin_flags = s_cand_cnt.p + nq;
        } else if (use_flat_tc_engine(nq, nprobe, k_base) && search_flat_tc(sp, nq, nprobe, Ksel, k_base, dbits != nullptr)) {
            flat_tc = true;
            fin_partial = s_cand.p;
            fin_stride = kTcCandCap;
            fin_n = kTcCandCap;
            fin_counts = s_cand_cnt.p;
        } else {
            launch_scan(sp, grid, Ksel, np_max, dbits != nullptr);
            if (cut_slices) {
                s_partial.ensure((size_t)nq * Ksel);
                large_k_select<uint64_t>(*this, s_partial2.p, fin_stride, fin_stride, 0u, Ksel, s_partial.p, Ksel, nq);
                fin_partial = s_partial.p;
                fin_stride = Ksel;
                fin_n = Ksel;
            }
        }
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev1, st));

        // ---- finalize: merge CTA lists, optional exact refine, labels.  With a communicator the local top-k goes to a
        //      staging buffer, ONE fused all-gather ships ids + distances of every shard, and the merge kernel writes the result.
        if (dist) ensure_gather_buffers(nq, k);
        {
            FinalizeParams fp{};
            fp.partial = fin_partial;
            fp.partial_stride = fin_stride;
            fp.n_partial = fin_n;
            fp.counts = fin_counts;
            fp.count_flags = fin_flags;
            fp.k_sel = flat_tc ? k_base + 16 : k_base;   // tensor-core IVF_FLAT: 3xTF32 keys, exact re-rank of the k+16 best
            fp.k_out = k;
            fp.rows = rows.p;
            fp.labels = labels.device();
            fp.rerank = (use_refine || flat_tc) ? 1 : 0;
            fp.raw = vecs.p;
            fp.raw16 = (is_pq && refine_kind) ? vecs16.p : nullptr;
            fp.raw16_kind = refine_kind;
            fp.raw_by_pos = 1;
            fp.queries = dq;
            fp.d = dim;
            fp.metric = metric;
            fp.out_ids = dist ? s_loc_ids.p : d_ids;
            fp.out_dist = dist ? s_loc_dist.p : d_dist;
            launch_finalize(*this, fp, nq);
        }
        if (dist) gather_merge(nq, k, d_ids, d_dist);
        unsigned long long* hc = (unsigned long long*)h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(hc, d_counter.p, 64, cudaMemcpyDeviceToHost, st));
        results_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        KB2_REQUIRE(hc[1] == 0 && hc[5] == 0, KB2_INTERNAL_ERROR, "ivfpq_scan_kernel: unexpected shared-memory window base");
        last.survivors = (int64_t)hc[2];
        last.flagged = (int64_t)hc[7];
        const unsigned long long scanned = hc[0];
        last.codes = (int64_t)scanned;
        last.code_bytes = (int64_t)scanned * (is_pq ? (int64_t)M : (int64_t)dim * 4);
        last.pairs = nq * nprobe;
        last_engine = (tc_engine || flat_tc) ? 1 : 0;
        if (timing) {
            KB2_CUDA_CHECK(cudaEventElapsedTime(&last_stage_ms, ev0, ev1));
            last_kernel_ms = last_stage_ms;
            if (tc_engine || flat_tc) KB2_CUDA_CHECK(cudaEventElapsedTime(&last_kernel_ms, ev2, ev3));
            last_comm_ms = 0.f;
            if (dist) {
                float a = 0.f, b = 0.f;
                KB2_CUDA_CHECK(cudaEventElapsedTime(&a, ev_c0, ev_c1));
                KB2_CUDA_CHECK(cudaEventElapsedTime(&b, ev_c2, ev_c3));
                last_comm_ms = a + b;
            }
        }
    }

    void
    get_vectors(const int64_t* ids, int64_t n, float* out) override {
        KB2_REQUIRE(keeps_vecs(), KB2_NOT_IMPLEMENTED, "index holds no raw data");
        KB2_REQUIRE(!labels.custom && shard_world == 1, KB2_NOT_IMPLEMENTED, "GetVectorByIds with custom ids / shards");
        seal();
        std::vector<int64_t> h(n);
        if (is_device_ptr(ids)) {
            KB2_CUDA_CHECK(cudaMemcpy(h.data(), ids, n * 8, cudaMemcpyDeviceToHost));
        } else {
            memcpy(h.data(), ids, n * 8);
        }
        std::vector<int32_t> hpos(n_total);
        KB2_CUDA_CHECK(cudaMemcpy(hpos.data(), pos_of_row.p, n_total * 4, cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < n; i++) {
            KB2_REQUIRE(h[i] >= 0 && h[i] < n_total, KB2_INVALID_ARGS, "id out of range");
            KB2_CUDA_CHECK(cudaMemcpyAsync(out + i * dim, vecs.p + (int64_t)hpos[h[i]] * dim, (size_t)dim * 4,
                                           cudaMemcpyDefault, stream));
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    // ---------------------------------------------------------------- import of an externally built index
    std::vector<int32_t> imp_assign;
    std::vector<int64_t> imp_labels;
    std::vector<uint8_t> imp_codes;
    void
    import_begin(int64_t nl, const float* cent, const float* pq_cent) {
        KB2_REQUIRE(n_total == 0, KB2_INVALID_ARGS, "import into a non-empty index");
        nlist = nl;
        centroids.alloc_exact((size_t)nlist * dim);
        KB2_CUDA_CHECK(cudaMemcpyAsync(centroids.p, cent, (size_t)nlist * dim * 4, cudaMemcpyDefault, stream));
        set_centroids_common();
        if (is_pq) {
            KB2_REQUIRE(pq_cent != nullptr, KB2_INVALID_ARGS, "IVF_PQ import needs pq centroids");
            KB2_REQUIRE(M > 0 && dim % M == 0 && nbits == 8, KB2_INVALID_ARGS, "IVF_PQ import: bad m / nbits");
            dsub = dim / M;
            pqc.alloc_exact((size_t)M * 256 * dsub);
            tc_ready = false;
            KB2_CUDA_CHECK(cudaMemcpyAsync(pqc.p, pq_cent, (size_t)M * 256 * dsub * 4, cudaMemcpyDefault, stream));
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        trained = true;
        imp_assign.clear();
        imp_labels.clear();
        imp_codes.clear();
    }
    void
    import_list(int64_t l, int64_t sz, const int64_t* ids, const uint8_t* cds) {
        KB2_REQUIRE(l >= 0 && l < nlist, KB2_INVALID_ARGS, "list number out of range");
        const size_t cs = is_pq ? (size_t)M : (size_t)dim * 4;
        imp_assign.insert(imp_assign.end(), (size_t)sz, (int32_t)l);
        imp_labels.insert(imp_labels.end(), ids, ids + sz);
        imp_codes.insert(imp_codes.end(), cds, cds + (size_t)sz * cs);
    }
    // raw (refine=true): [n_raw][dim] rows addressed by label, or — raw_in_import_order — by the order of the import_list calls
    void
    import_finish(const float* raw, int64_t n_raw, bool raw_in_import_order = false) {
        const int64_t n = (int64_t)imp_assign.size();
        std::vector<int32_t> orig_of_row;   // row -> position in the import stream (only when raw_in_import_order)
        // Rows were numbered in import (list) order.  The reference's ids are segment offsets 0..n-1 and a BitsetView /
        // GetVectorByIds address vectors by that id (bitsetview.h:131-175), so when the labels are a permutation of
        // 0..n-1 renumber the rows so that row == label: bitset tests, GetVectorByIds and add() then behave exactly as
        // on an index built here.  Within a list the scan order becomes ascending id (the reference's insertion order).
        {
            bool perm = n > 0;
            std::vector<uint8_t> seen((size_t)n, 0);
            for (int64_t i = 0; i < n && perm; i++) {
                const int64_t l = imp_labels[i];
                if (l < 0 || l >= n || seen[l]) perm = false; else seen[l] = 1;
            }
            if (perm) {
                const size_t cs = is_pq ? (size_t)M : (size_t)dim * 4;
                std::vector<int32_t> a2((size_t)n);
                std::vector<uint8_t> c2((size_t)n * cs);
                if (raw_in_import_order) orig_of_row.resize((size_t)n);
                for (int64_t i = 0; i < n; i++) {
                    const int64_t l = imp_labels[i];
                    if (raw_in_import_order) orig_of_row[l] = (int32_t)i;
                    a2[l] = imp_assign[i];
                    memcpy(c2.data() + (size_t)l * cs, imp_codes.data() + (size_t)i * cs, cs);
                }
                imp_assign.swap(a2);
                imp_codes.swap(c2);
                for (int64_t i = 0; i < n; i++) imp_labels[i] = i;
            }
            labels = RowLabels{};
            if (!perm) labels.append(0, imp_labels.data(), n, 0, true, stream);
        }
        f_assign_used = 0;
        dev_append(f_assign, f_assign_used, imp_assign.data(), (size_t)n, stream);
        if (is_pq) {
            f_codes_used = 0;
            dev_append(f_codes, f_codes_used, imp_codes.data(), imp_codes.size(), stream);
            if (refine) {
                KB2_REQUIRE(raw != nullptr, KB2_INVALID_ARGS, "refine=true import needs the raw vectors");
                // gather the raw vector of every row: raw[label[row]], or raw[import position of row]
                std::vector<int32_t> lab32(n);
                for (int64_t i = 0; i < n; i++) {
                    const int64_t src = raw_in_import_order ? (orig_of_row.empty() ? i : (int64_t)orig_of_row[i]) : imp_labels[i];
                    KB2_REQUIRE(src >= 0 && src < n_raw, KB2_INVALID_ARGS, "label outside raw data");
                    lab32[i] = (int32_t)src;
                }
                DevBuf<float> rbuf;
                const float* draw = to_device(raw, (size_t)n_raw * dim, rbuf, false);
                DevBuf<int32_t> dl;
                dl.ensure(n);
                KB2_CUDA_CHECK(cudaMemcpyAsync(dl.p, lab32.data(), n * 4, cudaMemcpyHostToDevice, stream));
                f_vecs.alloc_exact((size_t)n * dim);
                gather_rows_kernel<<<grid1d(n * 32, 256), 256, 0, stream>>>(draw, dl.p, n, dim, dim, f_vecs.p);
                f_vecs_used = (size_t)n * dim;
                KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
            }
        } else {
            f_vecs_used = 0;
            dev_append(f_vecs, f_vecs_used, (const float*)imp_codes.data(), (size_t)n * dim, stream);
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        n_total = n;
        imp_assign.clear(); imp_assign.shrink_to_fit();
        imp_labels.clear(); imp_labels.shrink_to_fit();
        imp_codes.clear(); imp_codes.shrink_to_fit();
        sealed = false;
    }
    // export one list in scan order (host buffers)
    void
    export_list(int64_t l, int64_t* ids, uint8_t* cds) {
        seal();
        KB2_REQUIRE(l >= 0 && l < nlist, KB2_INVALID_ARGS, "list number out of range");
        const int64_t off = h_list_off[l], len = h_list_len[l];
        if (len == 0) return;
        std::vector<int32_t> hrows(len);
        KB2_CUDA_CHECK(cudaMemcpy(hrows.data(), rows.p + off, len * 4, cudaMemcpyDeviceToHost));
        const std::vector<int64_t> hl = labels.host(n_total);
        for (int64_t i = 0; i < len; i++) ids[i] = hl.empty() ? hrows[i] : hl[hrows[i]];
        if (!is_pq) {
            KB2_CUDA_CHECK(cudaMemcpy(cds, vecs.p + off * dim, (size_t)len * dim * 4, cudaMemcpyDeviceToHost));
        } else if (G > 0) {
            std::vector<uint8_t> tmp((size_t)len * 16);
            for (int g = 0; g < G; g++) {
                KB2_CUDA_CHECK(cudaMemcpy(tmp.data(), codes.p + ((size_t)g * npad + off) * 16, (size_t)len * 16,
                                          cudaMemcpyDeviceToHost));
                for (int64_t i = 0; i < len; i++)
                    for (int s = 0; s < 16; s++)
                        cds[i * M + g * 16 + ((s + (off + i)) & 15)] = tmp[i * 16 + s];
            }
        } else {
            KB2_CUDA_CHECK(cudaMemcpy(cds, codes.p + (size_t)off * M, (size_t)len * M, cudaMemcpyDeviceToHost));
        }
    }

    void
    configure(const JsonObj& cfg) override {
        nlist = cfg.get_int("nlist", 128);
        KB2_REQUIRE(nlist >= 1 && nlist <= 65536 * 16, KB2_OUT_OF_RANGE_IN_JSON, "nlist out of range");
        if (!is_pq) return;
        KB2_REQUIRE(cfg.has("m"), KB2_INVALID_PARAM_IN_JSON, "IVF_PQ requires m");
        M = (int)cfg.get_int("m", 0);
        nbits = (int)cfg.get_int("nbits", 8);
        KB2_REQUIRE(M >= 1 && dim % M == 0, KB2_INVALID_ARGS, "dim must be a multiple of m");
        KB2_REQUIRE(nbits >= 1 && nbits <= 24, KB2_OUT_OF_RANGE_IN_JSON, "nbits out of range");
        refine = cfg.get_bool("refine", false);
        if (refine) {
            std::string rt = cfg.get_str("refine_type", "flat");
            for (auto& ch : rt) ch = (char)tolower((unsigned char)ch);
            if (rt == "flat" || rt == "fp32" || rt == "float32" || rt == "data_view") refine_kind = 0;
            else if (rt == "fp16" || rt == "float16") refine_kind = 1;
            else if (rt == "bf16" || rt == "bfloat16") refine_kind = 2;
            else throw Error(KB2_NOT_IMPLEMENTED, "refine_type " + rt + " is not implemented (flat / fp16 / bf16 are)");
        }
    }

    void
    save(BlobWriter& w) override {
        KB2_REQUIRE(trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        KB2_REQUIRE(shard_world == 1, KB2_NOT_IMPLEMENTED, "serialising a shard");
        seal();
        w.put<int64_t>(nlist);
        w.put<int32_t>(M);
        w.put<int32_t>(nbits);
        w.put<int32_t>(refine ? 1 + refine_kind : 0);   // 0 none, 1 fp32, 2 fp16, 3 bf16 refine store
        DevBuf<float> dec;
        const float* v32 = (is_pq && refine) ? vecs_f32(dec) : nullptr;
        if (v32) KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        std::vector<float> c((size_t)nlist * dim);
        KB2_CUDA_CHECK(cudaMemcpy(c.data(), centroids.p, c.size() * 4, cudaMemcpyDeviceToHost));
        w.put_bytes(c.data(), c.size() * 4);
        if (is_pq) {
            std::vector<float> pc((size_t)M * 256 * dsub);
            KB2_CUDA_CHECK(cudaMemcpy(pc.data(), pqc.p, pc.size() * 4, cudaMemcpyDeviceToHost));
            w.put_bytes(pc.data(), pc.size() * 4);
        }
        const size_t cs = is_pq ? (size_t)M : (size_t)dim * 4;
        for (int64_t l = 0; l < nlist; l++) {
            const int64_t len = h_list_len[l];
            w.put<int64_t>(len);
            if (!len) continue;
            std::vector<int64_t> ids(len);
            std::vector<uint8_t> cd((size_t)len * cs);
            export_list(l, ids.data(), cd.data());
            w.put_bytes(ids.data(), len * 8);
            w.put_bytes(cd.data(), cd.size());
            if (is_pq && refine) {
                std::vector<float> rv((size_t)len * dim);
                KB2_CUDA_CHECK(cudaMemcpy(rv.data(), v32 + h_list_off[l] * dim, rv.size() * 4, cudaMemcpyDeviceToHost));
                w.put_bytes(rv.data(), rv.size() * 4);
            }
        }
    }
    void
    load(BlobReader& r) override {
        const int64_t nl = r.get<int64_t>();
        M = r.get<int32_t>();
        nbits = r.get<int32_t>();
        const int rf = r.get<int32_t>();
        KB2_REQUIRE(rf >= 0 && rf <= 3, KB2_INVALID_BINARY_SET, "bad refine field in blob");
        refine = rf != 0;
        refine_kind = rf ? rf - 1 : 0;
        KB2_REQUIRE(nl >= 1 && (uint64_t)nl <= r.n / ((size_t)dim * 4), KB2_INVALID_BINARY_SET, "bad nlist in blob");
        if (is_pq) KB2_REQUIRE(M > 0 && dim % M == 0 && nbits == 8, KB2_INVALID_BINARY_SET, "bad m / nbits in blob");
        std::vector<float> c((size_t)nl * dim);
        memcpy(c.data(), r.get_bytes(c.size() * 4), c.size() * 4);
        std::vector<float> pc;
        if (is_pq) {
            pc.resize((size_t)M * 256 * (dim / M));
            memcpy(pc.data(), r.get_bytes(pc.size() * 4), pc.size() * 4);
        }
        import_begin(nl, c.data(), is_pq ? pc.data() : nullptr);
        const size_t cs = is_pq ? (size_t)M : (size_t)dim * 4;
        const bool with_raw = is_pq && refine;
        std::vector<float> raw_rows;  // import order
        for (int64_t l = 0; l < nl; l++) {
            const int64_t len = r.get<int64_t>();
            KB2_REQUIRE(len >= 0 && (uint64_t)len <= r.n / 8, KB2_INVALID_BINARY_SET, "bad list length in blob");
            if (!len) continue;
            std::vector<int64_t> ids(len);
            memcpy(ids.data(), r.get_bytes(len * 8), len * 8);
            const uint8_t* cd = r.get_bytes((size_t)len * cs);
            import_list(l, len, ids.data(), cd);
            if (with_raw) {
                const uint8_t* rv = r.get_bytes((size_t)len * dim * 4);
                const size_t o = raw_rows.size();
                raw_rows.resize(o + (size_t)len * dim);
                memcpy(raw_rows.data() + o, rv, (size_t)len * dim * 4);
            }
        }
        import_finish(with_raw ? raw_rows.data() : nullptr, with_raw ? (int64_t)(raw_rows.size() / dim) : 0, true);
    }

    void
    to_faiss(FaissIndexData& o) override {
        KB2_REQUIRE(trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        seal();
        o.nlist = nlist;
        o.nprobe = 1;
        o.centroids.resize((size_t)nlist * o.d);
        KB2_CUDA_CHECK(cudaMemcpy(o.centroids.data(), centroids.p, o.centroids.size() * 4, cudaMemcpyDeviceToHost));
        o.M = M;
        o.code_size = is_pq ? (uint64_t)M : (uint64_t)o.d * 4;
        if (is_pq) {
            KB2_REQUIRE(nbits == 8, KB2_NOT_IMPLEMENTED, "faiss stream: nbits != 8");
            o.pq_centroids.resize((size_t)256 * o.d);
            KB2_CUDA_CHECK(cudaMemcpy(o.pq_centroids.data(), pqc.p, o.pq_centroids.size() * 4, cudaMemcpyDeviceToHost));
        }
        o.list_ids.assign(nlist, {});
        o.list_codes.assign(nlist, {});
        for (int64_t l = 0; l < nlist; l++) {
            const int64_t len = h_list_len[l];
            if (!len) continue;
            o.list_ids[l].resize(len);
            o.list_codes[l].resize((size_t)len * o.code_size);
            export_list(l, o.list_ids[l].data(), o.list_codes[l].data());
        }
        o.has_refine = is_pq && refine;
        if (o.has_refine) {
            KB2_REQUIRE(!labels.custom, KB2_NOT_IMPLEMENTED, "faiss stream: refine store with custom ids");
            KB2_REQUIRE(refine_kind == 0, KB2_NOT_IMPLEMENTED, "faiss stream: only a flat fp32 refine store is written");
            // refine store in id order: row r lives at position pos_of_row[r]
            DevBuf<float> byrow;
            byrow.ensure((size_t)std::max<int64_t>(o.ntotal, 1) * o.d);
            gather_rows_kernel<<<grid1d(o.ntotal * 32, 256), 256, 0, stream>>>(vecs.p, pos_of_row.p, o.ntotal, o.d, o.d, byrow.p);
            o.refine_xb.resize((size_t)o.ntotal * o.d);
            KB2_CUDA_CHECK(cudaMemcpyAsync(o.refine_xb.data(), byrow.p, o.refine_xb.size() * 4, cudaMemcpyDeviceToHost, stream));
            KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
            o.k_factor = 1.f;
        }
    }
    void
    from_faiss(const FaissIndexData& o) override {
        KB2_REQUIRE(!o.cosine, KB2_NOT_IMPLEMENTED, "faiss stream: cosine IVF indexes are not supported");
        nlist = o.nlist;
        M = o.M;
        nbits = 8;
        refine = o.has_refine;
        import_begin(o.nlist, o.centroids.data(), is_pq ? o.pq_centroids.data() : nullptr);
        for (int64_t l = 0; l < o.nlist; l++)
            if (!o.list_ids[l].empty()) import_list(l, (int64_t)o.list_ids[l].size(), o.list_ids[l].data(), o.list_codes[l].data());
        import_finish(o.has_refine ? o.refine_xb.data() : nullptr, o.has_refine ? o.ntotal : 0);
    }

    void
    append_meta(std::string& s) const override {
        s += ", \"nlist\": " + std::to_string(nlist);
        if (is_pq) s += ", \"m\": " + std::to_string(M) + ", \"nbits\": " + std::to_string(nbits) + ", \"refine\": " + (refine ? "true" : "false");
    }
    // RangeSearch: the hits of the nprobe nearest lists, their positions mapped to rows
    std::vector<RangeHit>
    range_hits(const RangeParams& q, const JsonObj& cfg, int& nprobe) override {
        KB2_REQUIRE(trained, KB2_INDEX_NOT_TRAINED, "index not trained");
        seal();
        const int64_t nq = q.sp.nq;
        nprobe = search_nprobe(cfg);
        // above kMaxWindowProbes the queries run in groups whose probe arrays fit kProbeScratch
        const int64_t g = (nprobe > kMaxWindowProbes) ? std::max<int64_t>(1, std::min<int64_t>(nq, kProbeScratch / ((int64_t)nprobe * 12)))
                                                      : nq;
        s_probe_ids.ensure((size_t)g * nprobe);
        s_probe_dis.ensure((size_t)g * nprobe);
        std::vector<RangeHit> h;
        for (int64_t q0 = 0; q0 < nq; q0 += g) {
            const int64_t rows = std::min(g, nq - q0);
            const float* gq = q.sp.queries + q0 * dim;
            coarse_probes(gq, 0, rows, nprobe);
            RangeParams rp = list_params(gq, rows, nprobe, q.sp.bitset);
            rp.radius = q.radius;
            rp.range_filter = q.range_filter;
            // with max_empty_result_buckets on, a probe is empty when it adds no hit inside the radius, whatever range_filter
            // says (faiss range_search_preassigned): the scan emits the radius hits and range_search_index filters after the cut
            rp.has_filter = range_max_empty(cfg) > 0 ? 0 : q.has_filter;
            rp.sp.nsplit = (rows < 2 * num_sms()) ? (int)std::min<int64_t>(nprobe, (2 * num_sms() + rows - 1) / rows) : 1;
            rp.sp.nsplit = std::max(rp.sp.nsplit, (nprobe + kScanSliceProbes - 1) / kScanSliceProbes);
            const int np_max = (nprobe + rp.sp.nsplit - 1) / rp.sp.nsplit;
            size_t smem = (size_t)dim * 4 + 64 + (size_t)(np_max + 1) * 4 + (size_t)np_max * 12;
            if (is_pq) smem += (size_t)M * 1024;
            KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_NOT_IMPLEMENTED, "range search: m too large");
            std::vector<RangeHit> hg = range_scan(*this, rp, smem);
            if (q0 == 0) {
                h = std::move(hg);
            } else {
                for (RangeHit& e : hg) e.q += (int32_t)q0;   // the group's queries are numbered from 0
                h.insert(h.end(), hg.begin(), hg.end());
            }
        }
        std::vector<int32_t> hrows(npad);
        KB2_CUDA_CHECK(cudaMemcpy(hrows.data(), rows.p, npad * 4, cudaMemcpyDeviceToHost));
        for (RangeHit& e : h) e.pos = (uint32_t)hrows[e.pos];
        return h;
    }

    bool takes_emb_list() const override { return !is_pq; }
    std::pair<const float*, const int32_t*>
    emb_list_rows() override {
        seal();
        return {vecs.p, pos_of_row.p};
    }
};

}  // namespace kb2
