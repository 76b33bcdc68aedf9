// kb2_sparse.cuh — sparse float vectors: SPARSE_INVERTED_INDEX / SPARSE_WAND with the IP and BM25 metrics, and the sparse
// BruteForce (reference: src/index/sparse/sparse_index_node.cc, src/index/sparse/inverted_index.h,
// src/index/sparse/scorer.h, src/common/comp/brute_force.cc:1227-1340).
//
// Every search is exhaustive and exact (DESIGN §4.13): each posting of each kept query term is scored, so one definition
// serves both index types and every inverted_index_algo the reference offers.  Rows are CSR (indptr int64[n + 1], indices
// uint32[nnz] strictly ascending per row, values float32[nnz] finite and >= 0).  The index keeps the rows it was given
// (every add rebuilds the postings from all of them, so two adds equal one add of the concatenation) and, built from
// them, a term table (the sorted distinct indices), term-major postings (row int32, value f32) sorted by row within a
// term with int64 term offsets, and for BM25 the row sums L_r.
//
// A search prepares each query's kept (term id, weight) list (prep_queries_kernel), then scores one (query, tile of kTile
// rows) per CTA into a shared-memory accumulator (score_tile_kernel): the tile's segment of each kept term's posting list
// is found by binary search and walked in query order with a barrier between terms, so the sums have the definition's
// order whatever the schedule.  The tile's result then goes to the shared selection and finalize code: the best Ksel
// entries into the partial slots (k + 16 <= 1024), a dense key chunk for select_rows_kernel (larger k), or RangeSearch
// hits.  No [nq][n] score matrix is written on the top-k path.
#pragma once
#include <algorithm>
#include <cctype>
#include <cub/cub.cuh>
#include <string>
#include <vector>

#include "kb2_index.cuh"

namespace kb2 {

inline bool
is_sparse_type(const std::string& t) {
    return t == "SPARSE_INVERTED_INDEX" || t == "SPARSE_WAND";
}

namespace sparse {

constexpr int kTile = 16384;      // rows per scoring CTA: one fp32 accumulator each, 64 KB of shared memory
constexpr int kThreads = 256;
constexpr int kTermChunk = 128;   // query terms whose tile segments a CTA locates at once (two threads per term)
constexpr size_t kScoreSmem = (size_t)kTile * 4 + (size_t)kTermChunk * 20 + 288 * 4;
constexpr int64_t kMaxGridY = 65535;

// CSR validation status bits
enum : unsigned long long { kBadOffsets = 1, kBadIndices = 2, kBadValues = 4 };

// one thread per row: offsets inside [0, nnz] and non-decreasing, indices strictly ascending, values finite and >= 0
__global__ void
validate_csr_kernel(const int64_t* __restrict__ indptr, const uint32_t* __restrict__ indices, const float* __restrict__ values,
                    int64_t n, int64_t nnz, unsigned long long* status) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t lo = indptr[r], hi = indptr[r + 1];
        if (lo < 0 || lo > hi || hi > nnz) {
            atomicOr(status, kBadOffsets);
            continue;
        }
        unsigned long long bad = 0;
        for (int64_t j = lo; j < hi; j++) {
            if (j > lo && indices[j] <= indices[j - 1]) bad |= kBadIndices;
            const float v = values[j];
            if (!(v >= 0.f) || isinf(v)) bad |= kBadValues;
        }
        if (bad) atomicOr(status, bad);
    }
}

// sort keys (term << 32 | row) of every stored entry; with row_sum, also L_r = the fp32 sum of row r's values in index order
__global__ void
build_keys_kernel(const int64_t* __restrict__ indptr, const uint32_t* __restrict__ indices, const float* __restrict__ values,
                  int64_t n, uint64_t* __restrict__ keys, float* __restrict__ row_sum) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    float s = 0.f;
    for (int64_t j = indptr[r]; j < indptr[r + 1]; j++) {
        keys[j] = ((uint64_t)indices[j] << 32) | (uint64_t)r;
        if (row_sum) s = __fadd_rn(s, values[j]);
    }
    if (row_sum) row_sum[r] = s;
}

// after the sort: posting rows, and flags[i] = 1 where a new term starts
__global__ void
split_postings_kernel(const uint64_t* __restrict__ keys, int64_t nnz, int32_t* __restrict__ post_row, int64_t* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    post_row[i] = (int32_t)(uint32_t)keys[i];
    flags[i] = (i == 0 || (keys[i] >> 32) != (keys[i - 1] >> 32)) ? 1 : 0;
}

// term table and term offsets from the inclusive scan of the flags
__global__ void
term_table_kernel(const uint64_t* __restrict__ keys, const int64_t* __restrict__ scan, int64_t nnz, uint32_t* __restrict__ terms,
                  int64_t* __restrict__ term_off) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    if (i == 0 || scan[i] != scan[i - 1]) {
        terms[scan[i] - 1] = (uint32_t)(keys[i] >> 32);
        term_off[scan[i] - 1] = i;
    }
    if (i == nnz - 1) term_off[scan[i]] = nnz;
}

struct PrepParams {
    const int64_t* q_indptr;
    const uint32_t* q_indices;
    const float* q_values;
    const float* sorted;      // each query's values in ascending order (drop_ratio_search > 0), or null
    int64_t nq;
    float ratio;              // drop_ratio_search
    const uint32_t* terms;    // the index's term table
    int64_t nterms;
    const int64_t* term_off;
    int bm25;
    float p1;
    int32_t* q_term;          // [nnz_q] kept term ids, at the query's CSR offsets
    float* q_w;               // [nnz_q] kept weights: w (IP) or w * p1 (BM25)
    int32_t* q_cnt;           // [nq] kept entries
    unsigned long long* postings;   // += postings of the kept terms (last_search_counters)
};

// one warp per query: drop threshold (get_query_drop_threshold, inverted_index.h:151-162), term lookup, ordered compaction
__global__ void
prep_queries_kernel(PrepParams p) {
    const int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= p.nq) return;
    const int64_t lo = p.q_indptr[q], hi = p.q_indptr[q + 1];
    float thr = 0.f;
    if (p.sorted && hi > lo) {
        // c = (size_t)(float(ratio) * float(nnz_q)); ratio < 1, so only a product rounded up to nnz_q itself can reach it
        const uint64_t c = (uint64_t)__fmul_rn(p.ratio, (float)(hi - lo));
        if (c > 0) thr = p.sorted[lo + (int64_t)min(c, (uint64_t)(hi - lo - 1))];
    }
    int32_t kept = 0;
    unsigned long long post = 0;
    for (int64_t j0 = lo; j0 < hi; j0 += 32) {
        const int64_t j = j0 + lane;
        bool keep = false;
        int64_t tid = 0;
        float v = 0.f;
        if (j < hi) {
            v = p.q_values[j];
            if (v >= thr) {
                const uint32_t x = p.q_indices[j];
                int64_t a = 0, b = p.nterms;
                while (a < b) {
                    const int64_t m = (a + b) >> 1;
                    if (p.terms[m] < x) a = m + 1; else b = m;
                }
                tid = a;
                keep = a < p.nterms && p.terms[a] == x;
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const int64_t o = lo + kept + __popc(bal & ((1u << lane) - 1u));
            p.q_term[o] = (int32_t)tid;
            p.q_w[o] = p.bm25 ? __fmul_rn(v, p.p1) : v;
            post += (unsigned long long)(p.term_off[tid + 1] - p.term_off[tid]);
        }
        kept += __popc(bal);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) post += __shfl_xor_sync(0xffffffffu, post, o);
    if (lane == 0) {
        p.q_cnt[q] = kept;
        if (post) atomicAdd(p.postings, post);
    }
}

enum { kTopK = 0, kKeys = 1, kCount = 2, kEmit = 3 };

struct ScoreParams {
    // the index
    const int64_t* term_off;
    const int32_t* post_row;
    const float* post_val;
    const float* row_sum;     // BM25: L_r
    int64_t n;
    int bm25;
    float p2, p3;
    const uint8_t* bitset;
    // the prepared queries
    const int64_t* q_off;
    const int32_t* q_cnt;
    const int32_t* q_term;
    const float* q_w;
    int64_t q0, tile0;        // query and tile of blockIdx (0, 0)
    // kTopK: the tile's best ksel entries go to slot (slot0 + blockIdx.y) of the query's partial row
    uint64_t* partial;
    int64_t partial_stride;
    int slot0, ksel;
    // kKeys: key -s (or +inf) of row r at keys[(q - q0) * ldk + r - col0]
    float* keys;
    int64_t ldk, col0;
    // kCount / kEmit: hits radius < s <= range_filter; counts and offsets per (query, tile)
    float radius, range_filter;
    int has_filter;
    int64_t ntiles;
    int32_t* counts;
    const int64_t* hit_off;
    uint32_t* hit_key;        // f2ord(-s)
    int32_t* hit_row;
};

// The shared-memory counterpart of select_rows_kernel's radix select (same algorithm, entries from the accumulator):
// out[0..ksel) <- the ksel smallest (f2ord(-s) << 32 | row) entries of the tile's candidates (s > 0), unsorted, then kEmpty.
__device__ __forceinline__ uint64_t
tile_entry(const float* acc, int i, int64_t r0) {
    const float s = acc[i];
    return s > 0.f ? pack_kp(-s, (uint32_t)(r0 + i)) : kEmpty;
}

__device__ void
tile_select(const float* acc, int rows, int64_t r0, int K, uint64_t* __restrict__ out, uint32_t* hist, uint32_t* misc) {
    const int lane = threadIdx.x & 31;
    unsigned long long* s_prefix = reinterpret_cast<unsigned long long*>(misc);
    unsigned long long* s_mask = s_prefix + 1;
    uint32_t* s_need = misc + 4;
    uint32_t* s_done = misc + 5;
    uint32_t* s_cnt = misc + 6;
    if (threadIdx.x == 0) {
        *s_prefix = 0;
        *s_mask = 0;
        *s_need = (uint32_t)K;
        *s_done = 0;
        *s_cnt = 0;
    }
    uint64_t prefix = 0, mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (int i0 = 0; i0 < rows; i0 += blockDim.x) {
            const int i = i0 + threadIdx.x;
            uint32_t dig = 256;
            if (i < rows) {
                const uint64_t e = tile_entry(acc, i, r0);
                if (e != kEmpty && (e & mask) == prefix) dig = (uint32_t)(e >> shift) & 255u;
            }
            const unsigned grp = __match_any_sync(0xffffffffu, dig);
            if (dig != 256 && lane == __ffs(grp) - 1) atomicAdd(&hist[dig], (uint32_t)__popc(grp));
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t h[8], sum = 0;
#pragma unroll
            for (int t = 0; t < 8; t++) { h[t] = hist[lane * 8 + t]; sum += h[t]; }
            uint32_t incl = sum;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += v;
            }
            const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
            const uint32_t need = *s_need;
            if (total <= need) {
                if (lane == 0) *s_done = 1;
            } else if (incl - sum < need && need <= incl) {
                uint32_t c = incl - sum;
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    if (c + h[t] >= need) {
                        *s_prefix = prefix | ((uint64_t)(lane * 8 + t) << shift);
                        *s_mask = mask | (0xffull << shift);
                        *s_need = need - c;
                        *s_done = (h[t] == need - c) ? 1u : 0u;
                        break;
                    }
                    c += h[t];
                }
            }
        }
        __syncthreads();
        prefix = *s_prefix;
        mask = *s_mask;
        const bool done = *s_done != 0;
        __syncthreads();   // every thread has read the state before thread 0 of a next pass could change it
        if (done) break;
    }
    for (int i0 = 0; i0 < rows; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        uint64_t e = kEmpty;
        bool keep = false;
        if (i < rows) {
            e = tile_entry(acc, i, r0);
            keep = e != kEmpty && (e & mask) <= prefix;
        }
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        uint32_t base = 0;
        if (lane == 0 && b) base = atomicAdd(s_cnt, (uint32_t)__popc(b));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (keep) {
            const uint32_t slot = base + __popc(b & ((1u << lane) - 1u));
            if (slot < (uint32_t)K) out[slot] = e;
        }
    }
    __syncthreads();
    for (int i = (int)min(*s_cnt, (uint32_t)K) + threadIdx.x; i < K; i += blockDim.x) out[i] = kEmpty;
}

__device__ __forceinline__ bool
in_range(const ScoreParams& p, float s) {
    return s > 0.f && s > p.radius && (!p.has_filter || s <= p.range_filter);
}

// One CTA per (query q0 + blockIdx.x, tile tile0 + blockIdx.y).  Dynamic smem kScoreSmem, so three CTAs per SM; the
// minimum of three in the launch bounds is that occupancy (without it ptxas holds the kKeys instance to 40 registers and
// spills).
template <int MODE>
__global__ void __launch_bounds__(kThreads, 3)
score_tile_kernel(ScoreParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* acc = (float*)smem_raw;
    int64_t* s_lo = (int64_t*)(acc + kTile);
    int64_t* s_hi = s_lo + kTermChunk;
    float* s_w = (float*)(s_hi + kTermChunk);
    uint32_t* s_u = (uint32_t*)(s_w + kTermChunk);   // 256 histogram bins or warp totals, then 32 words of state
    const int64_t q = p.q0 + blockIdx.x;
    const int64_t t = p.tile0 + blockIdx.y;
    const int64_t r0 = t * kTile;
    const int rows = (int)min((int64_t)kTile, p.n - r0);
    for (int i = threadIdx.x; i < rows; i += kThreads) acc[i] = 0.f;
    const int64_t qb = p.q_off[q];
    const int cnt = p.q_cnt[q];
    for (int c0 = 0; c0 < cnt; c0 += kTermChunk) {
        const int m = min(kTermChunk, cnt - c0);
        __syncthreads();   // the previous chunk's segments are consumed (first chunk: the accumulator is zeroed)
        const int i = threadIdx.x >> 1;
        if (i < m) {
            const int32_t term = p.q_term[qb + c0 + i];
            int64_t lo = p.term_off[term], hi = p.term_off[term + 1];
            const int64_t target = (threadIdx.x & 1) ? r0 + rows : r0;
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if ((int64_t)p.post_row[mid] < target) lo = mid + 1; else hi = mid;
            }
            if (threadIdx.x & 1) {
                s_hi[i] = lo;
            } else {
                s_lo[i] = lo;
                s_w[i] = p.q_w[qb + c0 + i];
            }
        }
        __syncthreads();
        for (int j = 0; j < m; j++) {
            const int64_t lo = s_lo[j], hi = s_hi[j];
            if (lo == hi) continue;   // CTA-uniform
            const float w = s_w[j];
            for (int64_t e = lo + threadIdx.x; e < hi; e += kThreads) {
                const int64_t row = p.post_row[e];
                const int r = (int)(row - r0);
                assert(r >= 0 && r < rows);
                const float v = p.post_val[e];
                const float c = p.bm25 ? __fdiv_rn(__fmul_rn(w, v), __fadd_rn(__fadd_rn(v, p.p2), __fmul_rn(p.p3, p.row_sum[row])))
                                       : __fmul_rn(w, v);
                acc[r] = __fadd_rn(acc[r], c);   // a row occurs once per posting list: no other thread writes acc[r] now
            }
            __syncthreads();
        }
    }
    __syncthreads();
    if (p.bitset) {
        for (int i = threadIdx.x; i < rows; i += kThreads)
            if (bit_is_set(p.bitset, r0 + i)) acc[i] = 0.f;   // filtered rows are no candidates
        __syncthreads();
    }
    if (MODE == kTopK) {
        uint64_t* out = p.partial + q * p.partial_stride + (int64_t)(p.slot0 + blockIdx.y) * p.ksel;
        tile_select(acc, rows, r0, p.ksel, out, s_u, s_u + 256);
    } else if (MODE == kKeys) {
        float* out = p.keys + (q - p.q0) * p.ldk + (r0 - p.col0);
        for (int i = threadIdx.x; i < rows; i += kThreads) out[i] = acc[i] > 0.f ? -acc[i] : INFINITY;
    } else if (MODE == kCount) {
        uint32_t* s_cnt = s_u + 256;
        if (threadIdx.x == 0) *s_cnt = 0;
        __syncthreads();
        uint32_t c = 0;
        for (int i = threadIdx.x; i < rows; i += kThreads) c += in_range(p, acc[i]);
        if (c) atomicAdd(s_cnt, c);
        __syncthreads();
        if (threadIdx.x == 0) p.counts[q * p.ntiles + t] = (int32_t)*s_cnt;
    } else {
        // hits in row order: ballot + warp totals per round of kThreads rows
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        int64_t base = p.hit_off[q * p.ntiles + t];
        for (int i0 = 0; i0 < rows; i0 += kThreads) {
            const int i = i0 + threadIdx.x;
            const bool hit = i < rows && in_range(p, acc[i]);
            const unsigned b = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) s_u[warp] = __popc(b);
            __syncthreads();
            int64_t off = base + __popc(b & ((1u << lane) - 1u));
            int total = 0;
            for (int w = 0; w < kThreads / 32; w++) {
                if (w < warp) off += s_u[w];
                total += s_u[w];
            }
            if (hit) {
                p.hit_key[off] = f2ord(-acc[i]);
                p.hit_row[off] = (int32_t)(r0 + i);
            }
            base += total;
            __syncthreads();
        }
    }
}

}  // namespace sparse

// ============================================================================================
// SPARSE_INVERTED_INDEX / SPARSE_WAND (sparse_index_node.cc): metric IP or BM25; dim is 0
// ============================================================================================
struct SparseIndex : IndexBase {
    // the rows as added (CSR), kept on the host: every add rebuilds the postings from all of them, and the KB2I section
    // stores them
    std::vector<int64_t> h_indptr{0};
    std::vector<uint32_t> h_indices;
    std::vector<float> h_values;
    int64_t n = 0;
    // built from them on the device
    DevBuf<uint32_t> terms;      // [nterms] the sorted distinct indices
    DevBuf<int64_t> term_off;    // [nterms + 1]
    DevBuf<int32_t> post_row;
    DevBuf<float> post_val;
    DevBuf<float> row_sum;
    int64_t nterms = 0, sparse_dim = 0;
    // build keys (sparse_index_node.cc:121-126, sparse_index_config.h)
    bool has_bm25 = false;
    float k1 = 0.f, b = 0.f, avgdl = 0.f;
    // per-search scratch
    DevBuf<int64_t> s_qptr;
    DevBuf<uint32_t> s_qidx;
    DevBuf<float> s_qval, s_qsorted, s_qw;
    DevBuf<int32_t> s_qterm, s_qcnt;
    DevBuf<uint8_t> s_sort_tmp;

    bool bm25() const { return metric == KB2_METRIC_BM25; }
    int64_t count() const override { return n; }
    int64_t nnz() const { return (int64_t)h_indices.size(); }
    // device postings, term table and row sums, plus the host copy of the rows
    int64_t
    size_bytes() const override {
        return (int64_t)(terms.bytes() + term_off.bytes() + post_row.bytes() + post_val.bytes() + row_sum.bytes() +
                         h_indptr.size() * 8 + h_indices.size() * 4 + h_values.size() * 4);
    }
    bool is_trained() const override { return true; }
    bool has_raw() const override { return false; }

    // the dense entry points name the sparse ones
    void train(const float*, int64_t) override {
        throw Error(KB2_INVALID_ARGS, type + " holds sparse rows: build it with kb2_index_add_sparse (no training)");
    }
    void add(const float*, int64_t, const int64_t*) override {
        throw Error(KB2_INVALID_ARGS, type + " holds sparse rows: add them with kb2_index_add_sparse");
    }
    void search(const float*, int64_t, int, const JsonObj&, const uint8_t*, int64_t, int64_t*, float*) override {
        throw Error(KB2_INVALID_ARGS, type + " holds sparse rows: search it with kb2_index_search_sparse");
    }
    void
    refuse(Op op) const override {
        KB2_REQUIRE(op != kRangeSearch, KB2_INVALID_ARGS, type + " holds sparse rows: search it with kb2_index_range_search_sparse");
        KB2_REQUIRE(op != kShard, KB2_NOT_IMPLEMENTED, type + ": sharding is not implemented");
        KB2_REQUIRE(op != kEmbList, KB2_NOT_IMPLEMENTED, type + ": emb-lists are not implemented on sparse rows");
    }
    void
    to_faiss(FaissIndexData&) override {
        throw Error(KB2_NOT_IMPLEMENTED, type + ": the reference's sparse index has no faiss stream");
    }

    // the BM25 parameters of a build config: all three required for BM25 (sparse_index_node.cc:121-126), each in range
    static void
    check_bm25(float k1_, float b_, float avgdl_, int status) {
        KB2_REQUIRE(k1_ >= 0.f && k1_ <= 3.f, status, "bm25_k1 out of range [0, 3]");
        KB2_REQUIRE(b_ >= 0.f && b_ <= 1.f, status, "bm25_b out of range [0, 1]");
        KB2_REQUIRE(avgdl_ >= 0.f && avgdl_ <= FLT_MAX, status, "bm25_avgdl out of range [0, inf)");
    }
    void
    set_bm25(const JsonObj& cfg) {
        has_bm25 = cfg.has("bm25_k1") && cfg.has("bm25_b") && cfg.has("bm25_avgdl");
        KB2_REQUIRE(!bm25() || has_bm25, KB2_INVALID_ARGS, "BM25 needs bm25_k1, bm25_b and bm25_avgdl");
        k1 = (float)cfg.get_num("bm25_k1", 0.0);
        b = (float)cfg.get_num("bm25_b", 0.0);
        avgdl = (float)cfg.get_num("bm25_avgdl", 0.0);
        check_bm25(k1, b, avgdl, KB2_OUT_OF_RANGE_IN_JSON);
    }
    void
    configure(const JsonObj& cfg) override {
        set_bm25(cfg);
        std::string algo = cfg.get_str("inverted_index_algo", "");
        for (char& c : algo) c = (char)toupper((unsigned char)c);
        KB2_REQUIRE(algo.empty() || algo == "TAAT_NAIVE" || algo == "DAAT_WAND" || algo == "DAAT_MAXSCORE" ||
                        algo == "BLOCK_MAX_MAXSCORE" || algo == "BLOCK_MAX_WAND" || algo == "SINDI",
                    KB2_INVALID_ARGS,
                    "inverted_index_algo " + algo +
                        " not supported, supported: [TAAT_NAIVE DAAT_WAND DAAT_MAXSCORE BLOCK_MAX_MAXSCORE BLOCK_MAX_WAND SINDI]");
        const std::string qt = cfg.get_str("quant_type", "");
        if (!qt.empty()) {
            if (bm25())
                KB2_REQUIRE(qt == "u16" || qt == "u32", KB2_INVALID_ARGS, "quant_type for BM25 metric must be 'u16' or 'u32'");
            else
                KB2_REQUIRE(qt == "fp16" || qt == "fp32", KB2_INVALID_ARGS, "quant_type for IP metric must be 'fp16' or 'fp32'");
        }
    }
    void
    append_meta(std::string& s) const override {
        s += ", \"sparse_dim\": " + std::to_string(sparse_dim) + ", \"nnz\": " + std::to_string(nnz());
    }

    // ------------------------------------------------------------ input
    struct Csr {
        const int64_t* indptr;
        const uint32_t* indices;
        const float* values;
        int64_t n, nnz;
    };
    template <typename T>
    const T*
    staged(const T* src, size_t count, DevBuf<T>& buf) {
        if (count == 0 || is_device_ptr(src)) return src;
        buf.ensure(count);
        KB2_CUDA_CHECK(cudaMemcpyAsync(buf.p, src, count * sizeof(T), cudaMemcpyHostToDevice, stream));
        last.h2d += (int64_t)(count * sizeof(T));
        return buf.p;
    }
    // device view of a caller's CSR (each array host or device), checked before any kernel indexes by it
    Csr
    device_csr(const int64_t* ip, const uint32_t* ix, const float* val, int64_t rows, DevBuf<int64_t>& bp, DevBuf<uint32_t>& bi,
               DevBuf<float>& bv, const char* what) {
        KB2_REQUIRE(ip != nullptr && rows >= 0, KB2_INVALID_ARGS, std::string(what) + ": null indptr or negative row count");
        int64_t ends[2];
        if (is_device_ptr(ip)) {
            int64_t* h = (int64_t*)h_counter.p;
            KB2_CUDA_CHECK(cudaMemcpyAsync(h, ip, 8, cudaMemcpyDeviceToHost, stream));
            KB2_CUDA_CHECK(cudaMemcpyAsync(h + 1, ip + rows, 8, cudaMemcpyDeviceToHost, stream));
            KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
            ends[0] = h[0];
            ends[1] = h[1];
        } else {
            ends[0] = ip[0];
            ends[1] = ip[rows];
        }
        KB2_REQUIRE(ends[0] == 0 && ends[1] >= 0, KB2_INVALID_ARGS, std::string(what) + ": indptr must start at 0 and not decrease");
        Csr c{nullptr, nullptr, nullptr, rows, ends[1]};
        KB2_REQUIRE(c.nnz == 0 || (ix && val), KB2_INVALID_ARGS, std::string(what) + ": null indices or values");
        c.indptr = staged(ip, (size_t)rows + 1, bp);
        c.indices = staged(ix, (size_t)c.nnz, bi);
        c.values = staged(val, (size_t)c.nnz, bv);
        if (rows == 0) return c;
        KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p, 0, 8, stream));
        sparse::validate_csr_kernel<<<(unsigned)std::min<int64_t>((rows + 255) / 256, 8 * num_sms()), 256, 0, stream>>>(
            c.indptr, c.indices, c.values, rows, c.nnz, d_counter.p);
        KB2_CUDA_CHECK(cudaGetLastError());
        unsigned long long* h = (unsigned long long*)h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(h, d_counter.p, 8, cudaMemcpyDeviceToHost, stream));
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        KB2_REQUIRE(!(h[0] & sparse::kBadOffsets), KB2_INVALID_ARGS, std::string(what) + ": indptr must start at 0 and not decrease");
        KB2_REQUIRE(!(h[0] & sparse::kBadIndices), KB2_INVALID_ARGS,
                    std::string(what) + ": indices must be strictly ascending within a row");
        KB2_REQUIRE(!(h[0] & sparse::kBadValues), KB2_INVALID_ARGS, std::string(what) + ": values must be finite and >= 0");
        return c;
    }

    // ------------------------------------------------------------ build
    void
    add_rows(const int64_t* ip, const uint32_t* ix, const float* val, int64_t rows) {
        DevBuf<int64_t> bp;
        DevBuf<uint32_t> bi;
        DevBuf<float> bv;
        const Csr c = device_csr(ip, ix, val, rows, bp, bi, bv, "rows");
        KB2_REQUIRE(n + rows < (1ll << 31), KB2_INVALID_ARGS, "sparse index: at most 2^31 - 1 rows");
        if (rows == 0) return;
        const size_t p0 = h_indptr.size(), z0 = h_indices.size();
        const int64_t base = (int64_t)z0;
        h_indptr.resize(p0 + (size_t)rows);
        h_indices.resize(z0 + (size_t)c.nnz);
        h_values.resize(z0 + (size_t)c.nnz);
        // from the caller's arrays (host or device), now that they are checked
        KB2_CUDA_CHECK(cudaMemcpyAsync(h_indptr.data() + p0, ip + 1, (size_t)rows * 8, cudaMemcpyDefault, stream));
        if (c.nnz) {
            KB2_CUDA_CHECK(cudaMemcpyAsync(h_indices.data() + z0, ix, (size_t)c.nnz * 4, cudaMemcpyDefault, stream));
            KB2_CUDA_CHECK(cudaMemcpyAsync(h_values.data() + z0, val, (size_t)c.nnz * 4, cudaMemcpyDefault, stream));
        }
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (size_t i = p0; i < h_indptr.size(); i++) h_indptr[i] += base;
        n += rows;
        build_postings();
    }

    // the rows and everything built from them dropped (the BruteForce slot between calls)
    void
    clear_rows() {
        h_indptr.assign(1, 0);
        h_indices.clear();
        h_values.clear();
        h_indices.shrink_to_fit();
        h_values.shrink_to_fit();
        h_indptr.shrink_to_fit();
        n = nterms = sparse_dim = 0;
        term_off.release();
        terms.release();
        post_row.release();
        post_val.release();
        row_sum.release();
    }

    // term table, postings and row sums from all stored rows: a device sort of (term << 32 | row) keys with the values.
    // Every add re-sorts all rows, O(total nonzeros) per add.
    void
    build_postings() {
        const int64_t nnz = this->nnz();
        DevBuf<int64_t> d_indptr;
        DevBuf<uint32_t> d_indices;
        DevBuf<float> d_values;
        d_indptr.ensure((size_t)n + 1);
        d_indices.ensure((size_t)nnz);
        d_values.ensure((size_t)nnz);
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_indptr.p, h_indptr.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, stream));
        if (nnz) {
            KB2_CUDA_CHECK(cudaMemcpyAsync(d_indices.p, h_indices.data(), (size_t)nnz * 4, cudaMemcpyHostToDevice, stream));
            KB2_CUDA_CHECK(cudaMemcpyAsync(d_values.p, h_values.data(), (size_t)nnz * 4, cudaMemcpyHostToDevice, stream));
        }
        if (bm25()) {
            row_sum.alloc_exact((size_t)n);
        } else {
            row_sum.release();
        }
        DevBuf<uint64_t> keys, keys2;
        keys.ensure((size_t)nnz);
        keys2.ensure((size_t)nnz);
        sparse::build_keys_kernel<<<grid1d(n, 256), 256, 0, stream>>>(d_indptr.p, d_indices.p, d_values.p, n, keys.p,
                                                                       bm25() ? row_sum.p : nullptr);
        KB2_CUDA_CHECK(cudaGetLastError());
        nterms = 0;
        sparse_dim = 0;
        post_row.alloc_exact((size_t)nnz);
        post_val.alloc_exact((size_t)nnz);
        // the term table is written at the first entry of each term, so its scratch has one slot per nonzero; the index
        // keeps exact copies of nterms (+ 1) entries
        DevBuf<uint32_t> t_all;
        DevBuf<int64_t> off_all;
        t_all.ensure((size_t)nnz);
        off_all.ensure((size_t)nnz + 1);
        if (nnz > 0) {
            size_t bytes = 0;
            KB2_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys.p, keys2.p, d_values.p, post_val.p, nnz, 0, 64, stream));
            DevBuf<uint8_t> tmp;
            tmp.ensure(bytes);
            KB2_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, keys.p, keys2.p, d_values.p, post_val.p, nnz, 0, 64, stream));
            DevBuf<int64_t> flags, scan;
            flags.ensure((size_t)nnz);
            scan.ensure((size_t)nnz);
            sparse::split_postings_kernel<<<grid1d(nnz, 256), 256, 0, stream>>>(keys2.p, nnz, post_row.p, flags.p);
            size_t sbytes = 0;
            KB2_CUDA_CHECK(cub::DeviceScan::InclusiveSum(nullptr, sbytes, flags.p, scan.p, nnz, stream));
            DevBuf<uint8_t> stmp;
            stmp.ensure(sbytes);
            KB2_CUDA_CHECK(cub::DeviceScan::InclusiveSum(stmp.p, sbytes, flags.p, scan.p, nnz, stream));
            sparse::term_table_kernel<<<grid1d(nnz, 256), 256, 0, stream>>>(keys2.p, scan.p, nnz, t_all.p, off_all.p);
            KB2_CUDA_CHECK(cudaGetLastError());
            int64_t* h = (int64_t*)h_counter.p;
            KB2_CUDA_CHECK(cudaMemcpyAsync(h, scan.p + nnz - 1, 8, cudaMemcpyDeviceToHost, stream));
            KB2_CUDA_CHECK(cudaMemcpyAsync(h + 1, keys2.p + nnz - 1, 8, cudaMemcpyDeviceToHost, stream));
            KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
            nterms = h[0];
            sparse_dim = (int64_t)((uint64_t)h[1] >> 32) + 1;
        } else {
            KB2_CUDA_CHECK(cudaMemsetAsync(off_all.p, 0, 8, stream));
        }
        terms.alloc_exact((size_t)nterms);
        term_off.alloc_exact((size_t)nterms + 1);
        if (nterms) KB2_CUDA_CHECK(cudaMemcpyAsync(terms.p, t_all.p, (size_t)nterms * 4, cudaMemcpyDeviceToDevice, stream));
        KB2_CUDA_CHECK(cudaMemcpyAsync(term_off.p, off_all.p, ((size_t)nterms + 1) * 8, cudaMemcpyDeviceToDevice, stream));
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
    }

    // ------------------------------------------------------------ KB2I section: the BM25 keys and the rows
    void
    save(BlobWriter& w) override {
        w.put<int32_t>(has_bm25 ? 1 : 0);
        w.put<float>(k1);
        w.put<float>(b);
        w.put<float>(avgdl);
        w.put<int64_t>(n);
        w.put<int64_t>(nnz());
        if (n) w.put_bytes(h_indptr.data(), h_indptr.size() * 8);
        w.put_bytes(h_indices.data(), h_indices.size() * 4);
        w.put_bytes(h_values.data(), h_values.size() * 4);
    }
    void
    load(BlobReader& r) override {
        has_bm25 = r.get<int32_t>() != 0;
        k1 = r.get<float>();
        b = r.get<float>();
        avgdl = r.get<float>();
        KB2_REQUIRE(!bm25() || has_bm25, KB2_INVALID_BINARY_SET, "BM25 index without its parameters in blob");
        check_bm25(k1, b, avgdl, KB2_INVALID_BINARY_SET);
        const int64_t rows = r.get<int64_t>(), nnz = r.get<int64_t>();
        const uint64_t left = r.n - r.o;
        KB2_REQUIRE(rows >= 0 && nnz >= 0 && (uint64_t)rows <= left / 8 && (uint64_t)nnz <= left / 8, KB2_INVALID_BINARY_SET,
                    "bad sparse sizes in blob");
        std::vector<int64_t> hp(rows ? (size_t)rows + 1 : 0);
        std::vector<uint32_t> hi((size_t)nnz);
        std::vector<float> hv((size_t)nnz);
        // blob memory may be unaligned: copy out
        memcpy(hp.data(), r.get_bytes(hp.size() * 8), hp.size() * 8);
        memcpy(hi.data(), r.get_bytes(hi.size() * 4), hi.size() * 4);
        memcpy(hv.data(), r.get_bytes(hv.size() * 4), hv.size() * 4);
        KB2_REQUIRE(rows == 0 || hp[rows] == nnz, KB2_INVALID_BINARY_SET, "bad sparse offsets in blob");
        try {
            if (rows) add_rows(hp.data(), hi.data(), hv.data(), rows);
        } catch (const Error& e) {
            if (e.status != KB2_INVALID_ARGS) throw;
            throw Error(KB2_INVALID_BINARY_SET, std::string("bad sparse rows in blob: ") + e.what());
        }
    }

    // ------------------------------------------------------------ search
    // device query CSR -> s_qterm / s_qw / s_qcnt (kept terms in query order); returns the postings they hold
    int64_t
    prepare(const Csr& qc, float ratio, float p1) {
        KB2_REQUIRE(qc.nnz < (1ll << 31), KB2_INVALID_ARGS, "queries: at most 2^31 - 1 nonzeros per batch");
        const size_t nnzq = (size_t)std::max<int64_t>(qc.nnz, 1);
        s_qterm.ensure(nnzq);
        s_qw.ensure(nnzq);
        s_qcnt.ensure((size_t)qc.n);
        const float* sorted = nullptr;
        if (ratio > 0.f && qc.nnz > 0) {
            // each query's values in ascending order: a segmented sort, so no query length is capped
            s_qsorted.ensure(nnzq);
            size_t bytes = 0;
            KB2_CUDA_CHECK(cub::DeviceSegmentedSort::SortKeys(nullptr, bytes, qc.values, s_qsorted.p, (int)qc.nnz, (int)qc.n,
                                                              qc.indptr, qc.indptr + 1, stream));
            s_sort_tmp.ensure(bytes);
            KB2_CUDA_CHECK(cub::DeviceSegmentedSort::SortKeys(s_sort_tmp.p, bytes, qc.values, s_qsorted.p, (int)qc.nnz, (int)qc.n,
                                                              qc.indptr, qc.indptr + 1, stream));
            sorted = s_qsorted.p;
            last.launches++;
        }
        KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p + 1, 0, 8, stream));
        sparse::PrepParams pp{qc.indptr, qc.indices, qc.values, sorted, qc.n, ratio, terms.p, nterms, term_off.p, bm25() ? 1 : 0, p1,
                              s_qterm.p, s_qw.p, s_qcnt.p, d_counter.p + 1};
        sparse::prep_queries_kernel<<<grid1d(qc.n * 32, 256), 256, 0, stream>>>(pp);
        KB2_CUDA_CHECK(cudaGetLastError());
        last.launches++;
        int64_t* h = (int64_t*)h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(h, d_counter.p + 1, 8, cudaMemcpyDeviceToHost, stream));
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        return h[0];
    }

    // search keys: drop_ratio_search (index search only) and the BM25 parameters; fills the scoring parameters
    sparse::ScoreParams
    score_params(const Csr& qc, const JsonObj& cfg, bool brute_force, const uint8_t* dbits) {
        KB2_REQUIRE(!cfg.has("metric_type") || cfg.get_str("metric_type", "") == (bm25() ? "BM25" : "IP"), KB2_INVALID_METRIC_TYPE,
                    "search metric type must be same as built index");
        float ratio = 0.f;
        if (!brute_force) {
            const double r = cfg.get_num("drop_ratio_search", 0.0);
            KB2_REQUIRE(r >= 0.0 && r < 1.0, KB2_OUT_OF_RANGE_IN_JSON, "drop_ratio_search out of range [0, 1)");
            ratio = (float)r;
        }
        float p1 = 1.f, p2 = 0.f, p3 = 0.f;
        if (bm25()) {
            // sparse_index_node.cc:767-792: avgdl is a search key; k1 and b, if given, are the build values
            KB2_REQUIRE(cfg.has("bm25_avgdl"), KB2_INVALID_ARGS, "BM25 parameter avgdl must be set when searching");
            KB2_REQUIRE((!cfg.has("bm25_k1") || (float)cfg.get_num("bm25_k1", 0.0) == k1) &&
                            (!cfg.has("bm25_b") || (float)cfg.get_num("bm25_b", 0.0) == b),
                        KB2_INVALID_VALUE_IN_JSON, "BM25 parameters k1 and b in search config must be same as built index");
            const float avg = std::max((float)cfg.get_num("bm25_avgdl", 0.0), 1.f);
            p1 = k1 + 1.f;
            p2 = k1 * (1.f - b);
            p3 = (k1 * b) / avg;
        }
        const int64_t postings = prepare(qc, ratio, p1);
        last.pairs = postings;
        last.code_bytes = postings * 8;
        last.codes = qc.n * n;
        sparse::ScoreParams sp{};
        sp.term_off = term_off.p;
        sp.post_row = post_row.p;
        sp.post_val = post_val.p;
        sp.row_sum = row_sum.p;
        sp.n = n;
        sp.bm25 = bm25() ? 1 : 0;
        sp.p2 = p2;
        sp.p3 = p3;
        sp.bitset = dbits;
        sp.q_off = qc.indptr;
        sp.q_cnt = s_qcnt.p;
        sp.q_term = s_qterm.p;
        sp.q_w = s_qw.p;
        return sp;
    }

    // top-k of nq prepared queries (device CSR) into d_ids / d_dist [nq][k]
    void
    knn(const Csr& qc, int k, const JsonObj& cfg, bool brute_force, const uint8_t* dbits, int64_t* d_ids, float* d_dist) {
        const int64_t nq = qc.n;
        sparse::ScoreParams sp = score_params(qc, cfg, brute_force, dbits);
        const int64_t ntiles = (n + sparse::kTile - 1) / sparse::kTile;
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev0, stream));
        FinalizeParams fp{};
        fp.k_out = k;
        fp.metric = KB2_METRIC_IP;   // key = -s: the distance written is s, padding -FLT_MAX
        fp.out_ids = d_ids;
        fp.out_dist = d_dist;
        if (k + 16 <= kMaxK) {
            // each tile's best Ksel into a partial slot; full slot rows are reduced to one slot, as dense_candidates does
            const int Ksel = next_pow2(std::max(32, k + 16));
            const int S = (int)std::min<int64_t>(std::max(2, kMaxSortEntries / Ksel), ntiles);
            const int64_t stride = (int64_t)S * Ksel;
            s_partial.ensure((size_t)nq * stride);
            sp.partial = s_partial.p;
            sp.partial_stride = stride;
            sp.ksel = Ksel;
            int used = 0;
            for (int64_t t0 = 0; t0 < ntiles;) {
                if (used == S) {
                    const int n_in = used * Ksel;
                    launch<reduce_partials_kernel>((unsigned)nq, 256, (size_t)next_pow2(n_in) * 8, stream, s_partial.p, (int)stride, n_in,
                                                   next_pow2(n_in), Ksel);
                    last.launches++;
                    used = 1;
                }
                const int64_t tiles = std::min<int64_t>(ntiles - t0, S - used);
                sp.slot0 = used;
                sp.tile0 = t0;
                launch<sparse::score_tile_kernel<sparse::kTopK>>(dim3((unsigned)nq, (unsigned)tiles), sparse::kThreads,
                                                                 sparse::kScoreSmem, stream, sp);
                KB2_CUDA_CHECK(cudaGetLastError());
                last.launches++;
                used += (int)tiles;
                t0 += tiles;
            }
            fp.partial = s_partial.p;
            fp.partial_stride = stride;
            fp.n_partial = used * Ksel;
            fp.k_sel = k;
            launch_finalize(*this, fp, nq);
            last_engine = 5;
        } else {
            // k + 16 > 1024: dense key chunks, the running best set of select_rows_kernel and the large-k finalize (as FLAT)
            const int K = k;
            const int64_t g = large_k_group(nq, (int64_t)K * 32 + large_k_row_bytes(K));
            const int64_t max_key_elems = 64ll << 20;
            const int64_t chunk_tiles = std::max<int64_t>(1, std::min<int64_t>(std::min(ntiles, sparse::kMaxGridY),
                                                                                  max_key_elems / g / sparse::kTile));
            const int64_t ldk = chunk_tiles * sparse::kTile;
            s_keys.ensure((size_t)g * ldk);
            s_lk_rows.ensure((size_t)g * 4 * K);
            sp.keys = s_keys.p;
            sp.ldk = ldk;
            fp.k_sel = K;
            for (int64_t q0 = 0; q0 < nq; q0 += g) {
                const int64_t rows = std::min(g, nq - q0);
                uint64_t* A = s_lk_rows.p;
                uint64_t* B = A + (size_t)g * 2 * K;
                sp.q0 = q0;
                for (int64_t t0 = 0; t0 < ntiles; t0 += chunk_tiles) {
                    const int64_t tiles = std::min(chunk_tiles, ntiles - t0);
                    const int64_t col0 = t0 * sparse::kTile;
                    const int64_t cols = std::min(tiles * sparse::kTile, n - col0);
                    sp.tile0 = t0;
                    sp.col0 = col0;
                    launch<sparse::score_tile_kernel<sparse::kKeys>>(dim3((unsigned)rows, (unsigned)tiles), sparse::kThreads,
                                                                     sparse::kScoreSmem, stream, sp);
                    KB2_CUDA_CHECK(cudaGetLastError());
                    last.launches++;
                    if (t0 == 0) {
                        large_k_select<float>(*this, s_keys.p, ldk, cols, 0u, K, A, 2 * K, rows);
                    } else {
                        large_k_select<float>(*this, s_keys.p, ldk, cols, (uint32_t)col0, K, A + K, 2 * K, rows);
                        large_k_select<uint64_t>(*this, A, 2 * K, 2 * K, 0u, K, B, 2 * K, rows);
                        std::swap(A, B);
                    }
                }
                large_k_finalize(*this, fp, A, 2 * K, K, rows, q0);
            }
            last_engine = 2;
        }
        if (timing) {
            KB2_CUDA_CHECK(cudaEventRecord(ev1, stream));
            KB2_CUDA_CHECK(cudaEventSynchronize(ev1));
            KB2_CUDA_CHECK(cudaEventElapsedTime(&last_stage_ms, ev0, ev1));
            last_kernel_ms = last_stage_ms;
        }
    }

    // kb2_index_search_sparse / kb2_bruteforce_search_sparse
    void
    search_sparse(const int64_t* ip, const uint32_t* ix, const float* val, int64_t nq, int k, const JsonObj& cfg, const uint8_t* bitset,
                  int64_t nbits, int64_t* out_ids, float* out_dist, bool brute_force) {
        KB2_REQUIRE(k > 0 && k <= kMaxLargeK, KB2_INVALID_ARGS, "k out of range (1..16384)");
        KB2_REQUIRE(nq >= 0, KB2_INVALID_ARGS, "bad nq");
        KB2_REQUIRE(n > 0, KB2_EMPTY_INDEX, "index is empty");
        if (nq == 0) return;
        KB2_REQUIRE(out_ids && out_dist, KB2_INVALID_ARGS, "null buffer");
        KB2_REQUIRE(is_device_ptr(out_ids) == is_device_ptr(out_dist), KB2_INVALID_ARGS,
                    "out_ids and out_dist must both be host or both be device buffers");
        const Csr qc = device_csr(ip, ix, val, nq, s_qptr, s_qidx, s_qval, "queries");
        const uint8_t* dbits = bitset_to_device(bitset, nbits);
        int64_t* d_ids;
        float* d_dist;
        device_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        knn(qc, k, cfg, brute_force, dbits, d_ids, d_dist);
        results_out(nq, k, out_ids, out_dist, d_ids, d_dist);
    }

    // kb2_index_range_search_sparse: hits radius < s <= range_filter (one-sided without the filter), best first, ties by row
    void
    range_search_sparse(const int64_t* ip, const uint32_t* ix, const float* val, int64_t nq, float radius, float range_filter,
                        bool has_filter, const JsonObj& cfg, const uint8_t* bitset, int64_t nbits, int64_t** out_lims,
                        int64_t** out_ids, float** out_dist) {
        KB2_REQUIRE(n > 0, KB2_EMPTY_INDEX, "index is empty");
        KB2_REQUIRE(nq >= 0, KB2_INVALID_ARGS, "bad nq");
        const Csr qc = device_csr(ip, ix, val, nq, s_qptr, s_qidx, s_qval, "queries");
        const uint8_t* dbits = bitset_to_device(bitset, nbits);
        std::vector<int64_t> lims((size_t)nq + 1, 0);
        std::vector<uint32_t> hkey;
        std::vector<int32_t> hrow;
        last_engine = 5;
        last_stage_ms = last_kernel_ms = 0.f;
        if (nq > 0) {
            sparse::ScoreParams sp = score_params(qc, cfg, false, dbits);
            if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev0, stream));
            sp.radius = radius;
            sp.range_filter = range_filter;
            sp.has_filter = has_filter ? 1 : 0;
            const int64_t ntiles = (n + sparse::kTile - 1) / sparse::kTile;
            KB2_REQUIRE(ntiles <= sparse::kMaxGridY, KB2_INVALID_ARGS, "range search: too many rows");
            sp.ntiles = ntiles;
            DevBuf<int32_t> counts;
            counts.ensure((size_t)nq * ntiles);
            sp.counts = counts.p;
            launch<sparse::score_tile_kernel<sparse::kCount>>(dim3((unsigned)nq, (unsigned)ntiles), sparse::kThreads, sparse::kScoreSmem,
                                                              stream, sp);
            KB2_CUDA_CHECK(cudaGetLastError());
            std::vector<int32_t> hc((size_t)nq * ntiles);
            KB2_CUDA_CHECK(cudaMemcpyAsync(hc.data(), counts.p, hc.size() * 4, cudaMemcpyDeviceToHost, stream));
            KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
            std::vector<int64_t> off(hc.size());
            int64_t total = 0;
            for (int64_t q = 0; q < nq; q++) {
                for (int64_t t = 0; t < ntiles; t++) {
                    off[q * ntiles + t] = total;
                    total += hc[q * ntiles + t];
                }
                lims[q + 1] = total;
            }
            KB2_REQUIRE(total < (1ll << 31), KB2_INVALID_ARGS, "range search: more than 2^31 - 1 hits");
            if (total > 0) {
                DevBuf<int64_t> d_off, d_lims;
                DevBuf<uint32_t> key, key2;
                DevBuf<int32_t> row, row2;
                d_off.ensure(off.size());
                d_lims.ensure(lims.size());
                key.ensure((size_t)total);
                key2.ensure((size_t)total);
                row.ensure((size_t)total);
                row2.ensure((size_t)total);
                KB2_CUDA_CHECK(cudaMemcpyAsync(d_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice, stream));
                KB2_CUDA_CHECK(cudaMemcpyAsync(d_lims.p, lims.data(), lims.size() * 8, cudaMemcpyHostToDevice, stream));
                sp.hit_off = d_off.p;
                sp.hit_key = key.p;
                sp.hit_row = row.p;
                launch<sparse::score_tile_kernel<sparse::kEmit>>(dim3((unsigned)nq, (unsigned)ntiles), sparse::kThreads,
                                                                 sparse::kScoreSmem, stream, sp);
                KB2_CUDA_CHECK(cudaGetLastError());
                // hits arrive in row order per query; a stable sort by key gives (s descending, row ascending)
                size_t bytes = 0;
                KB2_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, bytes, key.p, key2.p, row.p, row2.p, (int)total, (int)nq,
                                                                        d_lims.p, d_lims.p + 1, 0, 32, stream));
                DevBuf<uint8_t> tmp;
                tmp.ensure(bytes);
                KB2_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortPairs(tmp.p, bytes, key.p, key2.p, row.p, row2.p, (int)total, (int)nq,
                                                                        d_lims.p, d_lims.p + 1, 0, 32, stream));
                hkey.resize((size_t)total);
                hrow.resize((size_t)total);
                KB2_CUDA_CHECK(cudaMemcpyAsync(hkey.data(), key2.p, (size_t)total * 4, cudaMemcpyDeviceToHost, stream));
                KB2_CUDA_CHECK(cudaMemcpyAsync(hrow.data(), row2.p, (size_t)total * 4, cudaMemcpyDeviceToHost, stream));
                KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
                last.d2h += total * 8;
            }
            last.launches += 4;
            if (timing) {
                KB2_CUDA_CHECK(cudaEventRecord(ev1, stream));
                KB2_CUDA_CHECK(cudaEventSynchronize(ev1));
                KB2_CUDA_CHECK(cudaEventElapsedTime(&last_stage_ms, ev0, ev1));
                last_kernel_ms = last_stage_ms;
            }
        }
        const size_t total = (size_t)lims[nq];
        int64_t* L = (int64_t*)malloc(lims.size() * 8);
        int64_t* I = (int64_t*)malloc(std::max<size_t>(total, 1) * 8);
        float* D = (float*)malloc(std::max<size_t>(total, 1) * 4);
        if (!L || !I || !D) {
            free(L);
            free(I);
            free(D);
            throw Error(KB2_MALLOC_ERROR, "malloc failed");
        }
        memcpy(L, lims.data(), lims.size() * 8);
        for (size_t i = 0; i < total; i++) {
            I[i] = hrow[i];
            D[i] = -ord2f(hkey[i]);
        }
        *out_lims = L;
        *out_ids = I;
        *out_dist = D;
    }
};

}  // namespace kb2
