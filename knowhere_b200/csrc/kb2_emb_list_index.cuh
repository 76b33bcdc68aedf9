// kb2_emb_list_index.cuh — emb-list (multi-vector) search on an HNSW or IVF_FLAT index with the MAX_SIM metrics, with the
// reference's TokenANN strategy (src/index/emb_list/emb_list_strategy_token_ann.cc:51-175, emb_list_strategy.cc:45-117,
// index_node.cc:275-324,453-507) or, on an index created with "emb_list_strategy": "muvera" (MuveraIndex, kb2_muvera.cuh),
// its MUVERA strategy (emb_list_strategy_muvera.cc:159-324).  DESIGN §4.11.
//
// The index holds every row of every document; the document offsets are attached afterwards (set_emb_list), and
// doc_of_row maps each row to its document on the device.  One driver, search_emb_list, runs both strategies over chunks
// of whole query lists; they differ only in how a chunk's lists find their candidate documents (stages 1 and 2):
//   TokenANN (token_ann_candidates)
//     1. stage 1: the handle's own search() of every query token with k = vec_topk = min(max(int(k * ratio), 1), rows);
//        HNSW checks ef >= k against the list-level k and searches with max(ef, vec_topk).  With a bitset,
//        row_bits_kernel first expands the document bitset into a row bitset, so the base search, its kAlpha and its
//        brute-force thresholds all see row counts, as the reference does;
//     2. cand_keys_kernel maps each stage-1 id to (list << 32) | document, one radix sort and one unique pass compact
//        them, and cand_off_kernel finds each list's run: a CSR of distinct documents per list, ascending.
//   MUVERA (muvera_candidates)
//     1. muvera_encode sums each list's raw tokens into its FDE row, and the base index (HNSW or IVF_FLAT over the
//        documents' FDE rows) returns ann_k = min(max(int(k * ratio), 1), n_docs) documents per list, the document
//        bitset applied directly;
//     2. muvera_cand_kernel keeps the ids that are documents with rows, as a CSR per list (none for an empty list).
// Then, for both:
//   3. re-rank: msim::rerank (kb2_maxsim.cuh), the BruteForce re-rank, packs each list's candidates into work items and
//      computes their exact MaxSim keys with msim::maxsim_rerank_kernel, over the query rows normalised under COSINE;
//   4. select: a segmented radix sort orders each list's (key, document) entries and el_emit_kernel writes the k best,
//      padded with id -1 and -FLT_MAX (larger is better) or FLT_MAX (MAX_SIM_L2), as emb_list_strategy.cc:111-114.
// Ties in the score are ordered by ascending document id (the reference's order follows unordered_set iteration).  With
// emb_list_rerank false, MUVERA takes ann_k = min(k, n_docs) and muvera_pass_kernel returns the base's ids and distances
// instead of stages 2-4, padded with -1 and -inf (IP, COSINE) or +inf (L2) (emb_list_strategy_muvera.cc:236-259).
// Largest E each base serves (E = R * 2^P * d, kMaxDynSmem = 227 KB of shared memory per CTA; DESIGN §4.11):
//   HNSW search      four-warp kernel while 4 * (4 E + 8 max(ef, k)) bytes fit (E <= 14336 at max(ef, k) <= 96), else one
//                    query per CTA while 4 E + 8 max(ef, k) + 42 M + 32 bytes fit (E <= 57 700 at ef 128, M 30);
//   HNSW build       the host build (under 20 000 documents) any E; the device build's link kernel holds 4 rows of
//                    8 E bytes beside 3456 bytes of slots: E <= 7156;
//   IVF_FLAT search  the query-major scan keeps the query (4 E bytes) beside its selection buffers (E <= 57 000 at
//                    k <= 32) and the finalize beside up to 8192 candidates: E <= 41 700; the list-major engine streams
//                    E in 32-column stages, and its split queries take 8 E bytes per (query, probe).
#pragma once
#include <cub/cub.cuh>

#include "kb2_hnsw.cuh"
#include "kb2_maxsim.cuh"
#include "kb2_muvera.cuh"

namespace kb2 {

constexpr uint32_t kEmbListTag = 0x54534c45;         // "ELST": emb-list section of a "KB2I" blob (kb2_range.cuh)
constexpr uint32_t kEmbListMuveraTag = 0x564d4c45;   // "ELMV": the same section of a MUVERA index
// 36 bytes of stage-1 and candidate scratch per (token, vec_topk) entry: at most this many entries per chunk of lists
constexpr int64_t kEmbListChunkEntries = 8ll << 20;
// MUVERA: at most this many floats of encoded query lists per chunk (64 MB; at least one list)
constexpr int64_t kMuveraChunkFloats = 16ll << 20;

struct EmbListState {
    int metric = KB2_METRIC_MAX_SIM_L2;   // KB2_METRIC_MAX_SIM_*
    std::vector<int64_t> lims;            // [n_docs + 1] document offsets (host)
    DevBuf<int64_t> d_lims;
    DevBuf<int32_t> doc_of_row;
    // per-search scratch (grow-only)
    DevBuf<float> q, s1_dist;
    DevBuf<int64_t> qlims, s1_ids, cand_cnt, cand_off;
    DevBuf<int32_t> row_list;
    DevBuf<uint64_t> keys, keys_sorted, cand, cand_key, cand_sorted;
    msim::RerankScratch rr;
    DevBuf<uint8_t> doc_bits, row_bits, tmp;
    DevBuf<unsigned long long> counters;   // [0] candidate pairs, [1] token x row distances, [2] unique count
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    float stage_ms[4] = {0.f, 0.f, 0.f, 0.f};   // last search: stage 1, candidates, re-rank, select (with timing on)
    int64_t n_docs() const { return (int64_t)lims.size() - 1; }
    ~EmbListState() {
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
};

__global__ void
doc_of_row_kernel(const int64_t* lims, int64_t n_docs, int32_t* doc_of_row) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_docs) return;
    for (int64_t r = lims[j]; r < lims[j + 1]; r++) doc_of_row[r] = (int32_t)j;
}

// byte b of the row bitset: bit i set when the document of row 8b + i is filtered out
__global__ void
row_bits_kernel(const uint8_t* doc_bits, const int32_t* doc_of_row, int64_t n, uint8_t* row_bits) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b * 8 >= n) return;
    uint32_t v = 0;
    for (int i = 0; i < 8 && b * 8 + i < n; i++)
        if (bit_is_set(doc_bits, doc_of_row[b * 8 + i])) v |= 1u << i;
    row_bits[b] = (uint8_t)v;
}

// entry e = (token, slot) of the stage-1 result -> (list of the token - l0) << 32 | document; kEmpty for id -1
__global__ void
cand_keys_kernel(const int64_t* ids, int64_t n, int vec_topk, const int32_t* row_list, int64_t r0, int64_t l0,
                 const int32_t* doc_of_row, uint64_t* keys) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int64_t id = ids[e];
    keys[e] = id < 0 ? kEmpty
                     : ((uint64_t)(row_list[r0 + e / vec_topk] - l0) << 32) | (uint64_t)(uint32_t)doc_of_row[id];
}

// off[l] = first of the nu sorted distinct keys with list >= l (the kEmpty sentinel sorts after every list)
__global__ void
cand_off_kernel(const uint64_t* ukeys, const unsigned long long* nu, int64_t nlists, int64_t* off) {
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l > nlists) return;
    const uint64_t key = (uint64_t)l << 32;
    int64_t lo = 0, hi = (int64_t)*nu;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (ukeys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    off[l] = lo;
}

template <int METRIC>
__global__ void
el_emit_kernel(const uint64_t* sorted, const int64_t* off, int64_t nlists, int k, int64_t l0, int64_t* out_ids,
               float* out_dist) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nlists * k) return;
    const int64_t l = e / k, r = e % k;
    const int64_t o = (l0 + l) * k + r;
    if (r < off[l + 1] - off[l]) {
        const uint64_t v = sorted[off[l] + r];
        const float key = unpack_key(v);
        out_ids[o] = (int64_t)unpack_pos(v);
        out_dist[o] = (METRIC == KB2_METRIC_L2) ? key : -key;
    } else {
        out_ids[o] = -1;
        out_dist[o] = (METRIC == KB2_METRIC_L2) ? FLT_MAX : -FLT_MAX;
    }
}

// MUVERA: list l's candidates are its stage-1 ids (ann_k per list, -1 past the base's hits) that are documents with rows,
// in stage-1 order; an empty query list has none.  Pass 1 (cand null) counts them into cnt[l], pass 2 writes them at off[l].
__global__ void
muvera_cand_kernel(const int64_t* ids, int64_t L, int ann_k, const int64_t* qlims, int64_t l0, const int64_t* xlims,
                   int64_t* cnt, const int64_t* off, uint64_t* cand) {
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L) return;
    int64_t c = 0;
    if (qlims[l0 + l + 1] > qlims[l0 + l])
        for (int j = 0; j < ann_k; j++) {
            const int64_t id = ids[l * ann_k + j];
            if (id < 0 || xlims[id + 1] == xlims[id]) continue;
            if (cand) cand[off[l] + c] = (uint64_t)id;
            c++;
        }
    if (!cand) cnt[l] = c;
}

// MUVERA without re-rank: the base's ann_k results of each list, padded to k with -1 and +inf (L2) or -inf
template <int METRIC>
__global__ void
muvera_pass_kernel(const int64_t* ids, const float* dist, int64_t L, int ann_k, int k, int64_t l0, int64_t* out_ids,
                   float* out_dist) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= L * k) return;
    const int64_t l = e / k, r = e % k, o = (l0 + l) * k + r;
    out_ids[o] = r < ann_k ? ids[l * ann_k + r] : -1;
    out_dist[o] = r < ann_k ? dist[l * ann_k + r] : (METRIC == KB2_METRIC_L2 ? INFINITY : -INFINITY);
}

// metric of the base index that an emb-list metric pairs with (MAX_SIM_L2 - L2, MAX_SIM_IP - IP, MAX_SIM_COSINE - COSINE)
inline bool
emb_list_metric_pairs(const IndexBase& ix, int metric) {
    if (metric == KB2_METRIC_MAX_SIM_L2) return ix.metric == KB2_METRIC_L2;
    if (metric == KB2_METRIC_MAX_SIM_IP) return ix.metric == KB2_METRIC_IP && !ix.cosine;
    if (metric == KB2_METRIC_MAX_SIM_COSINE) return ix.cosine;
    return false;
}

// Attach validated host offsets (lims.back() == ix.count()) to an HNSW or IVF_FLAT index.  A MUVERA index encodes its
// documents and builds its base here, or takes `muvera_base` (deserialisation).
inline void
set_emb_list(IndexBase& ix, std::vector<int64_t> lims, int metric, std::unique_ptr<IndexBase> muvera_base = nullptr) {
    KB2_REQUIRE(ix.takes_emb_list(), KB2_INVALID_METRIC_TYPE, "emb-lists are supported on HNSW and IVF_FLAT only");
    KB2_REQUIRE(metric == KB2_METRIC_MAX_SIM_L2 || metric == KB2_METRIC_MAX_SIM_IP || metric == KB2_METRIC_MAX_SIM_COSINE,
                KB2_INVALID_METRIC_TYPE, "metric must be MAX_SIM_L2, MAX_SIM_IP or MAX_SIM_COSINE");
    KB2_REQUIRE(emb_list_metric_pairs(ix, metric), KB2_INVALID_METRIC_TYPE,
                "the emb-list metric does not match the index metric (MAX_SIM_L2: L2, MAX_SIM_IP: IP, MAX_SIM_COSINE: COSINE)");
    KB2_REQUIRE(ix.shard_world == 1, KB2_NOT_IMPLEMENTED, "emb-lists on a sharded index");
    KB2_REQUIRE(!ix.labels.custom, KB2_NOT_IMPLEMENTED, "emb-lists with custom ids");
    const int64_t n = ix.count();
    KB2_REQUIRE(lims.size() >= 2 && lims.back() == n, KB2_INVALID_ARGS, "document offsets must end at the index's row count");
    KB2_REQUIRE(n > 0 && n < (1ll << 31) && (int64_t)lims.size() - 1 < (1ll << 31), KB2_INVALID_ARGS,
                "emb-list sizes out of range (rows 1 .. 2^31 - 1)");
    ix.emb_list_rows();   // the rows the re-rank reads exist from the attach on (IVF: its lists are sealed here)
    auto el = std::make_shared<EmbListState>();
    el->metric = metric;
    el->lims = std::move(lims);
    const int64_t nd = el->n_docs();
    el->d_lims.ensure(nd + 1);
    el->doc_of_row.ensure(n);
    KB2_CUDA_CHECK(cudaMemcpyAsync(el->d_lims.p, el->lims.data(), (nd + 1) * 8, cudaMemcpyHostToDevice, ix.stream));
    doc_of_row_kernel<<<grid1d(nd, 256), 256, 0, ix.stream>>>(el->d_lims.p, nd, el->doc_of_row.p);
    KB2_CUDA_CHECK(cudaGetLastError());
    for (cudaEvent_t& e : el->ev) KB2_CUDA_CHECK(cudaEventCreate(&e));
    el->counters.ensure(4);
    if (auto* mv = dynamic_cast<MuveraIndex*>(&ix)) mv->attach(nd, el->d_lims.p, std::move(muvera_base));
    KB2_CUDA_CHECK(cudaStreamSynchronize(ix.stream));
    ix.emb_list = std::move(el);
}

// emb_list_strategy_token_ann.cc:87-88, emb_list_strategy_muvera.cc:186-190: int32(k * ratio) in fp32, at least 1, at
// most n
inline int
emb_list_ann_k(int k, const JsonObj& cfg, int64_t n) {
    const float ratio = (float)cfg.get_num("retrieval_ann_ratio", 3.0);
    KB2_REQUIRE(ratio > 0.f, KB2_EMB_LIST_INNER_ERROR, "retrieval_ann_ratio could not be less than or equal to 0");
    const float prod = (float)k * ratio;
    const int64_t want = prod >= 2147483648.f ? (int64_t)INT32_MAX : (int64_t)(int32_t)prod;
    return (int)std::min<int64_t>(std::max<int64_t>(want, 1), n);
}

// TokenANN candidates of lists [l0, l0 + L), whose query rows are rows [r0, r0 + nt) of qn (normalised under COSINE):
// stage 1 of every token on the handle itself with k = vec_topk (rbits: the row bitset), ev[1], then the distinct
// (list, document) pairs of its hits as a CSR in el.cand / el.cand_off.  False for a chunk without tokens: no candidates.
inline bool
token_ann_candidates(IndexBase& ix, EmbListState& el, const float* qn, int64_t l0, int64_t L, int64_t r0, int64_t nt,
                     int vec_topk, const JsonObj& cfg, const uint8_t* rbits) {
    cudaStream_t st = ix.stream;
    const int64_t ne = nt * vec_topk;
    KB2_REQUIRE(ne < (1ll << 31), KB2_INVALID_ARGS, "emb-list search: one query list's tokens x vec_topk exceed 2^31 - 1");
    el.cand_off.ensure(L + 1);
    if (nt == 0) {
        KB2_CUDA_CHECK(cudaMemsetAsync(el.cand_off.p, 0, (L + 1) * 8, st));
        if (ix.timing) KB2_CUDA_CHECK(cudaEventRecord(el.ev[1], st));
        return false;
    }
    el.s1_ids.ensure(ne);
    el.s1_dist.ensure(ne);
    ix.search(qn + r0 * ix.dim, nt, vec_topk, cfg, rbits, rbits ? ix.count() : 0, el.s1_ids.p, el.s1_dist.p);
    if (ix.timing) KB2_CUDA_CHECK(cudaEventRecord(el.ev[1], st));
    el.keys.ensure(ne);
    el.keys_sorted.ensure(ne);
    el.cand.ensure(ne);
    cand_keys_kernel<<<grid1d(ne, 256), 256, 0, st>>>(el.s1_ids.p, ne, vec_topk, el.row_list.p, r0, l0, el.doc_of_row.p,
                                                      el.keys.p);
    // list bits up to the first that no list of the chunk sets: kEmpty (all ones) still sorts last
    int end_bit = 33;
    while ((1ll << (end_bit - 32)) <= L) end_bit++;
    size_t b1 = 0, b2 = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, b1, el.keys.p, el.keys_sorted.p, (int)ne, 0, end_bit, st);
    cub::DeviceSelect::Unique(nullptr, b2, el.keys_sorted.p, el.cand.p, el.counters.p + 2, (int)ne, st);
    el.tmp.ensure(std::max(b1, b2));
    b1 = el.tmp.n;
    KB2_CUDA_CHECK(cub::DeviceRadixSort::SortKeys(el.tmp.p, b1, el.keys.p, el.keys_sorted.p, (int)ne, 0, end_bit, st));
    b2 = el.tmp.n;
    KB2_CUDA_CHECK(cub::DeviceSelect::Unique(el.tmp.p, b2, el.keys_sorted.p, el.cand.p, el.counters.p + 2, (int)ne, st));
    cand_off_kernel<<<grid1d(L + 1, 256), 256, 0, st>>>(el.cand.p, el.counters.p + 2, L, el.cand_off.p);
    ix.last.launches += 7;
    return true;
}

// MUVERA candidates of lists [l0, l0 + L), whose query rows are rows [r0, r0 + nt) of q (raw): their encodings, the
// base's ann_k documents for each into el.s1_* (dbits: the document bitset), ev[1], then with re-rank each list's
// documents with rows as a CSR in el.cand / el.cand_off.  True with re-rank: the chunk has candidates to re-rank.
inline bool
muvera_candidates(MuveraIndex& mv, EmbListState& el, const float* q, int64_t l0, int64_t L, int64_t r0, int64_t nt, int ann_k,
                  const JsonObj& cfg, const uint8_t* dbits, bool rerank) {
    cudaStream_t st = mv.stream;
    IndexBase& base = mv.base_index();
    mv.fde.ensure((size_t)L * mv.E());
    muvera_encode(mv.mp, mv.dim, mv.proj.p, nt > 0 ? q + r0 * mv.dim : nullptr, nt, el.qlims.p, l0, L, false, mv.bucket, mv.fde.p,
                  st);
    el.s1_ids.ensure((size_t)L * ann_k);
    el.s1_dist.ensure((size_t)L * ann_k);
    base.search(base.cosine ? base.normalized(mv.fde.p, L) : mv.fde.p, L, ann_k, cfg, dbits, dbits ? el.n_docs() : 0, el.s1_ids.p,
                el.s1_dist.p);
    mv.last.launches += 2;
    if (mv.timing) KB2_CUDA_CHECK(cudaEventRecord(el.ev[1], st));
    if (!rerank) return false;
    el.cand_off.ensure(L + 1);
    el.cand_cnt.ensure(L + 1);
    KB2_CUDA_CHECK(cudaMemsetAsync(el.cand_cnt.p + L, 0, 8, st));
    muvera_cand_kernel<<<grid1d(L, 128), 128, 0, st>>>(el.s1_ids.p, L, ann_k, el.qlims.p, l0, el.d_lims.p, el.cand_cnt.p, nullptr,
                                                       nullptr);
    size_t b1 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b1, el.cand_cnt.p, el.cand_off.p, (int)(L + 1), st);
    el.tmp.ensure(b1);
    b1 = el.tmp.n;
    KB2_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(el.tmp.p, b1, el.cand_cnt.p, el.cand_off.p, (int)(L + 1), st));
    el.cand.ensure((size_t)L * ann_k);
    muvera_cand_kernel<<<grid1d(L, 128), 128, 0, st>>>(el.s1_ids.p, L, ann_k, el.qlims.p, l0, el.d_lims.p, nullptr, el.cand_off.p,
                                                       el.cand.p);
    KB2_CUDA_CHECK(cudaGetLastError());
    mv.last.launches += 8;
    return true;
}

// The search of either strategy (see the top of the file).  queries: host or device rows, ql: validated host offsets of
// the query lists; out_*: [lists][k], host or device.  stats: query lists, (list, document) candidates re-ranked,
// token x row distances computed.
inline void
search_emb_list(IndexBase& ix, const float* queries, const std::vector<int64_t>& ql, int k, const JsonObj& cfg,
                const uint8_t* bitset, int64_t nbits, int64_t* out_ids, float* out_dist, int64_t stats[3]) {
    auto* mv = dynamic_cast<MuveraIndex*>(&ix);
    EmbListState& el = *ix.emb_list;
    cudaStream_t st = ix.stream;
    const int64_t n = ix.count(), n_docs = el.n_docs(), n_lists = (int64_t)ql.size() - 1, nq_rows = ql.back();
    const int d = ix.dim;
    // doc_of_row and the offsets were built for the rows the index held when they were attached
    KB2_REQUIRE(el.lims.back() == n, KB2_EMB_LIST_INNER_ERROR, "the index's rows no longer match its emb-list offsets");
    // stage 1 takes ann_k rows per token (TokenANN) or documents per list (MUVERA, which without re-rank returns them)
    const bool rerank = !mv || cfg.get_bool("emb_list_rerank", true);
    const int ann_k = rerank ? emb_list_ann_k(k, cfg, mv ? n_docs : n) : (int)std::min<int64_t>(k, n_docs);
    JsonObj bcfg = cfg;
    (mv ? mv->base_index() : ix).emb_list_base_config(bcfg, k, ann_k);
    for (float& v : el.stage_ms) v = 0.f;
    if (n_lists == 0) return;

    // query rows on the device and, under COSINE, their normalised copy qn: TokenANN's stage 1 and every re-rank read
    // qn, MUVERA encodes the raw rows; list offsets, and TokenANN's list of every row
    const float *q = nullptr, *qn = nullptr;
    if (nq_rows > 0) {
        el.q.ensure((size_t)nq_rows * d);
        KB2_CUDA_CHECK(cudaMemcpyAsync(el.q.p, queries, (size_t)nq_rows * d * 4, cudaMemcpyDefault, st));
        q = el.q.p;
        qn = ix.cosine ? ix.normalized(q, nq_rows) : q;
        // h2d counts the host query rows of TokenANN under COSINE only (the accounting the search has always reported)
        if (!mv && ix.cosine && !is_device_ptr(queries)) ix.last.h2d += nq_rows * d * 4;
    }
    el.qlims.ensure(ql.size());
    KB2_CUDA_CHECK(cudaMemcpyAsync(el.qlims.p, ql.data(), ql.size() * 8, cudaMemcpyHostToDevice, st));
    const std::vector<int32_t> row_list = mv ? std::vector<int32_t>() : msim::upload_row_list(ql, el.row_list, st);

    // the document bitset: MUVERA's base searches documents; TokenANN's stage 1 takes it as a row bitset
    const uint8_t* bits = msim::doc_bits_to_device(bitset, nbits, n_docs, el.doc_bits, st);
    if (bits && !mv) {
        el.row_bits.ensure((size_t)((n + 7) / 8));
        row_bits_kernel<<<grid1d((n + 7) / 8, 256), 256, 0, st>>>(bits, el.doc_of_row.p, n, el.row_bits.p);
        KB2_CUDA_CHECK(cudaGetLastError());
        bits = el.row_bits.p;
    }

    int64_t* d_ids;
    float* d_dist;
    ix.device_out(n_lists, k, out_ids, out_dist, d_ids, d_dist);
    const auto [X, pos] = ix.emb_list_rows();
    const bool vec4 = (d & 3) == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0;
    KB2_CUDA_CHECK(cudaMemsetAsync(el.counters.p, 0, 2 * sizeof(unsigned long long), st));
    // lists [l0, l1) fit one chunk: TokenANN's stage-1 entries, MUVERA's encodings and stage-1 entries within the budgets
    auto fits = [&](int64_t l0, int64_t l1) {
        if (!mv) return (ql[l1] - ql[l0]) * ann_k <= kEmbListChunkEntries;
        return (l1 - l0) * mv->E() <= kMuveraChunkFloats && (l1 - l0) * ann_k <= kEmbListChunkEntries;
    };
    auto mark = [&](int from, int to) {   // the stage boundaries ev[from .. to) at this point of the stream
        for (int i = from; i < to; i++)
            if (ix.timing) KB2_CUDA_CHECK(cudaEventRecord(el.ev[i], st));
    };

    for (int64_t l0 = 0, l1; l0 < n_lists; l0 = l1) {
        // whole lists (at least one)
        l1 = l0 + 1;
        while (l1 < n_lists && fits(l0, l1 + 1)) l1++;
        const int64_t L = l1 - l0, r0 = ql[l0], nt = ql[l1] - r0;
        mark(0, 1);
        // 1. stage 1 and 2. each list's candidate documents
        const bool scored = mv ? muvera_candidates(*mv, el, q, l0, L, r0, nt, ann_k, bcfg, bits, rerank)
                               : token_ann_candidates(ix, el, qn, l0, L, r0, nt, ann_k, bcfg, bits);
        if (!rerank) {
            with_metric(ix.metric, [&](auto m) {
                muvera_pass_kernel<decltype(m)::value><<<grid1d(L * k, 256), 256, 0, st>>>(el.s1_ids.p, el.s1_dist.p, L, ann_k, k, l0,
                                                                                         d_ids, d_dist);
            });
            KB2_CUDA_CHECK(cudaGetLastError());
            mark(2, 4);
        } else {
            int64_t nu = 0;
            if (scored) {
                // 3. exact keys of every candidate (the plan ends the candidates stage and adds to counters[0..1])
                const msim::RerankParams rp{qn, el.qlims.p, X, pos, el.d_lims.p, d, l0, nullptr, el.cand.p, nullptr};
                nu = msim::rerank(ix, ix.metric, vec4, rp, el.cand_off.p, nullptr, L, el.cand_key, el.rr, el.counters.p,
                                  ix.timing ? el.ev[2] : nullptr);
                mark(3, 4);
            } else {
                mark(2, 4);
            }
            // 4. each list's candidates in (key, document) order, the k best
            el.cand_sorted.ensure(std::max<int64_t>(nu, 1));
            if (nu > 0) {
                size_t b4 = 0;
                cub::DeviceSegmentedRadixSort::SortKeys(nullptr, b4, el.cand_key.p, el.cand_sorted.p, (int)nu, (int)L, el.cand_off.p,
                                                        el.cand_off.p + 1, 0, 64, st);
                el.tmp.ensure(b4);
                b4 = el.tmp.n;
                KB2_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortKeys(el.tmp.p, b4, el.cand_key.p, el.cand_sorted.p, (int)nu, (int)L,
                                                                       el.cand_off.p, el.cand_off.p + 1, 0, 64, st));
            }
            with_metric(ix.metric, [&](auto m) {
                el_emit_kernel<decltype(m)::value><<<grid1d(L * k, 256), 256, 0, st>>>(el.cand_sorted.p, el.cand_off.p, L, k, l0, d_ids,
                                                                                      d_dist);
            });
            KB2_CUDA_CHECK(cudaGetLastError());
        }
        mark(4, 5);
        if (ix.timing) {
            KB2_CUDA_CHECK(cudaEventSynchronize(el.ev[4]));
            for (int i = 0; i < 4; i++) {
                float ms = 0.f;
                KB2_CUDA_CHECK(cudaEventElapsedTime(&ms, el.ev[i], el.ev[i + 1]));
                el.stage_ms[i] += ms;
            }
        }
    }
    unsigned long long* hc = (unsigned long long*)ix.h_counter.p + 12;
    KB2_CUDA_CHECK(cudaMemcpyAsync(hc, el.counters.p, 16, cudaMemcpyDeviceToHost, st));
    ix.results_out(n_lists, k, out_ids, out_dist, d_ids, d_dist);
    stats[0] = n_lists;
    stats[1] = (int64_t)hc[0];
    stats[2] = (int64_t)hc[1];
}

}  // namespace kb2
