// kb2_maxsim.cuh — BruteForce search over emb-lists (multi-vector rows) with the MAX_SIM metrics (DESIGN §4.10).
//
//   score(Q, D) = sum over q in Q of ( max over x in D of <q, x> )        MAX_SIM_IP, MAX_SIM / MAX_SIM_COSINE (unit rows)
//   score(Q, D) = sum over q in Q of ( min over x in D of |q - x|^2 )     MAX_SIM_L2 (smaller is better)
//
// Reference: src/common/comp/brute_force.cc:424-584 (one thread per query list builds the |Q| x |D| distance block of every
// document, then get_sum_max_sim), include/knowhere/emb_list_utils.h:28-107,154-176.
//
// Internally every score is a key, smaller is better: the sum over the query tokens of min over x of (-<q, x>) for IP,
// of |q - x|^2 for L2.  Three stages per chunk of query lists:
//   1. maxsim_filter_kernel: persistent, sm_90a.  The 3xTF32 wgmma contraction of gemm_keys_tc_kernel with query tokens on
//      M and base tokens on N; its epilogue takes each query token's extremum over every document of the base tile and sums
//      them over the tokens of each query list.  It writes one approximate key per (query list, document) to S, never the
//      token-by-token distances.
//   2. select_rows_kernel keeps the K = k + 16 best of each S row; rerank() recomputes their keys in fp32 on the CUDA
//      cores in a fixed order (maxsim_rerank_kernel); a segmented radix sort orders them by (key, document);
//      maxsim_emit_kernel writes the k best and certifies the list against the filter's error bound (maxsim_bound).
//   3. Lists that could not be certified are redone with exact keys for every document (rerank() with every unfiltered
//      document as a candidate), selected and emitted again.  dim % 4 != 0 (no TMA) takes that exact all-documents path
//      for every list.
// The index-level emb-list search (kb2_emb_list_index.cuh) re-ranks its gathered candidates through the same rerank().
#pragma once
#include "kb2_index.cuh"

namespace kb2 {
namespace msim {

constexpr int BM = tc::BM;        // query tokens per block: two consumer warpgroups of 64 rows
constexpr int BN = tc::BN;        // base rows per tile
constexpr int MAXD = 32;          // documents per work item
constexpr int STAGES = 3;
constexpr size_t SMEM_BYTES = (size_t)STAGES * tc::STAGE_BYTES + (size_t)MAXD * BM * 4 + 2 * MAXD * 4 + 2 * STAGES * 8 + 1024;

// A work item: base rows [row0, row0 + 128 * ntiles) holding the whole documents [doc0, doc0 + ndocs).  Either several
// documents in one tile, or one document longer than a tile over ntiles consecutive tiles.
struct Item {
    int32_t row0, ntiles, doc0, ndocs;
};

struct FilterParams {
    const Item* items;
    int nitems;
    const int64_t* xlims;      // [n_docs + 1] base list offsets
    const int64_t* qlims;      // [n_lists + 1] query list offsets
    const int32_t* row_list;   // [query rows] list of each query row
    const float* qn;           // |q|^2 per query row (L2)
    const float* xn;           // |x|^2 per base row (L2)
    int64_t r0, r1;            // query rows of the chunk (whole lists)
    int64_t l0;                // first list of the chunk: S row 0
    int d;
    const uint8_t* bitset;     // bit i: document i filtered out (its S entry stays +inf)
    float* S;                  // [lists of the chunk][lds] approximate keys
    int64_t lds;
};

// grid = persistent (min(#SMs, items)), block = tc::THREADS (two consumer warpgroups + the TMA producer warp), dynamic
// smem SMEM_BYTES.  Each CTA walks the items blockIdx.x, + gridDim.x, ...; for each item it walks the query blocks of the
// chunk in order, and for each block the item's tiles.  A tile's TMA box and the query box stay resident in L2 across the
// blocks, so the base is read from HBM once per chunk.  Per tile, thread rows keep their extremum over the columns of each
// document (one quad of lanes holds an accumulator row: a pass over the thread's columns and two shuffles), folded into
// R[doc][row] across the tiles of a long document.  After the last tile the tokens of each query list are summed over the
// rows in order; a list that continues into the next block carries its partial sums in `carry` (double-buffered by block
// parity).  Every S entry is written once, by one thread: the result does not depend on scheduling.
template <int METRIC>
__global__ void __launch_bounds__(tc::THREADS, 1)
maxsim_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                     const FilterParams p) {
    using namespace tc;
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t raw = smem_u32(smem_dyn);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* base_ptr = smem_dyn + (base - raw);
    float* R = reinterpret_cast<float*>(base_ptr + STAGES * STAGE_BYTES);   // [MAXD][BM]
    float* carry = R + MAXD * BM;                                           // [2][MAXD]
    const uint32_t bars = base + STAGES * STAGE_BYTES + (uint32_t)(MAXD * BM + 2 * MAXD) * 4u;
    auto bar_full = [&](int s) { return bars + 8u * s; };
    auto bar_empty = [&](int s) { return bars + 8u * (STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nkb = (p.d + BK - 1) / BK;
    const int64_t nqb = (p.r1 - p.r0 + BM - 1) / BM;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) {
            mbar_init(bar_full(s), 1);
            mbar_init(bar_empty(s), CONS_THREADS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            uint32_t it = 0;
            for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
                const Item w = p.items[item];
                for (int64_t qb = 0; qb < nqb; qb++)
                    for (int t = 0; t < w.ntiles; t++)
                        for (int kb = 0; kb < nkb; kb++, it++) {
                            const int s = (int)(it % STAGES);
                            const uint32_t ph = (it / STAGES) & 1u;
                            mbar_wait(bar_empty(s), ph ^ 1u);
                            const uint32_t st = base + (uint32_t)s * STAGE_BYTES;
                            mbar_expect_tx(bar_full(s), 2 * TILE_BYTES);
                            tma_load_2d(st, &tmap_q, kb * BK, (int)(p.r0 + qb * BM), bar_full(s));
                            tma_load_2d(st + TILE_BYTES, &tmap_x, kb * BK, w.row0 + t * BN, bar_full(s));
                        }
            }
        }
        return;
    }
    const int t = threadIdx.x;   // 0..255
    const int wg = t >> 7;
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // block rows of this thread: rl (acc i = 0) and rl + 8 (i = 1)
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0.f;
    uint32_t it = 0;
    for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
        const Item w = p.items[item];
        for (int64_t qb = 0; qb < nqb; qb++) {
            const int64_t b0 = p.r0 + qb * BM;
            float qq0 = 0.f, qq1 = 0.f;
            if (METRIC == KB2_METRIC_L2) {
                if (b0 + rl < p.r1) qq0 = p.qn[b0 + rl];
                if (b0 + rl + 8 < p.r1) qq1 = p.qn[b0 + rl + 8];
            }
            for (int tile = 0; tile < w.ntiles; tile++) {
                for (int kb = 0; kb < nkb; kb++, it++) {
                    const int s = (int)(it % STAGES);
                    const uint32_t ph = (it / STAGES) & 1u;
                    mbar_wait(bar_full(s), ph);
                    float4* hi = reinterpret_cast<float4*>(base_ptr + (size_t)s * STAGE_BYTES);
                    float4* lo = reinterpret_cast<float4*>(base_ptr + (size_t)s * STAGE_BYTES + 2 * TILE_BYTES);
#pragma unroll 4
                    for (int i = t; i < 2 * TILE_BYTES / 16; i += CONS_THREADS) {
                        float4 v = hi[i];
                        float4 h, l;
                        h.x = tf32_rn(v.x); l.x = tf32_rn(v.x - h.x);
                        h.y = tf32_rn(v.y); l.y = tf32_rn(v.y - h.y);
                        h.z = tf32_rn(v.z); l.z = tf32_rn(v.z - h.z);
                        h.w = tf32_rn(v.w); l.w = tf32_rn(v.w - h.w);
                        hi[i] = h;
                        lo[i] = l;
                    }
                    fence_proxy_async();
                    asm volatile("bar.sync 1, 256;" ::: "memory");
                    const uint32_t st = base + (uint32_t)s * STAGE_BYTES;
                    const uint32_t a_off = (uint32_t)wg * 64u * 128u;
                    fence_operand(acc);
                    wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < BK / 8; kk++) {
                        const uint32_t ko = (uint32_t)kk * 32u;
                        const uint64_t a_hi = make_desc(st + a_off + ko);
                        const uint64_t b_hi = make_desc(st + TILE_BYTES + ko);
                        const uint64_t a_lo = make_desc(st + 2 * TILE_BYTES + a_off + ko);
                        const uint64_t b_lo = make_desc(st + 3 * TILE_BYTES + ko);
                        wgmma_tf32_n128(acc, a_hi, b_hi, (kb > 0 || kk > 0) ? 1u : 0u);
                        wgmma_tf32_n128(acc, a_hi, b_lo, 1u);
                        wgmma_tf32_n128(acc, a_lo, b_hi, 1u);
                    }
                    wgmma_commit();
                    fence_operand(acc);
                    // the previous stage's wgmmas have retired once at most one group is pending: release its slot
                    wgmma_wait<1>();
                    if (kb > 0) mbar_arrive(bar_empty((int)((it - 1) % STAGES)));
                }
                wgmma_wait<0>();
                fence_operand(acc);
                mbar_arrive(bar_empty((int)((it - 1) % STAGES)));
                // ---- epilogue of the tile: per document, each row's extremum over the document's columns in this tile
                const int64_t trow0 = (int64_t)w.row0 + (int64_t)tile * BN;
                for (int dd = 0; dd < w.ndocs; dd++) {
                    const int64_t lo_c = p.xlims[w.doc0 + dd] - trow0, hi_c = p.xlims[w.doc0 + dd + 1] - trow0;
                    const int a = lo_c > 0 ? (int)lo_c : 0, b = hi_c < BN ? (int)hi_c : BN;
                    float m0 = INFINITY, m1 = INFINITY;
                    if (a < b) {
#pragma unroll
                        for (int j = 0; j < BN / 8; j++) {
#pragma unroll
                            for (int c = 0; c < 2; c++) {
                                const int col = j * 8 + 2 * (lane & 3) + c;
                                if (col >= a && col < b) {
                                    float k0, k1;
                                    if (METRIC == KB2_METRIC_L2) {
                                        const float xx = __ldg(p.xn + trow0 + col);
                                        k0 = qq0 + xx - 2.f * acc[4 * j + c];
                                        k1 = qq1 + xx - 2.f * acc[4 * j + 2 + c];
                                    } else {
                                        k0 = -acc[4 * j + c];
                                        k1 = -acc[4 * j + 2 + c];
                                    }
                                    m0 = fminf(m0, k0);
                                    m1 = fminf(m1, k1);
                                }
                            }
                        }
                    }
                    m0 = fminf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
                    m0 = fminf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
                    m1 = fminf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
                    m1 = fminf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
                    if ((lane & 3) == 0) {
                        float* Rd = R + dd * BM;
                        if (tile == 0) {
                            Rd[rl] = m0;
                            Rd[rl + 8] = m1;
                        } else {
                            Rd[rl] = fminf(Rd[rl], m0);
                            Rd[rl + 8] = fminf(Rd[rl + 8], m1);
                        }
                    }
                }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");   // R complete for this block
            // ---- sum over the tokens of each query list (segments of the block's rows), in row order
            const int cur = (int)(qb & 1);
            for (int task = t; task < BM * w.ndocs; task += CONS_THREADS) {
                const int dd = task / BM, r = task % BM;
                const int64_t g = b0 + r;
                if (g >= p.r1) continue;
                const int lst = p.row_list[g];
                if (r > 0 && p.row_list[g - 1] == lst) continue;   // not the first row of its segment
                const int64_t lbeg = p.qlims[lst], lend = p.qlims[lst + 1];
                float sum = (r == 0 && lbeg < b0) ? carry[(cur ^ 1) * MAXD + dd] : 0.f;
                const int rend = lend - b0 < BM ? (int)(lend - b0) : BM;
                for (int rr = r; rr < rend; rr++) sum += R[dd * BM + rr];
                if (lend > b0 + BM) {
                    carry[cur * MAXD + dd] = sum;
                } else {
                    const int64_t doc = (int64_t)w.doc0 + dd;
                    if (!(p.bitset && bit_is_set(p.bitset, doc))) p.S[(lst - p.l0) * p.lds + doc] = sum;
                }
            }
            // the next R / carry writes come after the first bar.sync of the next tile's contraction
        }
    }
}

// Error bound of the filter's key of list Q against any document, from its tokens' norms and M^2 = max |x|^2 over the
// base (DESIGN §4.10):  E = sum_t rel(d) a_t + |Q| 2^-22 sum_t a_t,  a_t = |q_t| M (IP, COSINE) or |q_t|^2 + M^2 (L2).
// rel(d) = fin_cert_rel(d) bounds one approximate distance against its exact value as for FLAT (kb2_topk.cuh); the
// extremum over a document is then off by at most the same, and the second term covers the fp32 sums over the tokens
// (filter and re-rank both: each extremum is at most 2 a_t in magnitude).
__device__ __forceinline__ float
maxsim_bound(float sum_a, int64_t ntok, int d) {
    return fin_cert_rel(d) * sum_a + (float)ntok * 0x1p-22f * sum_a;
}

// Row b of a chunk (list qlist[b], or l0 + b): the k best of its K sorted (exact key, document) entries, padded with -1 and
// the reference's values (brute_force.cc:566-581: FLT_MIN when larger is better, FLT_MAX for L2).  With `approx` (the
// filter's selection of the row), the list is certified: when the filter kept K entries, its k-th exact key must beat the
// largest approximate key kept by more than the bound, or the list is appended to cert[2..] (count in cert[1]) for the
// exact all-documents redo.  grid = rows, block 256.
struct EmitParams {
    const uint64_t* sorted;   // [rows][K]
    const uint64_t* approx;   // [rows][K] or nullptr
    int K, k;
    const float* Q;
    const int64_t* qlims;
    int d;
    uint32_t* cert;           // [0] max |x|^2 (float bits), [1] count, [2..] lists to redo
    int64_t l0;
    const uint32_t* qlist;
    int64_t* out_ids;
    float* out_dist;
};

template <int METRIC>
__global__ void __launch_bounds__(256)
maxsim_emit_kernel(const EmitParams p) {
    __shared__ uint32_t s_cnt, s_max;
    __shared__ float s_a[8];
    const int64_t b = blockIdx.x;
    const int64_t lst = p.qlist ? (int64_t)p.qlist[b] : p.l0 + b;
    const uint64_t* row = p.sorted + b * p.K;
    for (int r = threadIdx.x; r < p.k; r += blockDim.x) {
        const uint64_t e = row[r];
        const int64_t o = lst * p.k + r;
        if (e == kEmpty) {
            p.out_ids[o] = -1;
            p.out_dist[o] = (METRIC == KB2_METRIC_L2) ? FLT_MAX : FLT_MIN;
        } else {
            const float key = unpack_key(e);
            p.out_ids[o] = (int64_t)unpack_pos(e);
            p.out_dist[o] = (METRIC == KB2_METRIC_L2) ? key : -key;
        }
    }
    if (!p.approx) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { s_cnt = 0; s_max = 0; }
    __syncthreads();
    uint32_t cnt = 0, mx = 0;
    for (int j = threadIdx.x; j < p.K; j += blockDim.x) {
        const uint64_t e = p.approx[b * p.K + j];
        if (e != kEmpty) { cnt++; mx = max(mx, (uint32_t)(e >> 32)); }
    }
    atomicAdd(&s_cnt, cnt);
    atomicMax(&s_max, mx);
    const float M2 = __uint_as_float(p.cert[0]);
    const int64_t qa = p.qlims[lst], qe = p.qlims[lst + 1];
    float a = 0.f;
    for (int64_t tq = qa + warp; tq < qe; tq += 8) {
        float s = 0.f;
        for (int i = lane; i < p.d; i += kWarp) s = fmaf(p.Q[tq * p.d + i], p.Q[tq * p.d + i], s);
        s = warp_sum(s);
        a += (METRIC == KB2_METRIC_L2) ? s + M2 : sqrtf(s * M2);
    }
    if (lane == 0) s_a[warp] = a;
    __syncthreads();
    if (threadIdx.x != 0 || s_cnt < (uint32_t)p.K) return;   // fewer than K documents scored: nothing was cut
    float sum_a = 0.f;
    for (int w = 0; w < 8; w++) sum_a += s_a[w];
    const float E = maxsim_bound(sum_a * 1.0001f, qe - qa, p.d);
    const float kth = unpack_key(row[p.k - 1]);
    const float last = ord2f(s_max);
    if (kth <= last - E) return;
    p.cert[2 + atomicAdd(p.cert + 1, 1u)] = (uint32_t)lst;
}

// Work items from the base offsets: consecutive documents packed greedily into one 128-row tile (at most MAXD of them),
// and each document longer than a tile alone over consecutive tiles.  Empty documents are never scored.
inline std::vector<Item>
plan_items(const std::vector<int64_t>& xl) {
    std::vector<Item> items;
    const int64_t n_docs = (int64_t)xl.size() - 1;
    bool open = false;
    Item cur{};
    int64_t used = 0;
    auto close = [&] {
        if (open) items.push_back(cur);
        open = false;
    };
    for (int64_t j = 0; j < n_docs; j++) {
        const int64_t len = xl[j + 1] - xl[j];
        if (len > BN) {
            close();
            items.push_back(Item{(int32_t)xl[j], (int32_t)((len + BN - 1) / BN), (int32_t)j, 1});
            continue;
        }
        if (open && (used + len > BN || cur.ndocs == MAXD)) close();
        if (!open) {
            if (len == 0) continue;
            cur = Item{(int32_t)xl[j], 1, (int32_t)j, 0};
            used = 0;
            open = true;
        }
        cur.ndocs++;
        used += len;
    }
    close();
    return items;
}

// ---------------------------------------------------------------------------------------------------------------------
// Exact re-rank of (query list, document) candidates: the BruteForce candidates and all-documents rows (search() below)
// and the index-level emb-list search (kb2_emb_list_index.cuh; DESIGN §4.10, §4.11).
//
// A work item is one query list and a run of its candidate documents: up to RR_MAXD whole documents of at most RR_TR
// rows in all, or one longer document alone.  One CTA per item.  The list's tokens are taken RR_TQ at a time; for each
// token block the item's rows are taken RR_TR at a time, and the (token x row) block is contracted like an SGEMM over
// RR_DK-dimension stages (cp.async 16-byte copies into a double-buffered shared tile when rows are float4-aligned).
// Each thread owns a 4 x 4 (token x row) register tile and runs every one of its distances as one fmaf chain over
// dimensions 0..d-1 in order (get_sum_max_sim's order); the per-(token, document) extremum is order-free (fminf over the
// same values), and after each token block one thread per document adds the block's extrema to its running sum in token
// order.  A score therefore does not depend on how the candidates are packed into items.  Rows are read in place
// (BruteForce, HNSW) or at pos[row] (IVF_FLAT's list-order store).
constexpr int RR_TQ = 32;
constexpr int RR_TR = 128;
constexpr int RR_DK = 32;
constexpr int RR_LD = RR_DK + 4;   // row stride of the stage tiles: a warp's 8 tokens / 4 rows fall on distinct banks
constexpr int RR_MAXD = 32;
constexpr int RR_THREADS = 256;
constexpr size_t RR_SMEM = (size_t)(2 * (RR_TQ + RR_TR) * RR_LD + RR_TQ * RR_TR + RR_TQ * RR_MAXD + RR_MAXD) * 4 +
                           (size_t)(2 * RR_TR + RR_MAXD + 1) * 4;

struct RerankItem {
    int32_t list;    // query list, relative to RerankParams::l0
    int32_t c0;      // first candidate (index into cand)
    int32_t ndocs;   // candidates cand[c0 .. c0 + ndocs)
    int32_t nrows;   // their rows in all
};

struct RerankParams {
    const float* Q;             // query rows
    const int64_t* qlims;       // [lists + 1]
    const float* X;             // stored rows
    const int32_t* pos;         // row -> position in X, or nullptr (row r at X + r * d)
    const int64_t* xlims;       // [n_docs + 1]
    int d;
    int64_t l0;
    const RerankItem* items;
    const uint64_t* cand;       // low 32 bits: document
    uint64_t* out;              // [candidates] pack_kp(exact key, document)
};

__device__ __forceinline__ void
cp_async16(void* smem, const void* gmem, int src_bytes) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(src_bytes) : "memory");
}

template <int METRIC, bool VEC4>
__global__ void __launch_bounds__(RR_THREADS)
maxsim_rerank_kernel(const RerankParams p) {
    extern __shared__ __align__(16) unsigned char rr_smem[];
    float* sQ = reinterpret_cast<float*>(rr_smem);   // [2][RR_TQ][RR_LD]
    float* sX = sQ + 2 * RR_TQ * RR_LD;               // [2][RR_TR][RR_LD]
    float* sK = sX + 2 * RR_TR * RR_LD;               // [RR_TQ][RR_TR] keys of the current (token block, row tile)
    float* sE = sK + RR_TQ * RR_TR;                   // [RR_TQ][RR_MAXD] extremum per (token, document)
    float* sT = sE + RR_TQ * RR_MAXD;                 // [RR_MAXD] running token sums
    int32_t* sRow = reinterpret_cast<int32_t*>(sT + RR_MAXD);   // [RR_TR] position of each tile row in X, -1 past the end
    int32_t* sSlot = sRow + RR_TR;                               // [RR_TR] document slot of each tile row
    int32_t* sBeg = sSlot + RR_TR;                               // [RR_MAXD + 1] first item row of each document

    const RerankItem it = p.items[blockIdx.x];
    const int64_t lst = p.l0 + it.list;
    const int64_t qa = p.qlims[lst], qe = p.qlims[lst + 1];
    const int d = p.d;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int tg = lane & 7, rg = warp * 4 + (lane >> 3);   // this thread: tokens tg + 8i, rows rg + 32j (i, j < 4)
    if (t == 0) {
        int acc = 0;
        for (int s = 0; s < it.ndocs; s++) {
            sBeg[s] = acc;
            const int64_t doc = (int64_t)(uint32_t)p.cand[it.c0 + s];
            acc += (int)(p.xlims[doc + 1] - p.xlims[doc]);
        }
        sBeg[it.ndocs] = acc;
    }
    if (t < it.ndocs) sT[t] = 0.f;
    __syncthreads();

    const int ntiles = (it.nrows + RR_TR - 1) / RR_TR;
    const int nkc = (d + RR_DK - 1) / RR_DK;
    for (int64_t t0 = qa; t0 < qe; t0 += RR_TQ) {
        const int nt = qe - t0 < RR_TQ ? (int)(qe - t0) : RR_TQ;
        for (int tile = 0; tile < ntiles; tile++) {
            const int r0 = tile * RR_TR;
            if (t < RR_TR) {
                const int r = r0 + t;
                int32_t ps = -1, slot = 0;
                if (r < it.nrows) {
                    while (sBeg[slot + 1] <= r) slot++;
                    const int64_t doc = (int64_t)(uint32_t)p.cand[it.c0 + slot];
                    const int64_t row = p.xlims[doc] + (r - sBeg[slot]);
                    ps = p.pos ? p.pos[row] : (int32_t)row;
                }
                sRow[t] = ps;
                sSlot[t] = slot;
            }
            __syncthreads();
            // stage kc of dimensions [kc * RR_DK, +RR_DK) into buffer b; zero past d, past the list and past the item
            auto load = [&](int kc, int b) {
                float* q = sQ + b * RR_TQ * RR_LD;
                float* x = sX + b * RR_TR * RR_LD;
                const int k0 = kc * RR_DK;
                if (VEC4) {
                    {
                        const int tok = t >> 3, c = (t & 7) * 4;
                        const bool ok = tok < nt && k0 + c < d;
                        cp_async16(q + tok * RR_LD + c, ok ? p.Q + (t0 + tok) * d + k0 + c : p.Q, ok ? 16 : 0);
                    }
#pragma unroll
                    for (int i = 0; i < RR_TR * RR_DK / 4 / RR_THREADS; i++) {
                        const int e = t + i * RR_THREADS;
                        const int r = e >> 3, c = (e & 7) * 4;
                        const int32_t ps = sRow[r];
                        const bool ok = ps >= 0 && k0 + c < d;
                        cp_async16(x + r * RR_LD + c, ok ? p.X + (int64_t)ps * d + k0 + c : p.X, ok ? 16 : 0);
                    }
                    asm volatile("cp.async.commit_group;" ::: "memory");
                } else {
                    for (int e = t; e < RR_TQ * RR_DK; e += RR_THREADS) {
                        const int tok = e / RR_DK, c = e % RR_DK;
                        q[tok * RR_LD + c] = (tok < nt && k0 + c < d) ? p.Q[(t0 + tok) * d + k0 + c] : 0.f;
                    }
                    for (int e = t; e < RR_TR * RR_DK; e += RR_THREADS) {
                        const int r = e / RR_DK, c = e % RR_DK;
                        const int32_t ps = sRow[r];
                        x[r * RR_LD + c] = (ps >= 0 && k0 + c < d) ? p.X[(int64_t)ps * d + k0 + c] : 0.f;
                    }
                }
            };
            float acc[4][4];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
            load(0, 0);
            for (int kc = 0; kc < nkc; kc++) {
                if (kc + 1 < nkc) {
                    load(kc + 1, (kc + 1) & 1);
                    if (VEC4) asm volatile("cp.async.wait_group 1;" ::: "memory");
                } else if (VEC4) {
                    asm volatile("cp.async.wait_group 0;" ::: "memory");
                }
                __syncthreads();
                const float* q = sQ + (kc & 1) * RR_TQ * RR_LD;
                const float* x = sX + (kc & 1) * RR_TR * RR_LD;
                // zero-padded dimensions past d leave every chain unchanged: fmaf(0, 0, acc) == acc (acc is never -0)
#pragma unroll 8
                for (int kk = 0; kk < RR_DK; kk++) {
                    float qv[4], xv[4];
#pragma unroll
                    for (int i = 0; i < 4; i++) qv[i] = q[(tg + 8 * i) * RR_LD + kk];
#pragma unroll
                    for (int j = 0; j < 4; j++) xv[j] = x[(rg + 32 * j) * RR_LD + kk];
#pragma unroll
                    for (int i = 0; i < 4; i++)
#pragma unroll
                        for (int j = 0; j < 4; j++) {
                            if (METRIC == KB2_METRIC_L2) {
                                const float df = qv[i] - xv[j];
                                acc[i][j] = fmaf(df, df, acc[i][j]);
                            } else {
                                acc[i][j] = fmaf(qv[i], xv[j], acc[i][j]);
                            }
                        }
                }
                __syncthreads();
            }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++)
                    sK[(tg + 8 * i) * RR_TR + rg + 32 * j] = (METRIC == KB2_METRIC_L2) ? acc[i][j] : -acc[i][j];
            __syncthreads();
            // extremum of each (token, document) over the document's rows in this tile, folded over the tiles
            for (int task = t; task < RR_TQ * it.ndocs; task += RR_THREADS) {
                const int s = task / RR_TQ, tok = task % RR_TQ;
                if (tok >= nt) continue;
                const int a = max(sBeg[s], r0) - r0, b = min(sBeg[s + 1], r0 + RR_TR) - r0;
                if (a >= b) continue;
                float m = INFINITY;
                for (int r = a; r < b; r++) m = fminf(m, sK[tok * RR_TR + r]);
                float* e = sE + tok * RR_MAXD + s;
                *e = sBeg[s] >= r0 ? m : fminf(*e, m);
            }
            __syncthreads();
        }
        // sum of the block's extrema, in token order, onto each document's running sum
        if (t < it.ndocs) {
            float tot = sT[t];
            for (int tok = 0; tok < nt; tok++) tot += sE[tok * RR_MAXD + t];
            sT[t] = tot;
        }
        __syncthreads();
    }
    // an empty query list or document scores +inf, which no selection keeps
    if (t < it.ndocs)
        p.out[it.c0 + t] = pack_kp(qe > qa && sBeg[t + 1] > sBeg[t] ? sT[t] : INFINITY, (uint32_t)p.cand[it.c0 + t]);
}

template <int METRIC>
inline void
launch_rerank(bool vec4, unsigned nitems, cudaStream_t st, const RerankParams& rp) {
    if (vec4) launch<maxsim_rerank_kernel<METRIC, true>>(nitems, RR_THREADS, RR_SMEM, st, rp);
    else launch<maxsim_rerank_kernel<METRIC, false>>(nitems, RR_THREADS, RR_SMEM, st, rp);
}

// Items of the candidates of each list.  Row b's candidates are cand[cand_off[b] .. cand_off[b + 1]): documents in the
// low 32 bits, then possibly kEmpty padding, which is skipped (select_rows_kernel's rows).  Its query list is qlist[b],
// or l0 + b.  One thread per row packs the documents greedily: consecutive documents while they hold at most RR_TR rows and RR_MAXD documents, a longer document
// alone.  Pass 1 (items == nullptr) counts each row's items into cnt[b] and, with stats, adds the row's (candidate,
// |Q| x |D|) totals to stats[0..1]; pass 2 writes them at off[b].
__global__ void
rerank_plan_kernel(const int64_t* cand_off, const uint64_t* cand, const int64_t* xlims, const int64_t* qlims, int64_t l0,
                   const uint32_t* qlist, int64_t nlists, int32_t* cnt, const int32_t* off, RerankItem* items,
                   unsigned long long* stats) {
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= nlists) return;
    const int64_t lst = qlist ? (int64_t)qlist[l] : l0 + l;
    const int64_t c0 = cand_off[l];
    int64_t c1 = cand_off[l + 1];
    if (c1 > c0 && cand[c1 - 1] == kEmpty) {   // the padding starts at the first kEmpty: cut it off before the walk
        int64_t lo = c0, hi = c1 - 1;
        while (lo < hi) {
            const int64_t m = (lo + hi) >> 1;
            if (cand[m] == kEmpty) hi = m;
            else lo = m + 1;
        }
        c1 = lo;
    }
    int n = 0;
    int64_t o = items ? off[l] : 0;
    unsigned long long rows_all = 0;
    RerankItem cur{(int32_t)(lst - l0), 0, 0, 0};
    auto close = [&] {
        if (cur.ndocs == 0) return;
        if (items) items[o++] = cur;
        n++;
        cur.ndocs = 0;
    };
    for (int64_t c = c0; c < c1; c++) {
        const int64_t doc = (int64_t)(uint32_t)cand[c];
        const int len = (int)(xlims[doc + 1] - xlims[doc]);
        rows_all += (unsigned long long)len;
        if (cur.ndocs > 0 && (len > RR_TR || cur.nrows + len > RR_TR || cur.ndocs == RR_MAXD)) close();
        if (cur.ndocs == 0) {
            cur.c0 = (int32_t)c;
            cur.nrows = 0;
        }
        cur.ndocs++;
        cur.nrows += len;
        if (len > RR_TR) close();
    }
    close();
    if (!items) {
        cnt[l] = n;
        if (stats && c1 > c0) {
            atomicAdd(stats, (unsigned long long)(c1 - c0));
            atomicAdd(stats + 1, rows_all * (unsigned long long)(qlims[lst + 1] - qlims[lst]));
        }
    }
}

// Grow-only scratch of rerank().
struct RerankScratch {
    DevBuf<int32_t> cnt, off;
    DevBuf<RerankItem> items;
    DevBuf<uint8_t> tmp;
};

// Exact keys of the candidates of L rows (rerank_plan_kernel's rows: cand = rp.cand, list qlist[b] or rp.l0 + b):
// out[c] = pack_kp(exact key, document) for every entry c that is not kEmpty padding; the padding's slots are not
// written.  The plan's count pass, a cub::DeviceScan of the counts, one read-back of the item and candidate counts (the
// stream's only synchronisation here), the write pass and maxsim_rerank_kernel.  out is grown to the candidate count
// cand_off[L], which is returned.  stats: as rerank_plan_kernel's, or nullptr; `planned`, when given, is recorded
// between the plan and the re-rank.
inline int64_t
rerank(IndexBase& ix, int metric, bool vec4, RerankParams rp, const int64_t* cand_off, const uint32_t* qlist, int64_t L,
       DevBuf<uint64_t>& out, RerankScratch& rs, unsigned long long* stats, cudaEvent_t planned = nullptr) {
    cudaStream_t st = ix.stream;
    rs.cnt.ensure(L + 1);
    rs.off.ensure(L + 1);
    KB2_CUDA_CHECK(cudaMemsetAsync(rs.cnt.p + L, 0, 4, st));
    rerank_plan_kernel<<<grid1d(L, 128), 128, 0, st>>>(cand_off, rp.cand, rp.xlims, rp.qlims, rp.l0, qlist, L, rs.cnt.p,
                                                        nullptr, nullptr, stats);
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, rs.cnt.p, rs.off.p, (int)(L + 1), st);
    rs.tmp.ensure(bytes);
    bytes = rs.tmp.n;
    KB2_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(rs.tmp.p, bytes, rs.cnt.p, rs.off.p, (int)(L + 1), st));
    unsigned long long* hc = (unsigned long long*)ix.h_counter.p + 12;   // [0] items (int32), [1] candidates
    KB2_CUDA_CHECK(cudaMemcpyAsync(hc, rs.off.p + L, 4, cudaMemcpyDeviceToHost, st));
    KB2_CUDA_CHECK(cudaMemcpyAsync(hc + 1, cand_off + L, 8, cudaMemcpyDeviceToHost, st));
    KB2_CUDA_CHECK(cudaStreamSynchronize(st));
    const int64_t nitems = (int64_t)*(const int32_t*)hc, ncand = (int64_t)hc[1];
    rs.items.ensure(std::max<int64_t>(nitems, 1));
    out.ensure(std::max<int64_t>(ncand, 1));
    rerank_plan_kernel<<<grid1d(L, 128), 128, 0, st>>>(cand_off, rp.cand, rp.xlims, rp.qlims, rp.l0, qlist, L, nullptr,
                                                        rs.off.p, rs.items.p, nullptr);
    KB2_CUDA_CHECK(cudaGetLastError());
    if (planned) KB2_CUDA_CHECK(cudaEventRecord(planned, st));
    if (nitems > 0) {
        rp.items = rs.items.p;
        rp.out = out.p;
        with_metric(metric, [&](auto m) { launch_rerank<decltype(m)::value>(vec4, (unsigned)nitems, st, rp); });
        KB2_CUDA_CHECK(cudaGetLastError());
    }
    return ncand;
}

// ---------------------------------------------------------------------------------------------------------------------
// Host set-up of every emb-list search: the BruteForce search below and the index-level one (kb2_emb_list_index.cuh).

// The document bitset (host or device bits; none when null or nbits <= 0) on the device: checked to cover n_docs
// documents, a host bitset copied into buf
inline const uint8_t*
doc_bits_to_device(const uint8_t* bitset, int64_t nbits, int64_t n_docs, DevBuf<uint8_t>& buf, cudaStream_t st) {
    if (!bitset || nbits <= 0) return nullptr;
    KB2_REQUIRE(nbits >= n_docs, KB2_INVALID_ARGS, "bitset has fewer bits than the index has documents");
    if (is_device_ptr(bitset)) return bitset;
    buf.ensure((size_t)((n_docs + 7) / 8));
    KB2_CUDA_CHECK(cudaMemcpyAsync(buf.p, bitset, (size_t)((n_docs + 7) / 8), cudaMemcpyHostToDevice, st));
    return buf.p;
}

// Uploads into buf the list of every query row (ql: validated host offsets; at least one entry).  The returned host
// array is the copy's source: keep it until the stream has synchronised.
[[nodiscard]] inline std::vector<int32_t>
upload_row_list(const std::vector<int64_t>& ql, DevBuf<int32_t>& buf, cudaStream_t st) {
    std::vector<int32_t> row_list((size_t)std::max<int64_t>(ql.back(), 1));
    for (size_t l = 0; l + 1 < ql.size(); l++)
        for (int64_t r = ql[l]; r < ql[l + 1]; r++) row_list[r] = (int32_t)l;
    buf.ensure(row_list.size());
    KB2_CUDA_CHECK(cudaMemcpyAsync(buf.p, row_list.data(), row_list.size() * 4, cudaMemcpyHostToDevice, st));
    return row_list;
}

// ---------------------------------------------------------------------------------------------------------------------
// The BruteForce search.

// Scratch of one emb-list search, reused across calls (per-device BruteForce slot).
struct Scratch {
    DevBuf<int64_t> xlims, qlims, seg_off, doc_off;
    DevBuf<int32_t> row_list;
    DevBuf<uint32_t> kept;
    DevBuf<Item> items;
    DevBuf<uint64_t> cand, exact, sorted;
    DevBuf<uint8_t> bits, sort_tmp;
    RerankScratch rr;
};

// n entries of the all-documents mode's candidate rows: each row holds the n_kept documents kept[0 .. n_kept)
__global__ void
all_docs_kernel(const uint32_t* kept, int64_t n_kept, int64_t n, uint64_t* cand) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cand[i] = kept[i % n_kept];
}

// fi holds the base (fi.base, fi.norms = |x|^2, rows normalised for COSINE) and the stream; dq: device query rows
// (normalised for COSINE); xl / ql: validated host offsets; dbits: device bitset over documents or nullptr; d_ids /
// d_dist: device [n_lists][k].  metric: KB2_METRIC_L2 or KB2_METRIC_IP.  stats: lists, candidate slots re-ranked, lists
// scored exactly over all documents.
inline void
search(FlatIndex& fi, Scratch& sc, const float* dq, const std::vector<int64_t>& xl, const std::vector<int64_t>& ql, int d,
       int metric, int k, const uint8_t* dbits, int64_t* d_ids, float* d_dist, int64_t stats[3]) {
    cudaStream_t st = fi.stream;
    const int64_t n_docs = (int64_t)xl.size() - 1, n_lists = (int64_t)ql.size() - 1;
    const int64_t nb = xl.back(), nq_rows = ql.back();
    const float* X = fi.base.p;
    const float* xn = fi.norms.p;
    sc.xlims.ensure(xl.size());
    sc.qlims.ensure(ql.size());
    KB2_CUDA_CHECK(cudaMemcpyAsync(sc.xlims.p, xl.data(), xl.size() * 8, cudaMemcpyHostToDevice, st));
    KB2_CUDA_CHECK(cudaMemcpyAsync(sc.qlims.p, ql.data(), ql.size() * 8, cudaMemcpyHostToDevice, st));
    const std::vector<int32_t> row_list = upload_row_list(ql, sc.row_list, st);
    fi.s_qn.ensure(std::max<int64_t>(nq_rows, 1));
    if (metric == KB2_METRIC_L2 && nq_rows > 0)
        row_norms_kernel<<<grid1d(nq_rows * 32, 256), 256, 0, st>>>(dq, nq_rows, d, fi.s_qn.p);
    fi.s_cert.ensure((size_t)n_lists + 2);
    KB2_CUDA_CHECK(cudaMemsetAsync(fi.s_cert.p, 0, 8, st));
    pqtc::max_abs_kernel<<<2 * num_sms(), 256, 0, st>>>(xn, nb, fi.s_cert.p);

    CUtensorMap tq, tx;
    const bool use_tc = nq_rows > 0 && tc::make_tmap(&tq, dq, nq_rows, d) && tc::make_tmap(&tx, X, nb, d);
    const int K = k + 16;
    const int64_t lds = round_up(n_docs, 4);
    // lists per chunk: S within the 256 MB key budget of dense_candidates; the candidates, their exact keys, the sorted
    // rows and the re-rank items (at most one per candidate) within the large-k scratch
    const int64_t L = std::max<int64_t>(1, std::min<int64_t>({n_lists, (64ll << 20) / lds, large_k_group(n_lists, (int64_t)K * 40 + 16)}));
    // lists per all-documents group (at most L, so the K-entry buffers fit): the key rows within the same 64 M entries,
    // the candidate rows and their items within the large-k scratch; rows x n_docs < 2^31 as RerankItem::c0 is int32
    const int64_t La = std::max<int64_t>(1, std::min<int64_t>({L, (64ll << 20) / n_docs, large_k_group(n_lists, n_docs * 24)}));
    std::vector<Item> items;
    if (use_tc) {
        items = plan_items(xl);
        sc.items.ensure(std::max<size_t>(items.size(), 1));
        if (!items.empty())
            KB2_CUDA_CHECK(cudaMemcpyAsync(sc.items.p, items.data(), items.size() * sizeof(Item), cudaMemcpyHostToDevice, st));
        fi.s_keys.ensure((size_t)L * lds);
    }
    sc.cand.ensure((size_t)L * K);
    sc.sorted.ensure((size_t)L * K);
    sc.seg_off.ensure((size_t)L + 1);
    segment_offsets_kernel<<<grid1d(L + 1, 256), 256, 0, st>>>(sc.seg_off.p, L, K);
    size_t tmp_bytes = 0;
    cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp_bytes, sc.cand.p, sc.sorted.p, (int)(L * K), (int)L, sc.seg_off.p,
                                            sc.seg_off.p + 1, 0, 64, st);
    sc.sort_tmp.ensure(tmp_bytes);
    const bool vec4 = (d & 3) == 0 && (reinterpret_cast<uintptr_t>(dq) & 15) == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0;

    // exact keys of `rows` candidate rows of n entries in all into sc.exact; the slots of kEmpty padding stay kEmpty
    auto exact = [&](const uint64_t* cand, const int64_t* cand_off, int64_t n, int64_t rows, int64_t l0, const uint32_t* qlist) {
        sc.exact.ensure(n);
        KB2_CUDA_CHECK(cudaMemsetAsync(sc.exact.p, 0xFF, n * 8, st));
        const RerankParams rp{dq, sc.qlims.p, X, nullptr, sc.xlims.p, d, l0, nullptr, cand, nullptr};
        rerank(fi, metric, vec4, rp, cand_off, qlist, rows, sc.exact, sc.rr, nullptr);
        fi.last.launches += 4;
    };
    // sort the K entries of each row by (key, document) and emit the rows
    auto sort_emit = [&](const uint64_t* in, int64_t rows, int64_t l0, const uint32_t* qlist, const uint64_t* approx) {
        size_t bytes = tmp_bytes;
        KB2_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortKeys(sc.sort_tmp.p, bytes, in, sc.sorted.p, (int)(rows * K), (int)rows,
                                                               sc.seg_off.p, sc.seg_off.p + 1, 0, 64, st));
        EmitParams pp{sc.sorted.p, approx, K, k, dq, sc.qlims.p, d, fi.s_cert.p, l0, qlist, d_ids, d_dist};
        with_metric(metric, [&](auto m) { maxsim_emit_kernel<decltype(m)::value><<<(unsigned)rows, 256, 0, st>>>(pp); });
        fi.last.launches += 2;
        KB2_CUDA_CHECK(cudaGetLastError());
    };
    // exact keys of every document the bitset keeps for `rows` lists (at most La) -> their K best -> sorted, emitted.
    // The kept documents are listed on the host the first time: filtered ones are never scored.
    std::vector<uint32_t> kept;
    bool listed = false;
    auto exact_all = [&](int64_t rows, int64_t l0, const uint32_t* qlist) {
        if (!listed) {
            std::vector<uint8_t> bits(dbits ? (size_t)((n_docs + 7) / 8) : 0);
            if (dbits) {
                KB2_CUDA_CHECK(cudaMemcpyAsync(bits.data(), dbits, bits.size(), cudaMemcpyDeviceToHost, st));
                KB2_CUDA_CHECK(cudaStreamSynchronize(st));
            }
            for (int64_t j = 0; j < n_docs; j++)
                if (!dbits || !((bits[j >> 3] >> (j & 7)) & 1)) kept.push_back((uint32_t)j);
            sc.kept.ensure(std::max<size_t>(kept.size(), 1));
            KB2_CUDA_CHECK(cudaMemcpyAsync(sc.kept.p, kept.data(), kept.size() * 4, cudaMemcpyHostToDevice, st));
            listed = true;
        }
        const int64_t n_kept = (int64_t)kept.size(), n = rows * n_kept;
        sc.cand.ensure(n);
        sc.doc_off.ensure(rows + 1);
        if (n > 0) all_docs_kernel<<<grid1d(n, 256), 256, 0, st>>>(sc.kept.p, n_kept, n, sc.cand.p);
        segment_offsets_kernel<<<grid1d(rows + 1, 256), 256, 0, st>>>(sc.doc_off.p, rows, n_kept);
        fi.last.launches += 2;
        exact(sc.cand.p, sc.doc_off.p, n, rows, l0, qlist);
        large_k_select<uint64_t>(fi, sc.exact.p, n_kept, n_kept, 0u, K, sc.cand.p, K, rows);
        sort_emit(sc.cand.p, rows, l0, qlist, nullptr);
    };

    if (!use_tc) {
        for (int64_t l0 = 0; l0 < n_lists; l0 += La) exact_all(std::min(La, n_lists - l0), l0, nullptr);
        stats[0] += n_lists;
        stats[2] += n_lists;
        return;
    }
    for (int64_t l0 = 0; l0 < n_lists; l0 += L) {
        const int64_t rows = std::min(L, n_lists - l0);
        pqtc::fill_f32_kernel<<<grid1d(rows * lds, 256), 256, 0, st>>>(fi.s_keys.p, rows * lds, INFINITY);
        FilterParams fp{sc.items.p, (int)items.size(), sc.xlims.p, sc.qlims.p, sc.row_list.p, fi.s_qn.p, xn,
                        ql[l0], ql[l0 + rows], l0, d, dbits, fi.s_keys.p, lds};
        if (fp.r1 > fp.r0 && fp.nitems > 0) {
            const unsigned grid = (unsigned)std::min<int64_t>(num_sms(), fp.nitems);
            with_metric(metric, [&](auto m) {
                launch<maxsim_filter_kernel<decltype(m)::value>>(grid, tc::THREADS, SMEM_BYTES, st, tq, tx, fp);
            });
            fi.last.launches++;
            KB2_CUDA_CHECK(cudaGetLastError());
        }
        large_k_select<float>(fi, fi.s_keys.p, lds, n_docs, 0u, K, sc.cand.p, K, rows);
        exact(sc.cand.p, sc.seg_off.p, rows * K, rows, l0, nullptr);
        sort_emit(sc.exact.p, rows, l0, nullptr, sc.cand.p);
        stats[1] += rows * K;
    }
    int64_t nredo = 0;
    if (n_lists > 0) {
        uint32_t* hc = (uint32_t*)fi.h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(hc, fi.s_cert.p + 1, 4, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        nredo = hc[0];
        for (int64_t r0 = 0; r0 < nredo; r0 += La) exact_all(std::min(La, nredo - r0), 0, fi.s_cert.p + 2 + r0);
    }
    stats[0] += n_lists;
    stats[2] += nredo;
}

}  // namespace msim
}  // namespace kb2
