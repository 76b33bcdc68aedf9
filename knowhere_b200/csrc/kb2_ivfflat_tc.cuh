// kb2_ivfflat_tc.cuh — list-major tensor-core engine of the IVF_FLAT scan (batched queries).
//
// Reference path being replaced: IVFFlatScanner::scan_codes (exact distance of ONE query to every row of a probed
// list, K/IndexIVFFlat.cpp:139-232) under IndexIVF::search_preassigned (F/IndexIVF.cpp:401-768): the reference streams
// each probed list once per (query, list) pair — C2: 16.0 MB per query.
//
// Here the query x list distance is what it is, a dense contraction: the (query, probe) pairs are grouped by list
// (the list-major plan of kb2_listmajor.cuh), and every list is read ONCE per batch — a [128 rows] x [N queries of the list] x d
// tile product on the Hopper tensor cores (wgmma) with the operands brought by TMA.
//   * A operand: 128 consecutive rows of the list, fp32, straight from the list-order vector store (TMA, 128-byte swizzle).
//   * B operand: the item's queries, gathered pair-major beforehand and already split hi/lo (two TMA tiles).
//   * fp32 fidelity on the tf32 pipe: each consumer warpgroup splits its 64 rows of the A tile into hi = tf32(x),
//     lo = tf32(x - hi) and issues hi*hi + hi*lo + lo*hi (3 x wgmma m64nBROWSk8 tf32), error ~2^-21 relative
//     (kb2_gemm_tc.cuh); the split of k-block i+1 runs while the wgmmas of k-block i are in flight.
//   * accumulators: BROWS / 2 fp32 registers per thread; the producer keeps the stage ring full while the epilogue runs.
//   * epilogue: key = |q|^2 + |x|^2 - 2 acc (L2) / -acc (IP); keys within the per-query admission bound (exact k-th best
//     key of the query's nearest probed lists, from the query-major kernel, + a 3e-5 relative slack for the tf32 split)
//     are logged as survivors; finalize_kernel re-ranks the k+16 best of them EXACTLY from the fp32 rows, so the result
//     is the exact scan's (same guarantee as FLAT).
// Work item = (list, <= 32 or <= 128 of the queries probing it), drawn in descending-cost order from the ticket counter;
// survivors go to one log per CTA {query, position, f2ord(key), 0} and lm::scatter_survivors_kernel copies them into the
// per-query candidate rows as packed (key, position) entries.  One persistent CTA per SM, 288 threads:
//   warps 0-7 two consumer warpgroups (rows 0-63 | 64-127 of a tile: split, wgmma, epilogue) | warp 8 TMA producer.
#pragma once
#include "kb2_gemm_tc.cuh"
#include "kb2_listmajor.cuh"

namespace kb2 {
namespace fltc {

using lm::TM;                   // list rows per tile
constexpr int NQ_ITEM = 128;    // most queries per item
constexpr int BK = 32;          // floats per k-block (one 128-byte swizzle row)
constexpr int TILE_BYTES = 128 * BK * 4;        // 16 KB: 128 rows of one k-block
constexpr int THREADS = 288;
constexpr int PRODUCER_WARP = 8;
// item sequence of a CTA, shared by the two roles (< 16 items apart: the producer leads by at most STAGES k-blocks)
using ItemRing = lm::ItemRing<32>;
// BROWS = query rows per item the instance is built for (its B tiles are BROWS x 128 B): 32 -> 40 KB stages, 5 in flight
// (few queries per list: C2 has ~31); 128 -> 64 KB stages, 3 in flight.  The kernel is bound by the latency of the
// TMA -> convert -> MMA -> release chain of a stage, so the number of stages in flight sets the HBM rate it reaches.
template <int BROWS>
struct FlCfg {
    static constexpr int B_TILE_BYTES = BROWS * BK * 4;
    static constexpr int STAGE_BYTES = 2 * TILE_BYTES + 2 * B_TILE_BYTES;     // A_hi | A_lo | B_hi | B_lo
    static constexpr int STAGES = BROWS <= 32 ? 5 : 3;
    static constexpr int OFF_META = STAGES * STAGE_BYTES;                     // thr[128] | base[128] | qidx[128]
    static constexpr int OFF_BAR = OFF_META + 3 * NQ_ITEM * 4;
    static constexpr size_t SMEM_BYTES = OFF_BAR + 256 + ItemRing::BYTES + 1024 /*alignment slack*/;
    static_assert(SMEM_BYTES <= 227 * 1024, "IVF_FLAT tensor-core kernel shared memory");
};
constexpr float kSlack = 3e-5f;   // 3xTF32 contraction error, relative to |q|^2 + |x|^2 (measured 5e-6, tests/test_gemm_tc_gpu.py)

struct Params {
    int metric, d;
    const int32_t* n_items;
    int32_t* ticket;              // work counter (zeroed before the launch)
    const int32_t* item_list;
    const int32_t* item_q0;       // first pair of the item
    const int32_t* item_nq;
    const int32_t* pair_q;        // [pairs] query index, grouped by list
    const float* qnorm2;          // [nq] |q|^2
    const float* bound;           // [nq] admission bound on the key (+inf: none)
    const int64_t* list_off;
    const int32_t* list_len;
    const float* xnorm2;          // [npad] |x|^2 per position
    const uint8_t* bitset;
    const int32_t* rows;
    uint4* log;                   // [gridDim.x][log_cap] survivors {query, position, f2ord(key), 0}
    uint32_t* log_cnt;            // [gridDim.x] entries; [gridDim.x] = 1 when a log overflowed
    uint32_t log_cap;
    unsigned long long* counters; // [0] rows scanned (pairs x rows)
};

// pair-major copy of the queries, split for the 3xTF32 contraction: hi = tf32(q), lo = tf32(q - hi)   (warp per pair)
__global__ void __launch_bounds__(256)
gather_split_queries_kernel(const float* __restrict__ q, const int32_t* __restrict__ pair_q, int64_t npairs, int64_t npairs_pad, int d,
                            float* __restrict__ hi, float* __restrict__ lo) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= npairs_pad) return;
    const int32_t qi = i < npairs ? pair_q[i] : -1;
    for (int j = lane; j < d; j += kWarp) {
        const float v = qi >= 0 ? q[(int64_t)qi * d + j] : 0.f;
        const float h = tc::tf32_rn(v);
        hi[i * d + j] = h;
        lo[i * d + j] = tc::tf32_rn(v - h);
    }
}

// bound[q] = key of entry k-1 of the query's sorted phase-A row (+inf when it holds fewer than k entries)
__global__ void
extract_bound_kernel(const uint64_t* __restrict__ partial, int64_t stride, int k, int64_t nq, float* __restrict__ bound) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    const uint64_t e = partial[q * stride + k - 1];
    bound[q] = (e == kEmpty) ? INFINITY : unpack_key(e);
}

template <int BROWS>
__device__ __forceinline__ void
wgmma_tf32(float (&acc)[BROWS / 2], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    if constexpr (BROWS == 128) tc::wgmma_tf32_n128(acc, a_desc, b_desc, accumulate);
    else tc::wgmma_tf32_n32(acc, a_desc, b_desc, accumulate);
}

template <int METRIC, int BROWS>
__global__ void __launch_bounds__(THREADS, 1)
ivfflat_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_qhi,
                  const __grid_constant__ CUtensorMap tmap_qlo, Params p) {
    static_assert(BROWS == 32 || BROWS == 128, "wgmma N of the IVF_FLAT engine");
    using C = FlCfg<BROWS>;
    constexpr int STAGES = C::STAGES, STAGE_BYTES = C::STAGE_BYTES, B_TILE_BYTES = C::B_TILE_BYTES, OFF_META = C::OFF_META,
                  OFF_BAR = C::OFF_BAR;
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t raw = tc::smem_u32(smem_dyn);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* sm = smem_dyn + (base - raw);
    const uint32_t bars = base + OFF_BAR;
    // barriers: full[S] empty[S] | log cursor
    auto bar_full = [&](int s) { return bars + 8u * s; };
    auto bar_empty = [&](int s) { return bars + 8u * (STAGES + s); };
    uint32_t* log_cursor = (uint32_t*)(sm + OFF_BAR + 8 * (2 * STAGES));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_items = *p.n_items;
    const int nkb = p.d / BK;

    const ItemRing ring(sm + OFF_BAR + 256, p.ticket);
    ring.init();

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) {
            tc::mbar_init(bar_full(s), 1);
            tc::mbar_init(bar_empty(s), 256);
        }
        *log_cursor = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        // ================= TMA producer: per (item, tile, k-block) one stage = raw A tile + B_hi + B_lo =================
        if (lane == 0) {
            uint32_t it = 0;
            int seq = 0;
            for (int item = ring.at_thread(0); item < n_items; item = ring.at_thread(++seq)) {
                const int l = p.item_list[item];
                const int q0 = p.item_q0[item];
                const int64_t off = p.list_off[l];
                const int ntiles = (p.list_len[l] + TM - 1) / TM;
                for (int t = 0; t < ntiles; t++) {
                    for (int kb = 0; kb < nkb; kb++, it++) {
                        const int s = it % STAGES;
                        tc::mbar_wait(bar_empty(s), ((it / STAGES) & 1u) ^ 1u);
                        const uint32_t st = base + (uint32_t)s * STAGE_BYTES;
                        tc::mbar_expect_tx(bar_full(s), TILE_BYTES + 2 * B_TILE_BYTES);
                        tc::tma_load_2d(st, &tmap_x, kb * BK, (int)(off + (int64_t)t * TM), bar_full(s));
                        tc::tma_load_2d(st + 2 * TILE_BYTES, &tmap_qhi, kb * BK, q0, bar_full(s));
                        tc::tma_load_2d(st + 2 * TILE_BYTES + B_TILE_BYTES, &tmap_qlo, kb * BK, q0, bar_full(s));
                    }
                }
            }
        }
        return;
    }
    // ================= consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 of every tile; columns = the item's queries
    const int ct = threadIdx.x;          // 0..255
    const int wg = ct >> 7;
    const int w128 = ct & 127;
    float* m_thr = (float*)(sm + OFF_META);
    float* m_base = m_thr + NQ_ITEM;
    int* m_q = (int*)(m_base + NQ_ITEM);
    uint4* my_log = p.log + (size_t)blockIdx.x * p.log_cap;
    bool log_over = false;
    unsigned long long n_rows = 0;
    float acc[BROWS / 2];
#pragma unroll
    for (int i = 0; i < BROWS / 2; i++) acc[i] = 0.f;
    uint32_t it = 0;
    int seq = 0;
    for (int item = ring.at_warp(0); item < n_items; item = ring.at_warp(++seq)) {
        const int l = p.item_list[item];
        const int q0 = p.item_q0[item];
        const int nqi = p.item_nq[item];
        const int len = p.list_len[l];
        const int64_t off = p.list_off[l];
        const int ntiles = (len + TM - 1) / TM;
        asm volatile("bar.sync 1, 256;" ::: "memory");   // every consumer thread is done with the previous item's meta
        if (ct < NQ_ITEM) {
            // admit  <=>  key - slack * (|q|^2 + |x|^2) <= bound   (|q|^2 + |x|^2 >= 2 |q||x| bounds the 3xTF32 error scale)
            float thr = -INFINITY, bs = 0.f;
            int q = -1;
            if (ct < nqi) {
                q = p.pair_q[q0 + ct];
                bs = p.qnorm2[q];
                const float bnd = p.bound[q];
                thr = (bnd < INFINITY) ? bnd + kSlack * bs + 1e-30f : INFINITY;
            }
            m_thr[ct] = thr;
            m_base[ct] = bs;
            m_q[ct] = q;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (ct == 0) n_rows += (unsigned long long)len * (unsigned long long)nqi;
        for (int t = 0; t < ntiles; t++) {
            int pending = -1;   // stage whose wgmmas may still be in flight
            for (int kb = 0; kb < nkb; kb++, it++) {
                const int s = it % STAGES;
                tc::mbar_wait(bar_full(s), (it / STAGES) & 1u);
                // split this warpgroup's 64 rows of the raw A tile into hi (in place) and lo
                float4* hi = reinterpret_cast<float4*>(sm + (size_t)s * STAGE_BYTES + wg * (TILE_BYTES / 2));
                float4* lo = reinterpret_cast<float4*>(sm + (size_t)s * STAGE_BYTES + TILE_BYTES + wg * (TILE_BYTES / 2));
#pragma unroll 4
                for (int i = w128; i < TILE_BYTES / 32; i += 128) {
                    const float4 v = hi[i];
                    float4 h, w;
                    h.x = tc::tf32_rn(v.x); w.x = tc::tf32_rn(v.x - h.x);
                    h.y = tc::tf32_rn(v.y); w.y = tc::tf32_rn(v.y - h.y);
                    h.z = tc::tf32_rn(v.z); w.z = tc::tf32_rn(v.z - h.z);
                    h.w = tc::tf32_rn(v.w); w.w = tc::tf32_rn(v.w - h.w);
                    hi[i] = h;
                    lo[i] = w;
                }
                tc::fence_proxy_async();
                if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
                else asm volatile("bar.sync 3, 128;" ::: "memory");
                const uint32_t st = base + (uint32_t)s * STAGE_BYTES;
                const uint32_t a_off = (uint32_t)wg * (TILE_BYTES / 2);
                tc::fence_operand(acc);
                tc::wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < BK / 8; kk++) {
                    const uint32_t ko = (uint32_t)kk * 32u;
                    const uint64_t a_hi = tc::make_desc(st + a_off + ko);
                    const uint64_t a_lo = tc::make_desc(st + TILE_BYTES + a_off + ko);
                    const uint64_t b_hi = tc::make_desc(st + 2 * TILE_BYTES + ko);
                    const uint64_t b_lo = tc::make_desc(st + 2 * TILE_BYTES + B_TILE_BYTES + ko);
                    wgmma_tf32<BROWS>(acc, a_hi, b_hi, (kb > 0 || kk > 0) ? 1u : 0u);
                    wgmma_tf32<BROWS>(acc, a_hi, b_lo, 1u);
                    wgmma_tf32<BROWS>(acc, a_lo, b_hi, 1u);
                }
                tc::wgmma_commit();
                tc::fence_operand(acc);
                tc::wgmma_wait<1>();
                if (pending >= 0) tc::mbar_arrive(bar_empty(pending));
                pending = s;
            }
            tc::wgmma_wait<0>();
            tc::fence_operand(acc);
            if (pending >= 0) tc::mbar_arrive(bar_empty(pending));
            // ---- epilogue: this thread holds rows r0, r0 + 8 and columns 8 j + 2 (lane % 4) + c of the tile
            const int r0 = t * TM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int rel = r0 + 8 * i;
                const bool row_ok = rel < len;
                float xn = 0.f;
                if (row_ok) xn = __ldg(p.xnorm2 + off + rel);
                bool alive = row_ok;
                if (alive && p.bitset) alive = !bit_is_set(p.bitset, p.rows[off + rel]);
                const float xs = (METRIC == KB2_METRIC_L2) ? xn * (1.f - kSlack) : -kSlack * xn;   // (row part of the key) - slack * |x|^2
                uint32_t mask = 0;
                if (alive) {
#pragma unroll
                    for (int j = 0; j < BROWS / 8; j++) {
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            const int col = j * 8 + 2 * (lane & 3) + c;
                            const float a = acc[4 * j + 2 * i + c];
                            const float key = (METRIC == KB2_METRIC_L2) ? (m_base[col] + xs - 2.f * a) : (xs - a);
                            mask |= (col < nqi && key <= m_thr[col]) ? (1u << (2 * j + c)) : 0u;
                        }
                    }
                }
                const uint32_t cnt = __popc(mask);
                if (__any_sync(0xffffffffu, cnt != 0u)) {
                    uint32_t incl = cnt;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t tv = __shfl_up_sync(0xffffffffu, incl, o);
                        if (lane >= o) incl += tv;
                    }
                    uint32_t wbase = 0;
                    if (lane == 31) wbase = atomicAdd(log_cursor, incl);
                    wbase = __shfl_sync(0xffffffffu, wbase, 31);
                    uint32_t slot = wbase + incl - cnt;
#pragma unroll
                    for (int j = 0; j < BROWS / 8; j++) {   // static register indices (a data-dependent acc[u] would spill the tile)
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            if ((mask >> (2 * j + c)) & 1u) {
                                const int col = j * 8 + 2 * (lane & 3) + c;
                                const float a = acc[4 * j + 2 * i + c];
                                const float key = (METRIC == KB2_METRIC_L2) ? (m_base[col] + xn - 2.f * a) : -a;
                                if (slot < p.log_cap) {
                                    uint4 o;
                                    o.x = (uint32_t)m_q[col];
                                    o.y = (uint32_t)(off + rel);
                                    o.z = f2ord(key);
                                    o.w = 0u;
                                    my_log[slot] = o;
                                } else {
                                    log_over = true;
                                }
                                slot++;
                            }
                        }
                    }
                }
            }
        }
    }
    if (log_over) p.log_cnt[gridDim.x] = 1u;
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (ct == 0) {
        p.log_cnt[blockIdx.x] = min(*log_cursor, p.log_cap);
        if (p.counters) atomicAdd(p.counters, n_rows);
    }
}

// number of flagged queries (or every query when a log overflowed) -> *out
__global__ void
count_flags_kernel(const uint32_t* __restrict__ qflag, int64_t nq, const uint32_t* __restrict__ log_over, uint32_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && *log_over) atomicAdd(out, 1u);
    if (i < nq && qflag[i]) atomicAdd(out, 1u);
}

}  // namespace fltc
}  // namespace kb2
