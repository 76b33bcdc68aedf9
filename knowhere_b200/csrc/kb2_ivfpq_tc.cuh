// kb2_ivfpq_tc.cuh — list-major tensor-core engine of the IVF_PQ scan (large batches).
//
// Reference path being replaced: IVFPQScanner::scan_list_with_table (one table look-up chain per
// (query, code) pair; F/impl/pq_code_distance/IVFPQScanner_impl.h:110-185) under
// IndexIVF::search_preassigned (F/IndexIVF.cpp:401-768).
//
// Why a second engine.  The query-major LUT kernel (kb2_ivf.cuh) is bound by the shared-memory gather pipe:
// 16 wavefronts per 32 codes *per query*.  But the ADC inner term is a dot
// product, <q, r^(code)>, and at batch 10^4 x nprobe 64 every list is probed by ~150 queries.  Decoding a
// 128-code tile ONCE into bf16 and contracting it with all the queries of the list on the tensor cores replaces
// 16 gathers per (query, code) by 16 gathers per code + 128 x N x 128 MACs on the tensor pipe.
//
// Exactness.  The tensor-core value S' is only a FILTER.  With u = 2^-8 (bf16 round-to-nearest),
//     |S' - <q,r^>| <= (2u + u^2) |q| |r^| + (fp32 accumulation) <= 0.0085 |q| Rmax,   Rmax^2 = sum_m max_j |c_pq[m][j]|^2
// so with a per-query upper bound B_q of the K-th best key (taken from a LUT scan of the query's nearest lists,
// "phase A") every code with   key' <= B_q + |alpha| * 0.0085 |q| Rmax   is a *survivor*; survivors are
// re-evaluated with exactly the fp32 operations (and summation order) of the LUT kernel and kept when
// key <= B_q.  The final top-K is the same set with the same keys as the LUT engine returns
// (tests/test_ivf_gpu.py::test_ivfpq_tc_engine_matches_lut_engine).  Queries whose bound is missing (fewer
// than K codes in their nearest lists) or whose survivor buffer overflows are flagged and redone by the LUT kernel.
//
// sm_90a mapping (one persistent CTA per SM, 512 threads, <= 219.5 KB of shared memory):
//   warps 0-7  decoders : (two groups of 4 warps, one per A buffer, so two tiles are decoded concurrently)
//                         code tile -> A operand [128 codes x K] bf16 in the no-swizzle K-major wgmma layout (16-byte
//                         sub-vector of sub-quantizer m = one core-matrix row), via a bf16 copy of the PQ codebooks in
//                         shared memory, + the admission-test K-step [-r_hi, -r_mid, -r_lo, 1, 1, 1, 0, 0]; they also stage
//                         the B operand (bf16 queries of the item, gathered by index, + [1, 1, 1, h_hi, h_mid, h_lo, 0, 0])
//                         and the per-column meta data, one item ahead.
//   warps 8-15 consumers: two warpgroups, warpgroup e owns the tiles g % 2 == e (A buffer e).  A tile is contracted in
//                         blocks of 64 codes x at most MAXW queries, each exactly as wide as its share of the item's columns
//                         (K/16 + 1 x wgmma m64nNk16 bf16 into N / 2 registers per thread), the
//                         next block of the tile (of either 64-code half) is issued before the current one is tested; the accumulator
//                         holds D = S' + h - r, so "survives" is a clear sign bit, collected branch-free into per-row masks
//                         while the next block is in flight.  Once the tile is in registers the hits are expanded -> one
//                         shared-memory slot reservation per warp and half tile -> the group's private survivor log in global
//                         memory (plain stores, nothing on the critical path waits for a global round trip).
// Work item = (list, chunk of <= 256 of the queries probing it).  The plan, the cost-ordered ticket scheduling and the
// survivor logs are the list-major pipeline of kb2_listmajor.cuh (DESIGN.md 4.5); the log entries carry the key base's
// bits.  Then lm::scatter_survivors_kernel groups the logs by query, exact_eval_kernel recomputes the survivors' keys in fp32.
#pragma once
#include <cuda_bf16.h>

#include <type_traits>
#include <utility>

#include "kb2_gemm_tc.cuh"
#include "kb2_ivf.cuh"
#include "kb2_listmajor.cuh"

namespace kb2 {
namespace pqtc {

using lm::TM;                  // codes per tile
constexpr int NQT = 256;       // queries per item
constexpr int THREADS = 512;          // warps 0-7 decoders (2 groups), 8-15 consumers (2 warpgroups)
constexpr int GROUP_THREADS = 128;
// widest wgmma block of the consumers (columns).  Two blocks are in flight per warpgroup, and ptxas (CUDA 12.9) fits their
// accumulators under the kernel's 128-register cap only up to this width: wider blocks make it serialize the wgmmas
// (C7511 / C7512), and raising the consumers' budget with setmaxnreg does not change that.
constexpr int MAXW = 80;
constexpr int META_BYTES = 3 * NQT * 4;   // h | base | qidx
// geometry of one engine instance: G groups of 16 sub-quantizers of DSUB dimensions (K = 16 G DSUB).
// Instances: <1, 8> (m = 16, d = 128: BASELINE C3) and <3, 2> (m = 48, d = 96: BASELINE C5).
template <int G, int DSUB>
struct TcCfg {
    static constexpr int M = 16 * G;
    static constexpr int KD = M * DSUB;               // dimensions
    static_assert(KD % 16 == 0 && (DSUB == 2 || DSUB == 4 || DSUB == 8), "unsupported PQ geometry");
    static constexpr int XCHUNK = KD / 8;             // 16-byte chunk that carries the admission test (row term / column threshold)
    static constexpr int KSTEPS = KD / 16 + 1;        // the last K-step holds the test chunk + a zero chunk
    static constexpr int CHUNKS = 2 * KSTEPS;         // 16-byte chunks per operand row
    static constexpr int GRP_BYTES = CHUNKS * 128;    // one 8-row group of an operand: core matrices of 128 B (wgmma SBO)
    static constexpr int TAB_BYTES = M * 256 * DSUB * 2;   // bf16 codebooks
    static constexpr int A_BYTES = (TM / 8) * GRP_BYTES, B_BYTES = (NQT / 8) * GRP_BYTES;
    static constexpr int OFF_TAB = 0;
    static constexpr int OFF_A = TAB_BYTES;
    static constexpr int OFF_B = OFF_A + 2 * A_BYTES;
    static constexpr int OFF_META = OFF_B + B_BYTES;
    static constexpr int OFF_BAR = OFF_META + 2 * META_BYTES;
    static constexpr size_t SMEM_BYTES = OFF_BAR + 256 + 128 /*alignment slack*/;   // barriers 0..135, scheduler ring 144..239
    static_assert(SMEM_BYTES <= 227 * 1024, "filter kernel shared memory");
};
constexpr int KD = 128;                   // (phase-A kernels below are specific to the <1, 8> geometry)
constexpr float kErrCoef = 0.0085f;       // (2u + u^2) for bf16 operands + fp32 accumulation slack
constexpr float kAccCoef = 4e-5f;         // fp32 accumulation of the contraction incl. the threshold terms (x (|h| + max|r|))

struct Params {
    int metric;
    int nq, nprobe;
    const float* queries;          // [nq][128] fp32
    const __nv_bfloat16* qb16;     // [nq][128]
    const float* qnorm;            // [nq]
    // plan
    const int32_t* n_items;        // device scalar
    int32_t* ticket;               // work counter (zeroed before the launch): CTAs draw items from it in order, so a
                                   // CTA that got short items simply draws more
    const int32_t* item_list;      // [items]
    const int32_t* item_q0;        // [items] first pair of the chunk
    const int32_t* item_nq;        // [items]
    const int32_t* pair_q;         // [pairs] query index, grouped by list
    const float* pair_base;        // [pairs] key base: L2 |q-c|^2, IP -<q,c>
    // per-query bound from phase A
    const float* bound;            // [nq] upper bound of the k_need-th best key (+inf: none -> the LUT kernel redoes the query)
    int k_need;
    float margin_coef;             // |alpha| * kErrCoef * Rmax  (multiplied by |q|)
    float rmax;                    // max over the index of the row term |t1| / 2 (L2; 0 for IP)
    // index
    const int64_t* list_off;
    const int32_t* list_len;
    const uint4* codes;            // [G][npad] 16 code bytes per group, rotated by pos % 16 (kb2_ivf.cuh)
    const uint4* codes_plain;      // [G][npad] un-rotated copy (byte b = sub-quantizer 16 g + b); used by the decode when DSUB < 8
    int64_t npad;
    const float* t1;               // [npad] (L2)
    const float* pqc;              // [16][256][8] fp32
    const uint4* pqc16;            // [16][256] x 8 bf16
    const uint8_t* bitset;
    const int32_t* rows;
    // output
    uint4* log;                    // [2*gridDim.x][log_cap] survivors {query, position, key base bits, 0}: one log per
                                   // epilogue group
    uint32_t* log_cnt;             // [2*gridDim.x] entries per log; [2*gridDim.x] = 1 when any log overflowed
    uint32_t log_cap;              // entries per log
    uint32_t* qflag;               // [nq] 1: redo this query with the LUT kernel
    unsigned long long* counters;  // [0] codes scanned (pairs x codes), [2] survivors re-evaluated, [3] flagged
};

// f(std::integral_constant<int, I>{}) for I = 0 .. N-1, in order
template <typename F, int... I>
__device__ __forceinline__ void
static_for_impl(F&& f, std::integer_sequence<int, I...>) {
    (f(std::integral_constant<int, I>{}), ...);
}
template <int N, typename F>
__device__ __forceinline__ void
static_for(F&& f) {
    static_for_impl(f, std::make_integer_sequence<int, N>{});
}
// columns C0 .. C0 + W - 1 of an item, contracted in one wgmma block
template <int C0_, int W_>
struct BlockCols {
    static constexpr int C0 = C0_, W = W_;
};
// f(std::integral_constant<int, n>{}) for the run-time value n = LO .. HI (warp-uniform), by binary search
template <int LO, int HI, typename F>
__device__ __forceinline__ void
dispatch_range(int n, F&& f) {
    if constexpr (LO == HI) {
        f(std::integral_constant<int, LO>{});
    } else {
        constexpr int MID = (LO + HI) / 2;
        if (n <= MID) dispatch_range<LO, MID>(n, f);
        else dispatch_range<MID + 1, HI>(n, f);
    }
}

__device__ __forceinline__ void
bar_sync_epi() {
    asm volatile("bar.sync 1, 256;" ::: "memory");
}
// wgmma shared-memory descriptor, K-major, no swizzle: core matrix = 8 rows x 16 B (128 B contiguous);
// LBO = distance between the two core matrices of one K=16 step (128 B), SBO = distance between 8-row groups (GRP_BYTES)
__device__ __forceinline__ uint64_t
make_desc_ns(uint32_t smem_addr, uint32_t grp_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)(128 >> 4) << 16;
    d |= (uint64_t)(grp_bytes >> 4) << 32;
    return d;   // layout type 0 (no swizzle), base offset 0
}

// Cycle accounting of the filter kernel's roles, compiled in only with -DKB2_FILTER_STALLS (scripts/filter_stalls.py):
// one thread per group sums clock64() intervals into stall[slot] and stores them in g_filter_stalls at the end of the
// launch; filter_stalls_print_kernel, launched after the filter kernel, prints each CTA's sums over both groups of each
// role (a printf inside the filter kernel is a function call, and ptxas serializes the wgmmas of a kernel that makes
// one).  Without the macro these expand to nothing, so the default build is unchanged.
#ifdef KB2_FILTER_STALLS
#define KB2_STALL_BEGIN(v) const long long v = clock64()
#define KB2_STALL_END(slot, v) stall[slot] += clock64() - (v)
constexpr int kStallMaxCtas = 1024, kStallSlots = 8;
// [CTA][role: 0 decoders, 1 consumers][group][slot]
__device__ unsigned long long g_filter_stalls[kStallMaxCtas][2][2][kStallSlots];
__global__ void
filter_stalls_print_kernel(int ctas) {
    for (int b = 0; b < min(ctas, kStallMaxCtas); b++) {
        printf("KB2STALL cta=%d", b);
        for (int r = 0; r < 2; r++) {
            printf(r == 0 ? " dec=" : " cons=");
            for (int i = 0; i < kStallSlots; i++)
                printf(i ? ",%llu" : "%llu", g_filter_stalls[b][r][0][i] + g_filter_stalls[b][r][1][i]);
        }
        printf("\n");
    }
}
#else
#define KB2_STALL_BEGIN(v)
#define KB2_STALL_END(slot, v)
#endif

// x = hi + mid + lo with three bf16 terms (24 significant bits: exact for finite fp32 up to 2^-27 |x|); +-inf -> (+-inf, 0, 0)
__device__ __forceinline__ void
split3_bf16(float x, uint32_t& hi, uint32_t& mid, uint32_t& lo) {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    hi = (uint32_t)__bfloat16_as_ushort(h);
    if (!(fabsf(x) < INFINITY)) { mid = 0u; lo = 0u; return; }
    const float r1 = x - __bfloat162float(h);
    const __nv_bfloat16 m = __float2bfloat16_rn(r1);
    const float r2 = r1 - __bfloat162float(m);
    mid = (uint32_t)__bfloat16_as_ushort(m);
    lo = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(r2));
}

template <int METRIC, int G, int DSUB>
__global__ void __launch_bounds__(THREADS, 1)
ivfpq_tc_filter_kernel(Params p) {
    using C = TcCfg<G, DSUB>;
    constexpr int KD = C::KD, XCHUNK = C::XCHUNK, KSTEPS = C::KSTEPS, GRP_BYTES = C::GRP_BYTES, TAB_BYTES = C::TAB_BYTES;
    constexpr int A_BYTES = C::A_BYTES, OFF_TAB = C::OFF_TAB, OFF_A = C::OFF_A, OFF_B = C::OFF_B, OFF_META = C::OFF_META,
                  OFF_BAR = C::OFF_BAR;
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t raw = tc::smem_u32(smem_dyn);
    const uint32_t base = (raw + 127u) & ~127u;
    unsigned char* sm = smem_dyn + (base - raw);
    const uint32_t bars = base + OFF_BAR;
    // barriers: a_full[2] a_empty[2] (4..7 unused) b_full b_free meta_full[2] meta_free[2]
    auto bar_a_full = [&](int i) { return bars + 8u * i; };
    auto bar_a_empty = [&](int i) { return bars + 8u * (2 + i); };
    const uint32_t bar_b_full = bars + 8u * 8, bar_b_free = bars + 8u * 9;
    auto bar_meta_full = [&](int i) { return bars + 8u * (10 + i); };
    auto bar_meta_free = [&](int i) { return bars + 8u * (12 + i); };
    uint32_t* qcnt = (uint32_t*)(sm + OFF_BAR + 8 * 15);   // survivor counters: [epilogue group][own tile parity]

    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // role index, provably warp-uniform
    const int n_items = *p.n_items;

    // item sequence of this CTA, shared by the three roles (at most ~3 items apart)
    const lm::ItemRing<8> ring(sm + OFF_BAR + 144, p.ticket);
    ring.init();

    if (threadIdx.x == 0) {
        for (int i = 0; i < 2; i++) {
            tc::mbar_init(bar_a_full(i), GROUP_THREADS);
            tc::mbar_init(bar_a_empty(i), GROUP_THREADS);
            tc::mbar_init(bar_meta_full(i), 2 * GROUP_THREADS);
            tc::mbar_init(bar_meta_free(i), 2 * GROUP_THREADS);
        }
        tc::mbar_init(bar_b_full, 2 * GROUP_THREADS);
        tc::mbar_init(bar_b_free, 2 * GROUP_THREADS);
        qcnt[0] = qcnt[1] = qcnt[2] = qcnt[3] = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
#ifdef KB2_FILTER_STALLS
    long long stall[kStallSlots] = {0, 0, 0, 0, 0, 0, 0, 0};
    KB2_STALL_BEGIN(t_role);
#endif
    // bf16 codebooks -> shared memory
    {
        uint4* tab = (uint4*)(sm + OFF_TAB);
        for (int i = threadIdx.x; i < TAB_BYTES / 16; i += THREADS) tab[i] = __ldg(p.pqc16 + i);
    }
    __syncthreads();
    const float inv_alpha = (METRIC == KB2_METRIC_L2) ? 0.5f : 1.f;

    if (warp < 8) {
        // =========================== decoders: two groups of 4 warps, group d owns A buffer d (tiles g % 2 == d) =========
        const int dt = threadIdx.x;    // 0..255
        const int dg = dt >> 7;        // group
        const int tid = dt & 127;      // code row inside the tile
        const uint4* tab = (const uint4*)(sm + OFF_TAB);
        // per-column thresholds of one item -> meta buffer (it & 1), one column per decoder thread; written one item
        // AHEAD of its use so that the dependent global loads (pair -> bound, norm) stay off the critical path
        auto write_meta = [&](int item, int it) {
            KB2_STALL_BEGIN(t_meta);
            const int par = it & 1;
            tc::mbar_wait(bar_meta_free(par), (((uint32_t)it >> 1) & 1u) ^ 1u);
            const int q0 = p.item_q0[item];
            const int nqi = p.item_nq[item];
            float* m_h = (float*)(sm + OFF_META + par * META_BYTES);
            float* m_base = m_h + NQT;
            int* m_q = (int*)(m_base + NQT);
            const int j = dt;
            float h = -INFINITY, bs = 0.f;
            int q = -1;
            if (j < nqi) {
                q = p.pair_q[q0 + j];
                bs = p.pair_base[q0 + j];
                const float bnd = p.bound[q];
                if (!(bnd < INFINITY)) {
                    p.qflag[q] = 1u;   // no bound: the LUT kernel redoes this query
                    if (p.counters) atomicAdd(p.counters + 6, 1ull << 32);
                } else {
                    // pass  <=>  S' + h >= r  (S' bf16 contraction, r the row term); the margin covers the bf16 operand error,
                    // the extra term the fp32 accumulation of the K=144 contraction that now carries h and r as well
                    const float margin = p.margin_coef * p.qnorm[q] * 1.01f + 1e-30f;
                    const float h0 = (bnd + margin - bs) * inv_alpha;
                    h = h0 + kAccCoef * (fabsf(h0) + p.rmax) + 1e-30f;
                }
            }
            m_h[j] = h;
            m_base[j] = bs;
            m_q[j] = q;
            tc::mbar_arrive(bar_meta_full(par));
            KB2_STALL_END(5, t_meta);
        };
        uint32_t g0 = 0;   // global tile counter at the start of the item
        int it = 0;
        int item = ring.at_warp(0);
        if (item < n_items) write_meta(item, 0);
        for (; item < n_items; it++) {
            const int item_next = ring.at_warp(it + 1);
            const int l = p.item_list[item];
            const int nqi = p.item_nq[item];
            const int nmma = (nqi + 15) & ~15;
            const int len = p.list_len[l];
            const int64_t off = p.list_off[l];
            const int ntiles = (len + TM - 1) / TM;
            const int par = it & 1;
            const int t_first = (int)((dg - (int)(g0 & 1u)) & 1);   // this group's first tile of the item
            uint4 w_next[G];
#pragma unroll
            for (int g = 0; g < G; g++) w_next[g] = make_uint4(0, 0, 0, 0);
            float t_next = 0.f;
            const uint4* code_src = (DSUB == 8) ? p.codes : p.codes_plain;
            if (t_first < ntiles && off + (int64_t)t_first * TM + tid < p.npad) {
#pragma unroll
                for (int g = 0; g < G; g++) w_next[g] = ldg_stream_u4(code_src + (int64_t)g * p.npad + off + (int64_t)t_first * TM + tid);
                if (METRIC == KB2_METRIC_L2) t_next = __ldg(p.t1 + off + (int64_t)t_first * TM + tid);
            }
            auto decode_tile = [&](int t) {
                KB2_STALL_BEGIN(t_dec);
                const uint32_t g = g0 + (uint32_t)t;      // g & 1 == dg
                uint4 w[G];
#pragma unroll
                for (int gg = 0; gg < G; gg++) w[gg] = w_next[gg];
                const float tv = t_next;
                {
                    const int64_t pn = off + (int64_t)(t + 2) * TM + tid;
                    if (t + 2 < ntiles && pn < p.npad) {
#pragma unroll
                        for (int gg = 0; gg < G; gg++) w_next[gg] = ldg_stream_u4(code_src + (int64_t)gg * p.npad + pn);
                        if (METRIC == KB2_METRIC_L2) t_next = __ldg(p.t1 + pn);
                    }
                }
                // row term of the admission test, negated, as three bf16 terms; rows past the end of the list never pass
                float r = INFINITY;
                if (t * TM + tid < len) r = (METRIC == KB2_METRIC_L2) ? 0.5f * tv : 0.f;
                uint32_t rh, rm, rl;
                split3_bf16(-r, rh, rm, rl);
                // The chunks of the row are gathered from the codebook into registers BEFORE the A buffer is free: after
                // the consumers hand it back only the stores remain between them and the next tile.
                uint4 v[XCHUNK];
                if constexpr (DSUB == 8) {
                    // chunk = one sub-quantizer (8 bf16): 16 gathers per group through the rotated code bytes.  The table is
                    // laid out [code value][sub-quantizer] (16 B entries): the 8 lanes of a quarter-warp hold 8 consecutive
                    // sub-quantizers, i.e. 8 different 16-byte bank groups whatever their code values => every LDS.128 is
                    // conflict-free (a [sub-quantizer][code value] table costs ~3x the wavefronts with random codes).
                    // v[16 gg + s] is sub-quantizer 16 gg + (s + pos) % 16, pos % 16 == tid % 16.
#pragma unroll
                    for (int gg = 0; gg < G; gg++) {
                        const uint32_t ww[4] = {w[gg].x, w[gg].y, w[gg].z, w[gg].w};
#pragma unroll
                        for (int s = 0; s < 16; s++) {
                            const uint32_t byte = (ww[s >> 2] >> (8 * (s & 3))) & 255u;
                            v[gg * 16 + s] = tab[byte * (16 * G) + gg * 16 + ((s + tid) & 15)];
                        }
                    }
                } else {
                    // chunk = 8 / DSUB consecutive sub-quantizers, assembled from the un-rotated code bytes (static indices)
                    constexpr int SPC = 8 / DSUB;              // sub-quantizers per 16-byte chunk
                    constexpr int WPS = DSUB / 2;              // 32-bit words per sub-quantizer entry
                    const uint32_t* tab32 = reinterpret_cast<const uint32_t*>(tab);
#pragma unroll
                    for (int c = 0; c < XCHUNK; c++) {
                        uint32_t u[4];
#pragma unroll
                        for (int j = 0; j < SPC; j++) {
                            const int m = c * SPC + j;
                            const uint4 wg = w[m >> 4];
                            const int b = m & 15;
                            const uint32_t word = (b < 4) ? wg.x : (b < 8) ? wg.y : (b < 12) ? wg.z : wg.w;
                            const uint32_t byte = (word >> (8 * (b & 3))) & 255u;
#pragma unroll
                            for (int x = 0; x < WPS; x++) u[j * WPS + x] = tab32[(m * 256 + byte) * WPS + x];
                        }
                        v[c] = make_uint4(u[0], u[1], u[2], u[3]);
                    }
                }
                KB2_STALL_BEGIN(t_ae);
                tc::mbar_wait(bar_a_empty(dg), ((g >> 1) & 1u) ^ 1u);
                KB2_STALL_END(1, t_ae);
                unsigned char* A = sm + OFF_A + dg * A_BYTES + (tid >> 3) * GRP_BYTES + (tid & 7) * 16;
#pragma unroll
                for (int c = 0; c < XCHUNK; c++) {
                    const int chunk = (DSUB == 8) ? (c & ~15) + ((c + tid) & 15) : c;
                    *reinterpret_cast<uint4*>(A + chunk * 128) = v[c];
                }
                // test chunk: [-r_hi, -r_mid, -r_lo, 1, 1, 1, 0, 0] (bf16 1.0 = 0x3F80); then a zero chunk
                *reinterpret_cast<uint4*>(A + XCHUNK * 128) = make_uint4(rh | (rm << 16), rl | (0x3F80u << 16), 0x3F803F80u, 0u);
                *reinterpret_cast<uint4*>(A + (XCHUNK + 1) * 128) = make_uint4(0u, 0u, 0u, 0u);
                tc::fence_proxy_async();
                tc::mbar_arrive(bar_a_full(dg));
                KB2_STALL_END(3, t_dec);
            };
            // the first tile of each group only needs a free A buffer: decode it while the tensor pipe still works on
            // the previous item, then stage the B operand (which must wait for that item's last MMA)
            if (t_first < ntiles) decode_tile(t_first);
            // ---- B operand: the item's queries (bf16) gathered by index with cp.async, K-major no-swizzle layout,
            //      plus the threshold chunk [1, 1, 1, h_hi, h_mid, h_lo, 0, 0] of every column
            KB2_STALL_BEGIN(t_b);
            asm volatile("bar.sync 2, 256;" ::: "memory");          // meta[par] (thresholds, query indices) written by all decoders
            KB2_STALL_BEGIN(t_bf);
            tc::mbar_wait(bar_b_free, ((uint32_t)it & 1u) ^ 1u);
            KB2_STALL_END(2, t_bf);
            {
                const float* m_h = (const float*)(sm + OFF_META + par * META_BYTES);
                const int* m_q = (const int*)(m_h + 2 * NQT);
                const uint32_t Bs = base + OFF_B;
                unsigned char* B = sm + OFF_B;
                const int kc = tid >> 3;        // 16-byte chunk along K (0..15)
                const int rsub = tid & 7;
                for (int blk = dg; blk < nmma / 8 && kc < XCHUNK; blk += 2) {
                    const int row = blk * 8 + rsub;
                    const int q = m_q[row];
                    const uint32_t dst = (uint32_t)(blk * GRP_BYTES + kc * 128 + rsub * 16);
                    if (q >= 0) {
                        const void* src = reinterpret_cast<const uint4*>(p.qb16 + (int64_t)q * KD) + kc;
                        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(Bs + dst), "l"(src) : "memory");
                    } else {
                        *reinterpret_cast<uint4*>(B + dst) = make_uint4(0, 0, 0, 0);
                    }
                }
                if (dt < nmma) {   // one column per decoder thread
                    uint32_t hh, hm, hl;
                    split3_bf16(m_h[dt], hh, hm, hl);
                    unsigned char* Bc = B + (dt >> 3) * GRP_BYTES + (dt & 7) * 16;
                    *reinterpret_cast<uint4*>(Bc + XCHUNK * 128) = make_uint4(0x3F803F80u, 0x3F80u | (hh << 16), hm | (hl << 16), 0u);
                    *reinterpret_cast<uint4*>(Bc + (XCHUNK + 1) * 128) = make_uint4(0u, 0u, 0u, 0u);
                }
                asm volatile("cp.async.wait_all;" ::: "memory");
            }
            tc::fence_proxy_async();
            tc::mbar_arrive(bar_b_full);
            KB2_STALL_END(4, t_b);
            // thresholds of the NEXT item (other meta buffer)
            if (item_next < n_items) write_meta(item_next, it + 1);
            // ---- this group's remaining tiles
            for (int t = t_first + 2; t < ntiles; t += 2) decode_tile(t);
            g0 += (uint32_t)ntiles;
            item = item_next;
        }
    } else {
        // =========================== consumers: two warpgroups, warpgroup e owns A buffer e (tiles g % 2 == e) ==========
        // The accumulator holds D = S' + h_col - r_row: a (code, query) pair survives iff D >= 0, i.e. iff its sign bit is
        // clear.  The sign bits are packed into per-row masks while the next block is in flight; survivors are rare
        // (~0.1 %), and go straight to the group's survivor log in global memory (slot range reserved with one
        // shared-memory atomic per thread with survivors and tile; plain stores, nothing waits for them).
        const int et = threadIdx.x - 256;        // 0..255
        const int eg = et >> 7;                  // group
        const int e = et & 127;                  // thread inside the group
        const int we = warp & 3;                 // warp inside the warpgroup: rows 16 we .. 16 we + 15 of a 64-row half
        const uint32_t n_logs = 2u * gridDim.x;  // logs: one per epilogue group
        uint4* my_log = p.log + (size_t)(2 * blockIdx.x + eg) * p.log_cap;
        uint32_t* my_cursor = qcnt + eg;
        bool log_over = false;
        unsigned long long n_codes = 0;
        uint32_t g0 = 0;
        int it = 0;
        for (int item = ring.at_warp(0); item < n_items; item = ring.at_warp(++it)) {
            const int l = p.item_list[item];
            const int nqi = p.item_nq[item];
            // wgmma columns of the item, in 16-column units (1 .. NQT / 16).  The broadcast makes the width dispatch provably
            // warp-uniform: with a bound ptxas must treat as divergent it serializes the wgmmas (C7518).
            const int ncls = __shfl_sync(0xffffffffu, (nqi + 15) >> 4, 0);
            const int len = p.list_len[l];
            const int64_t off = p.list_off[l];
            const int ntiles = (len + TM - 1) / TM;
            const int par = it & 1;
            KB2_STALL_BEGIN(t_mf);
            tc::mbar_wait(bar_meta_full(par), ((uint32_t)it >> 1) & 1u);
            KB2_STALL_END(1, t_mf);
            const float* m_base = (const float*)(sm + OFF_META + par * META_BYTES) + NQT;
            const int* m_q = (const int*)(m_base + NQT);
            if (et == 0) n_codes += (unsigned long long)len * (unsigned long long)nqi;
            const int t_first = (int)((eg - (int)(g0 & 1u)) & 1);
            KB2_STALL_BEGIN(t_bfull);
            tc::mbar_wait(bar_b_full, (uint32_t)it & 1u);
            KB2_STALL_END(2, t_bfull);
            const uint32_t a0 = base + OFF_A + eg * A_BYTES;
            const uint32_t b0 = base + OFF_B;
            const uint32_t la0 = (uint32_t)make_desc_ns(a0, GRP_BYTES), lb0 = (uint32_t)make_desc_ns(b0, GRP_BYTES);
            constexpr uint64_t desc_hi = (uint64_t)(GRP_BYTES >> 4) << 32;   // high word of make_desc_ns (SBO)
            for (int t = t_first; t < ntiles; t += 2) {
                const uint32_t g = g0 + (uint32_t)t;   // g & 1 == eg
                KB2_STALL_BEGIN(t_af);
                tc::mbar_wait(bar_a_full(eg), (g >> 1) & 1u);
                KB2_STALL_END(3, t_af);
                // one block: the 64 codes of half h against the blk::W columns from column blk::C0, into the first W / 2
                // registers of acc
                auto issue = [&](auto& acc, int h, auto blk) {
                    using B = decltype(blk);
                    KB2_STALL_BEGIN(t_is);
                    // the operand descriptors of the wgmmas differ only in the start-address field (address >> 4) of the
                    // low word.  Every shared-memory address of the CTA lies below 2^18, so that 14-bit field never carries
                    // and an offset of x bytes is a 32-bit add of x / 16: one add per descriptor instead of rebuilding it.
                    uint32_t la = la0 + (uint32_t)(h * 8 * GRP_BYTES / 16), lb = lb0 + (uint32_t)(B::C0 / 8 * GRP_BYTES / 16);
                    // <1, 8>: computed here, not hoisted out of the tile loop, where the compiler would keep every K-step's
                    // descriptors in registers that the accumulators need (ptxas then serializes the wgmmas, C7511).  The
                    // <3, 2> geometry is the other way round: it serializes with this barrier and not without.
                    if constexpr (G == 1) asm volatile("" : "+r"(la), "+r"(lb));
                    tc::fence_operand(acc);
                    tc::wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < KSTEPS; ks++)
                        tc::wgmma_bf16<B::W>(acc, desc_hi | (la + ks * 16u), desc_hi | (lb + ks * 16u), ks > 0 ? 1u : 0u);
                    tc::wgmma_commit();
                    tc::fence_operand(acc);
                    KB2_STALL_END(6, t_is);
                };
                // sign test of one block -> bits C0 / 4 + 2 j + cc of the masks of the thread's two rows of half h (column
                // C0 + 8 j + 2 (lane % 4) + cc).  Every column of the block lies below the item's wgmma width, and the
                // columns past its queries fail through h = -inf, so no column mask is needed.  Branch-free: it runs between
                // the issue and the wait of the next block, where divergent code would make ptxas serialize the wgmmas.
                uint64_t mh[2][2] = {{0ull, 0ull}, {0ull, 0ull}};
                auto test = [&](const auto& v, int h, auto blk) {
                    using B = decltype(blk);
                    constexpr int NBIT = B::W / 4, HALF = NBIT / 2;   // bits per row, per chain
                    KB2_STALL_BEGIN(t_te);
                    // sign bit of column 8 j + cc (i = 2 j + cc) of the thread's first / second row -> bit i of n0 / n1.  A
                    // funnel shift (n << 1) | (x >> 31) appends one sign bit in one instruction; columns go in from the
                    // highest i down, in two chains per row (i < HALF, i >= HALF) for instruction-level parallelism.
                    uint32_t n0l = 0u, n0h = 0u, n1l = 0u, n1h = 0u;
#pragma unroll
                    for (int i = HALF - 1; i >= 0; i--) {
                        const int x = 4 * (i >> 1) + (i & 1);   // register of column i of the first row; + 2: second row
                        const int xh = 4 * ((i + HALF) >> 1) + ((i + HALF) & 1);
                        n0l = __funnelshift_l(__float_as_uint(v[x]), n0l, 1);
                        n0h = __funnelshift_l(__float_as_uint(v[xh]), n0h, 1);
                        n1l = __funnelshift_l(__float_as_uint(v[x + 2]), n1l, 1);
                        n1h = __funnelshift_l(__float_as_uint(v[xh + 2]), n1h, 1);
                    }
                    // a pair survives iff its sign bit is clear
                    constexpr uint32_t mask = (1u << NBIT) - 1u;
                    const uint32_t m0 = ~((n0h << HALF) | n0l) & mask, m1 = ~((n1h << HALF) | n1l) & mask;
                    mh[h][0] |= (uint64_t)m0 << (B::C0 / 4);   // h and C0 are compile-time (unrolled pipeline)
                    mh[h][1] |= (uint64_t)m1 << (B::C0 / 4);
                    KB2_STALL_END(7, t_te);
                };
                // survivors of the thread's four rows of the tile -> the group's log.  Survivors are rare (a few per warp and
                // tile), so each thread that has any reserves its own slot range with one shared-memory atomic.
                auto flush = [&]() {
                    const uint32_t total =
                        (uint32_t)(__popcll(mh[0][0]) + __popcll(mh[0][1]) + __popcll(mh[1][0]) + __popcll(mh[1][1]));
                    if (total != 0u) {
                        uint32_t slot = atomicAdd(my_cursor, total);
#pragma unroll
                        for (int h = 0; h < 2; h++) {
#pragma unroll
                            for (int i = 0; i < 2; i++) {
                                const int rel = t * TM + h * 64 + we * 16 + (lane >> 2) + 8 * i;
                                uint64_t m = mh[h][i];
                                while (m) {
                                    const int bit = __ffsll((long long)m) - 1;
                                    m &= m - 1;
                                    const int col = 8 * (bit >> 1) + 2 * (lane & 3) + (bit & 1);
                                    if (slot < p.log_cap) {
                                        uint4 o;
                                        o.x = (uint32_t)m_q[col];
                                        o.y = (uint32_t)(off + rel);
                                        o.z = __float_as_uint(m_base[col]);
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
                };
                // software pipeline over the blocks of the tile: each 64-code half is contracted in NB = ceil(width / MAXW)
                // blocks of near-equal width (half-major, va / vb alternating).  The wgmmas of block b+1 run while block b
                // is tested, across the boundary between the halves too; the survivors are expanded once the whole tile is
                // in registers.  The sequence is unrolled for each width, so every issue, wait and test sits in straight-line
                // code: with the wait inside a run-time loop ptxas cannot prove that the tested buffer has retired, and
                // serializes every wgmma of the kernel (C7514).
                dispatch_range<1, NQT / 16>(ncls, [&](auto nc) {
                    constexpr int NC = decltype(nc)::value, NB = (16 * NC + MAXW - 1) / MAXW, NBT = 2 * NB;
                    // block c of a half: U + (c < X) 16-column units from unit c U + min(c, X)
                    constexpr int U = NC / NB, X = NC % NB;
                    auto blk = [](auto cc) {
                        constexpr int c = decltype(cc)::value;
                        return BlockCols<16 * (c * U + (c < X ? c : X)), 16 * (U + (c < X ? 1 : 0))>{};
                    };
                    // the accumulators live only in here, sized for the widest block (block 0).  The first K-step of a
                    // block overwrites the registers it uses, so they need no initial value.
                    float va[8 * (U + (X > 0 ? 1 : 0))], vb[8 * (U + (X > 0 ? 1 : 0))];
                    issue(va, 0, blk(std::integral_constant<int, 0>{}));
                    static_for<NBT>([&](auto bc) {
                        constexpr int b = decltype(bc)::value;
                        if constexpr (b + 1 < NBT) {
                            constexpr auto bn = blk(std::integral_constant<int, (b + 1) % NB>{});
                            if constexpr ((b + 1) & 1) issue(vb, (b + 1) / NB, bn);
                            else issue(va, (b + 1) / NB, bn);
                            KB2_STALL_BEGIN(t_w);
                            tc::wgmma_wait<1>();
                            KB2_STALL_END(4, t_w);
                        } else {
                            KB2_STALL_BEGIN(t_w);
                            tc::wgmma_wait<0>();
                            KB2_STALL_END(4, t_w);
                        }
                        constexpr auto bb = blk(std::integral_constant<int, b % NB>{});
                        if constexpr (b & 1) {
                            tc::fence_operand(vb);
                            test(vb, b / NB, bb);
                        } else {
                            tc::fence_operand(va);
                            test(va, b / NB, bb);
                        }
                    });
                });
                tc::mbar_arrive(bar_a_empty(eg));   // every wgmma of this tile has retired: hand the A buffer back
                KB2_STALL_BEGIN(t_fl);
                flush();
                KB2_STALL_END(5, t_fl);
            }
            tc::mbar_arrive(bar_b_free);            // this group's wgmmas of the item have all retired
            tc::mbar_arrive(bar_meta_free(par));
            g0 += (uint32_t)ntiles;
        }
        if (log_over) p.log_cnt[n_logs] = 1u;
        if (eg == 0) asm volatile("bar.sync 3, 128;" ::: "memory"); else asm volatile("bar.sync 4, 128;" ::: "memory");
        if (e == 0) {
            const uint32_t n = min(*my_cursor, p.log_cap);
            p.log_cnt[2 * blockIdx.x + eg] = n;
            if (p.counters) atomicAdd(p.counters + 2, (unsigned long long)n);
        }
        if (et == 0 && p.counters) atomicAdd(p.counters, n_codes);
    }
#ifdef KB2_FILTER_STALLS
    // decoder slots: total, a_empty wait, b_free wait, decode_tile (incl. its a_empty wait), B staging (incl. its b_free
    // wait), write_meta
    // consumer slots: total, meta_full wait, b_full wait, a_full wait, wgmma_wait, flush, wgmma issue, sign test
    KB2_STALL_END(0, t_role);
    if ((threadIdx.x & 127) == 0 && blockIdx.x < kStallMaxCtas) {
        for (int i = 0; i < kStallSlots; i++)
            g_filter_stalls[blockIdx.x][warp >= 8][(threadIdx.x >> 7) & 1][i] = (unsigned long long)stall[i];
    }
#endif
}

// bf16 copy + norm of the queries (warp per query, d % 4 == 0)
__global__ void
prepare_queries_kernel(const float* __restrict__ q, int64_t nq, int d, __nv_bfloat16* __restrict__ qb16, float* __restrict__ qnorm) {
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= nq) return;
    float s = 0.f;
    for (int j = lane * 4; j < d; j += 128) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(q + w * d + j));
        __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
        uint2 o;
        o.x = *reinterpret_cast<uint32_t*>(&lo);
        o.y = *reinterpret_cast<uint32_t*>(&hi);
        *reinterpret_cast<uint2*>(qb16 + w * d + j) = o;
        s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    s = warp_sum(s);
    if (lane == 0) qnorm[w] = sqrtf(s) * 1.0001f;
}

// bf16 copy of the PQ codebooks + max_j |c[m][j]|^2 per sub-quantizer (grid = M, block = 256).  Layout: dsub == 8:
// [code value j][sub-quantizer m] (conflict-free gathers in the filter kernel's decode); dsub < 8: [m][j].
__global__ void __launch_bounds__(256)
prepare_tables_kernel(const float* __restrict__ pqc, int dsub, __nv_bfloat16* __restrict__ pqc16, float* __restrict__ maxn2) {
    const int m = blockIdx.x, j = threadIdx.x;
    const int M = gridDim.x;
    const float* c = pqc + ((size_t)m * 256 + j) * dsub;
    float n2 = 0.f;
    __nv_bfloat16* o = pqc16 + (dsub == 8 ? ((size_t)j * M + m) : ((size_t)m * 256 + j)) * dsub;
    for (int t = 0; t < dsub; t++) {
        n2 = fmaf(c[t], c[t], n2);
        o[t] = __float2bfloat16_rn(c[t]);
    }
    __shared__ float red[256];
    red[j] = n2;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (j < s) red[j] = fmaxf(red[j], red[j + s]);
        __syncthreads();
    }
    if (j == 0) maxn2[m] = red[0];
}
// un-rotated copy of the code bytes: plain[g][pos] byte b = sub-quantizer 16 g + b   (rotated: byte s = sub-quantizer (s + pos) % 16)
__global__ void
unrotate_codes_kernel(const uint8_t* __restrict__ rot, int64_t total_words /* G * npad */, int64_t npad, uint8_t* __restrict__ plain) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total_words * 16) return;
    const int s = (int)(t & 15);
    const int64_t word = t >> 4;
    const int64_t pos = word % npad;
    plain[word * 16 + ((s + (int)(pos & 15)) & 15)] = rot[t];
}

// Per-query ADC tables for the whole batch:  lut[q][j*16 + m] = scale * <q_m, c_pq[m][j]>  (scale -2 for L2, -1 for IP),
// each entry the same 8-term fma chain the LUT kernel uses when it builds its table itself, so every consumer
// (phase A, the exact re-evaluation, the LUT kernel's copy-in mode) sees bit-identical values.
// grid = number of SMs, block = 256 (thread = code value j, its 16 sub-vectors live in registers).
template <int METRIC>
__global__ void __launch_bounds__(256, 1)
lut_build_kernel(const float* __restrict__ queries, int64_t nq, const int32_t* __restrict__ qlist, const uint32_t* __restrict__ qcount,
                 const float* __restrict__ pqc, float* __restrict__ lut) {
    // qlist != NULL: table i belongs to query qlist[i], i < *qcount (the queries this rank runs phase A for)
    __shared__ __align__(16) float s_q[2][KD];
    const int j = threadIdx.x;
    const float scale = (METRIC == KB2_METRIC_L2) ? -2.f : -1.f;
    if (qlist) nq = (int64_t)*qcount;
    // thread j keeps the 16 sub-vectors c_pq[.][j] (128 floats) in registers for all the queries of this CTA
    float4 c[32];
#pragma unroll
    for (int m = 0; m < 16; m++) {
        const float* cp = pqc + ((size_t)m * 256 + j) * 8;
        c[2 * m] = __ldg(reinterpret_cast<const float4*>(cp));
        c[2 * m + 1] = __ldg(reinterpret_cast<const float4*>(cp + 4));
    }
    const int64_t per = (nq + gridDim.x - 1) / gridDim.x;
    const int64_t q_beg = (int64_t)blockIdx.x * per, q_end = min(nq, q_beg + per);
    auto qrow = [&](int64_t i) { return queries + (qlist ? (int64_t)qlist[i] : i) * KD; };
    if (q_beg < q_end && threadIdx.x < KD) s_q[0][threadIdx.x] = qrow(q_beg)[threadIdx.x];
    __syncthreads();
    for (int64_t q = q_beg; q < q_end; q++) {
        const int cur = (int)((q - q_beg) & 1);
        if (q + 1 < q_end && threadIdx.x < KD) s_q[cur ^ 1][threadIdx.x] = qrow(q + 1)[threadIdx.x];
        float* dst = lut + q * 4096 + j * 16;
#pragma unroll
        for (int m4 = 0; m4 < 16; m4 += 4) {
            float o[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int m = m4 + u;
                const float4 qa = *reinterpret_cast<const float4*>(&s_q[cur][m * 8]);
                const float4 qb = *reinterpret_cast<const float4*>(&s_q[cur][m * 8 + 4]);
                float a = 0.f;
                a = fmaf(qa.x, c[2 * m].x, a); a = fmaf(qa.y, c[2 * m].y, a); a = fmaf(qa.z, c[2 * m].z, a); a = fmaf(qa.w, c[2 * m].w, a);
                a = fmaf(qb.x, c[2 * m + 1].x, a); a = fmaf(qb.y, c[2 * m + 1].y, a); a = fmaf(qb.z, c[2 * m + 1].z, a); a = fmaf(qb.w, c[2 * m + 1].w, a);
                o[u] = a * scale;
            }
            *reinterpret_cast<float4*>(dst + m4) = make_float4(o[0], o[1], o[2], o[3]);
        }
        __syncthreads();
    }
}

// exact fp32 keys of the survivors: the LUT kernel's own values in its own order — every table entry is the 8-term fma
// chain of <q_m, c_pq[m][code]> times the scale, rounded once (never contracted into the sum), and the 16 entries are
// added into two interleaved accumulators over the stored byte order, key = base + (acc0 + acc1) — so both engines
// produce bit-identical keys.  The entries are recomputed from the fp32 codebook (L1/L2 resident) instead of read from
// a per-query table: no [nq][4096] table has to exist for the queries whose phase A ran on another rank.
// grid = nq, block = 128.  Survivors above the bound are dropped; with k_trim > 0 the row is cut to its k_trim best and compacted.
template <int METRIC, int G, int DSUB>
__global__ void __launch_bounds__(128)
exact_eval_kernel(const float* __restrict__ queries, const float* __restrict__ pqc, const float* __restrict__ lut,
                  const float* __restrict__ bound_of,
                  const uint4* __restrict__ codes, int64_t npad, const float* __restrict__ t1, const uint8_t* __restrict__ bitset,
                  const int32_t* __restrict__ rows, uint64_t* __restrict__ cand, uint32_t* __restrict__ cand_cnt, int cap,
                  uint32_t* __restrict__ qflag, const uint32_t* __restrict__ log_over, int k_trim = 0) {
    constexpr int KDIM = 16 * G * DSUB;
    __shared__ __align__(16) float s_q[KDIM];
    __shared__ uint32_t s_h[256];
    __shared__ float s_red[8];
    __shared__ uint32_t s_ctl[2];   // [0] crossing bin, [1] entries kept
    const int64_t q = blockIdx.x;
    if (*log_over) {
        if (threadIdx.x == 0) qflag[q] = 1u;
        return;
    }
    if (qflag[q]) return;
    const uint32_t n = min(cand_cnt[q], (uint32_t)cap);
    if (n == 0) return;
    // lut != NULL (<1, 8> geometry, single GPU): the batch's tables [nq][256][16] from lut_build_kernel hold exactly these
    // entries; otherwise they are recomputed from the codebook
    const bool use_lut = (G == 1 && DSUB == 8) && lut != nullptr;
    if (!use_lut) {
        for (int j = threadIdx.x; j < KDIM; j += 128) s_q[j] = queries[q * KDIM + j];
        __syncthreads();
    }
    const float* lq = lut + q * 4096;
    const float bound = bound_of[q];
    const float scale = (METRIC == KB2_METRIC_L2) ? -2.f : -1.f;
    uint64_t* row = cand + q * cap;
    // exact key of one logged survivor; returns the packed (key, position) entry, or kEmpty when it is above the bound / filtered
    auto eval = [&](uint64_t ent, float& key_out) -> uint64_t {
        const uint32_t pos = (uint32_t)ent;
        const float base = __uint_as_float((uint32_t)(ent >> 32));
        float acc0 = (METRIC == KB2_METRIC_L2) ? __ldg(t1 + pos) : 0.f, acc1 = 0.f;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const uint4 w = __ldg(codes + (int64_t)g * npad + pos);
            const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int s = 0; s < 16; s++) {
                const uint32_t byte = (ww[s >> 2] >> (8 * (s & 3))) & 255u;
                const uint32_t m = g * 16 + ((pos + s) & 15u);
                float v;
                if (use_lut) {
                    v = __ldg(lq + byte * 16 + m);
                } else {
                    const float* c = pqc + ((size_t)m * 256 + byte) * DSUB;
                    const float* qs = &s_q[m * DSUB];
                    float a = 0.f;
#pragma unroll
                    for (int t = 0; t < DSUB; t++) a = fmaf(qs[t], __ldg(c + t), a);
                    v = __fmul_rn(a, scale);
                }
                if (s & 1) acc1 = __fadd_rn(acc1, v); else acc0 = __fadd_rn(acc0, v);
            }
        }
        const float key = __fadd_rn(base, __fadd_rn(acc0, acc1));
        bool keep = key <= bound;
        if (keep && bitset) keep = !bit_is_set(bitset, rows[pos]);
        key_out = keep ? key : INFINITY;
        return keep ? pack_kp(key, pos) : kEmpty;
    };
    if (k_trim > 0 && n <= 512u && n > (uint32_t)k_trim) {   // CTA-uniform
        // Trim to the k_trim best.  Nearly every logged survivor passes `key <= bound` (the filter's margin is small), and the
        // bound itself comes from a sample of the codes, so a row holds ~4x the k' entries finalize needs (C3: 146 on average,
        // rows above 256 went to the CTA-wide finalize).  All exact keys of the row are here: a 256-bin histogram over their
        // range gives a cut that keeps the k_trim smallest (+ the rest of the crossing bin); the kept entries are compacted
        // to the front of the row (every thread holds its entries in registers before the first write) and the row's count is
        // rewritten.  Shared memory stays at ~1.5 KB so that the L1 keeps serving the table gathers.
        uint64_t pk[4];
        float kf[4];
        float lo = INFINITY, hi = -INFINITY;
        s_h[threadIdx.x] = 0;
        s_h[threadIdx.x + 128] = 0;
        if (threadIdx.x == 0) s_ctl[1] = 0;
#pragma unroll
        for (int it = 0; it < 4; it++) {
            const uint32_t i = threadIdx.x + it * 128;
            pk[it] = kEmpty;
            kf[it] = INFINITY;
            if (i < n) pk[it] = eval(row[i], kf[it]);
            if (kf[it] < INFINITY) { lo = fminf(lo, kf[it]); hi = fmaxf(hi, kf[it]); }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if ((threadIdx.x & 31) == 0) { s_red[threadIdx.x >> 5] = lo; s_red[4 + (threadIdx.x >> 5)] = hi; }
        __syncthreads();   // all entries of the row are in registers from here on
        lo = fminf(fminf(s_red[0], s_red[1]), fminf(s_red[2], s_red[3]));
        hi = fmaxf(fmaxf(s_red[4], s_red[5]), fmaxf(s_red[6], s_red[7]));
        const float sc = (hi > lo) ? 256.f / (hi - lo) : 0.f;
        int bin[4];
#pragma unroll
        for (int it = 0; it < 4; it++) {
            bin[it] = 256;
            if (kf[it] < INFINITY) {
                bin[it] = min(255, (int)((kf[it] - lo) * sc));
                atomicAdd(&s_h[bin[it]], 1u);
            }
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            const int lane = threadIdx.x;
            uint32_t h[8], sum = 0;
#pragma unroll
            for (int t = 0; t < 8; t++) { h[t] = s_h[lane * 8 + t]; sum += h[t]; }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const uint32_t excl = incl - sum;
            const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
            if (lane == 0 && total < (uint32_t)k_trim) s_ctl[0] = 255u;   // fewer than k_trim valid entries: keep them all
            if (excl < (uint32_t)k_trim && incl >= (uint32_t)k_trim) {
                uint32_t run = excl;
                int b = lane * 8 + 7;
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    run += h[t];
                    if (run >= (uint32_t)k_trim) { b = lane * 8 + t; break; }
                }
                s_ctl[0] = (uint32_t)b;
            }
        }
        __syncthreads();
        const int bstar = (int)s_ctl[0];
#pragma unroll
        for (int it = 0; it < 4; it++)
            if (bin[it] <= bstar) row[atomicAdd(&s_ctl[1], 1u)] = pk[it];
        __syncthreads();
        if (threadIdx.x == 0) cand_cnt[q] = s_ctl[1];
        return;
    }
    float lo = INFINITY, hi = -INFINITY;
    for (uint32_t i = threadIdx.x; i < n; i += 128) {
        float kf;
        row[i] = eval(row[i], kf);
        if (kf < INFINITY) { lo = fminf(lo, kf); hi = fmaxf(hi, kf); }
    }
    if (k_trim > 0 && k_trim <= 96 && n > 512u) {   // CTA-uniform
        // Long rows (queries in dense regions: up to `cap` logged survivors) are what the CTA-wide finalize spent its time on
        // (a 2048-entry bitonic sort for the 40 best).  Same cut as above, but the entries stay in global memory: every thread
        // re-reads the packed exact keys it has just written (its own stores), the kept ones are staged in shared memory
        // (at most 128, otherwise the row is left as it is) and written to the front of the row after a barrier.
        __shared__ uint64_t s_stage[128];
        s_h[threadIdx.x] = 0;
        s_h[threadIdx.x + 128] = 0;
        if (threadIdx.x == 0) { s_ctl[0] = 0xffffffffu; s_ctl[1] = 0; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if ((threadIdx.x & 31) == 0) { s_red[threadIdx.x >> 5] = lo; s_red[4 + (threadIdx.x >> 5)] = hi; }
        __syncthreads();
        lo = fminf(fminf(s_red[0], s_red[1]), fminf(s_red[2], s_red[3]));
        hi = fmaxf(fmaxf(s_red[4], s_red[5]), fmaxf(s_red[6], s_red[7]));
        const float sc = (hi > lo) ? 256.f / (hi - lo) : 0.f;
        for (uint32_t i = threadIdx.x; i < n; i += 128) {
            const uint64_t e = row[i];
            if (e != kEmpty) atomicAdd(&s_h[min(255, (int)((unpack_key(e) - lo) * sc))], 1u);
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            const int lane = threadIdx.x;
            uint32_t h[8], sum = 0;
#pragma unroll
            for (int t = 0; t < 8; t++) { h[t] = s_h[lane * 8 + t]; sum += h[t]; }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const uint32_t excl = incl - sum;
            if (excl < (uint32_t)k_trim && incl >= (uint32_t)k_trim) {
                uint32_t run = excl;
                int b = lane * 8 + 7;
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    run += h[t];
                    if (run >= (uint32_t)k_trim) { b = lane * 8 + t; break; }
                }
                if (run <= 128u) s_ctl[0] = (uint32_t)b;   // entries in bins [0, b]: they fit the staging buffer
            }
        }
        __syncthreads();
        const uint32_t bstar = s_ctl[0];
        if (bstar == 0xffffffffu) return;   // fewer than k_trim valid entries, or a crowded crossing bin: leave the row alone
        for (uint32_t i = threadIdx.x; i < n; i += 128) {
            const uint64_t e = row[i];
            if (e != kEmpty && (uint32_t)min(255, (int)((unpack_key(e) - lo) * sc)) <= bstar) s_stage[atomicAdd(&s_ctl[1], 1u)] = e;
        }
        __syncthreads();   // every read of the row is done
        const uint32_t nk = s_ctl[1];
        for (uint32_t i = threadIdx.x; i < nk; i += 128) row[i] = s_stage[i];
        if (threadIdx.x == 0) cand_cnt[q] = nk;
    }
}

// queries whose nearest list is owned by this rank -> compact list: this rank runs their phase A (one CTA; order is irrelevant)
__global__ void __launch_bounds__(1024)
compact_resp_kernel(const int64_t* __restrict__ probe_ids, int nprobe, int64_t nq, const int32_t* __restrict__ list_owner, int rank,
                    int32_t* __restrict__ list, uint32_t* __restrict__ count) {
    __shared__ uint32_t s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int64_t q = threadIdx.x; q < nq; q += 1024) {
        const int64_t l = probe_ids[q * nprobe];
        if (l >= 0 && list_owner[l] == rank) list[atomicAdd(&s_n, 1u)] = (int32_t)q;
    }
    __syncthreads();
    if (threadIdx.x == 0) *count = s_n;
}
__global__ void
fill_f32_kernel(float* __restrict__ out, int64_t n, float v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = v;
}
// max |x[i]| (one atomicMax on the bit pattern of a non-negative float)
__global__ void __launch_bounds__(256)
max_abs_kernel(const float* __restrict__ x, int64_t n, uint32_t* __restrict__ out) {
    float m = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(x[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}

// flagged queries -> compact list (one CTA; order is irrelevant)
__global__ void __launch_bounds__(1024)
compact_flags_kernel(const uint32_t* __restrict__ qflag, int64_t nq, int32_t* __restrict__ list, uint32_t* __restrict__ count) {
    __shared__ uint32_t s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int64_t q = threadIdx.x; q < nq; q += 1024)
        if (qflag[q]) list[atomicAdd(&s_n, 1u)] = (int32_t)q;
    __syncthreads();
    if (threadIdx.x == 0) *count = s_n;
}

// Phase A: exact keys of the codes in the nearest probed lists of every query — lists are taken in probe order until
// `min_codes` codes were seen (at most `p0_max` lists; lists of other shards have length 0 and cost nothing) —
// the k_need-th smallest key (rounded up to a histogram bin edge) -> entry k_need-1 of the query's row = the admission
// bound of the filter pass.  When the lists did not
// hold 4*k_need codes the bound would be loose (a large share of every probed list would survive): the row is left
// without a bound and the LUT kernel redoes that query.
// The query's table is copied from `lut` into a skewed shared layout: code value j owns a row of 32 words,
// row[w] = LUT[w % 16][j]; lane i reads word (i % 16) + s at step s, i.e. sub-quantizer (pos + s) % 16 — the address
// is one byte-permute plus an immediate (PRMT + LDS + FADD per look-up, like the LUT kernel), lanes i and i+16 share
// a bank (2 wavefronts per gather).  The keys go to shared memory and the bound is read off a 1024-bin histogram
// (no top-k structure at all).  grid = nq, block = NT (128 or 256); dynamic smem = bound_smem(bound_kmax(...)) (48 KB at C3).
#define KB2_BOUND_STEP(WORD, KB, S, ACC)                                                      \
    {                                                                                         \
        const uint32_t _x = __byte_perm((WORD), lane4, 0x6504u | ((KB) << 4));                \
        float _v;                                                                             \
        asm("ld.shared.f32 %0, [%1+%2];" : "=f"(_v) : "r"(_x >> 1), "n"(KB2_SMEM_BASE + 4 * (S))); \
        ACC += _v;                                                                            \
    }
// pqc [M][256][dsub] -> pqc_t [M/16][256][16][dsub] (the 16 sub-quantizers of a group adjacent: coalesced table builds)
__global__ void
transpose_codebook_kernel(const float* __restrict__ pqc, int M, int dsub, float* __restrict__ pqc_t) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)M * 256 * dsub;
    if (i >= n) return;
    const int x = (int)(i % dsub);
    const int j = (int)((i / dsub) % 256);
    const int m = (int)(i / ((int64_t)dsub * 256));
    pqc_t[((((int64_t)(m >> 4) * 256 + j) * 16) + (m & 15)) * dsub + x] = pqc[i];
}
constexpr int BOUND_KMAX = 6144;    // keys held per query (phase A looks at no more codes than this)
constexpr int BOUND_BINS = 1024;
// keys actually held for a launch: the requested number of codes rounded up (C3: 3000 -> 3008 keys = 12 KB instead of 24 KB, i.e.
// 48 KB per CTA and four CTAs per SM instead of three)
__host__ __device__ constexpr int bound_kmax(int min_codes, int k_need) {
    const int want = ((min_codes > k_need ? min_codes : k_need) + 63) & ~63;
    return want < BOUND_KMAX ? want : BOUND_KMAX;
}
// the 32 KB skewed table, the keys, the histogram and the reduction words
constexpr size_t bound_smem(int kmax) { return (size_t)32 * 1024 + (size_t)kmax * 4 + BOUND_BINS * 4 + 128; }

// G > 1 (m = 16 G sub-quantizers, e.g. m48 x dsub2): the groups are scanned one after the other through the same 32 KB
// table -- group g's table is built in the kernel from the query and the transposed codebook `pqc_t`
// ([g][code value][16 sub-quantizers][dsub], see transpose_codebook_kernel), the partial sums of the earlier groups wait in
// the shared key array.
// NT = threads per CTA: 128 (4 warps) or 256 (8 warps over the same tables: twice the gathers in flight per shared-memory byte)
template <int METRIC, int G, int DSUB, int NT>
__global__ void __launch_bounds__(NT)
bound_kernel(const float* __restrict__ lut, const int32_t* __restrict__ qlist, const uint32_t* __restrict__ qcount, int64_t nq,
             const int64_t* __restrict__ probe_ids, const float* __restrict__ probe_dis,
             int probe_stride, int p0_max, int min_codes, int k_need, const int64_t* __restrict__ list_off,
             const int32_t* __restrict__ list_len, const uint4* __restrict__ codes, const float* __restrict__ t1,
             const uint8_t* __restrict__ bitset, const int32_t* __restrict__ rows, float* __restrict__ out,
             unsigned long long* __restrict__ counters, int64_t npad = 0, const float* __restrict__ queries = nullptr,
             const float* __restrict__ pqc_t = nullptr) {
    static_assert(NT == 128 || NT == 256, "bound_kernel block size");
    constexpr int NW = NT / 32;               // warps
    constexpr int BPT = BOUND_BINS / NT;      // histogram bins owned by a thread
    // work list: table i / query qlist[i] for i < *qcount (qlist == NULL: query i, i < nq); CTAs stride the list
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_lut = (float*)smem_raw;                              // [256][32]
    const int key_cap = bound_kmax(min_codes, k_need);            // (the host sizes the shared memory with the same function)
    float* s_keys = (float*)(smem_raw + 32 * 1024);               // [key_cap]
    uint32_t* s_hist = (uint32_t*)(s_keys + key_cap);             // [BOUND_BINS]
    float* s_red = (float*)(s_hist + BOUND_BINS);                 // [32]: min [0,8) max [8,16) warp sums [16,24)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if ((uint32_t)__cvta_generic_to_shared(smem_raw) != (uint32_t)KB2_SMEM_BASE) {
        if (threadIdx.x == 0 && counters) atomicExch(counters + 1, 0xBAD5ull);   // layout assumption violated: host raises an error
        return;
    }
    const int64_t n_work = qlist ? (int64_t)*qcount : nq;
    for (int64_t wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
    const int64_t q = qlist ? (int64_t)qlist[wi] : wi;
    int seen = 0, n_tot = 0;
    float kmin = INFINITY, kmax = -INFINITY;
#pragma unroll 1
    for (int g = 0; g < G; g++) {
    __syncthreads();   // the previous iteration's readers of the shared tables are done
    if constexpr (G > 1 || DSUB != 8) {
        // table of group g from the query: entry (j, mm) = scale * <q_m, c_pq[m][j]>, m = 16 g + mm
        const float scale = (METRIC == KB2_METRIC_L2) ? -2.f : -1.f;
        const int mm = threadIdx.x & 15, jsub = threadIdx.x >> 4;   // 16 sub-quantizers x 8 code values per pass
        float qv[DSUB];
#pragma unroll
        for (int x = 0; x < DSUB; x++) qv[x] = queries[q * (int64_t)(16 * G * DSUB) + (g * 16 + mm) * DSUB + x];
        for (int j = jsub; j < 256; j += NT / 16) {
            const float* cp = pqc_t + (((size_t)g * 256 + j) * 16 + mm) * DSUB;
            float a = 0.f;
#pragma unroll
            for (int x = 0; x < DSUB; x++) a = fmaf(qv[x], __ldg(cp + x), a);
            a *= scale;
            s_lut[j * 32 + mm] = a;
            s_lut[j * 32 + 16 + mm] = a;
        }
    } else {
        // lut[q][j*16 + m] -> s_lut[j*32 + m] and s_lut[j*32 + 16 + m]
        const float4* src = reinterpret_cast<const float4*>(lut + wi * 4096);
#pragma unroll
        for (int i = 0; i < 1024 / NT; i++) {
            const int idx = threadIdx.x + i * NT;        // float4 index: j = idx / 4, m4 = (idx % 4) * 4
            const float4 v = __ldg(src + idx);
            float4* dst = reinterpret_cast<float4*>(s_lut + (idx >> 2) * 32 + (idx & 3) * 4);
            dst[0] = v;
            dst[4] = v;
        }
    }
    if (g == 0)
        for (int i = threadIdx.x; i < BOUND_BINS; i += NT) s_hist[i] = 0;
    __syncthreads();
    // PRMT builds (byte << 8) | (lane16 << 3) ; >> 1 = byte * 128 + lane16 * 4 (row pitch 128 B)
    const uint32_t lane4 = (uint32_t)(lane & 15) << 3;
    const uint4* gcodes = codes + (int64_t)g * npad;   // code plane of this group
    const bool first_g = (g == 0), last_g = (g == G - 1);
    seen = 0;
    n_tot = 0;
    const int code_cap = min(key_cap, max(min_codes, k_need));   // scan no more than the requested number of codes
    for (int j = 0; j < p0_max && seen < min_codes && n_tot < code_cap; j++) {
        const int64_t l = probe_ids[q * probe_stride + j];
        if (l < 0) continue;
        const int len_all = list_len[l];
        if (len_all == 0) continue;
        seen += len_all;
        const int len = min(len_all, code_cap - n_tot);   // any subset of the codes still yields a valid upper bound
        const int64_t off = list_off[l];
        const float dv = probe_dis[q * probe_stride + j];
        const float base = (METRIC == KB2_METRIC_L2) ? dv : -dv;
        // two chunks per iteration, software-pipelined: the code words / row terms of the NEXT iteration are in
        // flight while the gather chains of this one run (the kernel was latency bound on these loads)
        uint4 nA = make_uint4(0, 0, 0, 0), nB = nA;
        float ntA = 0.f, ntB = 0.f;
        auto load_iter = [&](int c0) {
            if (c0 < len) {
                nA = ldg_stream_u4(gcodes + off + c0 + lane);        // inside the padded position space even past len
                if (METRIC == KB2_METRIC_L2 && first_g) ntA = __ldg(t1 + off + c0 + lane);
                if (c0 + 32 < len) {
                    nB = ldg_stream_u4(gcodes + off + c0 + 32 + lane);
                    if (METRIC == KB2_METRIC_L2 && first_g) ntB = __ldg(t1 + off + c0 + 32 + lane);
                }
            }
        };
        load_iter(warp * 64);
        for (int c0 = warp * 64; c0 < len; c0 += NW * 64) {
            const int relA = c0 + lane, relB = c0 + 32 + lane;
            const bool okA = relA < len, okB = relB < len;
            const uint32_t posA = (uint32_t)(off + relA), posB = (uint32_t)(off + relB);
            const bool hasB = c0 + 32 < len;
            const uint4 wA = nA;
            const uint4 wB = hasB ? nB : nA;
            float a0 = ntA, a1 = 0.f, b0 = hasB ? ntB : 0.f, b1 = 0.f;
            load_iter(c0 + NW * 64);
            KB2_BOUND_STEP(wA.x, 0, 0, a0)  KB2_BOUND_STEP(wB.x, 0, 0, b0)  KB2_BOUND_STEP(wA.x, 1, 1, a1)  KB2_BOUND_STEP(wB.x, 1, 1, b1)
            KB2_BOUND_STEP(wA.x, 2, 2, a0)  KB2_BOUND_STEP(wB.x, 2, 2, b0)  KB2_BOUND_STEP(wA.x, 3, 3, a1)  KB2_BOUND_STEP(wB.x, 3, 3, b1)
            KB2_BOUND_STEP(wA.y, 0, 4, a0)  KB2_BOUND_STEP(wB.y, 0, 4, b0)  KB2_BOUND_STEP(wA.y, 1, 5, a1)  KB2_BOUND_STEP(wB.y, 1, 5, b1)
            KB2_BOUND_STEP(wA.y, 2, 6, a0)  KB2_BOUND_STEP(wB.y, 2, 6, b0)  KB2_BOUND_STEP(wA.y, 3, 7, a1)  KB2_BOUND_STEP(wB.y, 3, 7, b1)
            KB2_BOUND_STEP(wA.z, 0, 8, a0)  KB2_BOUND_STEP(wB.z, 0, 8, b0)  KB2_BOUND_STEP(wA.z, 1, 9, a1)  KB2_BOUND_STEP(wB.z, 1, 9, b1)
            KB2_BOUND_STEP(wA.z, 2, 10, a0) KB2_BOUND_STEP(wB.z, 2, 10, b0) KB2_BOUND_STEP(wA.z, 3, 11, a1) KB2_BOUND_STEP(wB.z, 3, 11, b1)
            KB2_BOUND_STEP(wA.w, 0, 12, a0) KB2_BOUND_STEP(wB.w, 0, 12, b0) KB2_BOUND_STEP(wA.w, 1, 13, a1) KB2_BOUND_STEP(wB.w, 1, 13, b1)
            KB2_BOUND_STEP(wA.w, 2, 14, a0) KB2_BOUND_STEP(wB.w, 2, 14, b0) KB2_BOUND_STEP(wA.w, 3, 15, a1) KB2_BOUND_STEP(wB.w, 3, 15, b1)
            float keyA = (first_g ? base : s_keys[n_tot + (okA ? relA : 0)]) + (a0 + a1);
            float keyB = (first_g ? base : s_keys[n_tot + ((hasB && okB) ? relB : 0)]) + (b0 + b1);
            if (okA) {
                if (last_g && bitset && bit_is_set(bitset, rows[posA])) keyA = INFINITY;
                s_keys[n_tot + relA] = keyA;
                if (last_g && keyA < INFINITY) { kmin = fminf(kmin, keyA); kmax = fmaxf(kmax, keyA); }
            }
            if (hasB && okB) {
                if (last_g && bitset && bit_is_set(bitset, rows[posB])) keyB = INFINITY;
                s_keys[n_tot + relB] = keyB;
                if (last_g && keyB < INFINITY) { kmin = fminf(kmin, keyB); kmax = fmaxf(kmax, keyB); }
            }
        }
        n_tot += len;
    }
    }   // groups
    // ---- K-th smallest key, rounded UP to the edge of one of 1024 linear bins over [min, max]: any value >= the
    //      k_need-th best is a valid admission bound, and a bin is far narrower than the filter's error margin
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        kmin = fminf(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
        kmax = fmaxf(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
    }
    if (lane == 0) { s_red[warp] = kmin; s_red[8 + warp] = kmax; }
    __syncthreads();
    float lo = s_red[0], hi = s_red[8];
#pragma unroll
    for (int w = 1; w < NW; w++) { lo = fminf(lo, s_red[w]); hi = fmaxf(hi, s_red[8 + w]); }
    const float scale = (hi > lo) ? (float)BOUND_BINS / (hi - lo) : 0.f;
    for (int i = threadIdx.x; i < n_tot; i += NT) {
        const float kv = s_keys[i];
        if (kv < INFINITY) atomicAdd(&s_hist[min(BOUND_BINS - 1, (int)((kv - lo) * scale))], 1u);
    }
    __syncthreads();
    // thread t owns bins [BPT t, BPT (t+1)): exclusive prefix over threads, then the owner of the crossing writes the bound
    uint32_t mine[BPT], tsum = 0;
#pragma unroll
    for (int b = 0; b < BPT; b++) { mine[b] = s_hist[threadIdx.x * BPT + b]; tsum += mine[b]; }
    uint32_t incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    uint32_t* s_wsum = (uint32_t*)(s_red + 16);
    if (lane == 31) s_wsum[warp] = incl;
    __syncthreads();
    uint32_t before = incl - tsum;
    for (int w = 0; w < warp; w++) before += s_wsum[w];
    uint32_t total = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) total += s_wsum[w];
    const uint32_t need = (uint32_t)k_need;
    if (total < need || seen < 4 * k_need) {
        if (threadIdx.x == 0) out[q] = INFINITY;   // no (or only a loose) bound: the LUT kernel redoes the query
    } else if (before < need && before + tsum >= need) {
        uint32_t cum = before;
        int b = 0;
#pragma unroll
        for (int bb = 0; bb < BPT; bb++) {
            if (cum < need) { cum += mine[bb]; b = bb; }
        }
        const float bound = (scale > 0.f) ? lo + ((float)(threadIdx.x * BPT + b) + 1.01f) / scale : hi;
        out[q] = fmaxf(bound, lo) + (G == 1 ? 4e-7f : 2e-6f) * fmaxf(fabsf(lo), fabsf(hi));
    }
    }   // work list
}
#undef KB2_BOUND_STEP

}  // namespace pqtc
}  // namespace kb2
