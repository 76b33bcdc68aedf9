// kb2_ivf.cuh — inverted-list scan kernels (IVF_FLAT exact scan, IVF_PQ LUT + ADC scan).
//
// Reference path being replaced (one CPU task per query):
//   IndexIVF::search_preassigned / scan_one_list          F/IndexIVF.cpp:401-768
//   IVFFlatScanner::scan_codes                            K/IndexIVFFlat.cpp:139-232
//   QueryTables::init_query / precompute_list_tables_*    F/impl/pq_code_distance/IVFPQ_QueryTables.cpp:44-192
//   IVFPQScanner::scan_list_with_table                    F/impl/pq_code_distance/IVFPQScanner_impl.h:110-185
//
// HBM layout (built by IvfIndex::seal()):
//   list l occupies positions [list_off[l], list_off[l] + list_len[l]) of the position space;
//   list_off is a multiple of 32 so that  (position % 32) == lane  inside the scan.
//   IVF_FLAT : vecs[pos][d] fp32 (list order)
//   IVF_PQ   : codes[g][pos] one uint4 per 16 sub-quantizers ("group" g), byte s of the uint4 holds
//              code[g*16 + ((s + pos) % 16)]  (bytes rotated by pos%16, see the LUT layout below)
//              t1[pos] fp32 (L2 only) = sum_m ( |c_pq[m][code_m]|^2 + 2 <c_list[m], c_pq[m][code_m]> )
//              which is exactly the reference's precomputed-table term summed over m
//              (F/IndexIVFPQ.cpp:407-513; IVFPQ_QueryTables.cpp:139-151) and depends on the stored
//              vector only, so it is folded at add() time.
//   rows[pos] int32 internal row id (insertion index) — read only for winners / bitset tests.
//
// ADC identity used (L2, by_residual):   |q - c - r^|^2 = |q-c|^2 + (|r^|^2 + 2<c,r^>) - 2<q,r^>
//   => key = dis0(q,l) + t1(pos) + sum_m LUT[m][code_m],   LUT[m][j] = -2 <q_m, c_pq[m][j]>
// The LUT therefore depends on the QUERY ONLY (one table per query instead of the reference's one
// table per (query, probed list): 64x less LUT work at nprobe=64).  IP: key = -(<q,c> + sum <q_m,c_pq>).
//
// Shared-memory LUT layout ("skewed, conflict-free"): for group g, code value j (0..255) owns a row of
// 64 floats at byte offset g*65536 + j*256; row[w] = LUT[g*16 + (w % 16)][j] for w = 0..63.
// Lane i at step s reads row word (i + s): bank = (i + s) % 32 is distinct for the 32 lanes no matter
// which code values they hold => every LDS is a single conflict-free wavefront (a plain [m][256]
// table costs ~3.4 wavefronts per gather with random codes).  Word (i+s) holds sub-quantizer
// (i+s)%16, which is why byte s of the stored code of position p is sub-quantizer (s+p)%16.
// Address = (code_byte << 8) | (lane << 2)  (+ 4*s as an immediate) comes from ONE byte-permute.
#pragma once
#include "kb2_topk.cuh"

namespace kb2 {

struct IvfScanParams {
    const float* queries;      // [nq][d]
    int nq, d;
    int metric;
    // probes from the coarse stage (finalize_kernel output)
    const int64_t* probe_ids;  // [nq][nprobe]
    const float* probe_dis;    // [nq][nprobe]  L2: |q-c|^2 ; IP: <q,c>
    int nprobe;
    const int64_t* list_off;   // [nlist]
    const int32_t* list_len;   // [nlist]  (0 for lists owned by another shard)
    int nsplit;                // CTAs per query
    int K, kout;               // per-warp list size / entries written per CTA
    uint64_t* partial;         // [nq][nsplit][kout]
    const uint8_t* bitset;     // internal-row bitmap or NULL
    const int32_t* rows;       // [npad]
    // IVF_FLAT
    const float* vecs;         // [npad][d]
    // IVF_PQ
    const float* pq_centroids; // [M][256][dsub]
    int M, dsub;
    const uint4* codes;        // [G][npad]
    int64_t npad;
    const float* t1;           // [npad] or NULL
    unsigned long long* counters;  // [0] codes scanned (optional, NULL to skip)
    const int32_t* qperm;          // [nq] visiting order of the queries (NULL: identity)
    int probe_stride;              // row stride of probe_ids/probe_dis (0: nprobe) — lets a pass scan only the first nprobe probes
    int64_t partial_stride;        // entries between the output rows of consecutive queries (0: nsplit*kout)
    const float* lut_global;       // [nq][G*4096] precomputed tables in the kernel's own enumeration ((g, j, m): m fastest), or NULL
    const uint32_t* only_flagged;  // non-NULL selects the redo pass of the tensor-core engine: a small grid walks
    const int32_t* flag_list;      //   the compacted list of flagged queries (flag_list[0..*flag_count)) x nsplit probe slices
    const uint32_t* flag_count;
    int clear_to;                  // the LAST probe slice fills its output with kEmpty from entry kout up to this entry count
};

// probe bookkeeping in shared memory
struct ProbeSmem {
    uint32_t* start;   // [np+1] first chunk index of probe j (chunks of 32 positions)
    uint32_t* off;     // [np]   list start position
    int32_t* len;      // [np]
    float* dis0;       // [np]   key base: L2 dis0, IP -<q,c>
};

__device__ __forceinline__ int
setup_probes(const IvfScanParams& p, int64_t q, int j0, int j1, ProbeSmem ps) {
    // serial prefix over <= a few hundred probes
    const int np = j1 - j0;
    const int64_t pstride = p.probe_stride ? p.probe_stride : p.nprobe;
    for (int j = threadIdx.x; j < np; j += blockDim.x) {
        const int64_t l = p.probe_ids[q * pstride + j0 + j];
        int len = 0;
        uint32_t off = 0;
        if (l >= 0) {
            len = p.list_len[l];
            off = (uint32_t)p.list_off[l];
        }
        ps.len[j] = len;
        ps.off[j] = off;
        const float dv = p.probe_dis[q * pstride + j0 + j];
        ps.dis0[j] = (p.metric == KB2_METRIC_L2) ? dv : -dv;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (int j = 0; j < np; j++) {
            ps.start[j] = acc;
            acc += (uint32_t)((ps.len[j] + 31) >> 5);
        }
        ps.start[np] = acc;
    }
    __syncthreads();
    return (int)ps.start[np];
}

// Shared-window address of the dynamic shared memory of a non-cluster CTA on sm_90 (as on every GPU since sm_80): the first
// 1 KB of the window is reserved by the system, so `extern __shared__` starts at 0x400.  The scan
// kernel checks this at run time (and reports through counters[1]) because the LUT gather folds
// the base into the LDS immediate:  LDS dst, [ (code<<8 | lane<<2) + KB2_SMEM_BASE + g*64K + 4*s ].
#define KB2_SMEM_BASE 1024

#define KB2_LUT_STEP(WORD, K, S, ACC)                                                         \
    {                                                                                         \
        const uint32_t _x = __byte_perm((WORD), lane4, 0x6504u | ((K) << 4));                 \
        float _v;                                                                             \
        asm("ld.shared.f32 %0, [%1+%2];" : "=f"(_v) : "r"(_x), "n"(KB2_SMEM_BASE + GRP * 65536 + 4 * (S))); \
        ACC += _v;                                                                            \
    }

// 16 conflict-free gathers of one 16-sub-quantizer group: PRMT + LDS + FADD per lookup
template <int GRP>
__device__ __forceinline__ void
pq_group_sum(const uint4& w, uint32_t lane4, float& acc0, float& acc1, float& acc2, float& acc3) {
    KB2_LUT_STEP(w.x, 0, 0, acc0)  KB2_LUT_STEP(w.x, 1, 1, acc1)  KB2_LUT_STEP(w.x, 2, 2, acc2)  KB2_LUT_STEP(w.x, 3, 3, acc3)
    KB2_LUT_STEP(w.y, 0, 4, acc0)  KB2_LUT_STEP(w.y, 1, 5, acc1)  KB2_LUT_STEP(w.y, 2, 6, acc2)  KB2_LUT_STEP(w.y, 3, 7, acc3)
    KB2_LUT_STEP(w.z, 0, 8, acc0)  KB2_LUT_STEP(w.z, 1, 9, acc1)  KB2_LUT_STEP(w.z, 2, 10, acc2) KB2_LUT_STEP(w.z, 3, 11, acc3)
    KB2_LUT_STEP(w.w, 0, 12, acc0) KB2_LUT_STEP(w.w, 1, 13, acc1) KB2_LUT_STEP(w.w, 2, 14, acc2) KB2_LUT_STEP(w.w, 3, 15, acc3)
}

// =====================================================================================
// IVF_PQ scan.  G = M/16 groups.  grid = nq * nsplit, block = 256.
// dynamic smem: G*65536 (LUT, first) | NW*2K*8 (candidate buffers) | probes | query | CTA bound block
// =====================================================================================
// one in-flight 32-code chunk of the software pipeline (all warp-uniform except w/t/pos/ok)
template <int G>
struct PqStage {
    uint4 w[G];
    float t;        // t1[pos]
    float d0;       // key base of the probe this chunk belongs to
    uint32_t pos;
    bool ok;        // lane's position is inside the list
    bool valid;     // stage holds a chunk (warp-uniform)
};

template <int G, int METRIC, bool HAS_BITSET>
__device__ __forceinline__ void
ivfpq_scan_body(const IvfScanParams& p, const int64_t bq, const int split) {
    constexpr int NW = kScanWarps;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned char* lut = smem_raw;
    uint64_t* lists = (uint64_t*)(smem_raw + (size_t)G * 65536);
    const int np_max = (p.nprobe + p.nsplit - 1) / p.nsplit;
    ProbeSmem ps;
    ps.start = (uint32_t*)(lists + NW * 2 * p.K);
    ps.off = ps.start + np_max + 1;
    ps.len = (int32_t*)(ps.off + np_max);
    ps.dis0 = (float*)(ps.len + np_max);
    float* s_q = ps.dis0 + np_max;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // queries are visited in the order given by qperm (sorted by nearest list => CTAs that run
    // together probe the same lists and hit them in L2)
    const int64_t q = p.qperm ? (int64_t)p.qperm[bq] : bq;
    const int j0 = min(p.nprobe, split * np_max), j1 = min(p.nprobe, j0 + np_max);
    const int np = j1 - j0;
    if ((uint32_t)__cvta_generic_to_shared(smem_raw) != (uint32_t)KB2_SMEM_BASE) {
        // layout assumption violated: flag it, the host turns this into an error (never a silent wrong answer)
        if (threadIdx.x == 0 && p.counters) atomicExch(p.counters + 1, 0xBAD5ull);
        return;
    }

    for (int i = threadIdx.x; i < p.d; i += blockDim.x) s_q[i] = p.queries[q * p.d + i];
    setup_probes(p, q, j0, j1, ps);  // contains __syncthreads
    if (p.counters && threadIdx.x == 0) {
        unsigned long long tot = 0;
        for (int j = 0; j < np; j++) tot += (unsigned long long)ps.len[j];
        atomicAdd(p.counters, tot);   // codes scanned by this CTA
    }

    // ---- LUT build: value(m, j) = scale * <q_m, c_pq[m][j]>, replicated at words m%16 + 16t.
    // Thread mapping chosen for conflict-free stores: within a warp, lanes 0-15 take the 16 sub-quantizers of
    // code value j, lanes 16-31 those of j+1 (same banks, one row = 64 words later), so the two half-warps
    // write DIFFERENT replicas in each of the four store steps (banks m+16r vs m+16(r^1)).
    {
        const float scale = (METRIC == KB2_METRIC_L2) ? -2.f : -1.f;
        const int dsub = p.dsub;
        const int half = lane >> 4;
        const int mm = threadIdx.x & 15;   // blockDim % 16 == 0: a thread keeps its sub-quantizer-in-group
        float qr[8];                       // its query sub-vector in registers when dsub <= 8 (no smem re-reads)
        int g_loaded = -1;
        for (int e = threadIdx.x; e < p.M * 256; e += blockDim.x) {
            // e enumerates (group g, code value j, sub-quantizer-in-group mm): mm fastest, then j
            const int j = (e >> 4) & 255;
            const int g = e >> 12;
            if (p.lut_global) {
                // tables of the whole batch were built by pqtc::lut_build_kernel (same fma chain): coalesced copy
                const float v = __ldg(p.lut_global + (int64_t)q * (p.M * 256) + e);
                float* row = (float*)(lut + (size_t)g * 65536 + (size_t)j * 256);
#pragma unroll
                for (int r = 0; r < 4; r++) row[mm + 16 * (r ^ half)] = v;
                continue;
            }
            const int m = g * 16 + mm;
            const float* c = p.pq_centroids + ((int64_t)m * 256 + j) * dsub;
            const float* qs = s_q + m * dsub;
            float acc = 0.f;
            if (dsub <= 8) {
                if (g != g_loaded) {
#pragma unroll
                    for (int t = 0; t < 8; t++) qr[t] = t < dsub ? qs[t] : 0.f;
                    g_loaded = g;
                }
                if (dsub == 8) {
                    const float4 c0 = *reinterpret_cast<const float4*>(c);
                    const float4 c1 = *reinterpret_cast<const float4*>(c + 4);
                    acc = fmaf(qr[0], c0.x, acc); acc = fmaf(qr[1], c0.y, acc);
                    acc = fmaf(qr[2], c0.z, acc); acc = fmaf(qr[3], c0.w, acc);
                    acc = fmaf(qr[4], c1.x, acc); acc = fmaf(qr[5], c1.y, acc);
                    acc = fmaf(qr[6], c1.z, acc); acc = fmaf(qr[7], c1.w, acc);
                } else {
#pragma unroll
                    for (int t = 0; t < 8; t++)
                        if (t < dsub) acc = fmaf(qr[t], c[t], acc);
                }
            } else if ((dsub & 3) == 0) {
                for (int t = 0; t < dsub; t += 4) {
                    const float4 cv = *reinterpret_cast<const float4*>(c + t);
                    acc = fmaf(qs[t], cv.x, acc);
                    acc = fmaf(qs[t + 1], cv.y, acc);
                    acc = fmaf(qs[t + 2], cv.z, acc);
                    acc = fmaf(qs[t + 3], cv.w, acc);
                }
            } else {
                for (int t = 0; t < dsub; t++) acc = fmaf(qs[t], c[t], acc);
            }
            acc *= scale;
            float* row = (float*)(lut + (size_t)g * 65536 + (size_t)j * 256);
#pragma unroll
            for (int r = 0; r < 4; r++) row[mm + 16 * (r ^ half)] = acc;
        }
    }
    WarpTopK tk;
    tk.init(lists + warp * 2 * p.K, p.K, lane);
    uint64_t* merge_tmp;
    uint32_t* merge_ctr;
    unsigned long long* sh_V_final;
    {
        // CTA-wide admission bound (see WarpTopK): 8-byte aligned block after the query
        unsigned long long* shb = (unsigned long long*)(((uintptr_t)(s_q + p.d) + 7) & ~(uintptr_t)7);
        tk.share(shb, shb + NW, NW, warp, lane);
        merge_tmp = (uint64_t*)(shb + NW + 2);      // 4K-entry compaction buffer for the final merge
        merge_ctr = (uint32_t*)(merge_tmp + 4 * p.K);
        sh_V_final = shb + NW;
    }
    __syncthreads();

    // ---- scan: the warps stride the 32-code chunks of all probed lists; three chunks in flight
    const uint32_t lane4 = (uint32_t)lane << 2;
    // chunk iterator (warp-uniform registers; probe arrays are touched only when the probe changes)
    int it_j = 0, it_ci = warp, it_nch = 0, it_len = 0;
    uint32_t it_off = 0;
    float it_d0 = 0.f;
    auto it_load = [&]() {
        while (it_j < np) {
            it_len = ps.len[it_j];
            it_nch = (it_len + 31) >> 5;
            if (it_ci < it_nch) {
                it_off = ps.off[it_j];
                it_d0 = ps.dis0[it_j];
                return;
            }
            it_ci -= it_nch;
            it_j++;
        }
    };
    it_load();

    auto fetch = [&](PqStage<G>& st) {
        st.valid = it_j < np;
        st.ok = false;
        if (!st.valid) return;
        const uint32_t rel = (uint32_t)it_ci * 32u + lane;
        st.pos = it_off + rel;
        st.ok = (int)rel < it_len;
        st.d0 = it_d0;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const uint4* cp = p.codes + (int64_t)g * p.npad + st.pos;
            st.w[g] = ldg_stream_u4(cp);
            // pull the chunk this warp will want four iterations from now into L2 (same list most of the
            // time; a stray prefetch into the next list or the tail padding is harmless)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(cp + 4 * NW * 32));
        }
        if (METRIC == KB2_METRIC_L2) {
            st.t = __ldg(p.t1 + st.pos);
            if (lane == 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.t1 + st.pos + 4 * NW * 32));
        } else {
            st.t = 0.f;
        }
        it_ci += NW;
        if (it_ci >= it_nch) it_load();
    };
    auto adc_key = [&](const PqStage<G>& st) -> float {
        float acc0 = st.t, acc1 = 0.f;
        pq_group_sum<0>(st.w[0], lane4, acc0, acc1, acc0, acc1);
        if (G > 1) pq_group_sum<1>(st.w[G > 1 ? 1 : 0], lane4, acc0, acc1, acc0, acc1);
        if (G > 2) pq_group_sum<2>(st.w[G > 2 ? 2 : 0], lane4, acc0, acc1, acc0, acc1);
        return st.d0 + (acc0 + acc1);
    };
    auto admit = [&](const PqStage<G>& st, float key, float bound) {
        bool pass = st.ok && key <= bound;            // one float compare on the hot path
        if (HAS_BITSET && pass) pass = !bit_is_set(p.bitset, p.rows[st.pos]);
        if (__any_sync(0xffffffffu, pass)) tk.push(pack_kp(key, st.pos), pass, lane);
    };
    // two chunks are evaluated together: 2 x 16 independent PRMT/LDS/FADD chains per warp hide the
    // shared-memory and ALU latencies that 24 resident warps alone cannot
    auto process2 = [&](const PqStage<G>& a, const PqStage<G>& b) {
        const float ka = adc_key(a);
        const float kb = b.valid ? adc_key(b) : 0.f;
        // hot path: one shared load + min; the exact (key,pos) test happens inside push()
        const float bound = fminf(tk.thr_key, tk.shared_key());
        admit(a, ka, bound);
        if (b.valid) admit(b, kb, fminf(tk.thr_key, bound));
    };

    PqStage<G> s0, s1, s2, s3;
    fetch(s0);
    fetch(s1);
    fetch(s2);
    fetch(s3);
    for (;;) {
        if (!s0.valid) break;
        process2(s0, s1);
        fetch(s0);
        fetch(s1);
        if (!s2.valid) break;
        process2(s2, s3);
        fetch(s2);
        fetch(s3);
    }

    uint64_t* out = p.partial_stride ? p.partial + (int64_t)q * p.partial_stride + (int64_t)split * p.kout
                                     : p.partial + ((int64_t)q * p.nsplit + split) * p.kout;
    if (split == p.nsplit - 1)   // only the last slice clears the rest of the row
        for (int i = p.kout + threadIdx.x; i < p.clear_to; i += blockDim.x) out[i] = kEmpty;
    tk.finish(lane);
    __syncthreads();
    block_emit_topk_bounded(lists, p.K, NW, *sh_V_final, merge_tmp, 4 * p.K, merge_ctr, out, p.kout);
}

template <int G, int METRIC, bool HAS_BITSET>
__global__ void __launch_bounds__(kScanThreads, G == 1 ? 3 : 1)
ivfpq_scan_kernel(IvfScanParams p) {
    if (p.only_flagged) {
        // redo pass of the tensor-core engine: a small grid walks the (query, probe slice) units and scans only the
        // flagged queries (every iteration is self-contained; the barrier keeps a fast warp out of the next unit's smem)
        const int64_t units = (int64_t)(*p.flag_count) * p.nsplit;
        for (int64_t w = blockIdx.x; w < units; w += gridDim.x) {
            const int64_t bq = p.flag_list[w / p.nsplit];
            const int split = (int)(w % p.nsplit);
            if (threadIdx.x == 0 && split == 0 && p.counters) atomicAdd(p.counters + 3, 1ull);   // queries redone by this pass
            ivfpq_scan_body<G, METRIC, HAS_BITSET>(p, bq, split);
            __syncthreads();
        }
        return;
    }
    ivfpq_scan_body<G, METRIC, HAS_BITSET>(p, (int64_t)(blockIdx.x / p.nsplit), (int)(blockIdx.x % p.nsplit));
}

// =====================================================================================
// IVF_PQ scan with a plain [M][256] table (M KB of shared memory, bank-conflicted gathers), any M, nbits=8.  Same math
// as ivfpq_scan_kernel in another summation order.  Used when M % 16 != 0 or M > 48 (G == 0: codes stored un-rotated as
// bytes codes_b[pos*M + m]), and as the fallback of the skewed kernel (G > 0: the rotated groups of p.codes) when its
// 64 KB per 16 sub-quantizers do not fit beside the candidate buffers of a large k or the probe arrays of many probes.
// dynamic smem: M*1024 | lists | probes | query
// =====================================================================================
template <int METRIC>
__device__ __forceinline__ void
ivfpq_scan_generic_body(const IvfScanParams& p, const uint8_t* __restrict__ codes_b, int G, const int64_t bq, const int split) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* lut = (float*)smem_raw;
    uint64_t* lists = (uint64_t*)(smem_raw + (size_t)p.M * 1024);
    const int np_max = (p.nprobe + p.nsplit - 1) / p.nsplit;
    ProbeSmem ps;
    ps.start = (uint32_t*)(lists + kScanWarps * 2 * p.K);
    ps.off = ps.start + np_max + 1;
    ps.len = (int32_t*)(ps.off + np_max);
    ps.dis0 = (float*)(ps.len + np_max);
    float* s_q = ps.dis0 + np_max;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = p.qperm ? (int64_t)p.qperm[bq] : bq;
    const int j0 = min(p.nprobe, split * np_max), j1 = min(p.nprobe, j0 + np_max);
    for (int i = threadIdx.x; i < p.d; i += blockDim.x) s_q[i] = p.queries[q * p.d + i];
    const int nchunks = setup_probes(p, q, j0, j1, ps);
    if (p.counters && threadIdx.x == 0) {
        unsigned long long tot = 0;
        for (int j = 0; j < j1 - j0; j++) tot += (unsigned long long)ps.len[j];
        atomicAdd(p.counters, tot);   // codes scanned by this CTA
    }
    const float scale = (METRIC == KB2_METRIC_L2) ? -2.f : -1.f;
    for (int e = threadIdx.x; e < p.M * 256; e += blockDim.x) {
        const int m = e >> 8;
        const float* c = p.pq_centroids + (int64_t)e * p.dsub;
        float acc = 0.f;
        for (int t = 0; t < p.dsub; t++) acc = fmaf(s_q[m * p.dsub + t], c[t], acc);
        lut[e] = acc * scale;
    }
    WarpTopK tk;
    tk.init(lists + warp * 2 * p.K, p.K, lane);
    __syncthreads();
    int cur = 0;
    for (int c = warp; c < nchunks; c += kScanWarps) {
        while (c >= (int)ps.start[cur + 1]) cur++;
        const uint32_t rel = ((uint32_t)c - ps.start[cur]) * 32u + lane;
        const uint32_t pos = ps.off[cur] + rel;
        bool valid = (int)rel < ps.len[cur];
        float acc = 0.f;
        if (valid) {
            acc = (METRIC == KB2_METRIC_L2) ? p.t1[pos] : 0.f;
            if (G > 0) {
                // byte s of group g's 16-byte word holds sub-quantizer g*16 + ((s + pos) % 16)
                for (int g = 0; g < G; g++) {
                    const uint8_t* cb = (const uint8_t*)(p.codes + (int64_t)g * p.npad + pos);
                    for (int s = 0; s < 16; s++) acc += lut[(g * 16 + ((s + pos) & 15)) * 256 + cb[s]];
                }
            } else {
                const uint8_t* cb = codes_b + (int64_t)pos * p.M;
                for (int m = 0; m < p.M; m++) acc += lut[m * 256 + cb[m]];
            }
            if (p.bitset) valid = !bit_is_set(p.bitset, p.rows[pos]);
        }
        tk.push(pack_kp(ps.dis0[cur] + acc, pos), valid, lane);
    }
    uint64_t* out = p.partial_stride ? p.partial + (int64_t)q * p.partial_stride + (int64_t)split * p.kout
                                     : p.partial + ((int64_t)q * p.nsplit + split) * p.kout;
    if (split == p.nsplit - 1)   // only the last slice clears the rest of the row
        for (int i = p.kout + threadIdx.x; i < p.clear_to; i += blockDim.x) out[i] = kEmpty;
    tk.finish(lane);
    block_emit_topk(lists, p.K, out, p.kout);
}

// codes_b: un-rotated bytes (G == 0) or unused (G > 0: p.codes)
template <int METRIC>
__global__ void __launch_bounds__(kScanThreads)
ivfpq_scan_generic_kernel(IvfScanParams p, const uint8_t* __restrict__ codes_b, int G) {
    if (p.only_flagged) {
        // redo pass of the tensor-core engine (see ivfpq_scan_kernel)
        const int64_t units = (int64_t)(*p.flag_count) * p.nsplit;
        for (int64_t w = blockIdx.x; w < units; w += gridDim.x) {
            const int64_t bq = p.flag_list[w / p.nsplit];
            const int split = (int)(w % p.nsplit);
            if (threadIdx.x == 0 && split == 0 && p.counters) atomicAdd(p.counters + 3, 1ull);
            ivfpq_scan_generic_body<METRIC>(p, codes_b, G, bq, split);
            __syncthreads();
        }
        return;
    }
    ivfpq_scan_generic_body<METRIC>(p, codes_b, G, (int64_t)(blockIdx.x / p.nsplit), (int)(blockIdx.x % p.nsplit));
}

// =====================================================================================
// IVF_FLAT exact scan (query-major).  One warp handles 32 consecutive positions per step, lanes
// stride the dimension with float4 loads; distances are the directly accumulated
// sum((q-x)^2) / sum(q*x) like fvec_L2sqr / fvec_inner_product (src/simd/distances_ref.cc:22-38).
// dynamic smem: lists | probes | query (16B aligned)
// =====================================================================================
template <int METRIC>
__global__ void __launch_bounds__(kScanThreads)
ivfflat_scan_kernel(IvfScanParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_q = (float*)smem_raw;                       // d floats, d % 4 == 0 (padded layout)
    uint64_t* lists = (uint64_t*)(s_q + p.d);
    const int np_max = (p.nprobe + p.nsplit - 1) / p.nsplit;
    ProbeSmem ps;
    ps.start = (uint32_t*)(lists + kScanWarps * 2 * p.K);
    ps.off = ps.start + np_max + 1;
    ps.len = (int32_t*)(ps.off + np_max);
    ps.dis0 = (float*)(ps.len + np_max);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.x / p.nsplit;
    const int split = blockIdx.x % p.nsplit;
    const int j0 = min(p.nprobe, split * np_max), j1 = min(p.nprobe, j0 + np_max);
    for (int i = threadIdx.x; i < p.d; i += blockDim.x) s_q[i] = p.queries[q * p.d + i];
    const int nchunks = setup_probes(p, q, j0, j1, ps);
    WarpTopK tk;
    tk.init(lists + warp * 2 * p.K, p.K, lane);
    __syncthreads();

    const int nv = p.d >> 2;  // float4 per row
    const float4* q4 = reinterpret_cast<const float4*>(s_q);
    int cur = 0;
    unsigned long long scanned = 0;
    for (int c = warp; c < nchunks; c += kScanWarps) {
        while (c >= (int)ps.start[cur + 1]) cur++;
        const uint32_t rel0 = ((uint32_t)c - ps.start[cur]) * 32u;
        const uint32_t pos0 = ps.off[cur] + rel0;
        const int nrows = min(32, ps.len[cur] - (int)rel0);
        float mykey = INFINITY;
        const float4* base = reinterpret_cast<const float4*>(p.vecs) + (int64_t)pos0 * nv;
        for (int r0 = 0; r0 < nrows; r0 += 4) {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            for (int v = lane; v < nv; v += kWarp) {
                const float4 qv = q4[v];
                float4 x[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    // rows past nrows are still inside the padded allocation (never selected)
                    x[u] = ldg_stream_f4(base + (int64_t)(r0 + u) * nv + v);
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (METRIC == KB2_METRIC_L2) {
                        float t;
                        t = qv.x - x[u].x; acc[u] = fmaf(t, t, acc[u]);
                        t = qv.y - x[u].y; acc[u] = fmaf(t, t, acc[u]);
                        t = qv.z - x[u].z; acc[u] = fmaf(t, t, acc[u]);
                        t = qv.w - x[u].w; acc[u] = fmaf(t, t, acc[u]);
                    } else {
                        acc[u] = fmaf(qv.x, x[u].x, acc[u]);
                        acc[u] = fmaf(qv.y, x[u].y, acc[u]);
                        acc[u] = fmaf(qv.z, x[u].z, acc[u]);
                        acc[u] = fmaf(qv.w, x[u].w, acc[u]);
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const float s = warp_sum(acc[u]);
                if (lane == r0 + u) mykey = (METRIC == KB2_METRIC_L2) ? s : -s;
            }
        }
        bool valid = lane < nrows;
        const uint32_t pos = pos0 + lane;
        if (p.bitset && valid) valid = !bit_is_set(p.bitset, p.rows[pos]);
        scanned += (lane < nrows) ? 1ull : 0ull;
        tk.push(pack_kp(mykey, pos), valid, lane);
    }
    if (p.counters) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) scanned += __shfl_xor_sync(0xffffffffu, scanned, o);
        if (lane == 0) atomicAdd(p.counters, scanned);
    }
    uint64_t* out = p.partial + ((int64_t)q * p.nsplit + split) * p.kout;
    tk.finish(lane);
    block_emit_topk(lists, p.K, out, p.kout);
}

// ============================================================================================
// Row scan with directly accumulated distances: RangeSearch (kb2_range.cuh) and the dense key rows of the large-k path.
// ============================================================================================
struct RangeParams {
    IvfScanParams sp;
    int kind;            // 0 vectors [pos][d], 1 PQ rotated groups, 2 PQ plain bytes
    int G;
    const uint8_t* codes_b;
    float radius, range_filter;
    int has_filter;
    RangeHit* hits;
    unsigned long long* count;
    unsigned long long cap;
    int64_t single_len;  // FLAT: one pseudo-list [0, single_len) (probe arrays unused)
    // Dense emission (the large-k path, kb2_large_k.cuh): instead of appending in-range hits, every probed row that is not
    // filtered writes (key, position) to a fixed slot of its query's row dense[i][*] (i = launch row): FLAT the position
    // itself, IVF the rank of its 32-row chunk among all the query's probed chunks (probe order) * 32 + lane.  Slots nobody
    // writes keep what the caller filled them with (kEmpty).  Row i is query qlist[i], or q0 + i without a list.
    uint64_t* dense;
    int64_t dense_ld;
    const uint32_t* qlist;
    int64_t q0;
    int64_t bit_base;    // bitset position of row 0 when rows are stored in row order (a FLAT or HNSW shard's shard_lo)
    unsigned long long* scanned;   // dense mode, optional: rows scanned
};

__device__ __forceinline__ bool
in_range(float dist, float radius, float range_filter, int has_filter, int metric) {
    if (metric == KB2_METRIC_L2) return dist < radius && (!has_filter || dist >= range_filter);
    return dist > radius && (!has_filter || dist <= range_filter);
}

static inline bool
in_range_host(float dist, float radius, float range_filter, bool has_filter, int metric) {
    if (metric == KB2_METRIC_L2) return dist < radius && (!has_filter || dist >= range_filter);
    return dist > radius && (!has_filter || dist <= range_filter);
}

// grid = rows * nsplit (rows = nq, or the dense mode's launch rows).  dynamic smem: query | [M*1024 LUT for PQ] | probes
__global__ void __launch_bounds__(kScanThreads)
range_scan_kernel(RangeParams rp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const IvfScanParams& p = rp.sp;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t qi = blockIdx.x / p.nsplit;
    const int64_t q = rp.qlist ? (int64_t)rp.qlist[qi] : rp.q0 + qi;
    const int split = blockIdx.x % p.nsplit;
    float* s_q = (float*)smem_raw;
    float* lut = s_q + p.d;
    const size_t lut_floats = (rp.kind == 0) ? 0 : (size_t)p.M * 256;
    const int np_max = (rp.single_len >= 0) ? 1 : (p.nprobe + p.nsplit - 1) / p.nsplit;
    ProbeSmem ps;
    ps.start = (uint32_t*)(lut + lut_floats);
    ps.off = ps.start + np_max + 1;
    ps.len = (int32_t*)(ps.off + np_max);
    ps.dis0 = (float*)(ps.len + np_max);

    for (int i = threadIdx.x; i < p.d; i += blockDim.x) s_q[i] = p.queries[q * p.d + i];
    int nchunks;
    int j0 = 0;
    uint32_t chunk_base = 0;   // dense IVF rows: chunks of the query's probes before this CTA's first one
    if (rp.single_len >= 0) {
        // FLAT: split the row range across the nsplit CTAs in multiples of 32 rows
        const int64_t per = ((rp.single_len + p.nsplit - 1) / p.nsplit + 31) / 32 * 32;
        const int64_t b = min((long long)rp.single_len, (long long)split * per);
        const int64_t e = min((long long)rp.single_len, (long long)(b + per));
        if (threadIdx.x == 0) {
            ps.start[0] = 0;
            ps.off[0] = (uint32_t)b;
            ps.len[0] = (int32_t)(e - b);
            ps.dis0[0] = 0.f;
            ps.start[1] = (uint32_t)((e - b + 31) / 32);
        }
        __syncthreads();
        nchunks = (int)ps.start[1];
    } else {
        j0 = min(p.nprobe, split * np_max);
        const int j1 = min(p.nprobe, j0 + np_max);
        nchunks = setup_probes(p, q, j0, j1, ps);
        if (rp.dense) {
            // block-wide sum over the probes before j0 (up to 65535 of them), accumulated in the word after the probe
            // arrays (inside the 64 bytes every IVF launch adds to them; no static shared memory, so that the launch
            // helper may raise the dynamic limit to kMaxDynSmem)
            uint32_t* s_chunk_base = (uint32_t*)(ps.dis0 + np_max);
            if (threadIdx.x == 0) *s_chunk_base = 0;
            __syncthreads();
            const int64_t pstride = p.probe_stride ? p.probe_stride : p.nprobe;
            uint32_t part = 0;
            for (int j = threadIdx.x; j < j0; j += blockDim.x) {
                const int64_t l = p.probe_ids[q * pstride + j];
                if (l >= 0) part += (uint32_t)((p.list_len[l] + 31) >> 5);
            }
            if (part) atomicAdd(s_chunk_base, part);
            __syncthreads();
            chunk_base = *s_chunk_base;
        }
    }
    if (rp.kind != 0) {
        const float scale = (p.metric == KB2_METRIC_L2) ? -2.f : -1.f;
        for (int e = threadIdx.x; e < p.M * 256; e += blockDim.x) {
            const int m = e >> 8;
            const float* c = p.pq_centroids + (int64_t)e * p.dsub;
            float acc = 0.f;
            for (int t = 0; t < p.dsub; t++) acc = fmaf(s_q[m * p.dsub + t], c[t], acc);
            lut[e] = acc * scale;
        }
    }
    __syncthreads();

    if (rp.scanned && threadIdx.x == 0) {
        unsigned long long rows_here = 0;
        const int np_here = (rp.single_len >= 0) ? 1 : min(p.nprobe, j0 + np_max) - j0;
        for (int j = 0; j < np_here; j++) rows_here += (unsigned long long)ps.len[j];
        if (rows_here) atomicAdd(rp.scanned, rows_here);
    }
    int cur = 0;
    for (int c = warp; c < nchunks; c += kScanWarps) {
        while (c >= (int)ps.start[cur + 1]) cur++;
        const uint32_t rel0 = ((uint32_t)c - ps.start[cur]) * 32u;
        const uint32_t pos0 = ps.off[cur] + rel0;
        const int nrows = min(32, ps.len[cur] - (int)rel0);
        float mykey = INFINITY;
        if (rp.kind == 0) {
            for (int r = 0; r < nrows; r++) {
                const float* x = p.vecs + (int64_t)(pos0 + r) * p.d;
                float acc = 0.f;
                if (p.metric == KB2_METRIC_L2) {
                    for (int j = lane; j < p.d; j += kWarp) {
                        const float t = s_q[j] - x[j];
                        acc = fmaf(t, t, acc);
                    }
                } else {
                    for (int j = lane; j < p.d; j += kWarp) acc = fmaf(s_q[j], x[j], acc);
                }
                acc = warp_sum(acc);
                if (lane == r) mykey = (p.metric == KB2_METRIC_L2) ? acc : -acc;
            }
        } else if (lane < nrows) {
            const uint32_t pos = pos0 + lane;
            float acc = (p.metric == KB2_METRIC_L2) ? p.t1[pos] : 0.f;
            if (rp.kind == 1) {
                for (int g = 0; g < rp.G; g++) {
                    const uint8_t* cb = (const uint8_t*)(p.codes + (int64_t)g * p.npad + pos);
                    for (int s = 0; s < 16; s++) acc += lut[(g * 16 + ((s + pos) & 15)) * 256 + cb[s]];
                }
            } else {
                const uint8_t* cb = rp.codes_b + (int64_t)pos * p.M;
                for (int m = 0; m < p.M; m++) acc += lut[m * 256 + cb[m]];
            }
            mykey = ps.dis0[cur] + acc;
        }
        if (rp.dense) {
            if (lane < nrows) {
                const uint32_t pos = pos0 + lane;
                const bool ok = !p.bitset || !bit_is_set(p.bitset, p.rows ? (int64_t)p.rows[pos] : rp.bit_base + (int64_t)pos);
                const int64_t slot = (rp.single_len >= 0) ? (int64_t)pos : ((int64_t)chunk_base + c) * 32 + lane;
                if (ok) rp.dense[qi * rp.dense_ld + slot] = pack_kp(mykey, pos);
            }
        } else if (lane < nrows) {
            const uint32_t pos = pos0 + lane;
            bool ok = true;
            if (p.bitset) ok = !bit_is_set(p.bitset, p.rows ? (int64_t)p.rows[pos] : rp.bit_base + (int64_t)pos);
            const float dist = (p.metric == KB2_METRIC_L2) ? mykey : -mykey;
            if (ok && in_range(dist, rp.radius, rp.range_filter, rp.has_filter, p.metric)) {
                const unsigned long long slot = atomicAdd(rp.count, 1ull);
                if (slot < rp.cap) {
                    RangeHit h;
                    h.q = (int32_t)q;
                    h.probe = j0 + cur;
                    h.pos = pos;
                    h.dist = dist;
                    rp.hits[slot] = h;
                }
            }
        }
    }
}

}  // namespace kb2
