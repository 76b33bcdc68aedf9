// kb2_topk.cuh — k-selection primitives shared by every scan kernel.
//
// Semantics we implement (documented deviation, see DESIGN.md "ties"): results are the k smallest
// under the TOTAL order (key, id).  The reference's binary heap admits a candidate only on strict
// improvement and evicts the (value,id)-largest root (K/impl/ResultHandler.h:238-245,
// F/utils/Heap.h:113-160), which yields the same set unless several candidates tie *exactly*
// with the k-th distance; the final ordering (distance, then id) is identical
// (heap_reorder, F/utils/Heap.h; F/IndexIVF.cpp:484-494).
#pragma once
#include <cuda_fp16.h>
#include <float.h>

#include "kb2_common.cuh"

namespace kb2 {

// --------------------------------------------------------------------------------------------
// Per-warp top-K, "append and prune".  The warp owns a buffer of 2K packed (key,pos) entries in
// shared memory.  Candidates below the warp-uniform threshold are appended (one ballot + one
// predicated store per 32 candidates); when the buffer would overflow it is bitonic-sorted in place
// and cut back to the best K, which also tightens the threshold to the K-th best seen so far.
// Cost: ~2 ln(N/K) prunes per warp instead of ~K ln(N/K) list updates.
// --------------------------------------------------------------------------------------------
struct WarpTopK {
    uint64_t* buf;   // shared memory, 2K entries
    int K;           // power of two, >= 32
    int cnt;         // entries in buf (warp-uniform)
    uint64_t thr;    // admission threshold (kEmpty until the first prune); warp-uniform
    float thr_key;   // key part of thr (+inf until the first prune): cheap float pre-filter `key <= thr_key`
    // CTA-wide bound exchange (optional): every warp publishes its (K/nwarps)-th best after a prune;
    // V = max over warps of those values has at least nwarps*(K/nwarps) = K distinct candidates at or
    // below it, so it is a valid admission bound for EVERY warp and ~nwarps times tighter (in quantile)
    // than a warp's own K-th best.  Published values only ever decrease, so stale reads stay valid.
    unsigned long long* sh_p;   // [nwarps] shared memory, or nullptr
    unsigned long long* sh_V;   // shared memory scalar
    float* sh_Vkey;             // key part of *sh_V (hot-path pre-filter reads only this)
    uint32_t sh_Vkey_addr;      // its shared-window address
    int nwarps, warp_id;

    __device__ __forceinline__ void
    init(uint64_t* b, int k, int lane) {
        buf = b;
        K = k;
        cnt = 0;
        thr = kEmpty;
        thr_key = INFINITY;
        sh_p = nullptr;
        sh_V = nullptr;
        sh_Vkey = nullptr;
        nwarps = 1;
        warp_id = 0;
        (void)lane;
    }
    // call before the first push; the caller zero-initialises nothing: slots start at kEmpty here
    __device__ __forceinline__ void
    share(unsigned long long* p, unsigned long long* V, int nw, int w, int lane) {
        if (K / nw < 1) return;
        sh_p = p;
        sh_V = V;
        sh_Vkey = reinterpret_cast<float*>(V + 1);
        sh_Vkey_addr = (uint32_t)__cvta_generic_to_shared(sh_Vkey);
        nwarps = nw;
        warp_id = w;
        if (lane == 0) sh_p[w] = kEmpty;
        if (w == 0 && lane == 0) { *sh_V = kEmpty; *sh_Vkey = INFINITY; }
    }
    // hot path: pre-filter key of the CTA-wide bound (one LDS; thr_key = min(own, shared) by the caller)
    // (requires share(); explicit shared-space load — a volatile generic load would compile to LD.E.STRONG.SYS)
    __device__ __forceinline__ float
    shared_key() const {
        float v;
        asm volatile("ld.volatile.shared.f32 %0, [%1];" : "=f"(v) : "r"(sh_Vkey_addr));
        return v;
    }
    // adopt the CTA-wide bound if it is tighter (one LDS.64 + compare)
    __device__ __forceinline__ void
    refresh() {
        if (sh_V) {
            unsigned long long v;
            asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"((uint32_t)__cvta_generic_to_shared(sh_V)));
            if (v < thr) {
                thr = v;
                thr_key = unpack_key(v);
            }
        }
    }

    // in-place ascending bitonic sort of the 2K-entry buffer by one warp (unused tail = kEmpty)
    __device__ __forceinline__ void
    prune(int lane) {
        const int n = 2 * K;
        for (int i = cnt + lane; i < n; i += kWarp) buf[i] = kEmpty;
        __syncwarp();
        for (int k2 = 2; k2 <= n; k2 <<= 1) {
            for (int j = k2 >> 1; j > 0; j >>= 1) {
                for (int t = lane; t < (n >> 1); t += kWarp) {
                    const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // index with bit j clear
                    const int p = i | j;
                    const uint64_t a = buf[i], b = buf[p];
                    const bool asc = ((i & k2) == 0);
                    if ((a > b) == asc) { buf[i] = b; buf[p] = a; }
                }
                __syncwarp();
            }
        }
        cnt = min(cnt, K);
        uint64_t nt = buf[K - 1];  // kEmpty while fewer than K candidates exist
        if (sh_p) {
            if (lane == 0) {
                sh_p[warp_id] = buf[K / nwarps - 1];
                unsigned long long V = 0;
                for (int w = 0; w < nwarps; w++) {
                    const unsigned long long pw = ((volatile unsigned long long*)sh_p)[w];
                    V = pw > V ? pw : V;
                }
                const unsigned long long old = atomicMin(sh_V, V);
                if (V < old) *(volatile float*)sh_Vkey = unpack_key(V);   // racy but monotone enough: any published
                                                                          // key belongs to a valid bound
            }
            __syncwarp();
            const unsigned long long v = *(volatile unsigned long long*)sh_V;
            nt = v < nt ? v : nt;
        }
        if (nt < thr) thr = nt;
        thr_key = (thr == kEmpty) ? INFINITY : unpack_key(thr);
    }

    // all 32 lanes must call; `valid` lanes offer `cand`
    __device__ __forceinline__ void
    push(uint64_t cand, bool valid, int lane) {
        refresh();
        bool pass = valid && cand < thr;
        unsigned m = __ballot_sync(0xffffffffu, pass);
        if (m == 0) return;
        if (cnt + __popc(m) > 2 * K) {
            prune(lane);
            pass = valid && cand < thr;
            m = __ballot_sync(0xffffffffu, pass);
            if (m == 0) return;
        }
        if (pass) buf[cnt + __popc(m & ((1u << lane) - 1u))] = cand;
        cnt += __popc(m);
    }

    // final prune: afterwards buf[0..K) is sorted ascending (kEmpty padded), buf[K..2K) = kEmpty
    __device__ __forceinline__ void
    finish(int lane) {
        __syncwarp();
        prune(lane);
        for (int i = K + lane; i < 2 * K; i += kWarp) buf[i] = kEmpty;
        __syncwarp();
    }
};

// --------------------------------------------------------------------------------------------
// CTA-wide bitonic sort of n (power of two) u64 keys in shared memory, ascending.
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ void
block_bitonic_sort(uint64_t* s, int n) {
    for (int k2 = 2; k2 <= n; k2 <<= 1) {
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                int ixj = i ^ j;
                if (ixj > i) {
                    uint64_t a = s[i], b = s[ixj];
                    bool asc = ((i & k2) == 0);
                    if ((a > b) == asc) { s[i] = b; s[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// After every warp called WarpTopK::finish(): the kScanWarps buffers (2K entries each, contiguous in
// `lists`) are sorted CTA-wide and the best `kout` written to out[0..kout).
__device__ __forceinline__ void
block_emit_topk(uint64_t* lists, int K, uint64_t* __restrict__ out, int kout, int nwarps = kScanWarps) {
    __syncthreads();
    block_bitonic_sort(lists, nwarps * 2 * K);
    for (int i = threadIdx.x; i < kout; i += blockDim.x) out[i] = lists[i];
}

// Cheaper CTA merge when the warps exchanged a CTA-wide bound V (WarpTopK::share): every entry of the final
// top-K is <= V and V is the max of the warps' (K/nwarps)-th best, so only the (typically K..2K) entries <= V
// need sorting.  They are compacted into `tmp` (capacity cap, power of two, >= K) and sorted there; if more than
// `cap` entries qualify the full sort is used.  `ctr` is one shared u32.  All threads of the CTA call this.
__device__ __forceinline__ void
block_emit_topk_bounded(uint64_t* lists, int K, int nwarps, unsigned long long V, uint64_t* tmp, int cap, uint32_t* ctr,
                        uint64_t* __restrict__ out, int kout) {
    __syncthreads();                      // every warp has finished (buffers sorted, [0,K) valid)
    if (threadIdx.x == 0) *ctr = 0;
    for (int i = threadIdx.x; i < cap; i += blockDim.x) tmp[i] = kEmpty;
    __syncthreads();
    for (int i = threadIdx.x; i < nwarps * K; i += blockDim.x) {
        const uint64_t e = lists[(i / K) * 2 * K + (i % K)];
        if (e != kEmpty && e <= V) {
            const uint32_t slot = atomicAdd(ctr, 1u);
            if (slot < (uint32_t)cap) tmp[slot] = e;
        }
    }
    __syncthreads();
    if (*ctr <= (uint32_t)cap) {          // CTA-uniform
        block_bitonic_sort(tmp, cap);
        for (int i = threadIdx.x; i < kout; i += blockDim.x) out[i] = i < cap ? tmp[i] : kEmpty;
    } else {
        block_bitonic_sort(lists, nwarps * 2 * K);
        for (int i = threadIdx.x; i < kout; i += blockDim.x) out[i] = lists[i];
    }
}

// --------------------------------------------------------------------------------------------
// Finalize: one CTA per query.
//   1. gather this query's partial candidate lists, CTA bitonic sort, keep the best k_sel
//   2. optional exact re-rank of those candidates from raw fp32 vectors (FLAT exactness,
//      IVF coarse dis0, IVF_PQ refine: K/IndexRefine.cpp:66-160)
//   3. order by (key, label) and emit k_out (ids int64, dist fp32); pad with -1 / +-FLT_MAX
// --------------------------------------------------------------------------------------------
struct FinalizeParams {
    const uint64_t* partial;   // [nq][partial_stride], first n_partial entries of each row are used
    int64_t partial_stride;
    int n_partial;             // entries per query
    int n_sort;                // next_pow2(n_partial) (<= 8192)
    int k_sel;                 // candidates kept after the sort (<= 1024)
    int k_out;                 // results written per query
    const int32_t* rows;       // pos -> internal row id (NULL: identity)
    const int64_t* labels;     // row -> label (NULL: identity)
    int rerank;                // 1: recompute keys exactly from `raw`
    const float* raw;          // [*][d] fp32
    const uint16_t* raw16;     // or [*][d] fp16 / bf16 (refine_type fp16 / bf16: src/index/refine/refine_utils.cc:99-160); NULL: use raw
    int raw16_kind;            // 1 fp16, 2 bf16
    int raw_by_pos;            // 1: raw indexed by pos, 0: by row
    const float* queries;      // [nq][d]
    int d;
    int metric;                // KB2_METRIC_L2 / KB2_METRIC_IP
    int64_t* out_ids;          // [nq][k_out]
    float* out_dist;           // [nq][k_out]
    int32_t* out_pos;          // optional [nq][k_out] positions (NULL: skip)
    const uint32_t* counts;    // optional [nq]: only the first min(counts[q], n_partial) entries of a row are valid ...
    const uint32_t* count_flags;   // ... unless count_flags[q] != 0 (then all n_partial are)
    int split_small;           // > 0: rows with at most this many valid entries were handled by finalize_warp_kernel: skip them
    int64_t row_loop_nq;       // > 0: finalize_kernel strides the rows [0, row_loop_nq) with its grid (0: row = blockIdx.x)
    uint32_t* cert;            // optional certification of an exact re-rank of norm-expanded keys (FLAT, see fin_certify):
                               //   [0] bits of max |x|^2 over the base (input); [1] count and [2..] list of the queries
                               //   whose result is not certified (output; requires rerank)
    const int32_t* qlist;      // optional: row i of the launch is query qlist[i] (the FLAT redo of uncertified queries)
};

// Relative error of the approximate FLAT keys |q|^2 + |x|^2 - 2 q.x (L2) and -q.x (IP), as a share of |q|^2 + max|x|^2 (L2)
// or |q| max|x| (IP): fin_cert_rel(d) = max(3e-5, (d + 8) 2^-22).
//  * (d + 8) 2^-22 comes from the rounding model of the contraction: every fp32 sum of the dot product and of the norms is
//    off by at most 2^-23 of the running magnitude, and each 3xTF32 product (hi*hi + hi*lo + lo*hi) by at most 3 * 2^-22 of
//    |q_i x_i|; summed over d terms and bounded with Cauchy-Schwarz that is below (d + 6) 2^-23 for the dot product, and the
//    L2 key adds d 2^-24 for the norms and 2^-22 for its two additions -- both then covered by doubling.  The tensor cores'
//    internal accumulation is not specified to the last bit, so for the 3xTF32 path this is a model, not a proof.
//  * 3e-5 is the IVF_FLAT tensor-core engine's admission slack (fltc::kSlack); the largest error measured at d = 128 is
//    5e-6.  It keeps the margin of short contractions, where the model's bound gets small.
constexpr float kCertSlack = 3e-5f;
__device__ __forceinline__ float
fin_cert_rel(int d) {
    return fmaxf(kCertSlack, (float)(d + 8) * 0x1p-22f);
}

// A row that the selection did not keep has an approximate key >= `last`, the largest one kept, so its exact key is at least
// last - err with err = fin_cert_rel(d) * (|q|^2 + max|x|^2) (L2) or fin_cert_rel(d) * |q| max|x| (IP).  The result is
// certified when its k-th exact key `kth` is at most that; when fewer candidates than k_sel existed (last = +inf) nothing
// was cut.  Otherwise the query is appended to the redo list.  When the norms are large against the distances (data with a
// large common offset) the fp32 key cancels and the re-ranked window can miss true neighbours: this is what catches it.
__device__ __forceinline__ void
fin_certify(const FinalizeParams& p, int64_t q, float last, float kth, float qq) {
    if (last == INFINITY || kth == INFINITY) return;
    const float xx = __uint_as_float(p.cert[0]);
    const float err = fin_cert_rel(p.d) * ((p.metric == KB2_METRIC_L2) ? qq + xx : sqrtf(qq * xx));
    if (kth <= last - err) return;
    p.cert[2 + atomicAdd(p.cert + 1, 1u)] = (uint32_t)q;
}

// Exact key of one candidate from the raw store (the re-rank of finalize_row and of the large-k finalize, kb2_large_k.cuh).
// fin_vec4(p): rows are read four floats at a time and a candidate is summed by 8 lanes, fin_exact_part8 giving lane
// `sub`'s share; otherwise by a whole warp, fin_exact_part32 giving lane `lane`'s share.  The caller adds the shares (in
// the same shuffle order everywhere, so every path gets the same bits) and negates for IP.  r = row of the raw store.
__device__ __forceinline__ bool
fin_vec4(const FinalizeParams& p) {
    return (p.d & 3) == 0 && (p.raw16 ? (reinterpret_cast<uintptr_t>(p.raw16) & 7) == 0
                                      : (reinterpret_cast<uintptr_t>(p.raw) & 15) == 0);
}
__device__ __forceinline__ float
fin_exact_part8(const FinalizeParams& p, const float4* q4, int64_t r, int sub) {
    float acc = 0.f;
    // a 16-bit store (refine_type fp16 / bf16) is decoded to fp32 and summed in the same order as the fp32
    // store, so it answers exactly like a flat store holding the rounded rows
    const float4* x4 = p.raw16 ? nullptr : reinterpret_cast<const float4*>(p.raw + r * (int64_t)p.d);
    const uint2* h4 = p.raw16 ? reinterpret_cast<const uint2*>(p.raw16 + r * (int64_t)p.d) : nullptr;
    for (int j = sub; j < (p.d >> 2); j += 8) {
        float4 xv;
        if (x4) {
            xv = __ldg(x4 + j);
        } else {
            const uint2 h = __ldg(h4 + j);
            if (p.raw16_kind == 1) {
                const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
                const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
                xv = make_float4(a.x, a.y, b.x, b.y);
            } else {
                xv = make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xffff0000u),
                                 __uint_as_float(h.y << 16), __uint_as_float(h.y & 0xffff0000u));
            }
        }
        const float4 qv = q4[j];
        if (p.metric == KB2_METRIC_L2) {
            float t;
            t = qv.x - xv.x; acc = fmaf(t, t, acc);
            t = qv.y - xv.y; acc = fmaf(t, t, acc);
            t = qv.z - xv.z; acc = fmaf(t, t, acc);
            t = qv.w - xv.w; acc = fmaf(t, t, acc);
        } else {
            acc = fmaf(qv.x, xv.x, acc); acc = fmaf(qv.y, xv.y, acc);
            acc = fmaf(qv.z, xv.z, acc); acc = fmaf(qv.w, xv.w, acc);
        }
    }
    return acc;
}
__device__ __forceinline__ float
fin_exact_part32(const FinalizeParams& p, const float* s_q, int64_t r, int lane) {
    float acc = 0.f;
    if (p.raw16) {
        const uint16_t* x16 = p.raw16 + r * (int64_t)p.d;
        for (int j = lane; j < p.d; j += kWarp) {
            const float xv = (p.raw16_kind == 1) ? __half2float(__ushort_as_half(x16[j]))
                                                 : __uint_as_float((uint32_t)x16[j] << 16);
            if (p.metric == KB2_METRIC_L2) {
                const float t = s_q[j] - xv;
                acc = fmaf(t, t, acc);
            } else {
                acc = fmaf(s_q[j], xv, acc);
            }
        }
    } else {
        const float* x = p.raw + r * (int64_t)p.d;
        if (p.metric == KB2_METRIC_L2) {
            for (int j = lane; j < p.d; j += kWarp) {
                float t = s_q[j] - x[j];
                acc = fmaf(t, t, acc);
            }
        } else {
            for (int j = lane; j < p.d; j += kWarp) acc = fmaf(s_q[j], x[j], acc);
        }
    }
    return acc;
}

// dynamic smem: n_sort*8 + k_sel*(4+8+4) + d*4
__device__ __forceinline__ void
finalize_row(FinalizeParams p, const int64_t q) {   // p by value: the variable-length branch edits its copy
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* s_sort = (uint64_t*)smem_raw;
    int64_t* s_label = (int64_t*)(s_sort + p.n_sort);
    float* s_key = (float*)(s_label + p.k_sel);
    uint32_t* s_pos = (uint32_t*)(s_key + p.k_sel);
    float* s_q = (float*)(s_pos + p.k_sel);

    const uint64_t* src = p.partial + q * p.partial_stride;
    if (p.counts && !(p.count_flags && p.count_flags[q])) {
        // variable-length row (tensor-core PQ engine): sort only what is there
        const int c = (int)min(p.counts[q], (uint32_t)p.n_partial);
        if (p.split_small > 0 && c <= p.split_small) return;
        p.n_partial = c;
        p.n_sort = c <= 2 ? 2 : (1 << (32 - __clz(c - 1)));
    }
    for (int i = threadIdx.x; i < p.n_sort; i += blockDim.x) s_sort[i] = (i < p.n_partial) ? src[i] : kEmpty;
    if (p.rerank)
        for (int i = threadIdx.x; i < p.d; i += blockDim.x) s_q[i] = p.queries[q * p.d + i];
    __syncthreads();
    if (p.n_sort <= (int)blockDim.x) {
        // small candidate sets (IVF coarse, tensor-core PQ survivors): rank by counting, one entry per thread.  The bitonic
        // network costs log^2(n) CTA barriers with most warps idle; this is n broadcast reads per thread and two barriers.
        const int i = threadIdx.x;
        const uint64_t mine = (i < p.n_sort) ? s_sort[i] : kEmpty;
        int rank = 0;
        if (i < p.n_partial) {
            for (int j = 0; j < p.n_partial; j++) {
                const uint64_t e = s_sort[j];
                rank += (e < mine) || (e == mine && j < i);
            }
        }
        __syncthreads();
        if (i < p.n_partial) s_sort[rank] = mine;   // a permutation of [0, n_partial); the kEmpty tail stays in place
        __syncthreads();
    } else {
        block_bitonic_sort(s_sort, p.n_sort);
    }

    const int ksel = p.k_sel;
    const uint64_t e_last = (ksel - 1 < p.n_sort) ? s_sort[ksel - 1] : kEmpty;   // largest approximate key kept (fin_certify)
    const float last = (e_last == kEmpty) ? INFINITY : unpack_key(e_last);
    for (int i = threadIdx.x; i < ksel; i += blockDim.x) {
        uint64_t e = (i < p.n_sort) ? s_sort[i] : kEmpty;
        if (e == kEmpty) {
            s_label[i] = INT64_MAX;
            s_key[i] = INFINITY;
            s_pos[i] = kNoPos;
        } else {
            uint32_t pos = unpack_pos(e);
            int64_t row = p.rows ? (int64_t)p.rows[pos] : (int64_t)pos;
            s_label[i] = p.labels ? p.labels[row] : row;
            s_key[i] = unpack_key(e);
            s_pos[i] = pos;
        }
    }
    __syncthreads();

    if (p.rerank) {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int nwarps = blockDim.x >> 5;
        if (fin_vec4(p)) {
            // four candidates per warp at a time (8 lanes each, 128 B per candidate and step): the re-rank is a chain of
            // dependent random-row round trips (L2 / HBM), so candidates in flight per warp are what sets its duration
            const int sub = lane & 7, grp = lane >> 3;
            const float4* q4 = reinterpret_cast<const float4*>(s_q);
            for (int i0 = warp * 4; i0 < ksel; i0 += nwarps * 4) {
                const int i = i0 + grp;
                const uint32_t pos = (i < ksel) ? s_pos[i] : kNoPos;
                float acc = 0.f;
                if (pos != kNoPos) {
                    const int64_t r = p.raw_by_pos ? (int64_t)pos : (p.rows ? (int64_t)p.rows[pos] : (int64_t)pos);
                    acc = fin_exact_part8(p, q4, r, sub);
                }
                acc += __shfl_xor_sync(0xffffffffu, acc, 4);
                acc += __shfl_xor_sync(0xffffffffu, acc, 2);
                acc += __shfl_xor_sync(0xffffffffu, acc, 1);
                if (sub == 0 && pos != kNoPos) s_key[i] = (p.metric == KB2_METRIC_L2) ? acc : -acc;
            }
            __syncthreads();
        } else {
        for (int i = warp; i < ksel; i += nwarps) {
            uint32_t pos = s_pos[i];
            if (pos == kNoPos) continue;
            int64_t r = p.raw_by_pos ? (int64_t)pos : (p.rows ? (int64_t)p.rows[pos] : (int64_t)pos);
            float acc = fin_exact_part32(p, s_q, r, lane);
            acc = warp_sum(acc);
            if (lane == 0) s_key[i] = (p.metric == KB2_METRIC_L2) ? acc : -acc;
        }
        __syncthreads();
        }
    }

    // rank by (key, label, slot)
    for (int i = threadIdx.x; i < ksel; i += blockDim.x) {
        const float ki = s_key[i];
        const int64_t li = s_label[i];
        int rank = 0;
        for (int j = 0; j < ksel; j++) {
            const float kj = s_key[j];
            const int64_t lj = s_label[j];
            rank += (kj < ki) || (kj == ki && (lj < li || (lj == li && j < i)));
        }
        if (rank < p.k_out) {
            const int64_t o = q * p.k_out + rank;
            if (s_pos[i] == kNoPos) {
                p.out_ids[o] = -1;
                p.out_dist[o] = (p.metric == KB2_METRIC_L2) ? FLT_MAX : -FLT_MAX;
                if (p.out_pos) p.out_pos[o] = -1;
            } else {
                p.out_ids[o] = li;
                p.out_dist[o] = (p.metric == KB2_METRIC_L2) ? ki : -ki;
                if (p.out_pos) p.out_pos[o] = (int32_t)s_pos[i];
            }
            if (p.cert && rank == p.k_out - 1) s_q[p.d] = ki;   // k-th exact key (in the spare word after the query)
        }
    }
    // k_out > k_sel cannot happen (host guarantees k_sel >= k_out)
    if (p.cert) {
        __syncthreads();
        if (threadIdx.x < kWarp) {
            float qq = 0.f;
            for (int j = threadIdx.x; j < p.d; j += kWarp) qq = fmaf(s_q[j], s_q[j], qq);
            qq = warp_sum(qq);
            if (threadIdx.x == 0) fin_certify(p, q, last, s_q[p.d], qq);
        }
    }
}

// grid = nq (one CTA per query), or -- p.row_loop_nq > 0 -- any grid striding the rows: as the tail pass after
// finalize_warp_kernel nearly every row is skipped, and launching one 256-thread CTA with ~17 KB of shared memory per query only
// to exit costs ~1.2 us per CTA and SM (measured at C3: 80 us for 10 000 empty CTAs)
__global__ void __launch_bounds__(256)
finalize_kernel(FinalizeParams p) {
    if (p.row_loop_nq > 0) {
        for (int64_t q = blockIdx.x; q < p.row_loop_nq; q += gridDim.x) {
            finalize_row(p, p.qlist ? (int64_t)p.qlist[q] : q);
            __syncthreads();
        }
    } else {
        finalize_row(p, p.qlist ? (int64_t)p.qlist[blockIdx.x] : (int64_t)blockIdx.x);
    }
}

// ------------------------------------------------------------------------------------------
// Finalize, small case (n_partial <= 128 candidates): ONE WARP per query, four queries per CTA.  Same contract and the same
// results as finalize_kernel; the CTA version spends its time in barriers and O(n^2) ranking loops (ncu r2: 12 k warp
// instructions per query, 75 % issue-active), this one sorts in registers (element i of the warp = lane * 4 + r):
//   1. bitonic sort of the packed (key, position) entries, 4 per lane
//   2. exact keys of the best k_sel from the raw rows, four candidates at a time (8 lanes each)
//   3. bitonic sort of (exact key, label) and the k_out best written out
// dynamic smem per warp: d floats + 128 * (8 + 4 + 8 + 4) bytes
// ------------------------------------------------------------------------------------------
struct FinEntry {
    float key;
    int64_t label;
    uint32_t pos;
};
__device__ __forceinline__ bool
fin_less(const FinEntry& a, const FinEntry& b) {
    return a.key < b.key || (a.key == b.key && a.label < b.label);
}
__device__ __forceinline__ FinEntry
fin_shfl_xor(const FinEntry& a, int m) {
    FinEntry o;
    o.key = __shfl_xor_sync(0xffffffffu, a.key, m);
    o.label = __shfl_xor_sync(0xffffffffu, a.label, m);
    o.pos = __shfl_xor_sync(0xffffffffu, a.pos, m);
    return o;
}
__device__ __forceinline__ uint64_t
fin_shfl_xor(uint64_t a, int m) {
    return __shfl_xor_sync(0xffffffffu, a, m);
}
__device__ __forceinline__ bool
fin_less(uint64_t a, uint64_t b) {
    return a < b;
}
// ascending bitonic sort of 32 * EPL elements held EPL per lane (index = lane * EPL + r)
template <typename T, int EPL>
__device__ __forceinline__ void
warp_bitonic(T (&v)[EPL], int lane) {
#pragma unroll
    for (int k2 = 2; k2 <= 32 * EPL; k2 <<= 1) {
#pragma unroll
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            if (j < EPL) {
#pragma unroll
                for (int r = 0; r < EPL; r++) {
                    if ((r ^ j) > r) {
                        const bool asc = (((lane * EPL + r) & k2) == 0);
                        const bool sw = fin_less(v[r ^ j], v[r]) == asc;   // out of order for this direction
                        const T a = v[r], b = v[r ^ j];
                        v[r] = sw ? b : a;
                        v[r ^ j] = sw ? a : b;
                    }
                }
            } else {
                const int m = j / EPL;
                const bool lower = (lane & m) == 0;
#pragma unroll
                for (int r = 0; r < EPL; r++) {
                    const bool asc = (((lane * EPL + r) & k2) == 0);
                    const T o = fin_shfl_xor(v[r], m);
                    const bool take_min = (lower == asc);
                    // equal elements: each side keeps its own copy
                    const bool take_o = take_min ? fin_less(o, v[r]) : fin_less(v[r], o);
                    v[r] = take_o ? o : v[r];
                }
            }
        }
    }
}

constexpr int kFinWarps = 4;
// step 1 of finalize_warp_kernel for one size class: sort this query's n packed entries (EPL per lane) and leave the best
// min(k_sel, 128) as (position, key, label) in shared memory
template <int EPL>
__device__ __forceinline__ void
finalize_warp_select(const FinalizeParams& p, const uint64_t* __restrict__ src, int n, int lane, uint32_t* s_pos, float* s_key,
                     int64_t* s_label) {
    uint64_t e[EPL];
#pragma unroll
    for (int r = 0; r < EPL; r++) {
        const int i = lane * EPL + r;
        e[r] = (i < n) ? src[i] : kEmpty;
    }
    warp_bitonic<uint64_t, EPL>(e, lane);
    const int ksel = p.k_sel;
#pragma unroll
    for (int r = 0; r < EPL; r++) {
        const int i = lane * EPL + r;
        if (i < 128) {
            const uint64_t v = e[r];
            uint32_t pos = kNoPos;
            float key = INFINITY;
            int64_t label = INT64_MAX;
            if (i < ksel && v != kEmpty) {
                pos = unpack_pos(v);
                key = unpack_key(v);
                const int64_t row = p.rows ? (int64_t)p.rows[pos] : (int64_t)pos;
                label = p.labels ? p.labels[row] : row;
            }
            s_pos[i] = pos;
            s_key[i] = key;
            s_label[i] = label;
        }
    }
}

template <int EPLMAX>   // largest size class compiled in: 4 (<= 128 candidates), 8 (<= 256) or 16 (<= 512)
__global__ void __launch_bounds__(kFinWarps * 32)
finalize_warp_kernel(FinalizeParams p, int64_t nq) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dpad = (p.d + 3) & ~3;
    const size_t per_warp = (size_t)dpad * 4 + 128 * 24;
    unsigned char* mine = smem_raw + (size_t)warp * per_warp;
    float* s_q = (float*)mine;
    int64_t* s_label = (int64_t*)(mine + (size_t)dpad * 4);
    uint64_t* s_e = (uint64_t*)(s_label + 128);
    float* s_key = (float*)(s_e + 128);
    uint32_t* s_pos = (uint32_t*)(s_key + 128);
    const int64_t row = (int64_t)blockIdx.x * kFinWarps + warp;
    if (row >= nq) return;
    const int64_t q = p.qlist ? (int64_t)p.qlist[row] : row;

    // ---- 1. approximate order
    int n = p.n_partial;
    if (p.counts && !(p.count_flags && p.count_flags[q])) n = (int)min(p.counts[q], (uint32_t)p.n_partial);
    if (n > 32 * EPLMAX) return;   // (only with p.split_small) left to finalize_kernel
    const uint64_t* src = p.partial + q * p.partial_stride;
    if (p.rerank)
        for (int j = lane; j < p.d; j += kWarp) s_q[j] = p.queries[q * p.d + j];
    if (EPLMAX >= 16 && n > 256) finalize_warp_select<(EPLMAX >= 16 ? 16 : 4)>(p, src, n, lane, s_pos, s_key, s_label);
    else if (EPLMAX >= 8 && n > 128) finalize_warp_select<(EPLMAX >= 8 ? 8 : 4)>(p, src, n, lane, s_pos, s_key, s_label);
    else finalize_warp_select<4>(p, src, n, lane, s_pos, s_key, s_label);
    const int ksel = p.k_sel;
    __syncwarp();
    const float last = p.cert ? s_key[ksel - 1] : INFINITY;   // largest approximate key kept (+inf: none), before the re-rank

    // ---- 2. exact keys (same arithmetic and summation order as finalize_kernel)
    if (p.rerank) {
        const bool vec4 = (p.d & 3) == 0 && (p.raw16 ? (reinterpret_cast<uintptr_t>(p.raw16) & 7) == 0
                                                      : (reinterpret_cast<uintptr_t>(p.raw) & 15) == 0);
        if (vec4) {
            // eight candidates per step (two groups of four, 8 lanes per row, 128 B per row and load): the re-rank is a chain of
            // dependent random-row round trips (L2 for the centroid table, HBM for the refine store), so what sets its duration
            // is the number of rows in flight per warp.  Per candidate the arithmetic and its order are unchanged.
            const int sub = lane & 7, grp = lane >> 3;
            const float4* q4 = reinterpret_cast<const float4*>(s_q);
            const int nj = p.d >> 2;
            auto load4 = [&](const float4* x4, const uint2* h4, int j) -> float4 {
                if (x4) return __ldg(x4 + j);
                const uint2 h = __ldg(h4 + j);
                if (p.raw16_kind == 1) {
                    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
                    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
                    return make_float4(a.x, a.y, b.x, b.y);
                }
                return make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xffff0000u), __uint_as_float(h.y << 16),
                                   __uint_as_float(h.y & 0xffff0000u));
            };
            auto accum = [&](float acc, const float4& qv, const float4& xv) -> float {
                if (p.metric == KB2_METRIC_L2) {
                    float t;
                    t = qv.x - xv.x; acc = fmaf(t, t, acc);
                    t = qv.y - xv.y; acc = fmaf(t, t, acc);
                    t = qv.z - xv.z; acc = fmaf(t, t, acc);
                    t = qv.w - xv.w; acc = fmaf(t, t, acc);
                } else {
                    acc = fmaf(qv.x, xv.x, acc); acc = fmaf(qv.y, xv.y, acc);
                    acc = fmaf(qv.z, xv.z, acc); acc = fmaf(qv.w, xv.w, acc);
                }
                return acc;
            };
            for (int i0 = 0; i0 < ksel; i0 += 8) {
                const int ia = i0 + grp, ib = i0 + 4 + grp;
                const uint32_t pa = (ia < ksel) ? s_pos[ia] : kNoPos;
                const uint32_t pb = (ib < ksel) ? s_pos[ib] : kNoPos;
                const int64_t ra = p.raw_by_pos ? (int64_t)pa : (p.rows && pa != kNoPos ? (int64_t)p.rows[pa] : (int64_t)pa);
                const int64_t rb = p.raw_by_pos ? (int64_t)pb : (p.rows && pb != kNoPos ? (int64_t)p.rows[pb] : (int64_t)pb);
                const float4* xa = (p.raw16 || pa == kNoPos) ? nullptr : reinterpret_cast<const float4*>(p.raw + ra * (int64_t)p.d);
                const float4* xb = (p.raw16 || pb == kNoPos) ? nullptr : reinterpret_cast<const float4*>(p.raw + rb * (int64_t)p.d);
                const uint2* ha = (p.raw16 && pa != kNoPos) ? reinterpret_cast<const uint2*>(p.raw16 + ra * (int64_t)p.d) : nullptr;
                const uint2* hb = (p.raw16 && pb != kNoPos) ? reinterpret_cast<const uint2*>(p.raw16 + rb * (int64_t)p.d) : nullptr;
                float acca = 0.f, accb = 0.f;
                for (int j = sub; j < nj; j += 8) {
                    float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
                    if (pa != kNoPos) va = load4(xa, ha, j);
                    if (pb != kNoPos) vb = load4(xb, hb, j);
                    const float4 qv = q4[j];
                    if (pa != kNoPos) acca = accum(acca, qv, va);
                    if (pb != kNoPos) accb = accum(accb, qv, vb);
                }
                acca += __shfl_xor_sync(0xffffffffu, acca, 4);
                accb += __shfl_xor_sync(0xffffffffu, accb, 4);
                acca += __shfl_xor_sync(0xffffffffu, acca, 2);
                accb += __shfl_xor_sync(0xffffffffu, accb, 2);
                acca += __shfl_xor_sync(0xffffffffu, acca, 1);
                accb += __shfl_xor_sync(0xffffffffu, accb, 1);
                if (sub == 0 && pa != kNoPos) s_key[ia] = (p.metric == KB2_METRIC_L2) ? acca : -acca;
                if (sub == 0 && pb != kNoPos) s_key[ib] = (p.metric == KB2_METRIC_L2) ? accb : -accb;
            }
        } else {
            for (int i = 0; i < ksel; i++) {
                const uint32_t pos = s_pos[i];
                if (pos == kNoPos) continue;
                const int64_t r = p.raw_by_pos ? (int64_t)pos : (p.rows ? (int64_t)p.rows[pos] : (int64_t)pos);
                float acc = 0.f;
                for (int j = lane; j < p.d; j += kWarp) {
                    float xv;
                    if (p.raw16) {
                        const uint16_t h = p.raw16[r * (int64_t)p.d + j];
                        xv = (p.raw16_kind == 1) ? __half2float(__ushort_as_half(h)) : __uint_as_float((uint32_t)h << 16);
                    } else {
                        xv = p.raw[r * (int64_t)p.d + j];
                    }
                    if (p.metric == KB2_METRIC_L2) {
                        const float t = s_q[j] - xv;
                        acc = fmaf(t, t, acc);
                    } else {
                        acc = fmaf(s_q[j], xv, acc);
                    }
                }
                acc = warp_sum(acc);
                if (lane == 0) s_key[i] = (p.metric == KB2_METRIC_L2) ? acc : -acc;
            }
        }
        __syncwarp();
    }

    // ---- 3. final order by (key, label); empty slots (key inf, label max) go last.  Sorted as packed (key, slot) words;
    //         only when two finite keys are bit-equal (rare) is the sort redone on (key, label) records.
    uint64_t f[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int i = lane * 4 + r;
        f[r] = ((uint64_t)f2ord(s_key[i]) << 32) | (uint32_t)i;
    }
    warp_bitonic<uint64_t, 4>(f, lane);
    bool tie = false;
    {
        const uint32_t kInf = f2ord(INFINITY);
        const uint32_t nxt = __shfl_down_sync(0xffffffffu, (uint32_t)(f[0] >> 32), 1);
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const uint32_t a = (uint32_t)(f[r] >> 32);
            const uint32_t b = (r < 3) ? (uint32_t)(f[r < 3 ? r + 1 : 3] >> 32) : nxt;
            if (a == b && a < kInf && !(r == 3 && lane == 31)) tie = true;
        }
    }
    if (__any_sync(0xffffffffu, tie)) {
        FinEntry g[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const int i = lane * 4 + r;
            g[r].key = s_key[i];
            g[r].label = s_label[i];
            g[r].pos = (uint32_t)i;   // slot
        }
        warp_bitonic<FinEntry, 4>(g, lane);
#pragma unroll
        for (int r = 0; r < 4; r++) f[r] = ((uint64_t)f2ord(g[r].key) << 32) | g[r].pos;
    }
    float kth = INFINITY;   // k-th exact key (fin_certify), held by lane (k_out - 1) / 4
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int i = lane * 4 + r;
        if (i < p.k_out) {
            const int64_t o = q * p.k_out + i;
            const int slot = (int)(uint32_t)f[r];
            const uint32_t pos = s_pos[slot];
            if (pos == kNoPos) {
                p.out_ids[o] = -1;
                p.out_dist[o] = (p.metric == KB2_METRIC_L2) ? FLT_MAX : -FLT_MAX;
                if (p.out_pos) p.out_pos[o] = -1;
            } else {
                const float key = s_key[slot];
                p.out_ids[o] = s_label[slot];
                p.out_dist[o] = (p.metric == KB2_METRIC_L2) ? key : -key;
                if (p.out_pos) p.out_pos[o] = (int32_t)pos;
                if (i == p.k_out - 1) kth = key;
            }
        }
    }
    if (p.cert) {
        kth = __shfl_sync(0xffffffffu, kth, (p.k_out - 1) >> 2);
        float qq = 0.f;
        for (int j = lane; j < p.d; j += kWarp) qq = fmaf(s_q[j], s_q[j], qq);
        qq = warp_sum(qq);
        if (lane == 0) fin_certify(p, q, last, kth, qq);
    }
}

// reduce [nq][n_in] partial entries to the best n_keep per query, in place at the front of each
// query's slot range (used when many base chunks accumulate more than 8192 candidates)
__global__ void __launch_bounds__(256)
reduce_partials_kernel(uint64_t* partial, int stride, int n_in, int n_sort, int n_keep) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* s = (uint64_t*)smem_raw;
    uint64_t* base = partial + (int64_t)blockIdx.x * stride;
    for (int i = threadIdx.x; i < n_sort; i += blockDim.x) s[i] = (i < n_in) ? base[i] : kEmpty;
    __syncthreads();
    block_bitonic_sort(s, n_sort);
    for (int i = threadIdx.x; i < n_keep; i += blockDim.x) base[i] = s[i];
}

// ------------------------------------------------------------------------------------------
// Merge of per-shard top-k lists after the all-gather: one CTA per query, rank by (key, id).
// in: [world][nq][k]; out: [nq][k]
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
merge_topk_kernel(int metric, int world, int64_t nq, int k, const int64_t* __restrict__ in_ids,
                  const float* __restrict__ in_dist, int64_t* __restrict__ out_ids, float* __restrict__ out_dist) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int n = world * k;
    int64_t* s_id = (int64_t*)smem_raw;
    float* s_key = (float*)(s_id + n);
    const int64_t q = blockIdx.x;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int w = i / k, j = i % k;
        const int64_t id = in_ids[((int64_t)w * nq + q) * k + j];
        const float d = in_dist[((int64_t)w * nq + q) * k + j];
        s_id[i] = id < 0 ? INT64_MAX : id;
        s_key[i] = id < 0 ? INFINITY : (metric == KB2_METRIC_L2 ? d : -d);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float ki = s_key[i];
        const int64_t li = s_id[i];
        int rank = 0;
        for (int j = 0; j < n; j++) {
            const float kj = s_key[j];
            const int64_t lj = s_id[j];
            rank += (kj < ki) || (kj == ki && (lj < li || (lj == li && j < i)));
        }
        if (rank < k) {
            const bool empty = (li == INT64_MAX);
            out_ids[q * k + rank] = empty ? -1 : li;
            out_dist[q * k + rank] = empty ? (metric == KB2_METRIC_L2 ? FLT_MAX : -FLT_MAX)
                                           : (metric == KB2_METRIC_L2 ? ki : -ki);
        }
    }
}


inline void
launch_merge_topk(int metric, int world, int64_t nq, int k, const int64_t* in_ids, const float* in_dist, int64_t* out_ids,
                  float* out_dist, cudaStream_t st) {
    const size_t smem = (size_t)world * k * 12 + 16;
    launch<merge_topk_kernel>((unsigned)nq, 256, smem, st, metric, world, nq, k, in_ids, in_dist, out_ids, out_dist);
    KB2_CUDA_CHECK(cudaGetLastError());
}

}  // namespace kb2
