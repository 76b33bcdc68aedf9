// kb2_large_k.cuh — the device half of search with a candidate window above kMaxK (1024) entries: an exact selection of
// each query's K best entries from rows of any length, and the finalize of those K candidates (exact re-rank, FLAT
// certification, labels, (distance, id) order).  The host half is large_k_* in kb2_index.cuh; DESIGN §4.9.
#pragma once
#include "kb2_topk.cuh"

namespace kb2 {

constexpr int kSelThreads = 1024;

template <typename T>
__device__ __forceinline__ uint64_t
sel_entry(const T* __restrict__ row, int64_t i, uint32_t pos_base);
// a key row of the dense contraction: (orderable key, pos_base + column)
template <>
__device__ __forceinline__ uint64_t
sel_entry<float>(const float* __restrict__ row, int64_t i, uint32_t pos_base) {
    return pack_kp(__ldg(row + i), pos_base + (uint32_t)i);
}
// packed (key, position) entries (dense IVF rows, the running best set of the FLAT key chunks)
template <>
__device__ __forceinline__ uint64_t
sel_entry<uint64_t>(const uint64_t* __restrict__ row, int64_t i, uint32_t) {
    return __ldg(reinterpret_cast<const unsigned long long*>(row) + i);
}

// Exact selection: out row b <- the min(K, valid) smallest entries of input row b, unsorted, then kEmpty.  An entry is
// valid when its key is below +inf (filtered keys of the contraction are +inf, unwritten slots of a dense row kEmpty).
// Entries are (orderable key << 32 | position), unique, so "smallest" is the (key, position) order: among equal keys the
// smallest positions are kept.  Radix select on the 64-bit entry, 8 bits per pass from the top: each pass histograms the
// entries that match the digits fixed so far (shared-memory bins, one atomic per distinct digit and warp) and fixes the
// digit holding the K-th entry; it stops as soon as that digit's bin is taken whole, usually once the key's 32 bits are
// fixed or earlier.  One last pass emits every entry whose fixed digits are at most the threshold's.
// grid = rows, block = kSelThreads, static smem only.  The row is re-read from global memory (L2) on every pass.
template <typename T>
__global__ void __launch_bounds__(kSelThreads)
select_rows_kernel(const T* __restrict__ in, int64_t ld, int64_t len, uint32_t pos_base, int K, uint64_t* __restrict__ out,
                   int64_t out_ld) {
    __shared__ uint32_t hist[256];
    __shared__ unsigned long long s_prefix, s_mask;
    __shared__ uint32_t s_need, s_done, s_cnt;
    const T* row = in + (int64_t)blockIdx.x * ld;
    uint64_t* o = out + (int64_t)blockIdx.x * out_ld;
    const uint32_t kInfOrd = f2ord(INFINITY);
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        s_prefix = 0;
        s_mask = 0;
        s_need = (uint32_t)K;
        s_done = 0;
        s_cnt = 0;
    }
    uint64_t prefix = 0, mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (int64_t i0 = 0; i0 < len; i0 += blockDim.x) {
            const int64_t i = i0 + threadIdx.x;
            uint32_t dig = 256;
            if (i < len) {
                const uint64_t e = sel_entry<T>(row, i, pos_base);
                if ((uint32_t)(e >> 32) < kInfOrd && (e & mask) == prefix) dig = (uint32_t)(e >> shift) & 255u;
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
            const uint32_t need = s_need;
            if (total <= need) {
                // every entry matching the fixed digits is kept (first pass: at most K valid entries in the row)
                if (lane == 0) s_done = 1;
            } else if (incl - sum < need && need <= incl) {
                uint32_t c = incl - sum;
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    if (c + h[t] >= need) {
                        s_prefix = prefix | ((uint64_t)(lane * 8 + t) << shift);
                        s_mask = mask | (0xffull << shift);
                        s_need = need - c;
                        s_done = (h[t] == need - c) ? 1u : 0u;
                        break;
                    }
                    c += h[t];
                }
            }
        }
        __syncthreads();
        prefix = s_prefix;
        mask = s_mask;
        if (s_done) break;
    }
    // emission: entries whose fixed digits are at most the threshold's (exactly min(K, valid) of them)
    for (int64_t i0 = 0; i0 < len; i0 += blockDim.x) {
        const int64_t i = i0 + threadIdx.x;
        uint64_t e = kEmpty;
        bool keep = false;
        if (i < len) {
            e = sel_entry<T>(row, i, pos_base);
            keep = (uint32_t)(e >> 32) < kInfOrd && (e & mask) <= prefix;
        }
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        uint32_t base = 0;
        if (lane == 0 && b) base = atomicAdd(&s_cnt, (uint32_t)__popc(b));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (keep) {
            const uint32_t slot = base + __popc(b & ((1u << lane) - 1u));
            if (slot < (uint32_t)K) o[slot] = e;
        }
    }
    __syncthreads();
    for (int i = (int)min(s_cnt, (uint32_t)K) + threadIdx.x; i < K; i += blockDim.x) o[i] = kEmpty;
}

// Scratch of the large finalize for one group of launch rows (row b is query qlist[b], or q0 + b).
struct LargeFin {
    const uint64_t* cand;   // [rows][cand_ld]: K entries per row, unsorted, kEmpty padded (select_rows_kernel)
    int64_t cand_ld;
    int K;
    int64_t q0;
    float* key;             // [rows][K] key of each candidate (exact when p.rerank), +inf for an empty slot
    int64_t* label;         // [rows][K] reported id, INT64_MAX for an empty slot
    int32_t* slot;          // [rows][K] 0..K-1 (sort values)
    uint32_t* okey;         // [rows][K] orderable key of the label-sorted candidates
    const int32_t* order;   // [rows][K] candidate slots in (key, label) order
    uint32_t* info;         // [rows][4]: [0] largest approximate key kept (orderable), [1] valid candidates, [2] |q|^2 bits
};

__device__ __forceinline__ int64_t
large_query(const FinalizeParams& p, const LargeFin& lf, int64_t b) {
    return p.qlist ? (int64_t)p.qlist[b] : lf.q0 + b;
}

// 1. key and label of every candidate; grid (rows, ceil(K / 256)), block 256, dynamic smem d*4 (+16).  The exact re-rank
//    runs the same per-candidate code as finalize_row.
__global__ void __launch_bounds__(256)
large_rerank_kernel(FinalizeParams p, LargeFin lf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_q = (float*)smem_raw;
    __shared__ uint32_t s_max, s_cnt;
    const int64_t b = blockIdx.x;
    const int64_t q = large_query(p, lf, b);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { s_max = 0; s_cnt = 0; }
    if (p.rerank || p.cert)
        for (int i = threadIdx.x; i < p.d; i += blockDim.x) s_q[i] = p.queries[q * p.d + i];
    __syncthreads();
    const int j = blockIdx.y * 256 + threadIdx.x;
    const uint64_t* row = lf.cand + b * lf.cand_ld;
    const uint64_t e = (j < lf.K) ? row[j] : kEmpty;
    const bool valid = e != kEmpty;
    if (j < lf.K) {
        int64_t lab = INT64_MAX;
        if (valid) {
            const uint32_t pos = unpack_pos(e);
            const int64_t r = p.rows ? (int64_t)p.rows[pos] : (int64_t)pos;
            lab = p.labels ? p.labels[r] : r;
        }
        lf.label[b * lf.K + j] = lab;
        lf.slot[b * lf.K + j] = j;
        if (!p.rerank) {
            const float k0 = valid ? unpack_key(e) : INFINITY;
            lf.key[b * lf.K + j] = (k0 == 0.f) ? 0.f : k0;   // -0 sorts as +0, as finalize_row's float compare does
        }
    }
    const unsigned vb = __ballot_sync(0xffffffffu, valid);
    uint32_t wmax = valid ? (uint32_t)(e >> 32) : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0 && vb) {
        atomicMax(&s_max, wmax);
        atomicAdd(&s_cnt, (uint32_t)__popc(vb));
    }
    if (p.rerank) {
        const int j0 = blockIdx.y * 256;
        if (fin_vec4(p)) {
            const int sub = lane & 7, grp = lane >> 3;
            const float4* q4 = reinterpret_cast<const float4*>(s_q);
            for (int i0 = warp * 4; i0 < 256; i0 += 32) {
                const int jj = j0 + i0 + grp;
                const uint64_t ej = (jj < lf.K) ? row[jj] : kEmpty;
                float acc = 0.f;
                if (ej != kEmpty) {
                    const uint32_t pos = unpack_pos(ej);
                    const int64_t r = p.raw_by_pos ? (int64_t)pos : (p.rows ? (int64_t)p.rows[pos] : (int64_t)pos);
                    acc = fin_exact_part8(p, q4, r, sub);
                }
                acc += __shfl_xor_sync(0xffffffffu, acc, 4);
                acc += __shfl_xor_sync(0xffffffffu, acc, 2);
                acc += __shfl_xor_sync(0xffffffffu, acc, 1);
                if (sub == 0 && jj < lf.K) {
                    const float k1 = (ej == kEmpty) ? INFINITY : ((p.metric == KB2_METRIC_L2) ? acc : -acc);
                    lf.key[b * lf.K + jj] = (k1 == 0.f) ? 0.f : k1;
                }
            }
        } else {
            for (int i0 = warp; i0 < 256; i0 += 8) {
                const int jj = j0 + i0;
                const uint64_t ej = (jj < lf.K) ? row[jj] : kEmpty;
                if (jj >= lf.K) break;
                float acc = 0.f;
                if (ej != kEmpty) {
                    const uint32_t pos = unpack_pos(ej);
                    const int64_t r = p.raw_by_pos ? (int64_t)pos : (p.rows ? (int64_t)p.rows[pos] : (int64_t)pos);
                    acc = warp_sum(fin_exact_part32(p, s_q, r, lane));
                }
                if (lane == 0) {
                    const float k1 = (ej == kEmpty) ? INFINITY : ((p.metric == KB2_METRIC_L2) ? acc : -acc);
                    lf.key[b * lf.K + jj] = (k1 == 0.f) ? 0.f : k1;
                }
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicMax(lf.info + b * 4, s_max);
        atomicAdd(lf.info + b * 4 + 1, s_cnt);
    }
    if (p.cert && blockIdx.y == 0 && warp == 0) {
        float qq = 0.f;
        for (int i = lane; i < p.d; i += kWarp) qq = fmaf(s_q[i], s_q[i], qq);
        qq = warp_sum(qq);
        if (lane == 0) lf.info[b * 4 + 2] = __float_as_uint(qq);
    }
}

// 2. between the two stable sorts: okey[b][i] = orderable key of the candidate in slot sorted_slot[b][i] (label order)
__global__ void
large_gather_keys_kernel(LargeFin lf, const int32_t* __restrict__ sorted_slot, int64_t n) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int64_t b = t / lf.K;
    lf.okey[t] = f2ord(lf.key[b * lf.K + sorted_slot[t]]);
}

// 3. the k_out best in (key, label) order (lf.order) to the result rows, padding, and the certification of FLAT results
//    (fin_certify, as finalize_row does it: `last` is the largest approximate key selected, +inf when nothing was cut)
__global__ void
large_emit_kernel(FinalizeParams p, LargeFin lf, int64_t rows) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= rows * p.k_out) return;
    const int64_t b = t / p.k_out;
    const int r = (int)(t % p.k_out);
    const int64_t q = large_query(p, lf, b);
    const int s = lf.order[b * lf.K + r];
    const bool valid = lf.cand[b * lf.cand_ld + s] != kEmpty;
    const float key = lf.key[b * lf.K + s];
    const int64_t o = q * p.k_out + r;
    if (!valid) {
        p.out_ids[o] = -1;
        p.out_dist[o] = (p.metric == KB2_METRIC_L2) ? FLT_MAX : -FLT_MAX;
    } else {
        p.out_ids[o] = lf.label[b * lf.K + s];
        p.out_dist[o] = (p.metric == KB2_METRIC_L2) ? key : -key;
    }
    if (p.cert && r == p.k_out - 1) {
        const uint32_t* inf = lf.info + b * 4;
        const float last = (inf[1] >= (uint32_t)lf.K) ? ord2f(inf[0]) : INFINITY;
        fin_certify(p, q, last, valid ? key : INFINITY, __uint_as_float(inf[2]));
    }
}

template <typename T>
__global__ void
segment_offsets_kernel(T* off, int64_t nseg, int64_t len) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t <= nseg) off[t] = (T)(t * len);
}

}  // namespace kb2
