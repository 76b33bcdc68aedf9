// kb2_hnsw.cuh — HNSW: graph container in the reference's layout, host-side construction, and the
// device search kernel (greedy descent on the upper levels + best-first beam on level 0).
//
// Reference path being replaced:
//   v2_hnsw_searcher::{search, greedy_search_top_levels, greedy_update_nearest,
//                      search_on_a_level, evaluate_single_node}   K/impl/HnswSearcher.h:116-432
//   NeighborSetPopList (sorted array, upper_bound insert, cursor)  K/impl/Neighbor.h:46-150
//   IndexHNSWWrapper::search (visited bitset per query, IP negation) src/index/hnsw/impl/IndexHNSWWrapper.cc:67-205
//   graph layout: neighbors/offsets/levels/cum_nneighbor_per_level   K/impl/HNSW.h, HNSW.cpp:53-89,202-225
//
// Device mapping: ONE WARP PER QUERY.  All <=32 link slots of the expanded node are examined
// at once (lane = slot), the visited test-and-set is one atomicOr per lane on a per-warp bitmap in
// HBM, distances are computed with the lanes striding the dimension (coalesced 128-bit row reads,
// two rows in flight), and the candidate pool is a sorted array in shared memory updated by
// warp-cooperative shifts.  The algorithm state after each expansion equals the reference's
// (same pool capacity max(ef,k), same strict/upper_bound tie rules), so with identical graph and
// distances the result is identical; distances differ by fp32 summation order only.  Pools too large for four per CTA
// (max(ef, k) up to 16384) run hnsw_wide_kernel: one query per CTA, same state after every expansion.
#pragma once
#include <omp.h>

#include <cmath>
#include <cub/cub.cuh>
#include <queue>

#include "kb2_blob.h"
#include "kb2_index.cuh"

namespace kb2 {

struct HnswSearchParams {
    const float* vecs;        // [n][d]
    int d;
    int64_t n;
    const int32_t* neighbors;
    const int64_t* offsets;   // [n+1]
    const int32_t* cum;       // cum_nneighbor_per_level
    int32_t entry_point, max_level;
    int metric;
    const float* queries;
    int nq, ef_cap, k;
    uint32_t* visited;        // [total_warps][nwords]
    int64_t nwords;
    int32_t* vis_log;         // [total_warps][log_cap]
    int log_cap;
    int* next_query;          // work counter
    const int64_t* labels;
    int64_t* out_ids;
    float* out_dist;
    unsigned long long* stats;  // [0] ndis, [1] nhops
    // filtered search / range search (hnsw_search_kernel<METRIC, true>, hnsw_wide_kernel<METRIC, true>)
    const uint8_t* bitset;      // bit set => node filtered out, bit index = internal id + bit_offset; or NULL
    int64_t bit_offset;         // first global row of this shard (graph-partition sharding), else 0
    float k_alpha;              // filter_ratio * 0.7 (faiss_hnsw.cc:1425)
    int range_mode;             // 0: top-k, 1: range search
    float radius_key;           // range: keep key < radius_key (key = L2 distance, or -ip)
    RangeHit* hits;             // range: global append buffer
    unsigned long long* hit_count;
    unsigned long long hit_cap;
    int32_t* bfs_queue;         // range: [total_warps][queue_cap]
    int queue_cap;
    uint32_t* q_overflow;       // range: [nq] 1 = the BFS queue overflowed (host reruns that query with a larger queue)
    const int32_t* q_list;      // optional: indices of the queries to run (second pass), nq = its length
    // construction (hnsw_search_kernel as the candidate generator of the batched GPU build)
    int beam_level;             // level the beam runs on (0 for searches); the greedy descent stops above it
    const int32_t* q_nodes;     // optional: query i is the stored vector of node q_nodes[i]
    const int32_t* node_rank;   // optional: insertion rank of every node; the descent only moves to nodes of rank < rank_limit
    int rank_limit;             //           (= nodes already linked on the beam level)
    int key8;                   // 1: level-0 expansion evaluates eight fresh neighbours per batch (KB2_HNSW_KEY8, opt-in)
};

constexpr int kHnswWarps = 4;  // warps (queries in flight) per CTA

// distance key of node v to the query held in shared memory (lanes stride the dimension)
template <int METRIC>
__device__ __forceinline__ float
hnsw_key(const float* __restrict__ vecs, int d, const float* s_q, int32_t v, int lane) {
    const float* x = vecs + (int64_t)v * d;
    float acc = 0.f;
    if ((d & 3) == 0) {
        const float4* x4 = reinterpret_cast<const float4*>(x);
        const float4* q4 = reinterpret_cast<const float4*>(s_q);
        for (int j = lane; j < (d >> 2); j += kWarp) {
            const float4 a = ldg_stream_f4(x4 + j);
            const float4 b = q4[j];
            if (METRIC == KB2_METRIC_L2) {
                float t;
                t = b.x - a.x; acc = fmaf(t, t, acc);
                t = b.y - a.y; acc = fmaf(t, t, acc);
                t = b.z - a.z; acc = fmaf(t, t, acc);
                t = b.w - a.w; acc = fmaf(t, t, acc);
            } else {
                acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
                acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
            }
        }
    } else {
        for (int j = lane; j < d; j += kWarp) {
            if (METRIC == KB2_METRIC_L2) {
                const float t = s_q[j] - x[j];
                acc = fmaf(t, t, acc);
            } else {
                acc = fmaf(s_q[j], x[j], acc);
            }
        }
    }
    acc = warp_sum(acc);
    return (METRIC == KB2_METRIC_L2) ? acc : -acc;  // NegativeDistanceComputer for IP
}

// two rows at once (independent loads in flight)
template <int METRIC>
__device__ __forceinline__ void
hnsw_key2(const float* __restrict__ vecs, int d, const float* s_q, int32_t v0, int32_t v1, int lane, float& k0,
          float& k1) {
    if ((d & 3) != 0) {
        k0 = hnsw_key<METRIC>(vecs, d, s_q, v0, lane);
        k1 = hnsw_key<METRIC>(vecs, d, s_q, v1, lane);
        return;
    }
    const float4* x0 = reinterpret_cast<const float4*>(vecs + (int64_t)v0 * d);
    const float4* x1 = reinterpret_cast<const float4*>(vecs + (int64_t)v1 * d);
    const float4* q4 = reinterpret_cast<const float4*>(s_q);
    float a0 = 0.f, a1 = 0.f;
    for (int j = lane; j < (d >> 2); j += kWarp) {
        const float4 a = ldg_stream_f4(x0 + j);
        const float4 c = ldg_stream_f4(x1 + j);
        const float4 b = q4[j];
        if (METRIC == KB2_METRIC_L2) {
            float t;
            t = b.x - a.x; a0 = fmaf(t, t, a0); t = b.y - a.y; a0 = fmaf(t, t, a0);
            t = b.z - a.z; a0 = fmaf(t, t, a0); t = b.w - a.w; a0 = fmaf(t, t, a0);
            t = b.x - c.x; a1 = fmaf(t, t, a1); t = b.y - c.y; a1 = fmaf(t, t, a1);
            t = b.z - c.z; a1 = fmaf(t, t, a1); t = b.w - c.w; a1 = fmaf(t, t, a1);
        } else {
            a0 = fmaf(a.x, b.x, a0); a0 = fmaf(a.y, b.y, a0); a0 = fmaf(a.z, b.z, a0); a0 = fmaf(a.w, b.w, a0);
            a1 = fmaf(c.x, b.x, a1); a1 = fmaf(c.y, b.y, a1); a1 = fmaf(c.z, b.z, a1); a1 = fmaf(c.w, b.w, a1);
        }
    }
    a0 = warp_sum(a0);
    a1 = warp_sum(a1);
    k0 = (METRIC == KB2_METRIC_L2) ? a0 : -a0;
    k1 = (METRIC == KB2_METRIC_L2) ? a1 : -a1;
}

// four rows at once: 4x the loads in flight per lane (the level-0 expansion is bound by the latency of random 3 KiB rows)
template <int METRIC>
__device__ __forceinline__ void
hnsw_key4(const float* __restrict__ vecs, int d, const float* s_q, int32_t v0, int32_t v1, int32_t v2, int32_t v3, int lane,
          float& k0, float& k1, float& k2, float& k3) {
    const float4* x0 = reinterpret_cast<const float4*>(vecs + (int64_t)v0 * d);
    const float4* x1 = reinterpret_cast<const float4*>(vecs + (int64_t)v1 * d);
    const float4* x2 = reinterpret_cast<const float4*>(vecs + (int64_t)v2 * d);
    const float4* x3 = reinterpret_cast<const float4*>(vecs + (int64_t)v3 * d);
    const float4* q4 = reinterpret_cast<const float4*>(s_q);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int j = lane; j < (d >> 2); j += kWarp) {
        const float4 a = ldg_stream_f4(x0 + j);
        const float4 b = ldg_stream_f4(x1 + j);
        const float4 c = ldg_stream_f4(x2 + j);
        const float4 e = ldg_stream_f4(x3 + j);
        const float4 q = q4[j];
        if (METRIC == KB2_METRIC_L2) {
            float t;
            t = q.x - a.x; a0 = fmaf(t, t, a0); t = q.y - a.y; a0 = fmaf(t, t, a0);
            t = q.z - a.z; a0 = fmaf(t, t, a0); t = q.w - a.w; a0 = fmaf(t, t, a0);
            t = q.x - b.x; a1 = fmaf(t, t, a1); t = q.y - b.y; a1 = fmaf(t, t, a1);
            t = q.z - b.z; a1 = fmaf(t, t, a1); t = q.w - b.w; a1 = fmaf(t, t, a1);
            t = q.x - c.x; a2 = fmaf(t, t, a2); t = q.y - c.y; a2 = fmaf(t, t, a2);
            t = q.z - c.z; a2 = fmaf(t, t, a2); t = q.w - c.w; a2 = fmaf(t, t, a2);
            t = q.x - e.x; a3 = fmaf(t, t, a3); t = q.y - e.y; a3 = fmaf(t, t, a3);
            t = q.z - e.z; a3 = fmaf(t, t, a3); t = q.w - e.w; a3 = fmaf(t, t, a3);
        } else {
            a0 = fmaf(a.x, q.x, a0); a0 = fmaf(a.y, q.y, a0); a0 = fmaf(a.z, q.z, a0); a0 = fmaf(a.w, q.w, a0);
            a1 = fmaf(b.x, q.x, a1); a1 = fmaf(b.y, q.y, a1); a1 = fmaf(b.z, q.z, a1); a1 = fmaf(b.w, q.w, a1);
            a2 = fmaf(c.x, q.x, a2); a2 = fmaf(c.y, q.y, a2); a2 = fmaf(c.z, q.z, a2); a2 = fmaf(c.w, q.w, a2);
            a3 = fmaf(e.x, q.x, a3); a3 = fmaf(e.y, q.y, a3); a3 = fmaf(e.z, q.z, a3); a3 = fmaf(e.w, q.w, a3);
        }
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2); a3 = warp_sum(a3);
    k0 = (METRIC == KB2_METRIC_L2) ? a0 : -a0;
    k1 = (METRIC == KB2_METRIC_L2) ? a1 : -a1;
    k2 = (METRIC == KB2_METRIC_L2) ? a2 : -a2;
    k3 = (METRIC == KB2_METRIC_L2) ? a3 : -a3;
}

// eight rows at once, three dimension chunks unrolled: 24 independent 128-bit loads in flight per lane (a 768-d row is six
// chunks per lane: two round trips per eight rows instead of four with two hnsw_key4 calls).  Per row the arithmetic and
// its order are those of hnsw_key4, so the keys are bit-identical.
template <int METRIC>
__device__ __forceinline__ void
hnsw_key8(const float* __restrict__ vecs, int d, const float* s_q, const int32_t (&v)[8], int lane, float (&k)[8]) {
    const float4* x[8];
#pragma unroll
    for (int r = 0; r < 8; r++) x[r] = reinterpret_cast<const float4*>(vecs + (int64_t)v[r] * d);
    const float4* q4 = reinterpret_cast<const float4*>(s_q);
    float acc[8];
#pragma unroll
    for (int r = 0; r < 8; r++) acc[r] = 0.f;
    const int nj = d >> 2;
    auto fold = [&](float& ac, const float4& q, const float4& a) {
        if (METRIC == KB2_METRIC_L2) {
            float t;
            t = q.x - a.x; ac = fmaf(t, t, ac); t = q.y - a.y; ac = fmaf(t, t, ac);
            t = q.z - a.z; ac = fmaf(t, t, ac); t = q.w - a.w; ac = fmaf(t, t, ac);
        } else {
            ac = fmaf(a.x, q.x, ac); ac = fmaf(a.y, q.y, ac);
            ac = fmaf(a.z, q.z, ac); ac = fmaf(a.w, q.w, ac);
        }
    };
    int j = lane;
    for (; j + 2 * kWarp < nj; j += 3 * kWarp) {   // three chunks of every row: all 24 loads first
        float4 a[3][8];
#pragma unroll
        for (int u = 0; u < 3; u++)
#pragma unroll
            for (int r = 0; r < 8; r++) a[u][r] = ldg_stream_f4(x[r] + j + u * kWarp);
#pragma unroll
        for (int u = 0; u < 3; u++) {
            const float4 q = q4[j + u * kWarp];
#pragma unroll
            for (int r = 0; r < 8; r++) fold(acc[r], q, a[u][r]);
        }
    }
    for (; j < nj; j += kWarp) {
        float4 a[8];
#pragma unroll
        for (int r = 0; r < 8; r++) a[r] = ldg_stream_f4(x[r] + j);
        const float4 q = q4[j];
#pragma unroll
        for (int r = 0; r < 8; r++) fold(acc[r], q, a[r]);
    }
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const float t = warp_sum(acc[r]);
        k[r] = (METRIC == KB2_METRIC_L2) ? t : -t;
    }
}

// greedy descent from max_level to level 1 (HnswSearcher.h:116-170,334-356): first strict minimum over the link slots
template <int METRIC>
__device__ __forceinline__ void
hnsw_descend(const HnswSearchParams& p, const float* s_q, int lane, int32_t& nearest, float& d_nearest,
             unsigned long long& ndis_tot, unsigned long long& nhops_tot) {
    for (int level = p.max_level; level > p.beam_level; level--) {
        for (;;) {
            const int32_t prev = nearest;
            const int64_t begin = p.offsets[prev] + p.cum[level];
            const int64_t end = p.offsets[prev] + p.cum[level + 1];
            bool done = false;
            for (int64_t b = begin; b < end && !done; b += kWarp) {
                const int32_t v = (b + lane < end) ? p.neighbors[b + lane] : -1;
                const unsigned neg = __ballot_sync(0xffffffffu, v < 0);
                const int cnt = neg ? (__ffs(neg) - 1) : kWarp;
                float myk = INFINITY;
                for (int j = 0; j < cnt; j += 2) {
                    const int32_t va = __shfl_sync(0xffffffffu, v, j);
                    float ka, kb = INFINITY;
                    if (j + 1 < cnt) {
                        const int32_t vb = __shfl_sync(0xffffffffu, v, j + 1);
                        hnsw_key2<METRIC>(p.vecs, p.d, s_q, va, vb, lane, ka, kb);
                    } else {
                        ka = hnsw_key<METRIC>(p.vecs, p.d, s_q, va, lane);
                    }
                    if (lane == j) myk = ka;
                    if (lane == j + 1) myk = kb;
                }
                ndis_tot += cnt;
                if (p.node_rank && lane < cnt && p.node_rank[v] >= p.rank_limit) myk = INFINITY;
                // sequential "if (dis < d_nearest)" over the slots == first strict minimum
                float bk = myk;
                int bl = lane;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float ok = __shfl_xor_sync(0xffffffffu, bk, o);
                    const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
                    if (ok < bk || (ok == bk && ol < bl)) { bk = ok; bl = ol; }
                }
                if (bk < d_nearest) {
                    d_nearest = bk;
                    nearest = __shfl_sync(0xffffffffu, v, bl);
                }
                if (cnt < kWarp) done = true;
            }
            nhops_tot++;
            if (nearest == prev) break;
        }
    }
}

// pos = upper_bound(key) in the sorted dist[0, size)
__device__ __forceinline__ int
hnsw_upper_bound(const float* dist, int size, float key, int lane) {
    int pos = 0;
    for (int base = 0; base < size; base += kWarp) {
        const int i = base + lane;
        const bool le = (i < size) && (dist[i] <= key);
        pos += __popc(__ballot_sync(0xffffffffu, le));
    }
    return pos;
}
// insert (key, idv) at pos < cap, dropping the last entry when full; returns the new size
__device__ __forceinline__ int
hnsw_shift_insert(float* dist, uint32_t* id, int size, int cap, int pos, float key, uint32_t idv, int lane) {
    const int newsize = min(size + 1, cap);
    for (int hi = newsize - 1; hi > pos; hi -= kWarp) {
        const int i = hi - lane;
        float td = 0.f;
        uint32_t ti = 0;
        if (i > pos) { td = dist[i - 1]; ti = id[i - 1]; }
        __syncwarp();
        if (i > pos) { dist[i] = td; id[i] = ti; }
        __syncwarp();
    }
    if (lane == 0) { dist[pos] = key; id[pos] = idv; }
    __syncwarp();
    return newsize;
}

// Greedy descent, then the beam's first entry: the node the descent ends on, marked visited and logged, goes to the valid
// pool (v_*) when it is a member, else to the invalid pool (i_*).  filter: the search has a bitset.  Returns whether it
// is a member.
template <int METRIC>
__device__ __forceinline__ bool
hnsw_enter(const HnswSearchParams& p, bool filter, const float* s_q, int lane, float* v_dist, uint32_t* v_id, float* i_dist,
           uint32_t* i_id, uint32_t* vis, int32_t* vlog, unsigned long long& ndis_tot, unsigned long long& nhops_tot) {
    int32_t nearest = p.entry_point;
    float d_nearest = hnsw_key<METRIC>(p.vecs, p.d, s_q, nearest, lane);
    hnsw_descend<METRIC>(p, s_q, lane, nearest, d_nearest, ndis_tot, nhops_tot);
    const bool member = !(filter && bit_is_set(p.bitset, nearest + p.bit_offset));
    if (lane == 0) {
        if (member) { v_dist[0] = d_nearest; v_id[0] = (uint32_t)nearest; }
        else { i_dist[0] = d_nearest; i_id[0] = (uint32_t)nearest; }
        atomicOr(&vis[nearest >> 5], 1u << (nearest & 31));
        vlog[0] = nearest;
    }
    return member;
}

// Link row [begin, end) in 32-slot chunks, lane = slot, up to its first -1: the visited test-and-set, and the fresh
// neighbours appended to the touched-id log (past log_cap they are only counted, and the clean-up clears the whole
// bitmap).  For each chunk with a fresh neighbour, body(v, fm, inv_m): v the lane's neighbour, fm the fresh mask, inv_m
// (FILTERED) the fresh neighbours the bitset filters out (filter: the search has a bitset).
template <bool FILTERED, typename Body>
__device__ __forceinline__ void
hnsw_scan_links(const HnswSearchParams& p, bool filter, uint32_t* vis, int32_t* vlog, int& logn, bool& log_overflow,
                int64_t begin, int64_t end, int lane, Body&& body) {
    bool done = false;
    for (int64_t b = begin; b < end && !done; b += kWarp) {
        const int32_t v = (b + lane < end) ? p.neighbors[b + lane] : -1;
        const unsigned neg = __ballot_sync(0xffffffffu, v < 0);
        const int cnt = neg ? (__ffs(neg) - 1) : kWarp;
        if (cnt < kWarp) done = true;
        bool fresh = false, member = true;
        if (lane < cnt) {
            const uint32_t bit = 1u << (v & 31);
            const uint32_t old = atomicOr(&vis[v >> 5], bit);
            fresh = !(old & bit);
            if (FILTERED && fresh && filter) member = !bit_is_set(p.bitset, v + p.bit_offset);
        }
        const unsigned fm = __ballot_sync(0xffffffffu, fresh);
        const int nf = __popc(fm);
        if (nf == 0) continue;
        if (logn + nf <= p.log_cap) {
            if (fresh) vlog[logn + __popc(fm & ((1u << lane) - 1))] = v;
        } else {
            log_overflow = true;
        }
        logn += nf;
        const unsigned inv_m = FILTERED ? __ballot_sync(0xffffffffu, fresh && !member) : 0u;
        body(v, fm, inv_m);
    }
}

// kAlpha budget (HnswSearcher.h:213-225): which of the filtered-out fresh neighbours inv still cost a distance, walked in
// slot order; alpha is the query's accumulated_alpha
__device__ __forceinline__ unsigned
hnsw_alpha_walk(unsigned inv, float k_alpha, float& alpha) {
    unsigned take = 0;
    while (inv) {
        const int j = __ffs(inv) - 1;
        inv &= inv - 1;
        alpha += k_alpha;
        if (alpha < 1.0f) continue;
        alpha -= 1.0f;
        take |= 1u << j;
    }
    return take;
}

// Keys of the neighbours v of the lanes in rem, evaluated in slot order in batches of eight (KB2_HNSW_KEY8), four, two
// and one row, the widest batch bounded by WIDEST.  Returns the lane's own key (INFINITY for lanes not in rem).
template <int METRIC, int WIDEST>
__device__ __forceinline__ float
hnsw_slot_keys(const HnswSearchParams& p, const float* s_q, int32_t v, unsigned rem, int lane) {
    float myk = INFINITY;
    if constexpr (WIDEST >= 8) {
        while (p.key8 && (p.d & 3) == 0 && __popc(rem) >= 8) {
            int js[8];
            int32_t vs[8];
            float ks[8];
#pragma unroll
            for (int r = 0; r < 8; r++) {
                js[r] = __ffs(rem) - 1;
                rem &= rem - 1;
                vs[r] = __shfl_sync(0xffffffffu, v, js[r]);
            }
            hnsw_key8<METRIC>(p.vecs, p.d, s_q, vs, lane, ks);
#pragma unroll
            for (int r = 0; r < 8; r++)
                if (lane == js[r]) myk = ks[r];
        }
    }
    if constexpr (WIDEST >= 4) {
        while ((p.d & 3) == 0 && __popc(rem) >= 4) {
            const int j0 = __ffs(rem) - 1; rem &= rem - 1;
            const int j1 = __ffs(rem) - 1; rem &= rem - 1;
            const int j2 = __ffs(rem) - 1; rem &= rem - 1;
            const int j3 = __ffs(rem) - 1; rem &= rem - 1;
            float q0, q1, q2, q3;
            hnsw_key4<METRIC>(p.vecs, p.d, s_q, __shfl_sync(0xffffffffu, v, j0), __shfl_sync(0xffffffffu, v, j1),
                              __shfl_sync(0xffffffffu, v, j2), __shfl_sync(0xffffffffu, v, j3), lane, q0, q1, q2, q3);
            if (lane == j0) myk = q0;
            if (lane == j1) myk = q1;
            if (lane == j2) myk = q2;
            if (lane == j3) myk = q3;
        }
    }
    while (rem) {
        const int ja = __ffs(rem) - 1;
        rem &= rem - 1;
        const int32_t va = __shfl_sync(0xffffffffu, v, ja);
        float ka, kb = INFINITY;
        int jb = -1;
        if (rem) {
            jb = __ffs(rem) - 1;
            rem &= rem - 1;
            const int32_t vb = __shfl_sync(0xffffffffu, v, jb);
            hnsw_key2<METRIC>(p.vecs, p.d, s_q, va, vb, lane, ka, kb);
        } else {
            ka = hnsw_key<METRIC>(p.vecs, p.d, s_q, va, lane);
        }
        if (lane == ja) myk = ka;
        if (lane == jb) myk = kb;
    }
    return myk;
}

// top-k row q from the sorted pool (HnswSearcher.h:414-428; IP sign restored as IndexHNSWWrapper.cc:198-204), padded
// with -1 / ±FLT_MAX; thread t of stride
template <int METRIC>
__device__ __forceinline__ void
hnsw_write_row(const HnswSearchParams& p, int q, const float* dist, const uint32_t* id, int size, int t, int stride) {
    const int len = min(size, p.k);
    for (int i = t; i < p.k; i += stride) {
        const int64_t o = (int64_t)q * p.k + i;
        if (i < len) {
            const int64_t idv = (int64_t)(id[i] & 0x7fffffffu);
            p.out_ids[o] = p.labels ? p.labels[idv] : idv;
            p.out_dist[o] = (METRIC == KB2_METRIC_L2) ? dist[i] : -dist[i];
        } else {
            p.out_ids[o] = -1;
            p.out_dist[o] = (METRIC == KB2_METRIC_L2) ? FLT_MAX : -FLT_MAX;
        }
    }
}

// clear the visited bits of a traversal: the logged words, or the whole bitmap when the log overflowed; thread t of stride
__device__ __forceinline__ void
hnsw_clear_visited(const HnswSearchParams& p, uint32_t* vis, const int32_t* vlog, int logn, bool log_overflow, int t,
                   int stride) {
    if (!log_overflow) {
        for (int i = t; i < logn; i += stride) vis[vlog[i] >> 5] = 0u;
    } else {
        for (int64_t i = t; i < p.nwords; i += stride) vis[i] = 0u;
    }
}

// ============================================================================================
// hnsw_search_kernel<METRIC, FILTERED>: one warp per query.  The reference always runs the two-pool searcher; FILTERED
// = false is its all-members special case, one pool (also the candidate generator of the GPU build: q_nodes, beam_level,
// node_rank).  FILTERED = true is the filtered top-k search and range search (a bitset that may be null):
//   NeighborSetDoublePopList                      K/impl/Neighbor.h:155-210
//   evaluate_single_node with kAlpha              K/impl/HnswSearcher.h:173-293 (:213-225 accumulated_alpha)
//   search / range_search                         K/impl/HnswSearcher.h:358-432, 435-553
// Valid pool: sorted array with a cursor and "checked" flags (capacity cap).  Invalid pool (filtered-out nodes that
// are still traversed): sorted array of capacity cap, popped from the front; a filtered node is admitted only while
// it is closer than the valid pool's back.  A filtered fresh neighbour costs a distance only every 1/kAlpha-th time
// (accumulated_alpha), evaluated in link-slot order like the reference.
// dynamic smem per warp: d floats (query, 16B aligned) + the valid pool, cap * (4 + 4), + FILTERED: the invalid pool,
// cap * (4 + 4)
// The launch bound keeps the allocation the two kernels had before they were one: 96 registers for the plain instances
// (five CTAs per SM, DESIGN §4.7), 80 for the two-pool ones (six).  Left to itself ptxas gives the folded two-pool L2
// instance 64 registers and spills in the expansion loop, and the filtered search then runs 20 % slower (DESIGN §4.7).
// ============================================================================================
template <int METRIC, bool FILTERED>
__global__ void __launch_bounds__(kHnswWarps * 32, FILTERED ? 6 : 5)
hnsw_search_kernel(HnswSearchParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dpad = (p.d + 3) & ~3;
    const int cap = p.ef_cap;
    // 16-byte aligned per-warp regions: the query row is read as float4 (an odd ef would misalign every other warp's)
    const size_t per_warp = ((size_t)dpad * 4 + (size_t)cap * (FILTERED ? 16 : 8) + 15) & ~(size_t)15;
    unsigned char* mine = smem_raw + (size_t)warp * per_warp;
    float* s_q = (float*)mine;
    float* v_dist = (float*)(mine + (size_t)dpad * 4);
    uint32_t* v_id = (uint32_t*)(v_dist + cap);   // bit31 = checked
    // the invalid pool: FILTERED only.  The plain instance's pointers lie past its region and are never dereferenced
    // (every node is a member there and inv_m is 0).
    float* i_dist = (float*)(v_id + cap);
    uint32_t* i_id = (uint32_t*)(i_dist + cap);
    const int level = FILTERED ? 0 : p.beam_level;

    const int64_t gw = (int64_t)blockIdx.x * kHnswWarps + warp;
    uint32_t* vis = p.visited + gw * p.nwords;
    int32_t* vlog = p.vis_log + gw * p.log_cap;
    int32_t* queue = (FILTERED && p.bfs_queue) ? p.bfs_queue + gw * (int64_t)p.queue_cap : nullptr;
    unsigned long long ndis_tot = 0, nhops_tot = 0;

    for (;;) {
        int qi = 0;
        if (lane == 0) qi = atomicAdd(p.next_query, 1);
        qi = __shfl_sync(0xffffffffu, qi, 0);
        if (qi >= p.nq) break;
        const int q = (FILTERED && p.q_list) ? p.q_list[qi] : qi;
        const float* qsrc = (!FILTERED && p.q_nodes) ? p.vecs + (int64_t)p.q_nodes[q] * p.d : p.queries + (int64_t)q * p.d;
        for (int j = lane; j < p.d; j += kWarp) s_q[j] = qsrc[j];
        __syncwarp();

        int v_size = 0, v_cur = 0, i_size = 0, logn = 1;
        bool log_overflow = false;
        const bool member =
            hnsw_enter<METRIC>(p, FILTERED && p.bitset, s_q, lane, v_dist, v_id, i_dist, i_id, vis, vlog, ndis_tot, nhops_tot);
        if (member) v_size = 1; else i_size = 1;
        __syncwarp();
        float alpha = 1.0f;   // initial_accumulated_alpha

        // ---- beam (HnswSearcher.h:296-332,390-432; Neighbor.h:46-210)
        for (;;) {
            bool take_inv = false;
            if (FILTERED) {
                const float back = (v_size < cap) ? FLT_MAX : v_dist[cap - 1];
                const bool has_res = v_cur < v_size, has_cand = i_size > 0;
                if (!(has_res || (has_cand && i_dist[0] < back))) break;
                take_inv = has_cand && (!has_res || i_dist[0] < v_dist[v_cur]);
            } else if (v_cur >= v_size) {
                break;
            }
            uint32_t cur_id;
            if (take_inv) {
                cur_id = i_id[0];
                __syncwarp();
                for (int base = 0; base < i_size - 1; base += kWarp) {   // pop front: shift left by one
                    const int i = base + lane;
                    float td = 0.f;
                    uint32_t ti = 0;
                    if (i < i_size - 1) { td = i_dist[i + 1]; ti = i_id[i + 1]; }
                    __syncwarp();
                    if (i < i_size - 1) { i_dist[i] = td; i_id[i] = ti; }
                    __syncwarp();
                }
                i_size--;
            } else {
                cur_id = v_id[v_cur] & 0x7fffffffu;
                __syncwarp();
                if (lane == 0) v_id[v_cur] |= 0x80000000u;
                __syncwarp();
                v_cur++;
                while (v_cur < v_size && (v_id[v_cur] & 0x80000000u)) v_cur++;
            }
            nhops_tot++;

            const int64_t begin = p.offsets[cur_id] + p.cum[level];
            const int64_t end = p.offsets[cur_id] + p.cum[level + 1];
            hnsw_scan_links<FILTERED>(p, p.bitset, vis, vlog, logn, log_overflow, begin, end, lane,
                                      [&](int32_t v, unsigned fm, unsigned inv_m) {
                const unsigned take_m = FILTERED ? (fm & ~inv_m) | hnsw_alpha_walk(inv_m, p.k_alpha, alpha) : fm;
                ndis_tot += __popc(take_m);
                const float myk = hnsw_slot_keys<METRIC, FILTERED ? 2 : 8>(p, s_q, v, take_m, lane);
                // insert in slot order (the reference inserts batch-4 results in the same order)
                unsigned ins = take_m;
                while (ins) {
                    const int j = __ffs(ins) - 1;
                    ins &= ins - 1;
                    const float key = __shfl_sync(0xffffffffu, myk, j);
                    const uint32_t id = (uint32_t)__shfl_sync(0xffffffffu, v, j);
                    if (!((inv_m >> j) & 1u)) {
                        const int pos = hnsw_upper_bound(v_dist, v_size, key, lane);
                        if (pos >= cap) continue;
                        v_size = hnsw_shift_insert(v_dist, v_id, v_size, cap, pos, key, id, lane);
                        if (pos < v_cur) v_cur = pos;
                    } else {
                        const float bk = (v_size < cap) ? FLT_MAX : v_dist[cap - 1];
                        if (!(key < bk)) continue;
                        const int pos = hnsw_upper_bound(i_dist, i_size, key, lane);
                        if (pos >= cap) continue;
                        i_size = hnsw_shift_insert(i_dist, i_id, i_size, cap, pos, key, id, lane);
                    }
                }
            });
        }

        __syncwarp();
        hnsw_clear_visited(p, vis, vlog, logn, log_overflow, lane, kWarp);
        __syncwarp();
        if (!FILTERED || !p.range_mode) {
            hnsw_write_row<METRIC>(p, q, v_dist, v_id, v_size, lane, kWarp);
            continue;
        }

        // ---- range search, second phase (HnswSearcher.h:497-545): closure of the in-range valid candidates over the
        //      level-0 links; a node is expanded iff it is a member with key < radius (so the result is order-free)
        int qh = 0, qt = 0;           // queue head / tail (entries [qh, qt) pending)
        bool q_over = false;
        logn = 0;
        log_overflow = false;
        auto emit = [&](uint32_t id, float key, bool mine_) {   // lanes with mine_ append one hit each
            const unsigned m = __ballot_sync(0xffffffffu, mine_);
            if (!m) return;
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(p.hit_count, (unsigned long long)__popc(m));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (mine_) {
                const unsigned long long slot = base + __popc(m & ((1u << lane) - 1));
                if (slot < p.hit_cap) {
                    RangeHit h;
                    h.q = q;
                    h.probe = 0;
                    h.pos = id;
                    h.dist = (METRIC == KB2_METRIC_L2) ? key : -key;
                    p.hits[slot] = h;
                }
                const int qs = qt + __popc(m & ((1u << lane) - 1));
                if (qs < p.queue_cap) queue[qs] = (int32_t)id; else q_over = true;
            }
            qt += __popc(m);
            q_over = __any_sync(0xffffffffu, q_over);
        };
        for (int base = 0; base < v_size; base += kWarp) {
            const int i = base + lane;
            const bool ok = i < v_size && v_dist[i] < p.radius_key;
            const uint32_t id = ok ? (v_id[i] & 0x7fffffffu) : 0u;
            if (ok) atomicOr(&vis[id >> 5], 1u << (id & 31));
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            if (logn + __popc(m) <= p.log_cap) {
                if (ok) vlog[logn + __popc(m & ((1u << lane) - 1))] = (int32_t)id;
            } else {
                log_overflow = true;
            }
            logn += __popc(m);
            emit(id, ok ? v_dist[i] : 0.f, ok);
        }
        while (qh < min(qt, p.queue_cap) && !q_over) {
            const int32_t cur = queue[qh++];
            const int64_t begin = p.offsets[cur] + p.cum[0];
            const int64_t end = p.offsets[cur] + p.cum[1];
            hnsw_scan_links<true>(p, p.bitset, vis, vlog, logn, log_overflow, begin, end, lane,
                                  [&](int32_t v, unsigned fm, unsigned inv_m) {
                const unsigned take_m = fm & ~inv_m;
                ndis_tot += __popc(take_m);
                const float myk = hnsw_slot_keys<METRIC, 2>(p, s_q, v, take_m, lane);
                const bool hit = ((take_m >> lane) & 1u) && myk < p.radius_key;
                emit((uint32_t)v, myk, hit);
            });
        }
        if (q_over && lane == 0) p.q_overflow[q] = 1u;
        __syncwarp();
        hnsw_clear_visited(p, vis, vlog, logn, log_overflow, lane, kWarp);
        __syncwarp();
    }
    if (p.stats && lane == 0) {
        atomicAdd(&p.stats[0], ndis_tot);
        atomicAdd(&p.stats[1], nhops_tot);
    }
}


// ============================================================================================
// One query per CTA: hnsw_wide_kernel<METRIC, FILTERED> runs the beams whose pools do not fit the four-warp layout of
// hnsw_search_kernel (DESIGN §4.7), max(ef, k) up to kMaxLargeK.  FILTERED is hnsw_search_kernel's of the same value
// (for FILTERED = true its top-k traversal: two pools, kAlpha budget).  The state after every expansion is theirs, and
// so the reference's:
//   * warp 0 reads the popped node's link row in 32-slot chunks and does the visited test-and-set, the touched-id log
//     and the kAlpha walk in slot order, exactly as the warp kernels; it lists the evaluated neighbours in slot order;
//   * every warp then computes keys of whole rows (hnsw_key4 / hnsw_key: the warp kernels' per-row arithmetic, so the
//     keys are bit-identical);
//   * the listed neighbours enter the pool in one CTA-wide merge (hnsw_wide_merge), which gives the pool of the one-by-one
//     upper_bound inserts in slot order;
//   * filtered: an invalid neighbour at slot j is admitted while its key is below the valid pool's back as it stands after
//     the valid neighbours of slots < j were inserted (thread 0 replays that back, see below).
// The valid pool lives in shared memory; the invalid pool, popped from the front, in a per-CTA global scratch of 2 * cap
// entries addressed through a head offset (compacted when the head passes cap).
// dynamic smem: 8 control ints | query (dpad floats) | valid pool (cap x (4 + 4)) | candidates (deg x 21 bytes)
// ============================================================================================
constexpr int kWideWarps = 8;
constexpr int kWideThreads = kWideWarps * 32;
constexpr int kWideItems = 4;   // pool entries each thread moves per step of the merge

struct HnswWideParams {
    HnswSearchParams s;
    int deg;              // level-0 link slots per node: bound on the neighbours one expansion evaluates
    float* inv_dist;      // FILTERED: [grid][2 * ef_cap] invalid pool of each CTA
    uint32_t* inv_id;
};

// Merges the candidates t < m with kind[t] == want (keys ck, ids cv, listed in link-slot order) into the sorted pool
// (dist, id) of `size` entries, keeping the first cap.  This is the pool the reference's one-by-one inserts build
// (Neighbor.h:46-150): each insert goes at upper_bound(key), i.e. after every equal key already present, earlier
// candidates of the same expansion included, so the final order is (key; old entries, then candidates in slot order),
// and dropping the last entry at every step keeps the same first cap entries as truncating once.  The smallest insert
// position of the sequence is the first position written here.  Returns it (cap if nothing enters).  Called by every
// thread with the same arguments; starts and ends at a barrier.
__device__ int
hnsw_wide_merge(float* dist, uint32_t* id, int& size, int cap, const float* ck, const int32_t* cv, const uint8_t* kind,
                int want, int m, int* c_dest, float* s_sorted, int* s_ctl) {
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid < kWarp) {
        int nsel = 0, p0 = cap;
        for (int base = 0; base < m; base += kWarp) {
            const int t = base + lane;
            const bool sel = t < m && kind[t] == want;
            int dest = INT_MAX;
            if (sel) {
                const float key = ck[t];
                int r = 0;   // rank among the selected candidates by (key, slot)
                for (int u = 0; u < m; u++) r += kind[u] == want && (ck[u] < key || (ck[u] == key && u < t));
                int lo = 0, hi = size;   // upper_bound(key) in the pool
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (dist[mid] <= key) lo = mid + 1; else hi = mid;
                }
                dest = lo + r;
                s_sorted[r] = key;
                p0 = min(p0, dest);
            }
            if (t < m) c_dest[t] = dest;
            nsel += __popc(__ballot_sync(0xffffffffu, sel));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) p0 = min(p0, __shfl_xor_sync(0xffffffffu, p0, o));
        if (lane == 0) { s_ctl[0] = nsel; s_ctl[1] = p0; }
    }
    __syncthreads();
    const int nsel = s_ctl[0], p0 = s_ctl[1];
    if (p0 < cap) {
        // entry i >= p0 moves up by the number of candidates with a smaller key; high chunks first, so every destination
        // has been read before it is written
        constexpr int kChunk = kWideThreads * kWideItems;
        for (int hi = min(size, cap); hi > p0; hi -= kChunk) {
            const int lo = max(p0, hi - kChunk);
            float dv[kWideItems];
            uint32_t iv[kWideItems];
            int to[kWideItems];
#pragma unroll
            for (int u = 0; u < kWideItems; u++) {
                const int i = lo + tid + u * kWideThreads;
                to[u] = -1;
                if (i < hi) {
                    dv[u] = dist[i];
                    iv[u] = id[i];
                    int a = 0, b = nsel;   // lower_bound(dv[u]) among the sorted candidate keys
                    while (a < b) {
                        const int mid = (a + b) >> 1;
                        if (s_sorted[mid] < dv[u]) a = mid + 1; else b = mid;
                    }
                    if (i + a < cap) to[u] = i + a;
                }
            }
            __syncthreads();
#pragma unroll
            for (int u = 0; u < kWideItems; u++)
                if (to[u] >= 0) { dist[to[u]] = dv[u]; id[to[u]] = iv[u]; }
            __syncthreads();
        }
        for (int t = tid; t < m; t += kWideThreads)
            if (c_dest[t] < cap) { dist[c_dest[t]] = ck[t]; id[c_dest[t]] = (uint32_t)cv[t]; }
    }
    __syncthreads();
    size = min(size + nsel, cap);
    return p0;
}

template <int METRIC, bool FILTERED>
__global__ void __launch_bounds__(kWideThreads)
hnsw_wide_kernel(HnswWideParams w) {
    const HnswSearchParams& p = w.s;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int dpad = (p.d + 3) & ~3;
    const int cap = p.ef_cap, deg = w.deg;
    int* s_ctl = (int*)smem_raw;
    float* s_q = (float*)(smem_raw + 32);
    float* v_dist = s_q + dpad;
    uint32_t* v_id = (uint32_t*)(v_dist + cap);   // bit31 = checked
    int32_t* c_v = (int32_t*)(v_id + cap);        // neighbours evaluated by this expansion, in slot order
    float* c_key = (float*)(c_v + deg);
    int* c_dest = (int*)(c_key + deg);
    float* s_sorted = (float*)(c_dest + deg);
    float* s_add = s_sorted + deg;
    uint8_t* c_kind = (uint8_t*)(s_add + deg);     // 0 member, 1 filtered and admitted, 2 filtered and not admitted

    uint32_t* vis = p.visited + (int64_t)blockIdx.x * p.nwords;
    int32_t* vlog = p.vis_log + (int64_t)blockIdx.x * p.log_cap;
    float* i_dist = FILTERED ? w.inv_dist + (int64_t)blockIdx.x * 2 * cap : nullptr;
    uint32_t* i_id = FILTERED ? w.inv_id + (int64_t)blockIdx.x * 2 * cap : nullptr;
    unsigned long long ndis_tot = 0, nhops_tot = 0;   // thread 0's are the CTA's
    int logn = 0;                                     // warp 0: touched-id log
    bool log_overflow = false;
    float alpha = 1.0f;                               // warp 0: accumulated_alpha

    for (;;) {
        if (tid == 0) s_ctl[0] = atomicAdd(p.next_query, 1);
        __syncthreads();
        const int q = s_ctl[0];
        if (q >= p.nq) break;
        for (int j = tid; j < p.d; j += kWideThreads) s_q[j] = p.queries[(int64_t)q * p.d + j];
        __syncthreads();

        if (warp == 0) {
            const bool member =
                hnsw_enter<METRIC>(p, FILTERED, s_q, lane, v_dist, v_id, i_dist, i_id, vis, vlog, ndis_tot, nhops_tot);
            if (lane == 0) s_ctl[1] = member ? 1 : 0;
            logn = 1;
            log_overflow = false;
            alpha = 1.0f;
        }
        __syncthreads();
        int v_size = 0, v_cur = 0, i_head = 0, i_size = 0;   // the same in every thread
        if (s_ctl[1]) v_size = 1; else i_size = 1;

        for (;;) {
            // ---- pop (Neighbor.h:46-150 / 155-210)
            bool take_inv = false;
            if (FILTERED) {
                const float back = (v_size < cap) ? FLT_MAX : v_dist[cap - 1];
                const bool has_res = v_cur < v_size, has_cand = i_size > 0;
                if (!(has_res || (has_cand && i_dist[i_head] < back))) break;
                take_inv = has_cand && (!has_res || i_dist[i_head] < v_dist[v_cur]);
            } else if (v_cur >= v_size) {
                break;
            }
            uint32_t cur;
            int popped = -1;
            if (take_inv) {
                cur = i_id[i_head];
                i_head++;
                if (--i_size == 0) i_head = 0;
            } else {
                cur = v_id[v_cur] & 0x7fffffffu;
                popped = v_cur++;
                while (v_cur < v_size && (v_id[v_cur] & 0x80000000u)) v_cur++;
            }
            nhops_tot++;

            // ---- warp 0: link row, visited test-and-set, kAlpha walk, in slot order
            if (warp == 0) {
                const int64_t begin = p.offsets[cur] + p.cum[0];
                const int64_t end = p.offsets[cur] + p.cum[1];
                int m = 0;
                hnsw_scan_links<FILTERED>(p, true, vis, vlog, logn, log_overflow, begin, end, lane,
                                          [&](int32_t v, unsigned fm, unsigned inv_m) {
                    const unsigned take_m = FILTERED ? (fm & ~inv_m) | hnsw_alpha_walk(inv_m, p.k_alpha, alpha) : fm;
                    ndis_tot += __popc(take_m);
                    if ((take_m >> lane) & 1u) {
                        const int t = m + __popc(take_m & ((1u << lane) - 1));
                        c_v[t] = v;
                        c_kind[t] = ((inv_m >> lane) & 1u) ? 1 : 0;
                    }
                    m += __popc(take_m);
                });
                if (lane == 0) s_ctl[2] = m;
            }
            __syncthreads();
            const int m = s_ctl[2];
            if (tid == 0 && popped >= 0) v_id[popped] |= 0x80000000u;

            // ---- keys: whole rows per warp, four at a time when every warp has work
            const int per = (m > kWideWarps && (p.d & 3) == 0) ? 4 : 1;
            for (int g = warp * per; g < m; g += kWideWarps * per) {
                if (per == 4 && g + 4 <= m) {
                    float k0, k1, k2, k3;
                    hnsw_key4<METRIC>(p.vecs, p.d, s_q, c_v[g], c_v[g + 1], c_v[g + 2], c_v[g + 3], lane, k0, k1, k2, k3);
                    if (lane == 0) { c_key[g] = k0; c_key[g + 1] = k1; c_key[g + 2] = k2; c_key[g + 3] = k3; }
                } else {
                    for (int t = g; t < min(g + per, m); t++) {
                        const float kt = hnsw_key<METRIC>(p.vecs, p.d, s_q, c_v[t], lane);
                        if (lane == 0) c_key[t] = kt;
                    }
                }
            }
            __syncthreads();
            if (m == 0) continue;

            // ---- filtered: admission of the invalid neighbours.  The back the reference compares against at slot j is
            //      the cap-th smallest key of the old valid pool plus the valid neighbours of slots < j (a valid neighbour
            //      that did not enter is not below that back, so counting it changes nothing); thread 0 keeps those keys
            //      sorted and reads the back off the merged tail.
            if (FILTERED) {
                if (tid == 0) {
                    int ns = 0;
                    for (int t = 0; t < m; t++) {
                        const float key = c_key[t];
                        if (c_kind[t] == 0) {
                            int j = ns++;
                            while (j > 0 && s_add[j - 1] > key) { s_add[j] = s_add[j - 1]; j--; }
                            s_add[j] = key;
                            continue;
                        }
                        float bk = FLT_MAX;
                        const int over = v_size + ns - cap;   // >= 0: the valid pool is full
                        if (over >= 0) {
                            int a = v_size - 1, b = ns - 1;   // drop the `over` largest of the union, then take its largest
                            for (int s = 0; s < over; s++) {
                                if (b >= 0 && (a < 0 || s_add[b] >= v_dist[a])) b--; else a--;
                            }
                            bk = (b >= 0 && (a < 0 || s_add[b] >= v_dist[a])) ? s_add[b] : v_dist[a];
                        }
                        c_kind[t] = key < bk ? 1 : 2;
                    }
                }
                __syncthreads();
            }

            // ---- merge into the pools
            const int p0 = hnsw_wide_merge(v_dist, v_id, v_size, cap, c_key, c_v, c_kind, 0, m, c_dest, s_sorted, s_ctl + 4);
            if (p0 < v_cur) v_cur = p0;
            if (FILTERED) {
                if (i_head > cap) {   // room for cap entries past the head: move the pool to the front
                    for (int i = tid; i < i_size; i += kWideThreads) {   // [head, head + size) and [0, size) are disjoint
                        i_dist[i] = i_dist[i_head + i];
                        i_id[i] = i_id[i_head + i];
                    }
                    __syncthreads();
                    i_head = 0;
                }
                hnsw_wide_merge(i_dist + i_head, i_id + i_head, i_size, cap, c_key, c_v, c_kind, 1, m, c_dest, s_sorted,
                                s_ctl + 4);
            }
        }

        hnsw_write_row<METRIC>(p, q, v_dist, v_id, v_size, tid, kWideThreads);
        // ---- clear the visited bits this query set (warp 0 kept the log)
        if (tid == 0) s_ctl[3] = log_overflow ? -1 : logn;
        __syncthreads();
        const int nlog = s_ctl[3];
        hnsw_clear_visited(p, vis, vlog, nlog, nlog < 0, tid, kWideThreads);
        __syncthreads();
    }
    if (p.stats && tid == 0) {
        atomicAdd(&p.stats[0], ndis_tot);
        atomicAdd(&p.stats[1], nhops_tot);
    }
}


// ============================================================================================
// GPU construction (SURVEY 8f rank 3; reference: K/IndexHNSW.cpp:83-215 hnsw_add_vertices, K/impl/HNSW.cpp:231-300
// shrink_neighbor_list, :302-420 add_links_starting_from).  The reference inserts one node at a time under per-node locks;
// here every level is built by BATCHED insertion in the reference's order (levels descending): for a batch of new nodes
//   1. hnsw_search_kernel (beam on that level, ef = efConstruction, entry from the finished upper levels) -> candidates
//   2. hnsw_select_kernel: shrink_neighbor_list (K/impl/HNSW.cpp:285-307): fewer candidates than the row holds are all
//      kept, else the heuristic (keep c unless some kept s has dist(c,s) < dist(c,q)); one (s << 32 | w) pair per link
//   3. cub::DeviceRadixSort of the pairs, so that each target s gets its arrivals in batch order
//   4. hnsw_link_kernel: one warp per target s appends the new nodes to s's row; a full row is re-shrunk with the heuristic
// Nodes of one batch do not see each other; batches grow with the graph (<= 1/4 of it), so the effect is that of a few
// concurrent inserters in the reference.  No step depends on scheduling, so a build is a function of the data and the
// parameters: tests/hnsw_build_model.py restates it and the device graph equals it bit for bit on small-integer data.
// ============================================================================================
struct HnswBuildParams {
    const float* vecs;
    int d, metric, level;
    int32_t* neighbors;
    const int64_t* offsets;
    const int32_t* cum;
    const int32_t* batch;        // [nb] node ids being inserted
    int nb, ef;
    const int64_t* cand_ids;     // [nb][ef] ascending by key (from the search kernel), -1 padded
    const float* cand_dist;      // [nb][ef] distances as Search reports them (IP un-negated)
    unsigned long long* pairs;   // [nb][64] (s << 32 | w) per selected neighbour s of batch[w], then pair_end
    const unsigned long long* sorted;   // the pairs, ascending
    unsigned long long pair_end; // (n << 32): sorts after every pair, its target is no node
};
constexpr int kBuildWarps = 4;

// keep candidate c (key kc to the centre) unless an already kept s is closer to c than the centre is
template <int METRIC>
__device__ __forceinline__ bool
hnsw_heuristic_keep(const float* __restrict__ vecs, int d, const float* s_c /* vector of c in smem */, float kc, const int32_t* s_sel,
                    int nsel, int lane) {
    int j = 0;
    if ((d & 3) == 0) {
        for (; j + 4 <= nsel; j += 4) {
            float k0, k1, k2, k3;
            hnsw_key4<METRIC>(vecs, d, s_c, s_sel[j], s_sel[j + 1], s_sel[j + 2], s_sel[j + 3], lane, k0, k1, k2, k3);
            if (k0 < kc || k1 < kc || k2 < kc || k3 < kc) return false;
        }
    }
    for (; j < nsel; j++)
        if (hnsw_key<METRIC>(vecs, d, s_c, s_sel[j], lane) < kc) return false;
    return true;
}

// dynamic smem per warp: d floats (candidate vector) + 64 ints
template <int METRIC>
__global__ void __launch_bounds__(kBuildWarps * 32)
hnsw_select_kernel(HnswBuildParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dpad = (p.d + 3) & ~3;
    unsigned char* mine = smem_raw + (size_t)warp * ((size_t)dpad * 4 + 256);
    float* s_c = (float*)mine;
    int32_t* s_sel = (int32_t*)(mine + (size_t)dpad * 4);
    const int w = blockIdx.x * kBuildWarps + warp;
    if (w >= p.nb) return;
    const int32_t q = p.batch[w];
    const int maxn = p.cum[p.level + 1] - p.cum[p.level];
    // the candidates are the pool up to its first -1, without q; fewer than maxn are all kept (K/impl/HNSW.cpp:290-292)
    int nvalid = 0;
    for (int base = 0; base < p.ef; base += kWarp) {
        const int64_t c = (base + lane < p.ef) ? p.cand_ids[(int64_t)w * p.ef + base + lane] : -1;
        nvalid += __popc(__ballot_sync(0xffffffffu, c >= 0 && c != q));
    }
    const bool keep_all = nvalid < maxn;
    int nsel = 0;
    for (int ci = 0; ci < p.ef && nsel < maxn; ci++) {
        const int64_t c = p.cand_ids[(int64_t)w * p.ef + ci];
        if (c < 0) break;
        if (c == q) continue;
        bool keep = keep_all;
        if (!keep) {
            const float dc = p.cand_dist[(int64_t)w * p.ef + ci];
            const float kc = (METRIC == KB2_METRIC_L2) ? dc : -dc;
            __syncwarp();
            for (int j = lane; j < p.d; j += kWarp) s_c[j] = p.vecs[c * p.d + j];
            __syncwarp();
            keep = hnsw_heuristic_keep<METRIC>(p.vecs, p.d, s_c, kc, s_sel, nsel, lane);
        }
        if (keep) {
            if (lane == 0) s_sel[nsel] = (int32_t)c;
            nsel++;
            __syncwarp();
        }
    }
    int32_t* row = p.neighbors + p.offsets[q] + p.cum[p.level];
    for (int j = lane; j < maxn; j += kWarp) row[j] = j < nsel ? s_sel[j] : -1;
    for (int j = lane; j < 64; j += kWarp)
        p.pairs[(int64_t)w * 64 + j] = j < nsel ? ((unsigned long long)s_sel[j] << 32) | (unsigned)w : p.pair_end;
}

// reverse links: warp i takes sorted pair i when it starts the run of its target s, and adds the new nodes batch[w] of
// the run to s's row in ascending w; a full row is re-selected among its members + the new node with the heuristic,
// centre s.  One warp owns each row, so no order between warps shows in the graph.  dynamic smem per warp: 2 * d floats
// + 3 * kLinkSlots words (a full row of 2M = 64 members plus the new node is 65 candidates)
constexpr int kLinkSlots = 72;
template <int METRIC>
__global__ void __launch_bounds__(kBuildWarps * 32)
hnsw_link_kernel(HnswBuildParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dpad = (p.d + 3) & ~3;
    unsigned char* mine = smem_raw + (size_t)warp * ((size_t)dpad * 8 + 3 * kLinkSlots * 4);
    float* s_s = (float*)mine;                       // vector of the centre s
    float* s_c = s_s + dpad;                         // vector of the candidate being tested
    int32_t* s_id = (int32_t*)(s_c + dpad);          // [kLinkSlots] candidate ids (sorted by key to s)
    float* s_key = (float*)(s_id + kLinkSlots);      // [kLinkSlots]
    int32_t* s_sel = (int32_t*)(s_key + kLinkSlots); // [kLinkSlots] kept ids
    const int64_t npairs = (int64_t)p.nb * 64;
    const int64_t i0 = (int64_t)blockIdx.x * kBuildWarps + warp;
    if (i0 >= npairs) return;
    const unsigned long long head = p.sorted[i0];
    if (head >= p.pair_end || (i0 > 0 && (p.sorted[i0 - 1] >> 32) == (head >> 32))) return;
    const int32_t s = (int32_t)(head >> 32);
    const int cap = p.cum[p.level + 1] - p.cum[p.level];   // <= 64 (M <= 32)
    int32_t* row = p.neighbors + p.offsets[s] + p.cum[p.level];
    for (int j = lane; j < p.d; j += kWarp) s_s[j] = p.vecs[(int64_t)s * p.d + j];
    for (int64_t i = i0; i < npairs && (p.sorted[i] >> 32) == (head >> 32); i++) {
        const int32_t q = p.batch[(uint32_t)p.sorted[i]];
        // current members (compact, -1 terminated)
        int cnt = 0;
        for (int j0 = 0; j0 < cap; j0 += kWarp) {
            const int32_t v = (j0 + lane < cap) ? row[j0 + lane] : -1;
            const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
            if (v >= 0) s_id[j0 + lane] = v;
            cnt += __popc(m);
        }
        __syncwarp();
        if (cnt < cap) {
            if (lane == 0) row[cnt] = q;
        } else {
            // full: candidates = members + q, keys to s, sort, heuristic, rewrite
            if (lane == 0) s_id[cnt] = q;
            __syncwarp();
            const int nc = cnt + 1;
            for (int j = 0; j < nc; j++) {
                const float kj = hnsw_key<METRIC>(p.vecs, p.d, s_s, s_id[j], lane);
                if (lane == 0) s_key[j] = kj;
            }
            __syncwarp();
            // rank by (key, id): nc <= 65 elements, two per lane at most three
            int32_t my_id[3];
            float my_key[3];
            int my_rank[3];
            for (int t = 0; t < 3; t++) {
                const int j = lane + 32 * t;
                my_rank[t] = -1;
                if (j < nc) {
                    my_id[t] = s_id[j];
                    my_key[t] = s_key[j];
                    int r = 0;
                    for (int x = 0; x < nc; x++) {
                        const float kx = s_key[x];
                        const int32_t ix = s_id[x];
                        r += (kx < my_key[t]) || (kx == my_key[t] && ix < my_id[t]);
                    }
                    my_rank[t] = r;
                }
            }
            __syncwarp();
            for (int t = 0; t < 3; t++)
                if (my_rank[t] >= 0) { s_id[my_rank[t]] = my_id[t]; s_key[my_rank[t]] = my_key[t]; }
            __syncwarp();
            int nsel = 0;
            for (int ci = 0; ci < nc && nsel < cap; ci++) {
                const int32_t c = s_id[ci];
                const float kc = s_key[ci];
                __syncwarp();
                for (int j = lane; j < p.d; j += kWarp) s_c[j] = p.vecs[(int64_t)c * p.d + j];
                __syncwarp();
                if (hnsw_heuristic_keep<METRIC>(p.vecs, p.d, s_c, kc, s_sel, nsel, lane)) {
                    if (lane == 0) s_sel[nsel] = c;
                    nsel++;
                    __syncwarp();
                }
            }
            for (int j = lane; j < cap; j += kWarp) row[j] = j < nsel ? s_sel[j] : -1;
        }
        __syncwarp();   // the row as this arrival left it is what the next one reads
    }
}

// number of set bits among the first nbits of a bitmap (grid-stride, one atomic per CTA)
__global__ void __launch_bounds__(256)
bitset_count_kernel(const uint8_t* __restrict__ bits, int64_t nbits, unsigned long long* __restrict__ out) {
    unsigned long long acc = 0;
    const int64_t nbytes = (nbits + 7) >> 3;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nbytes; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t b = bits[i];
        if (i == nbytes - 1 && (nbits & 7)) b &= (1u << (nbits & 7)) - 1u;
        acc += __popc(b);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}
// set bits among bit positions [first, first + count)
__global__ void __launch_bounds__(256)
bitset_count_range_kernel(const uint8_t* __restrict__ bits, int64_t first, int64_t count, unsigned long long* __restrict__ out) {
    unsigned long long acc = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        acc += bit_is_set(bits, first + i) ? 1ull : 0ull;
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}
// queries whose result row holds fewer than min(k, n_valid) ids -> compact list (brute-force fallback, faiss_hnsw.cc:1464-1478)
__global__ void __launch_bounds__(256)
short_rows_kernel(const int64_t* __restrict__ ids, int64_t nq, int k, int64_t n_valid, int32_t* __restrict__ list,
                  uint32_t* __restrict__ count) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    int real = 0;
    for (int j = 0; j < k; j++) real += ids[q * k + j] >= 0;
    if (real < k && real < n_valid) list[atomicAdd(count, 1u)] = (int32_t)q;
}
__global__ void
scatter_result_rows_kernel(const int64_t* __restrict__ src_ids, const float* __restrict__ src_dist, const int32_t* __restrict__ list,
                           int64_t n, int k, int64_t* __restrict__ dst_ids, float* __restrict__ dst_dist) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * k) return;
    const int64_t i = t / k, j = t % k;
    dst_ids[(int64_t)list[i] * k + j] = src_ids[t];
    dst_dist[(int64_t)list[i] * k + j] = src_dist[t];
}

// ============================================================================================
struct HnswIndex : IndexBase {
    int M = 30, efConstruction = 360;
    int64_t n = 0;
    int32_t entry_point = -1, max_level = -1;
    // host copies (reference layout)
    std::vector<float> h_vecs;
    std::vector<int32_t> h_levels, h_neighbors, h_cum;
    std::vector<int64_t> h_offsets;
    // device
    DevBuf<float> d_vecs, d_norms, s_bf_q, s_bf_dist;
    DevBuf<int32_t> d_neighbors, d_cum, d_vlog, s_short, d_queue;
    DevBuf<int64_t> s_bf_ids;
    DevBuf<uint32_t> d_qover;
    DevBuf<int64_t> d_offsets;
    DevBuf<uint32_t> d_visited;
    DevBuf<float> d_inv_dist;      // hnsw_wide_kernel<*, true>: per-CTA invalid pools
    DevBuf<uint32_t> d_inv_id;
    DevBuf<int> d_next;
    bool uploaded = false;
    int64_t last_ndis = 0, last_nhops = 0;

    void train(const float*, int64_t) override {}
    bool is_trained() const override { return true; }
    bool has_raw() const override { return true; }
    int64_t count() const override { return n; }
    int64_t size_bytes() const override {
        return (int64_t)(h_vecs.size() * 4 + h_neighbors.size() * 4 + h_offsets.size() * 8 + h_levels.size() * 4);
    }

    void
    set_default_cum(int nlevels) {
        // K/impl/HNSW.cpp:78-89 set_default_probas: level 0 has 2*M links, upper levels M
        h_cum.assign(1, 0);
        for (int l = 0; l < nlevels; l++) h_cum.push_back(h_cum.back() + (l == 0 ? 2 * M : M));
    }

    // ------------------------------------------------------------ host-side construction
    inline float
    host_key(const float* a, const float* b) const {
        float acc = 0.f;
        if (metric == KB2_METRIC_L2) {
            for (int j = 0; j < dim; j++) { const float t = a[j] - b[j]; acc += t * t; }
            return acc;
        }
        for (int j = 0; j < dim; j++) acc += a[j] * b[j];
        return -acc;
    }
    struct Cand { float key; int32_t id; };
    struct CandLess { bool operator()(const Cand& a, const Cand& b) const { return a.key < b.key; } };
    struct CandGreater { bool operator()(const Cand& a, const Cand& b) const { return a.key > b.key; } };

    int32_t* links(int32_t i, int level) { return h_neighbors.data() + h_offsets[i] + h_cum[level]; }
    int nlinks(int level) const { return h_cum[level + 1] - h_cum[level]; }

    // heuristic neighbour selection (HNSW paper alg. 4; reference shrink_neighbor_list, K/impl/HNSW.cpp:231-300)
    void
    select_neighbors(std::vector<Cand>& cands /* ascending */, int maxn, std::vector<Cand>& out) const {
        out.clear();
        for (const Cand& c : cands) {
            bool good = true;
            for (const Cand& s : out) {
                if (host_key(&h_vecs[(size_t)c.id * dim], &h_vecs[(size_t)s.id * dim]) < c.key) { good = false; break; }
            }
            if (good) {
                out.push_back(c);
                if ((int)out.size() >= maxn) return;
            }
        }
    }
    void
    search_layer(const float* qv, int32_t ep, float ep_key, int ef, int level, std::vector<omp_lock_t>& locks,
                 std::vector<uint32_t>& vis_tag, uint32_t tag, std::vector<Cand>& result) {
        std::priority_queue<Cand, std::vector<Cand>, CandGreater> cand;   // min-heap
        std::priority_queue<Cand, std::vector<Cand>, CandLess> best;      // max-heap
        cand.push({ep_key, ep});
        best.push({ep_key, ep});
        vis_tag[ep] = tag;
        std::vector<int32_t> nb;
        while (!cand.empty()) {
            Cand c = cand.top();
            if (c.key > best.top().key && (int)best.size() >= ef) break;
            cand.pop();
            nb.clear();
            omp_set_lock(&locks[c.id]);
            {
                const int32_t* l = links(c.id, level);
                for (int j = 0; j < nlinks(level); j++) { if (l[j] < 0) break; nb.push_back(l[j]); }
            }
            omp_unset_lock(&locks[c.id]);
            for (int32_t v : nb) {
                if (vis_tag[v] == tag) continue;
                vis_tag[v] = tag;
                const float kv = host_key(qv, &h_vecs[(size_t)v * dim]);
                if ((int)best.size() < ef || kv < best.top().key) {
                    cand.push({kv, v});
                    best.push({kv, v});
                    if ((int)best.size() > ef) best.pop();
                }
            }
        }
        result.clear();
        while (!best.empty()) { result.push_back(best.top()); best.pop(); }
        std::reverse(result.begin(), result.end());
    }
    void
    add_link(int32_t src, int32_t dst, float key, int level) {
        int32_t* l = links(src, level);
        const int cap = nlinks(level);
        if (l[cap - 1] < 0) {
            int j = 0;
            while (l[j] >= 0) j++;
            l[j] = dst;
            return;
        }
        std::vector<Cand> cands;
        cands.push_back({key, dst});
        for (int j = 0; j < cap; j++)
            cands.push_back({host_key(&h_vecs[(size_t)src * dim], &h_vecs[(size_t)l[j] * dim]), l[j]});
        std::sort(cands.begin(), cands.end(), [](const Cand& a, const Cand& b) { return a.key < b.key; });
        std::vector<Cand> sel;
        select_neighbors(cands, cap, sel);
        for (int j = 0; j < cap; j++) l[j] = j < (int)sel.size() ? sel[j].id : -1;
    }

    // IndexNode::Add for HNSW == build (faiss_hnsw.cc:2073-2178 -> K/IndexHNSW.cpp:83-215)
    void
    add(const float* x, int64_t nadd, const int64_t* ids) override {
        KB2_REQUIRE(n == 0, KB2_NOT_IMPLEMENTED, "HNSW: incremental add after the first build is not implemented");
        KB2_REQUIRE(nadd > 0 && nadd < (1ll << 31), KB2_INVALID_ARGS, "bad row count");
        // graph-partition sharding (SURVEY 8e, option 2): this rank builds an independent sub-graph over the contiguous row
        // slice [lo, hi); every shard is searched with the same ef and the per-shard top-k are all-gathered and merged
        const auto [lo, hi] = shard_slice(nadd);
        n_global = nadd;
        shard_lo = lo;
        const int64_t nloc = hi - lo;
        KB2_REQUIRE(nloc > 0, KB2_INVALID_ARGS, "HNSW shard without rows");
        h_vecs.resize((size_t)nloc * dim);
        KB2_CUDA_CHECK(cudaMemcpy(h_vecs.data(), x + lo * dim, h_vecs.size() * 4, cudaMemcpyDefault));
        labels.append(0, ids ? ids + lo : nullptr, nloc, lo, shard_world > 1, stream);
        nadd = nloc;
        n = nadd;
        // levels: floor(-ln(U) / ln(M)), RNG seed 12345 (K/impl/HNSW.cpp:60-63,92-105)
        std::mt19937 rng(12345);
        std::uniform_real_distribution<double> uni(0.0, 1.0);
        const double mult = 1.0 / std::log((double)M);
        h_levels.resize(n);
        int top = 0;
        for (int64_t i = 0; i < n; i++) {
            double u = uni(rng);
            if (u <= 0) u = 1e-12;
            const int lv = (int)(-std::log(u) * mult);
            h_levels[i] = lv + 1;
            top = std::max(top, lv);
        }
        set_default_cum(top + 1);
        h_offsets.assign(n + 1, 0);
        for (int64_t i = 0; i < n; i++) h_offsets[i + 1] = h_offsets[i] + h_cum[h_levels[i]];
        h_neighbors.assign(h_offsets[n], -1);
        // insertion order: highest level first (K/IndexHNSW.cpp:112-166)
        std::vector<int32_t> order(n);
        for (int64_t i = 0; i < n; i++) order[i] = (int32_t)i;
        std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return h_levels[a] > h_levels[b]; });
        entry_point = order[0];
        max_level = h_levels[order[0]] - 1;
        if (gpu_build_wanted(n, M)) {
            build_graph_gpu(order);
            return;
        }
        std::vector<omp_lock_t> locks(n);
        for (auto& l : locks) omp_init_lock(&l);
        // host threads: the affinity / OpenMP default, capped by the cgroup CPU quota (a 128-thread box leased with a 16-CPU
        // quota runs 128 threads 8x oversubscribed otherwise)
        int nthreads = omp_get_max_threads();
        if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
            char a[64], b[64];
            if (fscanf(f, "%63s %63s", a, b) == 2 && strcmp(a, "max") != 0) {
                const double q = atof(a) / std::max(1.0, atof(b));
                if (q >= 1.0) nthreads = std::max(1, std::min(nthreads, (int)(q + 0.5)));
            }
            fclose(f);
        }
        std::vector<std::vector<uint32_t>> tags(nthreads, std::vector<uint32_t>(n, 0));
        std::vector<uint32_t> tagc(nthreads, 0);
        omp_lock_t global;
        omp_init_lock(&global);
        int64_t start = 1;
        while (start < n) {
            int64_t stop = start;
            const int lv = h_levels[order[start]];
            while (stop < n && h_levels[order[stop]] == lv) stop++;
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthreads)
            for (int64_t t = start; t < stop; t++) {
                const int tid = omp_get_thread_num();
                const int32_t pt = order[t];
                const int pt_level = h_levels[pt] - 1;
                const float* qv = &h_vecs[(size_t)pt * dim];
                int32_t nearest;
                int cur_max;
                omp_set_lock(&global);
                nearest = entry_point;
                cur_max = max_level;
                omp_unset_lock(&global);
                float d_nearest = host_key(qv, &h_vecs[(size_t)nearest * dim]);
                for (int level = cur_max; level > pt_level; level--) {
                    bool changed = true;
                    while (changed) {
                        changed = false;
                        std::vector<int32_t> nb;
                        omp_set_lock(&locks[nearest]);
                        const int32_t* l = links(nearest, level);
                        for (int j = 0; j < nlinks(level); j++) { if (l[j] < 0) break; nb.push_back(l[j]); }
                        omp_unset_lock(&locks[nearest]);
                        for (int32_t v : nb) {
                            const float kv = host_key(qv, &h_vecs[(size_t)v * dim]);
                            if (kv < d_nearest) { d_nearest = kv; nearest = v; changed = true; }
                        }
                    }
                }
                std::vector<Cand> res, sel;
                for (int level = std::min(pt_level, cur_max); level >= 0; level--) {
                    search_layer(qv, nearest, d_nearest, efConstruction, level, locks, tags[tid], ++tagc[tid], res);
                    // drop self if present
                    res.erase(std::remove_if(res.begin(), res.end(), [&](const Cand& c) { return c.id == pt; }), res.end());
                    select_neighbors(res, nlinks(level), sel);  // K/impl/HNSW.cpp add_links_starting_from: M = nb_neighbors(level)
                    omp_set_lock(&locks[pt]);
                    {
                        int32_t* l = links(pt, level);
                        for (int j = 0; j < (int)sel.size() && j < nlinks(level); j++) l[j] = sel[j].id;
                    }
                    omp_unset_lock(&locks[pt]);
                    for (const Cand& s : sel) {
                        omp_set_lock(&locks[s.id]);
                        add_link(s.id, pt, s.key, level);
                        omp_unset_lock(&locks[s.id]);
                    }
                    if (!res.empty()) { nearest = res[0].id; d_nearest = res[0].key; }
                }
            }
            if (lv - 1 > max_level) { max_level = lv - 1; entry_point = order[start]; }
            start = stop;
        }
        for (auto& l : locks) omp_destroy_lock(&l);
        omp_destroy_lock(&global);
        uploaded = false;
    }

    // ------------------------------------------------------------ device-side construction (see hnsw_select_kernel)
    static constexpr int64_t kBuildBatch = 16384;   // most nodes inserted per batch (also at most a quarter of those linked)
    static bool
    gpu_build_wanted(int64_t n_rows, int M_) {
        if (2 * M_ > 64) return false;   // the link kernel keeps a row in 64 slots
        const char* e = getenv("KB2_HNSW_BUILD");
        if (e && !strcmp(e, "host")) return false;
        if (e && !strcmp(e, "gpu")) return true;
        return n_rows >= 20000;
    }
    void
    build_graph_gpu(const std::vector<int32_t>& order) {
        cudaStream_t st = stream;
        const int ef = std::max(efConstruction, 2 * M);
        d_vecs.alloc_exact(h_vecs.size());
        d_neighbors.alloc_exact(h_neighbors.size());
        d_offsets.alloc_exact(h_offsets.size());
        d_cum.alloc_exact(h_cum.size() + 1);
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_vecs.p, h_vecs.data(), h_vecs.size() * 4, cudaMemcpyHostToDevice, st));
        KB2_CUDA_CHECK(cudaMemsetAsync(d_neighbors.p, 0xff, h_neighbors.size() * 4, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_offsets.p, h_offsets.data(), h_offsets.size() * 8, cudaMemcpyHostToDevice, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_cum.p, h_cum.data(), h_cum.size() * 4, cudaMemcpyHostToDevice, st));
        std::vector<int32_t> rank(n);
        for (int64_t i = 0; i < n; i++) rank[order[i]] = (int32_t)i;
        DevBuf<int32_t> d_order, d_rank;
        DevBuf<int64_t> d_cand_ids;
        DevBuf<float> d_cand_dist;
        DevBuf<unsigned long long> d_pairs, d_sorted;
        DevBuf<unsigned char> d_sort_tmp;
        d_order.alloc_exact((size_t)n);
        d_rank.alloc_exact((size_t)n);
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_order.p, order.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_rank.p, rank.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        const int64_t maxb = std::min<int64_t>(kBuildBatch, n);
        d_cand_ids.alloc_exact((size_t)maxb * ef);
        d_cand_dist.alloc_exact((size_t)maxb * ef);
        // the link pairs (s << 32 | w) sort on their low 32 + bit_width(n) bits, so the end marker n << 32 sorts last
        int sort_bits = 32;
        while ((1ll << (sort_bits - 32)) <= n) sort_bits++;
        d_pairs.alloc_exact((size_t)maxb * 64);
        d_sorted.alloc_exact((size_t)maxb * 64);
        size_t sort_bytes = 0;
        KB2_CUDA_CHECK(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, d_pairs.p, d_sorted.p, (int)(maxb * 64), 0,
                                                      sort_bits, st));
        d_sort_tmp.alloc_exact(sort_bytes);
        d_next.ensure(1);
        const int dpad = (dim + 3) & ~3;
        const size_t smem_sel = (size_t)kBuildWarps * ((size_t)dpad * 4 + 256);
        const size_t smem_link = (size_t)kBuildWarps * ((size_t)dpad * 8 + 3 * kLinkSlots * 4);
        KB2_REQUIRE(smem_link <= (size_t)kMaxDynSmem, KB2_INVALID_ARGS, "HNSW GPU build: dim too large");
        int64_t level_count[64] = {0};   // nodes with (levels - 1) >= L
        for (int L = 0; L <= max_level && L < 64; L++) {
            int64_t c = 0;
            while (c < n && h_levels[order[c]] - 1 >= L) c++;
            level_count[L] = c;
        }
        int64_t n_batches = 0;
        for (int L = max_level; L >= 0; L--) {
            const int64_t cntL = level_count[L];
            int64_t inserted = 1;   // the entry point (order[0]) is on every level
            while (inserted < cntL) {
                const int64_t nb = std::min<int64_t>(std::min<int64_t>(maxb, std::max<int64_t>(1, inserted / 4)), cntL - inserted);
                const Launch La = plan_launch(nb, ef, false);
                KB2_CUDA_CHECK(cudaMemsetAsync(d_next.p, 0, 4, st));
                HnswSearchParams p = base_params(nullptr, nb, ef, ef, La, nullptr, 0);
                p.labels = nullptr;
                p.q_nodes = d_order.p + inserted;
                p.beam_level = L;
                p.node_rank = d_rank.p;
                p.rank_limit = (int)inserted;
                p.out_ids = d_cand_ids.p;
                p.out_dist = d_cand_dist.p;
                HnswBuildParams b{};
                b.vecs = d_vecs.p;
                b.d = dim;
                b.metric = metric;
                b.level = L;
                b.neighbors = d_neighbors.p;
                b.offsets = d_offsets.p;
                b.cum = d_cum.p;
                b.batch = d_order.p + inserted;
                b.nb = (int)nb;
                b.ef = ef;
                b.cand_ids = d_cand_ids.p;
                b.cand_dist = d_cand_dist.p;
                b.pairs = d_pairs.p;
                b.sorted = d_sorted.p;
                b.pair_end = (unsigned long long)n << 32;
                const int gb = (int)((nb + kBuildWarps - 1) / kBuildWarps);
                with_metric(metric, [&](auto m) {
                    constexpr int MM = decltype(m)::value;
                    launch<hnsw_search_kernel<MM, false>>(La.grid, kHnswWarps * 32, La.smem, st, p);
                    launch<hnsw_select_kernel<MM>>(gb, kBuildWarps * 32, smem_sel, st, b);
                    KB2_CUDA_CHECK(cub::DeviceRadixSort::SortKeys(d_sort_tmp.p, sort_bytes, d_pairs.p, d_sorted.p,
                                                                  (int)(nb * 64), 0, sort_bits, st));
                    launch<hnsw_link_kernel<MM>>((int)(nb * 64 / kBuildWarps), kBuildWarps * 32, smem_link, st, b);
                });
                inserted += nb;
                n_batches++;
            }
        }
        KB2_CUDA_CHECK(cudaGetLastError());
        KB2_CUDA_CHECK(cudaMemcpyAsync(h_neighbors.data(), d_neighbors.p, h_neighbors.size() * 4, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        last.launches = 4 * n_batches;   // search, select, the pair sort (counted once), link
        // rows are compact (-1 only at the tail) by construction of the two kernels; validate the structure once
        validate_graph();
        uploaded = false;
    }

    void
    import_graph(int64_t nn, const float* vectors, const int32_t* levels, const int64_t* offsets, const int32_t* neighbors,
                 const int32_t* cum, int n_cum, int32_t ep, int32_t ml) {
        KB2_REQUIRE(nn > 0 && n_cum >= 2, KB2_INVALID_ARGS, "bad graph");
        n = nn;
        h_vecs.assign(vectors, vectors + (size_t)nn * dim);
        h_levels.assign(levels, levels + nn);
        h_offsets.assign(offsets, offsets + nn + 1);
        h_neighbors.assign(neighbors, neighbors + offsets[nn]);
        h_cum.assign(cum, cum + n_cum);
        entry_point = ep;
        max_level = ml;
        KB2_REQUIRE(max_level + 1 < n_cum, KB2_INVALID_ARGS, "cum_nneighbor_per_level shorter than max_level");
        validate_graph();
        uploaded = false;
    }

    // structural checks of an externally supplied graph (the search kernel trusts these arrays)
    void
    validate_graph() const {
        const int ncum = (int)h_cum.size();
        KB2_REQUIRE(n > 0 && ncum >= 2 && h_cum[0] == 0, KB2_INVALID_BINARY_SET, "HNSW: bad graph header");
        for (int l = 0; l + 1 < ncum; l++) KB2_REQUIRE(h_cum[l + 1] > h_cum[l], KB2_INVALID_BINARY_SET, "HNSW: cum_nneighbor not increasing");
        KB2_REQUIRE(max_level >= 0 && max_level + 1 < ncum, KB2_INVALID_BINARY_SET, "HNSW: max_level outside cum_nneighbor");
        KB2_REQUIRE(entry_point >= 0 && entry_point < n, KB2_INVALID_BINARY_SET, "HNSW: entry point out of range");
        KB2_REQUIRE((int64_t)h_offsets.size() == n + 1 && h_offsets[0] == 0, KB2_INVALID_BINARY_SET, "HNSW: bad offsets");
        for (int64_t i = 0; i < n; i++) {
            const int lv = h_levels[i];
            KB2_REQUIRE(lv >= 1 && lv < ncum && h_offsets[i + 1] - h_offsets[i] == h_cum[lv], KB2_INVALID_BINARY_SET,
                        "HNSW: offsets do not match the levels");
        }
        KB2_REQUIRE((int64_t)h_neighbors.size() == h_offsets[n], KB2_INVALID_BINARY_SET, "HNSW: neighbor array size");
        KB2_REQUIRE(h_levels[entry_point] - 1 >= max_level, KB2_INVALID_BINARY_SET, "HNSW: entry point below max_level");
        for (int32_t v : h_neighbors) KB2_REQUIRE(v >= -1 && v < n, KB2_INVALID_BINARY_SET, "HNSW: neighbor id out of range");
    }

    void
    upload() {
        if (uploaded) return;
        d_vecs.alloc_exact(h_vecs.size());
        d_neighbors.alloc_exact(h_neighbors.size());
        d_offsets.alloc_exact(h_offsets.size());
        d_cum.alloc_exact(h_cum.size() + 1);
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_vecs.p, h_vecs.data(), h_vecs.size() * 4, cudaMemcpyHostToDevice, stream));
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_neighbors.p, h_neighbors.data(), h_neighbors.size() * 4, cudaMemcpyHostToDevice, stream));
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_offsets.p, h_offsets.data(), h_offsets.size() * 8, cudaMemcpyHostToDevice, stream));
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_cum.p, h_cum.data(), h_cum.size() * 4, cudaMemcpyHostToDevice, stream));
        d_next.ensure(1);
        d_norms.alloc_exact((size_t)n);   // brute-force fallback over the stored vectors
        row_norms_kernel<<<grid1d(n * 32, 256), 256, 0, stream>>>(d_vecs.p, n, dim, d_norms.p);
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        uploaded = true;
    }

    // exact scan of the stored vectors (the reference's brute-force wrapper: IndexConditionalWrapper.cc:103-200), certified
    // like FLAT's; last.flagged keeps counting the short rows this completes, not the queries dense_knn redoes
    void
    brute_force(const float* dq, int64_t nq, int k, const uint8_t* dbits, int64_t* d_ids, float* d_dist) {
        dense_knn(*this, dq, nq, d_vecs.p, d_norms.p, n, dim, metric, k, k + 16, dbits, shard_world > 1 ? shard_lo : 0,
                  labels.device(), d_ids, d_dist, true);
    }

    // set bits among the first n of the (device) bitmap
    int64_t
    count_filtered(const uint8_t* dbits) {
        if (!dbits) return 0;
        KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p + 4, 0, 8, stream));
        bitset_count_range_kernel<<<std::min<int64_t>(1024, (n + 255) / 256), 256, 0, stream>>>(dbits, shard_world > 1 ? shard_lo : 0, n,
                                                                                         d_counter.p + 4);
        unsigned long long* hc = (unsigned long long*)h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(hc, d_counter.p + 4, 8, cudaMemcpyDeviceToHost, stream));
        KB2_CUDA_CHECK(cudaStreamSynchronize(stream));
        return (int64_t)hc[0];
    }

    struct Launch {
        int grid;
        int64_t total_warps, nwords;
        int log_cap;
        size_t smem;
    };
    // shared memory of one hnsw_search_kernel CTA (layout at the kernel): per warp the query and one or two pools
    size_t
    warp_smem(int ef_cap, bool two_pools) const {
        const int dpad = (dim + 3) & ~3;
        return kHnswWarps * (size_t)round_up((int64_t)dpad * 4 + (int64_t)ef_cap * (two_pools ? 16 : 8), 16);
    }
    // grow the per-warp (per-CTA) visited bitmaps, zeroed, and touched-id logs to what L needs
    void
    ensure_visited(const Launch& L) {
        if (d_visited.n < (size_t)(L.total_warps * L.nwords)) {
            d_visited.ensure((size_t)(L.total_warps * L.nwords));
            KB2_CUDA_CHECK(cudaMemsetAsync(d_visited.p, 0, (size_t)(L.total_warps * L.nwords) * 4, stream));
        }
        d_vlog.ensure((size_t)(L.total_warps * L.log_cap));
    }
    Launch
    plan_launch(int64_t nq, int ef_cap, bool two_pools) {
        Launch L;
        L.smem = warp_smem(ef_cap, two_pools);
        KB2_REQUIRE(L.smem <= (size_t)kMaxDynSmem, KB2_OUT_OF_RANGE_IN_JSON, "ef / dim too large for shared memory");
        const int ctas_per_sm = (int)std::max<size_t>(1, std::min<size_t>(8, (size_t)kMaxDynSmem / std::max<size_t>(L.smem, 1)));
        L.grid = (int)std::min<int64_t>((nq + kHnswWarps - 1) / kHnswWarps, (int64_t)num_sms() * ctas_per_sm);
        L.total_warps = (int64_t)L.grid * kHnswWarps;
        L.nwords = (n + 31) / 32;
        L.log_cap = (int)std::min<int64_t>(n, (int64_t)ef_cap * h_cum[1] * 4 + 256);
        ensure_visited(L);
        return L;
    }
    // shared memory of one hnsw_wide_kernel CTA (layout at the kernel)
    size_t
    wide_smem(int ef_cap, int dpad) const {
        return (size_t)round_up(32 + (int64_t)dpad * 4 + (int64_t)ef_cap * 8 + (int64_t)h_cum[1] * 21, 16);
    }
    // one query per CTA: one visited bitmap and log per CTA, and for filtered search one invalid pool of 2 * ef_cap entries
    Launch
    plan_wide(int64_t nq, int ef_cap, bool filtered) {
        const int dpad = (dim + 3) & ~3;
        Launch L;
        L.smem = wide_smem(ef_cap, dpad);
        if (ef_cap > kMaxLargeK)
            throw Error(KB2_OUT_OF_RANGE_IN_JSON, "HNSW: max(ef, k) = " + std::to_string(ef_cap) +
                                                      " out of range (the graph search keeps at most 16384 candidates)");
        if (L.smem > (size_t)kMaxDynSmem) {
            int dmax = 0;
            while (wide_smem(ef_cap, dmax + 4) <= (size_t)kMaxDynSmem) dmax += 4;
            throw Error(KB2_OUT_OF_RANGE_IN_JSON, "HNSW: dim " + std::to_string(dim) + " too large for max(ef, k) = " +
                                                      std::to_string(ef_cap) + " (at most " + std::to_string(dmax) + ")");
        }
        const int ctas_per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (size_t)kMaxDynSmem / L.smem));
        L.grid = (int)std::min<int64_t>(nq, (int64_t)num_sms() * ctas_per_sm);
        L.total_warps = L.grid;
        L.nwords = (n + 31) / 32;
        // past nwords touched ids, clearing the whole bitmap is the cheaper of the two
        L.log_cap = (int)std::min<int64_t>(n, std::max<int64_t>(L.nwords, 1024));
        ensure_visited(L);
        if (filtered) {
            d_inv_dist.ensure((size_t)L.grid * 2 * ef_cap);
            d_inv_id.ensure((size_t)L.grid * 2 * ef_cap);
        }
        return L;
    }
    // dbits: the search's bitset (device) or null; n_filtered: its set bits among the index's rows
    HnswSearchParams
    base_params(const float* dq, int64_t nq, int ef_cap, int k, const Launch& L, const uint8_t* dbits, int64_t n_filtered) {
        HnswSearchParams p{};
        p.vecs = d_vecs.p;
        p.d = dim;
        p.n = n;
        p.neighbors = d_neighbors.p;
        p.offsets = d_offsets.p;
        p.cum = d_cum.p;
        p.entry_point = entry_point;
        p.max_level = max_level;
        p.metric = metric;
        p.queries = dq;
        p.nq = (int)nq;
        p.ef_cap = ef_cap;
        p.k = k;
        p.visited = d_visited.p;
        p.nwords = L.nwords;
        p.vis_log = d_vlog.p;
        p.log_cap = L.log_cap;
        p.next_query = d_next.p;
        p.labels = labels.device();
        p.stats = d_counter.p;
        p.bitset = dbits;
        p.bit_offset = shard_world > 1 ? shard_lo : 0;
        p.k_alpha = (float)((double)n_filtered / (double)n) * 0.7f;   // faiss_hnsw.cc:1425
        static const int key8 = [] { const char* e = getenv("KB2_HNSW_KEY8"); return (e && atoi(e) != 0) ? 1 : 0; }();
        p.key8 = key8;
        return p;
    }

    void
    search(const float* q, int64_t nq, int k, const JsonObj& cfg, const uint8_t* bitset, int64_t nbits, int64_t* out_ids,
           float* out_dist) override {
        KB2_REQUIRE(n > 0 && entry_point >= 0, KB2_EMPTY_INDEX, "index is empty");
        upload();
        // base_hnsw_config.h:40-71: search key is "ef", default max(k,16), must be >= k
        int ef = (int)cfg.get_int("ef", std::max(k, 16));
        KB2_REQUIRE(ef >= k, KB2_OUT_OF_RANGE_IN_JSON, "ef must be >= k");
        const int ef_cap = std::max(ef, k);
        cudaStream_t st = stream;
        const float* dq = to_device(q, (size_t)nq * dim, s_q);
        const uint8_t* dbits = bitset_to_device(bitset, nbits);
        int64_t* d_ids;
        float* d_dist;
        device_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        // with a communicator the shard's top-k goes to a staging buffer; one all-gather + the merge kernel produce the result
        const bool dist = distributed();
        int64_t* const final_ids = d_ids;
        float* const final_dist = d_dist;
        if (dist) {
            KB2_REQUIRE((int64_t)shard_world * k <= kMaxSortEntries, KB2_INVALID_ARGS, "world * k too large for the merge");
            ensure_gather_buffers(nq, k);
            d_ids = s_loc_ids.p;
            d_dist = s_loc_dist.p;
        }
        // WhetherPerformBruteForceSearch (IndexConditionalWrapper.cc:35-62): huge k or an almost-all-filtered bitset
        const int64_t n_filtered = count_filtered(dbits);
        const int64_t n_valid = n - n_filtered;
        bool bf = (double)k >= (double)n * 0.5;
        if (dbits) bf = bf || (double)n_filtered >= (double)n * 0.93 || (double)k >= (double)n_valid * 0.5;
        KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p, 0, 16, st));
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev0, st));
        // a pool the four-warp kernels cannot hold runs one query per CTA (a collective search over a communicator keeps the
        // warp kernels' limit; a shard searched on its own does not)
        const bool wide = !bf && !dist && warp_smem(ef_cap, dbits != nullptr) > (size_t)kMaxDynSmem;
        if (bf) {
            KB2_REQUIRE(k <= kMaxLargeK, KB2_INVALID_ARGS, "k out of range (1..16384)");
            brute_force(dq, nq, k, dbits, d_ids, d_dist);
        } else if (wide) {
            const Launch L = plan_wide(nq, ef_cap, dbits != nullptr);
            KB2_CUDA_CHECK(cudaMemsetAsync(d_next.p, 0, 4, st));
            HnswWideParams w{};
            w.s = base_params(dq, nq, ef_cap, k, L, dbits, n_filtered);
            w.s.out_ids = d_ids;
            w.s.out_dist = d_dist;
            w.deg = h_cum[1] - h_cum[0];
            if (dbits) {
                w.inv_dist = d_inv_dist.p;
                w.inv_id = d_inv_id.p;
            }
            with_metric(metric, [&](auto m) {
                constexpr int MM = decltype(m)::value;
                if (dbits)
                    launch<hnsw_wide_kernel<MM, true>>(L.grid, kWideThreads, L.smem, st, w);
                else
                    launch<hnsw_wide_kernel<MM, false>>(L.grid, kWideThreads, L.smem, st, w);
            });
            last.launches++;
            KB2_CUDA_CHECK(cudaGetLastError());
        } else {
            const Launch L = plan_launch(nq, ef_cap, dbits != nullptr);
            KB2_CUDA_CHECK(cudaMemsetAsync(d_next.p, 0, 4, st));
            HnswSearchParams p = base_params(dq, nq, ef_cap, k, L, dbits, n_filtered);
            p.out_ids = d_ids;
            p.out_dist = d_dist;
            with_metric(metric, [&](auto m) {
                constexpr int MM = decltype(m)::value;
                if (dbits)
                    launch<hnsw_search_kernel<MM, true>>(L.grid, kHnswWarps * 32, L.smem, st, p);
                else
                    launch<hnsw_search_kernel<MM, false>>(L.grid, kHnswWarps * 32, L.smem, st, p);
            });
            last.launches++;
            KB2_CUDA_CHECK(cudaGetLastError());
        }
        last_engine = wide ? 3 : 0;   // set once the search's kernel was launched
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev1, st));
        // rows with fewer than k results although more valid vectors exist: exact fallback (faiss_hnsw.cc:1464-1478)
        if (dbits && !bf && !cfg.get_bool("disable_fallback_brute_force", false) && k <= kMaxLargeK) {
            s_short.ensure((size_t)nq + 1);
            KB2_CUDA_CHECK(cudaMemsetAsync(s_short.p, 0, 4, st));
            short_rows_kernel<<<grid1d(nq, 256), 256, 0, st>>>(d_ids, nq, k, n_valid, s_short.p + 1, (uint32_t*)s_short.p);
            uint32_t* hc = (uint32_t*)h_counter.p + 8;
            KB2_CUDA_CHECK(cudaMemcpyAsync(hc, s_short.p, 4, cudaMemcpyDeviceToHost, st));
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
            const int64_t ns = hc[0];
            if (ns > 0) {
                s_bf_q.ensure((size_t)ns * dim);
                s_bf_ids.ensure((size_t)ns * k);
                s_bf_dist.ensure((size_t)ns * k);
                gather_rows_kernel<<<grid1d(ns * 32, 256), 256, 0, st>>>(dq, s_short.p + 1, ns, dim, dim, s_bf_q.p);
                brute_force(s_bf_q.p, ns, k, dbits, s_bf_ids.p, s_bf_dist.p);
                scatter_result_rows_kernel<<<grid1d(ns * k, 256), 256, 0, st>>>(s_bf_ids.p, s_bf_dist.p, s_short.p + 1, ns, k, d_ids,
                                                                             d_dist);
                KB2_CUDA_CHECK(cudaGetLastError());
                last.flagged = ns;
            }
        }
        if (dist) {
            gather_merge(nq, k, final_ids, final_dist);
            d_ids = final_ids;
            d_dist = final_dist;
        }
        unsigned long long* hs = (unsigned long long*)h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(hs, d_counter.p, 16, cudaMemcpyDeviceToHost, st));
        results_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        last_ndis = bf ? nq * n_valid : (int64_t)hs[0];
        last_nhops = bf ? 0 : (int64_t)hs[1];
        last.codes = last_ndis;
        last.code_bytes = last_ndis * (int64_t)dim * 4 + last_nhops * (int64_t)h_cum[1] * 4;
        last.pairs = last_nhops;
        if (timing) KB2_CUDA_CHECK(cudaEventElapsedTime(&last_kernel_ms, ev0, ev1));
    }

    // RangeSearch (faiss_hnsw.cc:1631-1800 -> IndexHNSWWrapper.cc:207-400 -> HnswSearcher.h:435-553): the graph's hits
    // within radius and range_filter; queries whose BFS queue overflowed are rerun with a queue of n entries.  Where the
    // reference would run the brute-force range search instead (IndexConditionalWrapper.cc:68-97), the exact scan.
    std::vector<RangeHit>
    range_hits(const RangeParams& rp, const JsonObj& cfg, int&) override {
        KB2_REQUIRE(n > 0 && entry_point >= 0, KB2_EMPTY_INDEX, "index is empty");
        upload();
        const float* dq = rp.sp.queries;
        const int64_t nq = rp.sp.nq;
        const uint8_t* dbits = rp.sp.bitset;
        const int ef = (int)cfg.get_int("ef", 16);
        KB2_REQUIRE(ef >= 1, KB2_OUT_OF_RANGE_IN_JSON, "ef must be positive");
        const int64_t n_filtered = count_filtered(dbits);
        const int64_t n_valid = n - n_filtered;
        bool bf = (double)ef >= (double)n * 0.5;
        if (dbits) bf = bf || (double)n_filtered >= (double)n * 0.97 || (double)ef >= (double)n_valid * 0.97;
        if (bf) return range_scan_rows(*this, rp, d_vecs.p, n);
        cudaStream_t st = stream;
        DevBuf<RangeHit> hits;
        uint64_t pass0_hits = 0;
        const Launch L = plan_launch(nq, ef, true);
        d_qover.ensure((size_t)nq);
        DevBuf<unsigned long long> cnt;
        cnt.ensure(1);
        unsigned long long cap = (unsigned long long)std::max<int64_t>(1 << 20, nq * 256);
        std::vector<uint32_t> h_over(nq);
        std::vector<int32_t> redo;
        uint64_t found = 0;
        for (int pass = 0; pass < 2; pass++) {
            const int64_t nrun = pass == 0 ? nq : (int64_t)redo.size();
            if (nrun == 0) break;
            // pass 1 (overflowed queries only): a queue that can hold every node, as many warps as ~2 GB of queues allow
            const int64_t qcap = pass == 0 ? std::min<int64_t>(n, 16384) : n;
            int grid = L.grid;
            if (pass == 1) {
                const int64_t max_warps = std::max<int64_t>(kHnswWarps, (int64_t)(2ll << 30) / (qcap * 4));
                grid = (int)std::min<int64_t>(std::min<int64_t>(L.grid, (nrun + kHnswWarps - 1) / kHnswWarps), max_warps / kHnswWarps);
            }
            d_queue.ensure((size_t)grid * kHnswWarps * qcap);
            DevBuf<int32_t> d_redo;
            if (pass == 1) {
                d_redo.ensure(redo.size());
                KB2_CUDA_CHECK(cudaMemcpyAsync(d_redo.p, redo.data(), redo.size() * 4, cudaMemcpyHostToDevice, st));
            }
            const uint64_t found_before = found;
            for (int attempt = 0; attempt < 2; attempt++) {
                hits.ensure(cap);   // NOTE: grow-only without preserving contents: pass 1 appends after a copy (below)
                KB2_CUDA_CHECK(cudaMemsetAsync(cnt.p, 0, 8, st));
                if (pass == 0) KB2_CUDA_CHECK(cudaMemsetAsync(d_qover.p, 0, (size_t)nq * 4, st));
                KB2_CUDA_CHECK(cudaMemsetAsync(d_next.p, 0, 4, st));
                KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p, 0, 16, st));
                HnswSearchParams p = base_params(dq, nrun, ef, 1, L, dbits, n_filtered);
                p.range_mode = 1;
                p.radius_key = (metric == KB2_METRIC_L2) ? rp.radius : -rp.radius;
                p.hits = hits.p + found_before;
                p.hit_count = cnt.p;
                p.hit_cap = cap - found_before;
                p.bfs_queue = d_queue.p;
                p.queue_cap = (int)qcap;
                p.q_overflow = d_qover.p;
                p.q_list = pass == 1 ? d_redo.p : nullptr;
                with_metric(metric, [&](auto m) {
                    launch<hnsw_search_kernel<decltype(m)::value, true>>(grid, kHnswWarps * 32, L.smem, st, p);
                });
                last.launches++;
                KB2_CUDA_CHECK(cudaGetLastError());
                unsigned long long got = 0;
                KB2_CUDA_CHECK(cudaMemcpyAsync(&got, cnt.p, 8, cudaMemcpyDeviceToHost, st));
                KB2_CUDA_CHECK(cudaStreamSynchronize(st));
                if (found_before + got <= cap) { found = found_before + got; break; }
                // the hit buffer was too small: grow it (keeping the hits of the previous pass) and run the pass again
                KB2_REQUIRE(attempt == 0, KB2_INTERNAL_ERROR, "range search: hit buffer overflow after resizing");
                DevBuf<RangeHit> bigger;
                cap = found_before + got;
                bigger.ensure(cap);
                if (found_before)
                    KB2_CUDA_CHECK(cudaMemcpyAsync(bigger.p, hits.p, found_before * sizeof(RangeHit), cudaMemcpyDeviceToDevice, st));
                KB2_CUDA_CHECK(cudaStreamSynchronize(st));
                hits = std::move(bigger);
            }
            if (pass == 0) {
                pass0_hits = found;
                KB2_CUDA_CHECK(cudaMemcpy(h_over.data(), d_qover.p, (size_t)nq * 4, cudaMemcpyDeviceToHost));
                for (int64_t i = 0; i < nq; i++)
                    if (h_over[i]) redo.push_back((int32_t)i);
            }
        }
        std::vector<RangeHit> h = hits_to_host(*this, hits.p, found);
        size_t w = 0;
        for (size_t i = 0; i < h.size(); i++) {
            // pass-0 hits of a query whose BFS queue overflowed are incomplete: the rerun (later entries) has them all
            if (i < pass0_hits && h_over[h[i].q]) continue;
            if (!in_range_host(h[i].dist, rp.radius, rp.range_filter, rp.has_filter, metric)) continue;
            h[w++] = h[i];
        }
        h.resize(w);
        return h;
    }

    void
    get_vectors(const int64_t* ids, int64_t cnt, float* out) override {
        KB2_REQUIRE(!labels.custom, KB2_NOT_IMPLEMENTED, "GetVectorByIds with custom ids");
        std::vector<int64_t> h(cnt);
        KB2_CUDA_CHECK(cudaMemcpy(h.data(), ids, cnt * 8, cudaMemcpyDefault));
        for (int64_t i = 0; i < cnt; i++) {
            KB2_REQUIRE(h[i] >= 0 && h[i] < n, KB2_INVALID_ARGS, "id out of range");
            KB2_CUDA_CHECK(cudaMemcpy(out + i * dim, &h_vecs[(size_t)h[i] * dim], (size_t)dim * 4, cudaMemcpyDefault));
        }
    }

    void
    configure(const JsonObj& cfg) override {
        M = (int)cfg.get_int("M", 30);
        efConstruction = (int)cfg.get_int("efConstruction", 360);
        KB2_REQUIRE(M >= 2 && M <= 2048, KB2_OUT_OF_RANGE_IN_JSON, "M out of range");
    }

    void
    save(BlobWriter& w) override {
        w.put<int32_t>(M);
        w.put<int32_t>(efConstruction);
        w.put<int64_t>(n);
        w.put<int32_t>(entry_point);
        w.put<int32_t>(max_level);
        w.put<int32_t>((int32_t)h_cum.size());
        w.put<int32_t>(labels.custom ? 1 : 0);
        w.put_bytes(h_cum.data(), h_cum.size() * 4);
        w.put_bytes(h_levels.data(), h_levels.size() * 4);
        w.put_bytes(h_offsets.data(), h_offsets.size() * 8);
        w.put_bytes(h_neighbors.data(), h_neighbors.size() * 4);
        w.put_bytes(h_vecs.data(), h_vecs.size() * 4);
        const std::vector<int64_t> l = labels.host(n);
        w.put_bytes(l.data(), l.size() * 8);
    }
    void
    load(BlobReader& r) override {
        M = r.get<int32_t>();
        efConstruction = r.get<int32_t>();
        n = r.get<int64_t>();
        entry_point = r.get<int32_t>();
        max_level = r.get<int32_t>();
        const int ncum = r.get<int32_t>();
        const bool custom = r.get<int32_t>() != 0;
        KB2_REQUIRE(n > 0 && n < (1ll << 31) && ncum >= 2 && ncum < 64 && (uint64_t)n <= r.n / 4, KB2_INVALID_BINARY_SET,
                    "HNSW: bad header in blob");
        h_cum.resize(ncum);
        memcpy(h_cum.data(), r.get_bytes((size_t)ncum * 4), (size_t)ncum * 4);
        h_levels.resize(n);
        memcpy(h_levels.data(), r.get_bytes((size_t)n * 4), (size_t)n * 4);
        h_offsets.resize(n + 1);
        memcpy(h_offsets.data(), r.get_bytes((size_t)(n + 1) * 8), (size_t)(n + 1) * 8);
        KB2_REQUIRE(h_offsets[n] >= 0 && (uint64_t)h_offsets[n] <= r.n / 4, KB2_INVALID_BINARY_SET, "HNSW: bad offsets in blob");
        h_neighbors.resize(h_offsets[n]);
        memcpy(h_neighbors.data(), r.get_bytes(h_neighbors.size() * 4), h_neighbors.size() * 4);
        h_vecs.resize((size_t)n * dim);
        memcpy(h_vecs.data(), r.get_bytes(h_vecs.size() * 4), h_vecs.size() * 4);
        if (custom) labels.append(0, (const int64_t*)r.get_bytes((size_t)n * 8), n, 0, false, stream);
        validate_graph();
        uploaded = false;
    }

    void
    to_faiss(FaissIndexData& o) override {
        KB2_REQUIRE(!labels.custom, KB2_NOT_IMPLEMENTED, "faiss stream: HNSW with custom ids");
        o.xb = h_vecs;
        o.levels = h_levels;
        o.neighbors = h_neighbors;
        o.offsets.assign(h_offsets.begin(), h_offsets.end());
        o.entry_point = entry_point;
        o.max_level = max_level;
        o.efConstruction = efConstruction;
        // K/impl/HNSW.cpp:78-89 set_default_probas(M, 1 / ln M): the full level table, of which h_cum is a prefix
        const double mult = 1.0 / std::log((double)M);
        int nn = 0;
        o.cum.assign(1, 0);
        for (int level = 0;; level++) {
            const double proba = std::exp(-level / mult) * (1 - std::exp(-1 / mult));
            if (proba < 1e-9) break;
            o.assign_probas.push_back(proba);
            nn += level == 0 ? M * 2 : M;
            o.cum.push_back(nn);
        }
        KB2_REQUIRE(o.cum.size() >= h_cum.size(), KB2_INTERNAL_ERROR, "HNSW level table shorter than the graph's");
        for (size_t i = 0; i < h_cum.size(); i++)
            KB2_REQUIRE(o.cum[i] == h_cum[i], KB2_NOT_IMPLEMENTED, "faiss stream: non-default HNSW link counts");
    }
    void
    from_faiss(const FaissIndexData& o) override {
        M = o.cum.size() >= 2 ? o.cum[1] / 2 : 16;
        efConstruction = o.efConstruction;
        std::vector<int64_t> off(o.offsets.begin(), o.offsets.end());
        std::vector<float> normed;
        const float* xb = o.xb.data();
        if (o.cosine) {   // the reference keeps raw rows + norms (IHN9); this core keeps unit rows
            normed = o.xb;
            for (int64_t i = 0; i < o.ntotal; i++) {
                double s2 = 0;
                for (int j = 0; j < o.d; j++) s2 += (double)normed[i * o.d + j] * normed[i * o.d + j];
                const float inv = s2 > 0 ? (float)(1.0 / std::sqrt(s2)) : 1.f;
                for (int j = 0; j < o.d; j++) normed[i * o.d + j] *= inv;
            }
            xb = normed.data();
        }
        import_graph(o.ntotal, xb, o.levels.data(), off.data(), o.neighbors.data(), o.cum.data(), (int)o.cum.size(), o.entry_point,
                     o.max_level);
    }

    void
    append_meta(std::string& s) const override {
        s += ", \"M\": " + std::to_string(M) + ", \"efConstruction\": " + std::to_string(efConstruction) +
             ", \"max_level\": " + std::to_string(max_level) + ", \"entry_point\": " + std::to_string(entry_point);
    }
    bool takes_emb_list() const override { return true; }
    std::pair<const float*, const int32_t*>
    emb_list_rows() override {
        upload();
        return {d_vecs.p, nullptr};
    }
    void
    emb_list_base_config(JsonObj& base, int k, int vec_topk) const override {
        // base_hnsw_config.h:60-72 checks ef against the list-level k; the base search keeps max(ef, vec_topk)
        const int64_t ef = base.get_int("ef", std::max(k, 16));
        KB2_REQUIRE(ef >= k, KB2_OUT_OF_RANGE_IN_JSON, "ef(" + std::to_string(ef) + ") should be larger than k(" + std::to_string(k) + ")");
        base.kv["ef"] = std::to_string(std::max<int64_t>(ef, vec_topk));
    }
};

}  // namespace kb2
