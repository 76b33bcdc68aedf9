// kb2_listmajor.cuh — the pipeline around the list-major tensor-core engines (IVF_PQ: kb2_ivfpq_tc.cuh, IVF_FLAT:
// kb2_ivfflat_tc.cuh; DESIGN.md 4.2, 4.4, 4.5).
//
//   1. plan: the (query, probe) pairs are grouped by list (count_pairs_kernel -> plan_kernel -> fill_pairs_kernel), and each
//      list's queries are cut into work items = (list, chunk of <= item_cap of the queries probing it);
//   2. the items are sorted by descending estimated cost (item_cost_kernel -> 16-bit radix sort -> deal_items_kernel);
//   3. one persistent CTA per SM draws the items in that order from a global ticket counter; the roles of a CTA share the
//      draws through an ItemRing in shared memory;
//   4. survivors go to per-group global logs (entry {query, position, high word of the candidate entry, 0}; log_cnt[g] =
//      entries of log g, log_cnt[n_logs] = 1 when any log overflowed);
//   5. scatter_survivors_kernel copies the logs into per-query candidate rows.
#pragma once
#include <cub/block/block_scan.cuh>

#include "kb2_common.cuh"

namespace kb2 {
namespace lm {

constexpr int TM = 128;   // list rows per tile of both engines (two wgmma M = 64 halves); the unit of the cost model

// ---------------------------------------------------------------- plan: (query, probe) pairs grouped by list
__global__ void
count_pairs_kernel(const int64_t* __restrict__ probe_ids, int64_t npairs, const int32_t* __restrict__ list_len,
                   int32_t* __restrict__ lcount) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    const int64_t l = probe_ids[i];
    if (l >= 0 && list_len[l] > 0) atomicAdd(lcount + l, 1);
}

// one CTA: exclusive scans over the lists -> first pair of each list, item table (list, chunk of <= item_cap queries)
__global__ void __launch_bounds__(1024)
plan_kernel(const int32_t* __restrict__ lcount, int nlist, int item_cap, int32_t* __restrict__ lstart, int32_t* __restrict__ item_list,
            int32_t* __restrict__ item_q0, int32_t* __restrict__ item_nq, int32_t* __restrict__ n_items) {
    typedef cub::BlockScan<int, 1024> Scan;
    __shared__ typename Scan::TempStorage tmp_a, tmp_b;
    __shared__ int carry_a, carry_b;
    if (threadIdx.x == 0) carry_a = carry_b = 0;
    __syncthreads();
    for (int b0 = 0; b0 < nlist; b0 += 1024) {
        const int l = b0 + threadIdx.x;
        const int c = l < nlist ? lcount[l] : 0;
        const int nch = (c + item_cap - 1) / item_cap;
        int ex_a, ex_b, tot_a, tot_b;
        Scan(tmp_a).ExclusiveSum(c, ex_a, tot_a);
        Scan(tmp_b).ExclusiveSum(nch, ex_b, tot_b);
        const int ca = carry_a, cb = carry_b;
        if (l < nlist) {
            lstart[l] = ca + ex_a;
            if (nch > 0) {
                // even chunks, multiples of 16 queries (the wgmma N granularity; item_cap is one too); full chunks when
                // rounding would leave the last one empty (an item without queries would be an N = 0 MMA)
                int per = ((c + nch - 1) / nch + 15) & ~15;
                if ((nch - 1) * per >= c) per = item_cap;
                for (int ch = 0; ch < nch; ch++) {
                    const int i = cb + ex_b + ch;
                    item_list[i] = l;
                    item_q0[i] = ca + ex_a + ch * per;
                    item_nq[i] = max(0, min(per, c - ch * per));
                }
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            carry_a = ca + tot_a;
            carry_b = cb + tot_b;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *n_items = carry_b;
}

// ---- load balancing of the persistent kernels.  Item costs have a heavy tail (list length x queries per list), and the
// launch lasts as long as its slowest CTA.  Items are therefore sorted by descending cost estimate and drawn in that order
// from the ticket counter (longest processing time first): a CTA that got short items simply draws more.
__global__ void
item_cost_kernel(const int32_t* __restrict__ n_items, const int32_t* __restrict__ item_list, const int32_t* __restrict__ item_nq,
                 const int32_t* __restrict__ list_len, int64_t max_items, int tile_cost, int col_cost, uint32_t* __restrict__ key,
                 int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= max_items) return;
    uint32_t k = 0xffffu;   // unused slots sort to the end; 16-bit keys = two radix passes
    if (i < *n_items) {
        const long long tiles = (list_len[item_list[i]] + TM - 1) / TM;
        const long long c = (tiles * (tile_cost + (long long)col_cost * ((item_nq[i] + 15) & ~15))) >> 5;
        k = 0xfffeu - (uint32_t)min(c, 0xfff0ll);   // ascending key = descending cost
    }
    key[i] = k;
    idx[i] = (int32_t)i;
}
__global__ void
deal_items_kernel(const int32_t* __restrict__ n_items, const int32_t* __restrict__ sorted_idx, const int32_t* __restrict__ in_list,
                  const int32_t* __restrict__ in_q0, const int32_t* __restrict__ in_nq, int32_t* __restrict__ out_list,
                  int32_t* __restrict__ out_q0, int32_t* __restrict__ out_nq) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;   // rank by descending cost
    if (j >= *n_items) return;
    const int src = sorted_idx[j];
    out_list[j] = in_list[src];
    out_q0[j] = in_q0[src];
    out_nq[j] = in_nq[src];
}

__global__ void
fill_pairs_kernel(const int64_t* __restrict__ probe_ids, const float* __restrict__ probe_dis, int64_t npairs, int nprobe,
                  int metric, const int32_t* __restrict__ list_len, const int32_t* __restrict__ lstart,
                  int32_t* __restrict__ lcursor, int32_t* __restrict__ pair_q, float* __restrict__ pair_base) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    const int64_t l = probe_ids[i];
    if (l < 0 || list_len[l] <= 0) return;
    const int slot = lstart[l] + atomicAdd(lcursor + l, 1);
    pair_q[slot] = (int32_t)(i / nprobe);
    const float dv = probe_dis[i];
    pair_base[slot] = (metric == KB2_METRIC_L2) ? dv : -dv;
}

// ---------------------------------------------------------------- item sequence of a CTA
// The roles of a CTA walk the same item sequence independently, so the seq-th draw is published through a ring of R slots
// in shared memory: whoever needs it first claims the slot (atomicCAS), takes a ticket from the global counter and
// publishes it; the others read it.  The roles must stay fewer than R draws apart.
template <int R>
struct ItemRing {
    static constexpr int BYTES = 3 * R * 4;   // claim[R] | item[R] | ready[R]
    int* claim;
    int* item;
    volatile int* ready;
    int* ticket;
    __device__ __forceinline__ ItemRing(unsigned char* at, int* ticket_)
        : claim((int*)at), item((int*)at + R), ready((volatile int*)at + 2 * R), ticket(ticket_) {}
    // before the CTA barrier that precedes the first draw
    __device__ __forceinline__ void
    init() const {
        if (threadIdx.x < R) {
            claim[threadIdx.x] = (int)threadIdx.x - R;
            ready[threadIdx.x] = -1;
        }
    }
    __device__ __forceinline__ int
    at_thread(int seq) const {
        const int sl = seq & (R - 1);
        if (ready[sl] != seq) {
            if (atomicCAS(claim + sl, seq - R, seq) == seq - R) {
                const int t = atomicAdd(ticket, 1);
                ((volatile int*)item)[sl] = t;
                __threadfence_block();
                ready[sl] = seq;
            } else {
                while (ready[sl] != seq) {}
            }
        }
        __threadfence_block();
        return ((volatile int*)item)[sl];
    }
    // warp-uniform call: lane 0 draws, the warp gets its result
    __device__ __forceinline__ int
    at_warp(int seq) const {
        int v = 0;
        if ((threadIdx.x & 31) == 0) v = at_thread(seq);
        return __shfl_sync(0xffffffffu, v, 0);
    }
};

// ---------------------------------------------------------------- survivor logs -> per-query candidate rows
// thread per log entry, grid = (x, number of logs).  The candidate entry is (log word 2 << 32) | position; a row that is full
// flags its query (and counts it in counters[6] when counters is set).
__global__ void
scatter_survivors_kernel(const uint4* __restrict__ log, const uint32_t* __restrict__ log_cnt, uint32_t log_cap,
                         uint64_t* __restrict__ cand, uint32_t* __restrict__ cand_cnt, int cap, uint32_t* __restrict__ qflag,
                         unsigned long long* __restrict__ counters) {
    const uint32_t n = min(log_cnt[blockIdx.y], log_cap);
    const uint4* src = log + (size_t)blockIdx.y * log_cap;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4 e = src[i];
        const uint32_t slot = atomicAdd(cand_cnt + e.x, 1u);
        if (slot < (uint32_t)cap) cand[(int64_t)e.x * cap + slot] = ((uint64_t)e.z << 32) | e.y;
        else {
            qflag[e.x] = 1u;
            if (counters) atomicAdd(counters + 6, 1ull);
        }
    }
}

}  // namespace lm
}  // namespace kb2
