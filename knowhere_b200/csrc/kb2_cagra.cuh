// kb2_cagra.cuh — GPU_CAGRA: a fixed-degree graph index built on the device and searched by a batched itopk kernel
// (DESIGN §4.12).  The reference's GPU_CAGRA node (src/index/gpu_cuvs/gpu_cuvs_cagra.cc) adapts cuVS; this index follows
// the same parameters (gpu_cuvs_cagra_config.h) with its own build and search, defined exactly so that the result can
// be checked against a numpy model of the definition.
//
// Build, m = min(intermediate_graph_degree, n - 1), g = min(graph_degree, m):
//   1. G0[i]: the m rows nearest to row i, best first, ties by ascending id (dense_knn over row chunks, k = m + 1, then
//      row i removed where it appears, else the last entry dropped); or, with build_algo NN_DESCENT, the NN-descent
//      graph defined at cagra_nnd_join_kernel.
//   2. detour(i, b) = #{a < b : G0[i][b] in G0[G0[i][a]][0:b]}                          (cagra_prune_kernel)
//   3. P[i]: the g entries of G0[i] with the smallest (detour, b), in that order         (cagra_prune_kernel)
//   4. R[v]: the sources i of the edges i -> v = P[i][p], ordered by (p, i)              (one cub radix sort)
//   5. row i: P[i][0:g/2], then R[i] in order, then P[i][g/2:], skipping ids present, up to g  (cagra_merge_kernel)
// The graph is one level of the reference's HNSW layout (levels 1, cum {0, g}, entry point 0), so CagraIndex is an
// HnswIndex: export, the IHNf writer, the exact scan, the visited bitmaps and the key arithmetic are HNSW's.
//
// Search (cagra_search_kernel, one query per CTA, persistent CTAs on an atomic counter):
//   * seeds j < s = min(n, max(1, num_random_samplings * search_width * g)): row splitmix64(j) mod n;
//   * pool T: the itopk best (key, id) of the evaluated rows, each with an expanded flag;
//   * iteration: the first <= search_width unexpanded entries of T are the parents; their g neighbours that are not yet
//     visited are evaluated; T becomes the first itopk of merge(T, candidates) by (key, id); stop when no entry is
//     unexpanded or after max_iterations (> 0) iterations;
//   * the visited set is exact (per-CTA bitmap + touched-id log, cleared after each query), so a row costs one distance;
//   * the result: the first k entries of T the bitset does not filter out (filtered rows route but are not returned).
#pragma once
#include <cub/cub.cuh>
#include <numeric>

#include "kb2_hnsw.cuh"

namespace kb2 {

constexpr int kCagraMaxIgd = 1007;      // igd + 1 must stay on dense_knn's kMaxK path (k + 16 <= 1024)
constexpr int kCagraMaxGd = 256;        // the reverse-edge sort keeps the slot in 8 bits
constexpr int kCagraMaxItopk = 1024;
constexpr int kCagraMaxCand = 4096;     // search_width * graph_degree: candidates of one iteration (shared memory)
constexpr int kCagraThreads = 256;
constexpr int kCagraPruneThreads = 256;
constexpr int kCagraHash = 2048;        // id -> rank table of one G0 row (m <= 1007: load below one half)
constexpr uint32_t kExpanded = 0x80000000u;

// seed j of every query (splitmix64 of j + 1)
__host__ __device__ __forceinline__ uint64_t
cagra_seed(uint64_t j) {
    uint64_t z = (j + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// ============================================================================================ build
// G0 row i <- the m + 1 nearest ids of row i without i (or without the last one when i is not among them); with g0_key,
// their keys too (dist: the dense_knn distances, negated for IP)
__global__ void __launch_bounds__(256)
cagra_drop_self_kernel(const int64_t* __restrict__ knn, const float* __restrict__ dist, int ip, int64_t rows, int64_t row0,
                       int m, int32_t* __restrict__ g0, float* __restrict__ g0_key) {
    const int64_t r = (int64_t)blockIdx.x * (blockDim.x / kWarp) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const int64_t self = row0 + r;
    const int64_t* in = knn + r * (m + 1);
    int32_t* out = g0 + self * m;
    // position of self in the list (m + 1 if absent: then entries 0..m-1 are kept)
    int pos = m + 1;
    for (int b = 0; b < m + 1; b += kWarp) {
        const bool hit = b + lane < m + 1 && in[b + lane] == self;
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (bal) { pos = b + __ffs(bal) - 1; break; }
    }
    for (int c = lane; c < m; c += kWarp) {
        const int s = c < pos ? c : c + 1;
        out[c] = (int32_t)in[s];
        if (g0_key) g0_key[self * m + c] = ip ? -dist[r * (m + 1) + s] : dist[r * (m + 1) + s];
    }
}

// Steps 2-3, one CTA per row i: detour counts through an id -> rank table of G0[i] in shared memory (each warp reads
// whole rows G0[G0[i][a]], coalesced), then the g best (detour, b) by a block radix sort of detour << 10 | b.
__global__ void __launch_bounds__(kCagraPruneThreads)
cagra_prune_kernel(const int32_t* __restrict__ g0, int64_t n, int m, int g, int32_t* __restrict__ pruned) {
    __shared__ int32_t h_id[kCagraHash];
    __shared__ int16_t h_rank[kCagraHash];
    __shared__ int32_t row[1024];
    __shared__ int32_t det[1024];
    using Sort = cub::BlockRadixSort<uint32_t, kCagraPruneThreads, 4>;
    __shared__ typename Sort::TempStorage sort_tmp;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t i = blockIdx.x;
    for (int t = tid; t < kCagraHash; t += kCagraPruneThreads) h_id[t] = -1;
    __syncthreads();
    for (int b = tid; b < m; b += kCagraPruneThreads) {
        const int32_t v = g0[i * m + b];
        row[b] = v;
        det[b] = 0;
        uint32_t h = ((uint32_t)v * 2654435761u) & (kCagraHash - 1);
        while (atomicCAS(&h_id[h], -1, v) != -1) h = (h + 1) & (kCagraHash - 1);
        h_rank[h] = (int16_t)b;
    }
    __syncthreads();
    for (int a = warp; a < m; a += kCagraPruneThreads / kWarp) {
        const int32_t* r = g0 + (int64_t)row[a] * m;
        // only positions c < b with b > a count, and b < m: c < m - 1
        for (int c = lane; c < m - 1; c += kWarp) {
            const int32_t w = r[c];
            uint32_t h = ((uint32_t)w * 2654435761u) & (kCagraHash - 1);
            int b = -1;
            for (;;) {
                const int32_t s = h_id[h];
                if (s == w) { b = h_rank[h]; break; }
                if (s < 0) break;
                h = (h + 1) & (kCagraHash - 1);
            }
            if (b > a && b > c) atomicAdd(&det[b], 1);
        }
    }
    __syncthreads();
    uint32_t keys[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int b = tid * 4 + u;
        keys[u] = b < m ? ((uint32_t)det[b] << 10) | (uint32_t)b : 0xffffffffu;
    }
    Sort(sort_tmp).Sort(keys, 0, 20);
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int p = tid * 4 + u;
        if (p < g) pruned[i * g + p] = row[keys[u] & 1023u];
    }
}

// reverse-edge sort input: key (v << 8 | p) and value i of every edge i -> v = P[i][p]
__global__ void
cagra_edge_keys_kernel(const int32_t* __restrict__ pruned, int64_t n, int g, uint64_t* __restrict__ key, int32_t* __restrict__ src) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n * g) return;
    key[e] = ((uint64_t)(uint32_t)pruned[e] << 8) | (uint64_t)(e % g);
    src[e] = (int32_t)(e / g);
}

// rstart[v] = first sorted edge whose target is >= v (v = 0..n)
__global__ void
cagra_reverse_offsets_kernel(const uint64_t* __restrict__ key, int64_t ne, int64_t n, int64_t* __restrict__ rstart) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > ne) return;
    const int64_t hi = t < ne ? (int64_t)(key[t] >> 8) : n;
    const int64_t lo = t > 0 ? (int64_t)(key[t - 1] >> 8) + 1 : 0;
    for (int64_t v = lo; v <= hi && v <= n; v++) rstart[v] = t;
}

// Step 5, one warp per row: P[i][0:g/2], then R[i], then P[i][g/2:], each id appended once, up to g ids.
constexpr int kMergeWarps = 8;
__global__ void __launch_bounds__(kMergeWarps * kWarp)
cagra_merge_kernel(const int32_t* __restrict__ pruned, const int32_t* __restrict__ rsrc, const int64_t* __restrict__ rstart,
                   int64_t n, int g, int32_t* __restrict__ graph) {
    __shared__ int32_t s_out[kMergeWarps][kCagraMaxGd];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kMergeWarps + warp;
    if (i >= n) return;
    int32_t* out = s_out[warp];
    const int half = g / 2;
    for (int c = lane; c < half; c += kWarp) out[c] = pruned[i * g + c];
    __syncwarp();
    int len = half;
    // candidates in 32-wide chunks; within a chunk, lanes are appended in order (an id repeats only across sources)
    auto append = [&](const int32_t* src, int64_t cnt) {
        for (int64_t b = 0; b < cnt && len < g; b += kWarp) {
            const int32_t v = b + lane < cnt ? src[b + lane] : -1;
            bool fresh = v >= 0;
            for (int c = 0; c < len; c++) fresh = fresh && out[c] != v;   // smem broadcast-free compare: len <= 256
            unsigned fm = __ballot_sync(0xffffffffu, fresh);
            const int pos = len + __popc(fm & ((1u << lane) - 1));
            if (fresh && pos < g) out[pos] = v;
            len = min(g, len + __popc(fm));
            __syncwarp();
        }
    };
    append(rsrc + rstart[i], rstart[i + 1] - rstart[i]);
    append(pruned + i * g + half, g - half);
    for (int c = lane; c < g; c += kWarp) graph[i * g + c] = out[c];
}

// ============================================================================================ NN-descent (step 1)
// With build_algo NN_DESCENT, G0 is the NN-descent graph (DESIGN §4.12; tests/cagra_nnd_model.py restates it).
// m = min(igd, n - 1), S = min(32, m).  Row i keeps L[i]: m entries (key, id, new), best first by (key, id), distinct ids,
// never i.
//   init:  L[i][j] = (i + 1 + (o_i + j * stride) mod (n - 1)) mod n, o_i = cagra_seed(i) mod (n - 1), stride the first
//          integer >= max(1, floor(0.618 (n - 1))) coprime to n - 1; every entry new.
//   iteration t < niter:
//     forward  new_f(i) / old_f(i): the first <= S entries of L[i] flagged new / old; the sampled new entries become old;
//     reverse  new_r(i) / old_r(i): the <= S sources j with i in new_f(j) / old_f(j) of smallest (nnd_hash(j, i, t), j);
//     join     C_new = new_f u new_r, C_old = old_f u old_r; every pair {u, v}, u != v, u in C_new, v in C_new u C_old,
//              proposes (key(u, v), v) to u and (key(u, v), u) to v;
//     update   L[u] <- the best m of L[u] u proposals(u) by (key, id), one entry per id; entries that enter are new;
//     stop     when updates(t) = #new entries <= 1e-4 n m.
//   G0[i]: the ids of L[i].
// Every key comes from nnd_gram (3xTF32 mma.sync with the lower id in the A role), so a pair has the same key bits in
// every kernel that computes it; the update is then the top m of a totally ordered set, and a proposal is only dropped
// unlocked when it is worse than the live m-th key of its target (which only improves): the graph does not depend on
// the order in which the joins run.
__device__ __forceinline__ bool cagra_less(float ka, uint32_t ia, float kb, uint32_t ib);
__device__ __forceinline__ int cagra_rank(const float* key, const uint32_t* id, int len, float k, uint32_t i);

constexpr int kNndS = 32;
constexpr int kNndMaxC = 4 * kNndS;          // candidates of one join: |C_new|, |C_old| <= 2S
constexpr int kNndThreads = 256;
constexpr int kNndWarps = kNndThreads / kWarp;
constexpr int kNndKc = 32;                   // dims staged per Gram step
constexpr int kNndXld = kNndKc + 4;          // staged row stride (fragment loads hit 32 distinct banks)
constexpr int kNndKld = kNndMaxC + 4;        // key tile row stride
constexpr uint32_t kNndNew = 0x80000000u;    // "new" flag of a list entry's id (cagra_less ignores it)
constexpr uint32_t kNndIdMask = 0x7fffffffu;
constexpr double kNndDelta = 1e-4;           // termination threshold (updates <= delta n m), cuVS's default

// priority of source j among the reverse samples of target i at iteration t (smaller first; ties by j)
__host__ __device__ __forceinline__ uint32_t
nnd_hash(uint32_t src, uint32_t tgt, int t) {
    return (uint32_t)(cagra_seed(cagra_seed((uint64_t)t) ^ (((uint64_t)src << 32) | tgt)) >> 32);
}

__device__ __forceinline__ void
nnd_split(float x, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(__fsub_rn(x, __uint_as_float(hi))));
}
__device__ __forceinline__ void
nnd_mma(float* c, const uint32_t* a, const uint32_t* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// key of a pair from the lower id's norm, the higher id's norm and their dot product; + 0 turns -0 into +0
template <int METRIC>
__device__ __forceinline__ float
nnd_key(float n_lo, float n_hi, float dot) {
    return __fadd_rn(METRIC == KB2_METRIC_L2 ? __fmaf_rn(-2.f, dot, __fadd_rn(n_lo, n_hi)) : -dot, 0.f);
}
// float -> uint32 with the same order
__device__ __forceinline__ uint32_t
nnd_ord(float k) {
    const uint32_t u = __float_as_uint(k);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float
nnd_unord(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// CTA-wide: the keys of the pairs r < c < C of the candidates s_id[0, C) (C <= kNndMaxC, ascending distinct ids) into
// s_key[r][c] and s_key[c][r].  focus >= 0: only the tiles holding row or column `focus` are needed.  Rows are gathered
// kNndKc dims at a time with cp.async (zero-filled past d and past C) and contracted in 16 x 8 tiles on the tensor cores,
// hi.hi + hi.lo + lo.hi per k-step of 8, fp32 accumulation.  Tile (r, c) always has the lower id in the A role and runs
// the same k-steps in the same order, so a pair's key has the same bits in every call.  Starts and ends at a barrier.
template <int METRIC>
__device__ __forceinline__ void
nnd_gram(const float* __restrict__ x, int d, const uint32_t* s_id, const float* s_norm, int C, int focus, float* s_x,
         float* s_key) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int cp = (C + 15) & ~15;
    const int nct = cp >> 3, ntiles = (cp >> 4) * nct;
    constexpr int kTiles = (kNndMaxC / 16) * (kNndMaxC / 8) / kNndWarps;   // tiles per warp at most
    auto live = [&](int q) {
        const int rt = q / nct, ct = q % nct;
        if (q >= ntiles || 8 * ct + 7 <= 16 * rt) return false;   // every (r, c) of the tile has r >= c
        return focus < 0 || (focus >> 4) == rt || (focus >> 3) == ct;
    };
    float acc[kTiles][4];
#pragma unroll
    for (int j = 0; j < kTiles; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int k0 = 0; k0 < d; k0 += kNndKc) {
        for (int e = tid; e < cp * kNndKc; e += kNndThreads) {
            const int r = e / kNndKc, kk = e % kNndKc;
            const bool ok = r < C && k0 + kk < d;
            const float* src = ok ? x + (int64_t)s_id[r] * d + k0 + kk : x;
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(s_x + r * kNndXld + kk);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(ok ? 4 : 0) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kTiles; j++) {
            const int q = warp + kNndWarps * j;
            if (!live(q)) continue;
            const float* A = s_x + ((q / nct) * 16 + g) * kNndXld + t4;
            const float* B = s_x + ((q % nct) * 8 + g) * kNndXld + t4;
#pragma unroll
            for (int ks = 0; ks < kNndKc; ks += 8) {
                uint32_t ah[4], al[4], bh[2], bl[2];
                nnd_split(A[ks], ah[0], al[0]);
                nnd_split(A[8 * kNndXld + ks], ah[1], al[1]);
                nnd_split(A[ks + 4], ah[2], al[2]);
                nnd_split(A[8 * kNndXld + ks + 4], ah[3], al[3]);
                nnd_split(B[ks], bh[0], bl[0]);
                nnd_split(B[ks + 4], bh[1], bl[1]);
                nnd_mma(acc[j], ah, bh);
                nnd_mma(acc[j], ah, bl);
                nnd_mma(acc[j], al, bh);
            }
        }
        __syncthreads();
    }
    // accumulator e of a tile: row g + 8 (e >> 1), column 2 t4 + (e & 1)
#pragma unroll
    for (int j = 0; j < kTiles; j++) {
        const int q = warp + kNndWarps * j;
        if (!live(q)) continue;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int r = (q / nct) * 16 + g + 8 * (e >> 1), c = (q % nct) * 8 + 2 * t4 + (e & 1);
            if (r < c && c < C) {
                const float k = nnd_key<METRIC>(s_norm[r], s_norm[c], acc[j][e]);
                s_key[r * kNndKld + c] = k;
                s_key[c * kNndKld + r] = k;
            }
        }
    }
    __syncthreads();
}

// CTA-wide: s_out[rank] = s_in[e] in ascending order (ties by position), s_perm[rank] = e if given.  Ends at a barrier.
__device__ __forceinline__ void
nnd_rank_sort(const uint32_t* s_in, int C, uint32_t* s_out, int16_t* s_perm) {
    for (int e = threadIdx.x; e < C; e += kNndThreads) {
        const uint32_t v = s_in[e];
        int r = 0;
        for (int f = 0; f < C; f++) {
            const uint32_t w = s_in[f];
            r += (w < v) || (w == v && f < e);
        }
        s_out[r] = v;
        if (s_perm) s_perm[r] = (int16_t)e;
    }
    __syncthreads();
}

// shared memory of the init and join kernels: key tile | staged rows | candidate norms, ids (+ per-warp lists and batches)
__host__ __device__ constexpr size_t
nnd_smem_common() {
    return (size_t)kNndMaxC * kNndKld * 4 + (size_t)kNndMaxC * kNndXld * 4 + (size_t)kNndMaxC * 4 * 4 + 256;
}

// L[i] <- the initial list of row i, best first: one CTA per row; the m ids are keyed in chunks of kNndMaxC - 1 together
// with i (the Gram tiles holding i only), then sorted by (key, id).  Dynamic smem: nnd_smem_common() + 8 KB.
template <int METRIC>
__global__ void __launch_bounds__(kNndThreads)
cagra_nnd_init_kernel(const float* __restrict__ x, const float* __restrict__ norms, int64_t n, int d, int m, int64_t stride,
                      float* __restrict__ lkey, uint32_t* __restrict__ lid) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_key = (float*)smem_raw;
    float* s_x = s_key + kNndMaxC * kNndKld;
    float* s_norm = s_x + kNndMaxC * kNndXld;
    uint32_t* s_raw = (uint32_t*)(s_norm + kNndMaxC);
    uint32_t* s_id = s_raw + kNndMaxC;
    int16_t* s_perm = (int16_t*)(s_id + kNndMaxC);
    int* s_focus = (int*)(s_perm + kNndMaxC);
    float* s_lk = (float*)(smem_raw + nnd_smem_common());   // 1024 keys, then 1024 ids
    uint32_t* s_li = (uint32_t*)(s_lk + 1024);
    const int tid = threadIdx.x;
    const int64_t i = blockIdx.x;
    const uint64_t nm1 = (uint64_t)(n - 1);
    const uint64_t o = cagra_seed((uint64_t)i) % nm1;
    for (int j = tid; j < m; j += kNndThreads) s_li[j] = (uint32_t)(((uint64_t)i + 1 + (o + (uint64_t)j * (uint64_t)stride) % nm1) % (uint64_t)n);
    __syncthreads();
    for (int j0 = 0; j0 < m; j0 += kNndMaxC - 1) {
        const int cnt = min(kNndMaxC - 1, m - j0);
        for (int e = tid; e <= cnt; e += kNndThreads) s_raw[e] = e == 0 ? (uint32_t)i : s_li[j0 + e - 1];
        __syncthreads();
        nnd_rank_sort(s_raw, cnt + 1, s_id, s_perm);
        for (int e = tid; e <= cnt; e += kNndThreads) {
            s_norm[e] = METRIC == KB2_METRIC_L2 ? norms[s_id[e]] : 0.f;
            if (s_perm[e] == 0) *s_focus = e;
        }
        __syncthreads();
        const int f = *s_focus;
        nnd_gram<METRIC>(x, d, s_id, s_norm, cnt + 1, f, s_x, s_key);
        for (int e = tid; e <= cnt; e += kNndThreads)
            if (e != f) s_lk[j0 + s_perm[e] - 1] = s_key[e * kNndKld + f];
        __syncthreads();
    }
    // best first by (key, id): one block radix sort of (ordered key, id), its storage over the key tile
    using Sort = cub::BlockRadixSort<uint64_t, kNndThreads, 4>;
    static_assert(sizeof(typename Sort::TempStorage) <= (size_t)kNndMaxC * kNndKld * 4, "sort storage");
    uint64_t k[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int j = tid * 4 + u;
        k[u] = j < m ? ((uint64_t)nnd_ord(s_lk[j]) << 32) | s_li[j] : ~0ull;
    }
    Sort(*reinterpret_cast<typename Sort::TempStorage*>(s_key)).Sort(k);
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int j = tid * 4 + u;
        if (j < m) {
            lkey[i * m + j] = nnd_unord((uint32_t)(k[u] >> 32));
            lid[i * m + j] = (uint32_t)k[u] | kNndNew;
        }
    }
}

// Forward samples of row i (one warp per row): fwd[i][0, S) the first <= S new entries (then flagged old), fwd[i][32,
// 32 + S) the first <= S old ones, ~0 past the counts.  Each sample j -> v also writes its reverse-sort entry: key
// v << 33 | old << 32 | nnd_hash(i, v, t), value i (~0 keys for the unused slots sort last).
__global__ void __launch_bounds__(256)
cagra_nnd_sample_kernel(uint32_t* __restrict__ lid, int64_t n, int m, int S, int t, uint32_t* __restrict__ fwd,
                        uint64_t* __restrict__ rkey, uint32_t* __restrict__ rsrc) {
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x / kWarp) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    uint32_t* L = lid + i * m;
    uint32_t* F = fwd + i * 2 * kNndS;
    uint64_t* K = rkey + i * 2 * kNndS;
    const unsigned lt = (1u << lane) - 1;
    int cn = 0, co = 0;
    for (int b = 0; b < m && (cn < S || co < S); b += kWarp) {
        const int q = b + lane;
        const uint32_t v = q < m ? L[q] : 0u;
        const bool isn = q < m && (v & kNndNew), iso = q < m && !(v & kNndNew);
        const unsigned bn = __ballot_sync(0xffffffffu, isn), bo = __ballot_sync(0xffffffffu, iso);
        const int pn = cn + __popc(bn & lt), po = co + __popc(bo & lt);
        const uint32_t tgt = v & kNndIdMask;
        if (isn && pn < S) {
            F[pn] = tgt;
            L[q] = tgt;
            K[pn] = ((uint64_t)tgt << 33) | nnd_hash((uint32_t)i, tgt, t);
        }
        if (iso && po < S) {
            F[kNndS + po] = tgt;
            K[kNndS + po] = ((uint64_t)tgt << 33) | (1ull << 32) | nnd_hash((uint32_t)i, tgt, t);
        }
        cn = min(S, cn + __popc(bn));
        co = min(S, co + __popc(bo));
    }
    for (int s = lane; s < 2 * kNndS; s += kWarp) {
        if ((s < kNndS && s >= cn) || (s >= kNndS && s - kNndS >= co)) {
            F[s] = ~0u;
            K[s] = ~0ull;
        }
        rsrc[i * 2 * kNndS + s] = (uint32_t)i;
    }
}

// rs[2 v + o] = the first sorted reverse entry of target v with old flag >= o (v = 0..n; rs[2 n] ends the real ones)
__global__ void
cagra_nnd_offsets_kernel(const uint64_t* __restrict__ key, int64_t ne, int64_t n, int64_t* __restrict__ rs) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > 2 * n) return;
    const uint64_t probe = ((uint64_t)(t >> 1) << 33) | ((uint64_t)(t & 1) << 32);
    int64_t lo = 0, hi = ne;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (key[mid] < probe) lo = mid + 1; else hi = mid;
    }
    rs[t] = lo;
}

// bounded spin (~3 s of SM clocks): a protocol bug must end the launch with an error, never hang the GPU
__device__ __forceinline__ void
nnd_lock(int* l) {
    if (atomicCAS(l, 0, 1) != 0) {
        const long long t0 = clock64();
        while (atomicCAS(l, 0, 1) != 0) {
            __nanosleep(64);
            if (clock64() - t0 > 6000000000ll) __trap();
        }
    }
    __threadfence();
}

struct NndJoinParams {
    const float* x;
    const float* norms;
    int64_t n;
    int d, m, S;
    const uint32_t* fwd;     // n x 2 kNndS forward samples
    const uint32_t* rsrc;    // sorted reverse sources
    const int64_t* rs;       // 2 n + 1 offsets into rsrc
    float* lkey;             // n x m lists
    uint32_t* lid;
    int* lock;               // n row locks
};

// per-warp shared memory of the join: the target's list (m keys, m ids), a batch (kNndMaxC keys, ids, ranks)
__host__ __device__ constexpr size_t
nnd_join_warp_smem(int m) {
    return ((size_t)m * 8 + (size_t)kNndMaxC * 12 + 15) & ~(size_t)15;
}

// One join per CTA (row i): the candidates (C_new before C_old, sorted by id, deduplicated keeping the new copy), their
// key tile (nnd_gram), then one warp per candidate u: the proposals to u that pass the live m-th key of L[u], sorted by
// (key, id), merged into L[u] under the row lock (one lane takes it; a warp holds one lock at a time and waits on none
// while it holds it).
template <int METRIC>
__global__ void __launch_bounds__(kNndThreads, 2)
cagra_nnd_join_kernel(NndJoinParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_key = (float*)smem_raw;
    float* s_x = s_key + kNndMaxC * kNndKld;
    float* s_norm = s_x + kNndMaxC * kNndXld;
    uint32_t* s_raw = (uint32_t*)(s_norm + kNndMaxC);
    uint32_t* s_sorted = s_raw + kNndMaxC;
    uint32_t* s_id = s_sorted + kNndMaxC;
    int* s_ctl = (int*)(s_id + kNndMaxC);
    uint8_t* s_new = (uint8_t*)(s_ctl + 4);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const unsigned lt = (1u << lane) - 1;
    const int m = p.m;
    unsigned char* wbase = smem_raw + nnd_smem_common() + (size_t)warp * nnd_join_warp_smem(m);
    float* wl_key = (float*)wbase;
    uint32_t* wl_id = (uint32_t*)(wl_key + m);
    float* wb_key = (float*)(wl_id + m);
    uint32_t* wb_id = (uint32_t*)(wb_key + kNndMaxC);
    int* wr = (int*)(wb_id + kNndMaxC);
    const int64_t i = blockIdx.x;

    // candidates: slots [0, 32) new_f, [32, 64) new_r, [64, 96) old_f, [96, 128) old_r as id << 1 | old (~0: none)
    if (tid < kNndMaxC) {
        const int part = tid >> 5, s = tid & 31;
        uint32_t v = ~0u;
        if (s < p.S) {
            if (part == 0 || part == 2) {
                const uint32_t f = p.fwd[i * 2 * kNndS + (part >> 1) * kNndS + s];
                if (f != ~0u) v = (f << 1) | (uint32_t)(part >> 1);
            } else {
                const int64_t a = p.rs[2 * i + (part >> 1)], b = p.rs[2 * i + (part >> 1) + 1];
                if (a + s < b) v = (p.rsrc[a + s] << 1) | (uint32_t)(part >> 1);
            }
        }
        s_raw[tid] = v;
    }
    __syncthreads();
    nnd_rank_sort(s_raw, kNndMaxC, s_sorted, nullptr);
    if (warp == 0) {
        int C = 0;
        for (int b = 0; b < kNndMaxC; b += kWarp) {
            const uint32_t v = s_sorted[b + lane];
            const bool ok = v != ~0u && (b + lane == 0 || (s_sorted[b + lane - 1] >> 1) != (v >> 1));
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            if (ok) {
                const int pos = C + __popc(bal & lt);
                s_id[pos] = v >> 1;
                s_new[pos] = (uint8_t)!(v & 1u);
            }
            C += __popc(bal);
        }
        if (lane == 0) s_ctl[0] = C;
    }
    __syncthreads();
    const int C = s_ctl[0];
    if (C < 2) return;
    for (int e = tid; e < C; e += kNndThreads) s_norm[e] = METRIC == KB2_METRIC_L2 ? p.norms[s_id[e]] : 0.f;
    __syncthreads();
    nnd_gram<METRIC>(p.x, p.d, s_id, s_norm, C, -1, s_x, s_key);

    for (int r = warp; r < C; r += kNndWarps) {
        const uint32_t u = s_id[r];
        const bool rnew = s_new[r] != 0;
        float* Lk = p.lkey + (int64_t)u * m;
        uint32_t* Li = p.lid + (int64_t)u * m;
        const float thr = __ldcg(Lk + m - 1);   // the live m-th key: it only improves, so worse proposals cannot enter
        int B = 0;
        for (int c0 = 0; c0 < C; c0 += kWarp) {
            const int c = c0 + lane;
            float k = 0.f;
            bool ok = c < C && c != r && (rnew || s_new[c]);
            if (ok) {
                k = s_key[r * kNndKld + c];
                ok = k <= thr;
            }
            const unsigned bal = __ballot_sync(0xffffffffu, ok);
            if (ok) {
                const int pos = B + __popc(bal & lt);
                wb_key[pos] = k;
                wb_id[pos] = s_id[c];
            }
            B += __popc(bal);
        }
        if (B == 0) continue;
        // bitonic sort of the batch by (key, id), padded to a power of two >= 32
        int len = kWarp;
        while (len < B) len <<= 1;
        for (int q = B + lane; q < len; q += kWarp) { wb_key[q] = INFINITY; wb_id[q] = kNndIdMask; }
        __syncwarp();
        for (int size = 2; size <= len; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int t = lane; t < (len >> 1); t += kWarp) {
                    const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                    const bool up = (lo & size) == 0;
                    const float ka = wb_key[lo], kb = wb_key[hi];
                    const uint32_t ia = wb_id[lo], ib = wb_id[hi];
                    if (cagra_less(kb, ib, ka, ia) == up) {
                        wb_key[lo] = kb; wb_id[lo] = ib;
                        wb_key[hi] = ka; wb_id[hi] = ia;
                    }
                }
                __syncwarp();
            }
        }
        if (lane == 0) nnd_lock(p.lock + u);
        __syncwarp();
        for (int q = lane; q < m; q += kWarp) {
            wl_key[q] = __ldcg(Lk + q);
            wl_id[q] = __ldcg(Li + q);
        }
        __syncwarp();
        // rank of each proposal in L[u]; drop those already present (same id means same key bits) or ranked past m
        int nb = 0;
        for (int b0 = 0; b0 < B; b0 += kWarp) {
            const int b = b0 + lane;
            float k = 0.f;
            uint32_t v = 0;
            int rk = m;
            bool keep = false;
            if (b < B) {
                k = wb_key[b];
                v = wb_id[b];
                rk = cagra_rank(wl_key, wl_id, m, k, v);
                keep = rk < m && !(wl_key[rk] == k && (wl_id[rk] & kNndIdMask) == v);
            }
            __syncwarp();
            const unsigned bal = __ballot_sync(0xffffffffu, keep);
            if (keep) {
                const int pos = nb + __popc(bal & lt);
                wb_key[pos] = k;
                wb_id[pos] = v;
                wr[pos] = rk;
            }
            nb += __popc(bal);
            __syncwarp();
        }
        if (nb > 0) {
            // merge: list entry q moves to q + #{proposals ranked <= q}; proposal b lands at wr[b] + b; past m drops out
            for (int q = wr[0] + lane; q < m; q += kWarp) {
                int lo = 0, hi = nb;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (wr[mid] <= q) lo = mid + 1; else hi = mid;
                }
                if (q + lo < m) {
                    __stcg(Lk + q + lo, wl_key[q]);
                    __stcg(Li + q + lo, wl_id[q]);
                }
            }
            for (int b = lane; b < nb; b += kWarp) {
                if (wr[b] + b < m) {
                    __stcg(Lk + wr[b] + b, wb_key[b]);
                    __stcg(Li + wr[b] + b, wb_id[b] | kNndNew);
                }
            }
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) atomicExch(p.lock + u, 0);
    }
}

// updates(t): the entries flagged new
__global__ void
cagra_nnd_count_kernel(const uint32_t* __restrict__ lid, int64_t total, unsigned long long* __restrict__ out) {
    unsigned c = 0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x)
        c += lid[e] >> 31;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

__global__ void
cagra_nnd_ids_kernel(const uint32_t* __restrict__ lid, int64_t total, int32_t* __restrict__ g0) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < total) g0[e] = (int32_t)(lid[e] & kNndIdMask);
}

// ============================================================================================ search
struct CagraSearchParams {
    HnswSearchParams s;    // vecs, d, n, neighbors (n x g), queries, nq, k, visited / log, work counter, outputs, bitset
    int g, itopk, width, max_iter, cand_cap;   // cand_cap: power of two >= width * g
    int64_t n_seeds;
};

__device__ __forceinline__ bool
cagra_less(float ka, uint32_t ia, float kb, uint32_t ib) {
    return ka < kb || (ka == kb && (ia & ~kExpanded) < (ib & ~kExpanded));
}

// bitonic sort of (key, id)[0, len), len a power of two; all threads; starts and ends at a barrier
__device__ __forceinline__ void
cagra_bitonic(float* key, uint32_t* id, int len) {
    for (int size = 2; size <= len; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < (len >> 1); t += blockDim.x) {
                const int lo = 2 * t - (t & (stride - 1));
                const int hi = lo + stride;
                const bool up = (lo & size) == 0;
                const float ka = key[lo], kb = key[hi];
                const uint32_t ia = id[lo], ib = id[hi];
                if (cagra_less(kb, ib, ka, ia) == up) {
                    key[lo] = kb; id[lo] = ib;
                    key[hi] = ka; id[hi] = ia;
                }
            }
            __syncthreads();
        }
    }
}

// entries of the sorted (key, id)[0, len) that come before (k, i)
__device__ __forceinline__ int
cagra_rank(const float* key, const uint32_t* id, int len, float k, uint32_t i) {
    int lo = 0, hi = len;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cagra_less(key[mid], id[mid], k, i)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// dynamic smem: 16 control ints | query (dpad floats) | T, T' (2 x itopk x 8) | candidates (cand_cap x 8) | parents
template <int METRIC>
__global__ void __launch_bounds__(kCagraThreads)
cagra_search_kernel(CagraSearchParams c) {
    const HnswSearchParams& p = c.s;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int dpad = (p.d + 3) & ~3;
    const int cap = c.itopk;
    int* s_ctl = (int*)smem_raw;
    float* s_q = (float*)(smem_raw + 64);
    float* t_key = s_q + dpad;
    uint32_t* t_id = (uint32_t*)(t_key + cap);
    float* u_key = (float*)(t_id + cap);
    uint32_t* u_id = (uint32_t*)(u_key + cap);
    float* c_key = (float*)(u_id + cap);
    uint32_t* c_id = (uint32_t*)(c_key + c.cand_cap);
    int32_t* s_par = (int32_t*)(c_id + c.cand_cap);

    uint32_t* vis = p.visited + (int64_t)blockIdx.x * p.nwords;
    int32_t* vlog = p.vis_log + (int64_t)blockIdx.x * p.log_cap;
    unsigned long long ndis_tot = 0, nhops_tot = 0;   // thread 0's are the CTA's

    for (;;) {
        if (tid == 0) s_ctl[0] = atomicAdd(p.next_query, 1);
        __syncthreads();
        const int q = s_ctl[0];
        if (q >= p.nq) break;
        for (int j = tid; j < p.d; j += kCagraThreads) s_q[j] = p.queries[(int64_t)q * p.d + j];
        if (tid == 0) s_ctl[1] = 0;
        __syncthreads();
        int size = 0, logn = 0;   // the same in every thread
        bool log_overflow = false;

        // Candidates c_id[0, nc) (ids the visited test-and-set found fresh): keys, sort, and T <- first cap of merge(T, C)
        auto absorb = [&]() {
            const int nc = s_ctl[1];
            __syncthreads();
            if (logn + nc > p.log_cap) log_overflow = true;
            logn += nc;
            if (tid == 0) { ndis_tot += nc; s_ctl[1] = 0; }
            if (nc == 0) return;
            const int per = (nc > 8 && (p.d & 3) == 0) ? 4 : 1;
            for (int g0 = warp * per; g0 < nc; g0 += (kCagraThreads / kWarp) * per) {
                if (per == 4 && g0 + 4 <= nc) {
                    float k0, k1, k2, k3;
                    hnsw_key4<METRIC>(p.vecs, p.d, s_q, (int32_t)c_id[g0], (int32_t)c_id[g0 + 1], (int32_t)c_id[g0 + 2],
                                      (int32_t)c_id[g0 + 3], lane, k0, k1, k2, k3);
                    if (lane == 0) { c_key[g0] = k0; c_key[g0 + 1] = k1; c_key[g0 + 2] = k2; c_key[g0 + 3] = k3; }
                } else {
                    for (int t = g0; t < min(g0 + per, nc); t++) {
                        const float kt = hnsw_key<METRIC>(p.vecs, p.d, s_q, (int32_t)c_id[t], lane);
                        if (lane == 0) c_key[t] = kt;
                    }
                }
            }
            int len = 32;
            while (len < nc) len <<= 1;
            for (int t = nc + tid; t < len; t += kCagraThreads) { c_key[t] = INFINITY; c_id[t] = 0x7fffffffu; }
            __syncthreads();
            cagra_bitonic(c_key, c_id, len);
            // merge path by ranks: (key, id) pairs are distinct (a row enters T at most once)
            for (int t = tid; t < size; t += kCagraThreads) {
                const int to = t + cagra_rank(c_key, c_id, nc, t_key[t], t_id[t]);
                if (to < cap) { u_key[to] = t_key[t]; u_id[to] = t_id[t]; }
            }
            for (int t = tid; t < nc; t += kCagraThreads) {
                const int to = t + cagra_rank(t_key, t_id, size, c_key[t], c_id[t]);
                if (to < cap) { u_key[to] = c_key[t]; u_id[to] = c_id[t]; }
            }
            __syncthreads();
            size = min(cap, size + nc);
            for (int t = tid; t < size; t += kCagraThreads) { t_key[t] = u_key[t]; t_id[t] = u_id[t]; }
            __syncthreads();
        };
        // visited test-and-set of row v; a fresh row is listed as a candidate and logged
        auto visit = [&](int32_t v) {
            const uint32_t bit = 1u << (v & 31);
            if (atomicOr(&vis[v >> 5], bit) & bit) return;
            const int t = atomicAdd(&s_ctl[1], 1);
            c_id[t] = (uint32_t)v;
            if (logn + t < p.log_cap) vlog[logn + t] = v;
        };

        // ---- seeds, cand_cap at a time
        for (int64_t j0 = 0; j0 < c.n_seeds; j0 += c.cand_cap) {
            const int64_t j1 = min(c.n_seeds, j0 + (int64_t)c.cand_cap);
            for (int64_t j = j0 + tid; j < j1; j += kCagraThreads) visit((int32_t)(cagra_seed((uint64_t)j) % (uint64_t)p.n));
            __syncthreads();
            absorb();
        }

        // ---- iterations
        for (int it = 0; c.max_iter == 0 || it < c.max_iter; it++) {
            if (warp == 0) {   // parents: the first <= width unexpanded entries of T, marked expanded
                int np = 0;
                for (int b = 0; b < size && np < c.width; b += kWarp) {
                    const int t = b + lane;
                    const bool un = t < size && !(t_id[t] & kExpanded);
                    const unsigned m = __ballot_sync(0xffffffffu, un);
                    const int r = np + __popc(m & ((1u << lane) - 1));
                    if (un && r < c.width) {
                        s_par[r] = (int32_t)t_id[t];
                        t_id[t] |= kExpanded;
                    }
                    np = min(c.width, np + __popc(m));
                }
                if (lane == 0) s_ctl[2] = np;
            }
            __syncthreads();
            const int np = s_ctl[2];
            if (np == 0) break;
            if (tid == 0) nhops_tot += np;
            for (int t = tid; t < np * c.g; t += kCagraThreads) {
                const int32_t v = p.neighbors[(int64_t)s_par[t / c.g] * c.g + t % c.g];
                if (v >= 0) visit(v);
            }
            __syncthreads();
            absorb();
        }

        // ---- result: the first k entries of T the bitset does not filter out
        if (warp == 0) {
            int cnt = 0;
            for (int b = 0; b < size && cnt < p.k; b += kWarp) {
                const int t = b + lane;
                const uint32_t v = t < size ? (t_id[t] & ~kExpanded) : 0u;
                const bool ok = t < size && !(p.bitset && bit_is_set(p.bitset, (int64_t)v));
                const unsigned m = __ballot_sync(0xffffffffu, ok);
                const int r = cnt + __popc(m & ((1u << lane) - 1));
                if (ok && r < p.k) {
                    p.out_ids[(int64_t)q * p.k + r] = (int64_t)v;
                    p.out_dist[(int64_t)q * p.k + r] = (METRIC == KB2_METRIC_L2) ? t_key[t] : -t_key[t];
                }
                cnt = min(p.k, cnt + __popc(m));
            }
            if (lane == 0) s_ctl[3] = cnt;
        }
        __syncthreads();
        for (int r = s_ctl[3] + tid; r < p.k; r += kCagraThreads) {
            p.out_ids[(int64_t)q * p.k + r] = -1;
            p.out_dist[(int64_t)q * p.k + r] = (METRIC == KB2_METRIC_L2) ? FLT_MAX : -FLT_MAX;
        }
        hnsw_clear_visited(p, vis, vlog, logn, log_overflow, tid, kCagraThreads);
        __syncthreads();
    }
    if (p.stats && tid == 0) {
        atomicAdd(&p.stats[0], ndis_tot);
        atomicAdd(&p.stats[1], nhops_tot);
    }
}

// ============================================================================================ host
struct CagraIndex : HnswIndex {
    int igd = 128, gd = 64;   // build keys (gpu_cuvs_cagra_config.h); the graph's degree is min(gd, igd, n - 1)
    bool nn_descent = false;  // build_algo NN_DESCENT: step 1 is the NN-descent graph, else the exact k-NN graph
    int nnd_niter = 20;       // nn_descent_niter: NN-descent's iteration cap
    std::vector<int64_t> nnd_updates;   // updates(t) of each NN-descent iteration of the last build
    float build_ms[3] = {0.f, 0.f, 0.f};   // k-NN graph, pruning, merge (CUDA events)

    int degree() const { return h_cum.size() >= 2 ? h_cum[1] : 0; }

    void
    add(const float* x, int64_t nadd, const int64_t* ids) override {
        KB2_REQUIRE(n == 0, KB2_NOT_IMPLEMENTED, "GPU_CAGRA implements no extend method: rows are added once, by the build");
        KB2_REQUIRE(ids == nullptr, KB2_NOT_IMPLEMENTED, "GPU_CAGRA: custom ids are not implemented");
        KB2_REQUIRE(shard_world == 1, KB2_NOT_IMPLEMENTED, "GPU_CAGRA: sharding is not implemented");
        KB2_REQUIRE(nadd > 0 && nadd < (1ll << 31), KB2_INVALID_ARGS, "bad row count");
        const int m = (int)std::min<int64_t>(igd, nadd - 1);
        const int g = std::min(gd, m);
        // the reverse-edge sort takes an int count of edges
        KB2_REQUIRE(nadd * g < (1ll << 31), KB2_INVALID_ARGS,
                    "GPU_CAGRA: rows x graph_degree must stay below 2^31 (" + std::to_string(nadd) + " x " + std::to_string(g) + ")");
        cudaStream_t st = stream;
        n = nadd;
        const int width = std::max(g, 1);   // n = 1: one empty slot (the HNSW layout needs a positive degree)
        h_vecs.resize((size_t)n * dim);
        KB2_CUDA_CHECK(cudaMemcpy(h_vecs.data(), x, h_vecs.size() * 4, cudaMemcpyDefault));
        d_vecs.alloc_exact(h_vecs.size());
        KB2_CUDA_CHECK(cudaMemcpyAsync(d_vecs.p, h_vecs.data(), h_vecs.size() * 4, cudaMemcpyHostToDevice, st));
        d_norms.alloc_exact((size_t)n);
        row_norms_kernel<<<grid1d(n * 32, 256), 256, 0, st>>>(d_vecs.p, n, dim, d_norms.p);
        h_neighbors.assign((size_t)n * width, -1);
        KB2_CUDA_CHECK(cudaEventRecord(ev0, st));
        if (g > 0) build_graph(m, g);
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        KB2_CUDA_CHECK(cudaGetLastError());
        h_levels.assign(n, 1);
        h_offsets.resize(n + 1);
        for (int64_t i = 0; i <= n; i++) h_offsets[i] = i * width;
        h_cum = {0, width};
        entry_point = 0;
        max_level = 0;
        M = std::max(1, width / 2);
        efConstruction = igd;
        validate_graph();
        uploaded = false;
    }

    void
    build_graph(int m, int g) {
        cudaStream_t st = stream;
        DevBuf<int32_t> g0, pruned, src, src_sorted, graph;
        DevBuf<int64_t> rstart;
        DevBuf<uint64_t> key, key_sorted;
        DevBuf<uint8_t> tmp;
        // 1. the intermediate graph
        g0.alloc_exact((size_t)n * m);
        knn_graph(m, g0.p, nullptr);
        KB2_CUDA_CHECK(cudaEventRecord(ev1, st));
        // 2-3. detour counts and the pruned rows
        pruned.alloc_exact((size_t)n * g);
        cagra_prune_kernel<<<(unsigned)n, kCagraPruneThreads, 0, st>>>(g0.p, n, m, g, pruned.p);
        KB2_CUDA_CHECK(cudaGetLastError());
        KB2_CUDA_CHECK(cudaEventRecord(ev2, st));
        g0.release();
        // 4. reverse edges: one radix sort of (target, slot) keys with the sources as values (stable: sources ascending)
        const int64_t ne = n * g;
        key.alloc_exact((size_t)ne);
        key_sorted.alloc_exact((size_t)ne);
        src.alloc_exact((size_t)ne);
        src_sorted.alloc_exact((size_t)ne);
        cagra_edge_keys_kernel<<<grid1d(ne, 256), 256, 0, st>>>(pruned.p, n, g, key.p, src.p);
        int vbits = 1;
        while ((1ll << vbits) < n) vbits++;
        size_t tb = 0;
        KB2_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, tb, key.p, key_sorted.p, src.p, src_sorted.p, (int)ne, 0, 8 + vbits, st));
        tmp.alloc_exact(tb);
        KB2_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, key.p, key_sorted.p, src.p, src_sorted.p, (int)ne, 0, 8 + vbits, st));
        rstart.alloc_exact((size_t)n + 1);
        cagra_reverse_offsets_kernel<<<grid1d(ne + 1, 256), 256, 0, st>>>(key_sorted.p, ne, n, rstart.p);
        // 5. final rows
        graph.alloc_exact((size_t)ne);
        cagra_merge_kernel<<<(unsigned)((n + kMergeWarps - 1) / kMergeWarps), kMergeWarps * kWarp, 0, st>>>(
            pruned.p, src_sorted.p, rstart.p, n, g, graph.p);
        KB2_CUDA_CHECK(cudaGetLastError());
        KB2_CUDA_CHECK(cudaEventRecord(ev3, st));
        KB2_CUDA_CHECK(cudaMemcpyAsync(h_neighbors.data(), graph.p, (size_t)ne * 4, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        KB2_CUDA_CHECK(cudaEventElapsedTime(&build_ms[0], ev0, ev1));
        KB2_CUDA_CHECK(cudaEventElapsedTime(&build_ms[1], ev1, ev2));
        KB2_CUDA_CHECK(cudaEventElapsedTime(&build_ms[2], ev2, ev3));
        last.launches = 0;
    }

    // Step 1 over the n rows of d_vecs: G0 (n x m int32, best first) and, if g0_key is given, its keys.  The exact k-NN
    // graph, or with build_algo NN_DESCENT the NN-descent graph (nnd_updates: updates(t) of each iteration run).
    void
    knn_graph(int m, int32_t* g0, float* g0_key) {
        nnd_updates.clear();
        if (nn_descent) {
            nnd_graph(m, g0, g0_key);
            return;
        }
        cudaStream_t st = stream;
        // a bounded batch of rows at a time (dense_knn's scratch grows with the batch)
        const int64_t chunk = std::min<int64_t>(n, 4096);
        DevBuf<int64_t> knn_ids;
        DevBuf<float> knn_dist;
        knn_ids.alloc_exact((size_t)chunk * (m + 1));
        knn_dist.alloc_exact((size_t)chunk * (m + 1));
        for (int64_t r0 = 0; r0 < n; r0 += chunk) {
            const int64_t rows = std::min(chunk, n - r0);
            dense_knn(*this, d_vecs.p + r0 * dim, rows, d_vecs.p, d_norms.p, n, dim, metric, m + 1, m + 17, nullptr, 0, nullptr,
                      knn_ids.p, knn_dist.p, true);
            cagra_drop_self_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(knn_ids.p, knn_dist.p, metric == KB2_METRIC_IP,
                                                                                rows, r0, m, g0, g0_key);
            KB2_CUDA_CHECK(cudaGetLastError());
        }
    }

    // NN-descent (definition at cagra_nnd_join_kernel).  Memory: the lists (8 B per entry), the forward samples and the
    // reverse-sample sort (2 x 64 entries of 12 B per row, double-buffered): O(n m).
    void
    nnd_graph(int m, int32_t* g0, float* g0_key) {
        cudaStream_t st = stream;
        const int S = std::min(kNndS, m);
        const int64_t nm = n * m, ne = n * 2 * kNndS;
        KB2_REQUIRE(ne < (1ll << 31), KB2_INVALID_ARGS,
                    "GPU_CAGRA NN_DESCENT: at most " + std::to_string((1ll << 31) / (2 * kNndS) - 1) + " rows");
        DevBuf<float> lkey;
        DevBuf<uint32_t> lid, fwd, rsrc[2];
        DevBuf<uint64_t> rkey[2];
        DevBuf<int64_t> rs;
        DevBuf<int> lock;
        DevBuf<uint8_t> tmp;
        DevBuf<unsigned long long> cnt;
        lkey.alloc_exact((size_t)nm);
        lid.alloc_exact((size_t)nm);
        fwd.alloc_exact((size_t)ne);
        for (int b = 0; b < 2; b++) {
            rkey[b].alloc_exact((size_t)ne);
            rsrc[b].alloc_exact((size_t)ne);
        }
        rs.alloc_exact((size_t)(2 * n + 1));
        lock.alloc_exact((size_t)n);
        cnt.alloc_exact(1);
        KB2_CUDA_CHECK(cudaMemsetAsync(lock.p, 0, (size_t)n * 4, st));
        int64_t stride = std::max<int64_t>(1, (n - 1) * 618 / 1000);
        while (std::gcd(stride, n - 1) != 1) stride++;
        const size_t smem_init = nnd_smem_common() + 8192;
        const size_t smem_join = nnd_smem_common() + (size_t)kNndWarps * nnd_join_warp_smem(m);
        with_metric(metric, [&](auto mt) {
            launch<cagra_nnd_init_kernel<decltype(mt)::value>>((unsigned)n, kNndThreads, smem_init, st, d_vecs.p, d_norms.p, n,
                                                               dim, m, stride, lkey.p, lid.p);
        });
        KB2_CUDA_CHECK(cudaGetLastError());
        int vbits = 1;
        while ((1ll << vbits) <= n) vbits++;   // 2^vbits > n: the ~0 keys of unused slots sort after every target
        cub::DoubleBuffer<uint64_t> dk(rkey[0].p, rkey[1].p);
        cub::DoubleBuffer<uint32_t> dv(rsrc[0].p, rsrc[1].p);
        size_t tb = 0;
        KB2_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)ne, 0, 33 + vbits, st));
        tmp.alloc_exact(tb);
        unsigned long long* hc = (unsigned long long*)h_counter.ensure(64);
        const unsigned rows_per_cta = 256 / kWarp;
        for (int t = 0; t < nnd_niter; t++) {
            dk.selector = 0;
            dv.selector = 0;
            cagra_nnd_sample_kernel<<<(unsigned)((n + rows_per_cta - 1) / rows_per_cta), 256, 0, st>>>(lid.p, n, m, S, t, fwd.p,
                                                                                                       rkey[0].p, rsrc[0].p);
            KB2_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, dk, dv, (int)ne, 0, 33 + vbits, st));
            cagra_nnd_offsets_kernel<<<grid1d(2 * n + 1, 256), 256, 0, st>>>(dk.Current(), ne, n, rs.p);
            NndJoinParams jp{d_vecs.p, d_norms.p, n, dim, m, S, fwd.p, dv.Current(), rs.p, lkey.p, lid.p, lock.p};
            with_metric(metric, [&](auto mt) {
                launch<cagra_nnd_join_kernel<decltype(mt)::value>>((unsigned)n, kNndThreads, smem_join, st, jp);
            });
            KB2_CUDA_CHECK(cudaGetLastError());
            KB2_CUDA_CHECK(cudaMemsetAsync(cnt.p, 0, 8, st));
            cagra_nnd_count_kernel<<<(unsigned)std::min<int64_t>((nm + 255) / 256, 4096), 256, 0, st>>>(lid.p, nm, cnt.p);
            KB2_CUDA_CHECK(cudaMemcpyAsync(hc, cnt.p, 8, cudaMemcpyDeviceToHost, st));
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
            nnd_updates.push_back((int64_t)hc[0]);
            if ((double)hc[0] <= kNndDelta * (double)n * (double)m) break;
        }
        cagra_nnd_ids_kernel<<<grid1d(nm, 256), 256, 0, st>>>(lid.p, nm, g0);
        KB2_CUDA_CHECK(cudaGetLastError());
        if (g0_key) KB2_CUDA_CHECK(cudaMemcpyAsync(g0_key, lkey.p, (size_t)nm * 4, cudaMemcpyDeviceToDevice, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
    }

    // shared memory of one cagra_search_kernel CTA (layout at the kernel)
    size_t
    search_smem(int itopk, int cand_cap, int width) const {
        const int dpad = (dim + 3) & ~3;
        return (size_t)round_up(64 + (int64_t)dpad * 4 + (int64_t)itopk * 16 + (int64_t)cand_cap * 8 + (int64_t)width * 4, 16);
    }

    void
    search(const float* q, int64_t nq, int k, const JsonObj& cfg, const uint8_t* bitset, int64_t nbits, int64_t* out_ids,
           float* out_dist) override {
        KB2_REQUIRE(n > 0, KB2_EMPTY_INDEX, "index is empty");
        KB2_REQUIRE(k > 0 && k <= kMaxLargeK, KB2_INVALID_ARGS, "k out of range (1..16384)");
        // gpu_cuvs_cagra_config.h: itopk_size (a multiple of 32), search_width, max_iterations, num_random_samplings
        int itopk = (int)cfg.get_int("itopk_size", std::max(k, 64));
        const int width = (int)cfg.get_int("search_width", std::max((k + 31) / 32, 1));
        const int max_iter = (int)cfg.get_int("max_iterations", 0);
        const int nrs = (int)cfg.get_int("num_random_samplings", 1);
        KB2_REQUIRE(itopk >= 1 && width >= 1 && max_iter >= 0 && nrs >= 1, KB2_OUT_OF_RANGE_IN_JSON,
                    "itopk_size, search_width and num_random_samplings must be positive, max_iterations >= 0");
        if (!cfg.has("itopk_size")) itopk = std::min(itopk, kCagraMaxItopk);
        itopk = (int)round_up(itopk, 32);
        KB2_REQUIRE(itopk <= kCagraMaxItopk, KB2_OUT_OF_RANGE_IN_JSON, "itopk_size out of range (at most 1024)");
        KB2_REQUIRE(std::max(itopk, 32 * width) >= k, KB2_OUT_OF_RANGE_IN_JSON, "max(itopk_size, 32 * search_width) must be >= k");
        const int g = degree();
        upload();
        cudaStream_t st = stream;
        const float* dq = to_device(q, (size_t)nq * dim, s_q);
        const uint8_t* dbits = bitset_to_device(bitset, nbits);
        int64_t* d_ids;
        float* d_dist;
        device_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        // HNSW's rule (IndexConditionalWrapper.cc:35-62): huge k or an almost-all-filtered bitset take the exact scan
        const int64_t n_filtered = count_filtered(dbits);
        const int64_t n_valid = n - n_filtered;
        bool bf = (double)k >= (double)n * 0.5;
        if (dbits) bf = bf || (double)n_filtered >= (double)n * 0.93 || (double)k >= (double)n_valid * 0.5;
        KB2_REQUIRE(bf || k <= kCagraMaxItopk, KB2_OUT_OF_RANGE_IN_JSON, "GPU_CAGRA: k above 1024 on the graph search");
        KB2_CUDA_CHECK(cudaMemsetAsync(d_counter.p, 0, 16, st));
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev0, st));
        if (bf) {
            brute_force(dq, nq, k, dbits, d_ids, d_dist);
        } else {
            KB2_REQUIRE((int64_t)width * g <= kCagraMaxCand, KB2_OUT_OF_RANGE_IN_JSON,
                        "search_width * graph_degree = " + std::to_string((int64_t)width * g) + " above " +
                            std::to_string(kCagraMaxCand) + " (the candidates of one iteration live in shared memory)");
            int cand_cap = 32;
            while (cand_cap < width * g) cand_cap <<= 1;
            const size_t smem = search_smem(itopk, cand_cap, width);
            KB2_REQUIRE(smem <= (size_t)kMaxDynSmem, KB2_OUT_OF_RANGE_IN_JSON, "GPU_CAGRA: dim too large for shared memory");
            // resident CTAs per SM from the registers and shared memory of the instance (the visited bitmaps are per CTA)
            int ctas_per_sm = 0;
            with_metric(metric, [&](auto m) {
                const void* fn = (const void*)cagra_search_kernel<decltype(m)::value>;
                KB2_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
                KB2_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, fn, kCagraThreads, smem));
            });
            ctas_per_sm = std::max(1, ctas_per_sm);
            Launch L;
            L.smem = smem;
            L.grid = (int)std::min<int64_t>(nq, (int64_t)num_sms() * ctas_per_sm);
            L.total_warps = L.grid;
            L.nwords = (n + 31) / 32;
            L.log_cap = (int)std::min<int64_t>(n, std::max<int64_t>(L.nwords, 1024));
            ensure_visited(L);
            KB2_CUDA_CHECK(cudaMemsetAsync(d_next.p, 0, 4, st));
            CagraSearchParams c{};
            c.s = base_params(dq, nq, itopk, k, L, dbits, n_filtered);
            c.s.labels = nullptr;
            c.s.out_ids = d_ids;
            c.s.out_dist = d_dist;
            c.g = g;
            c.itopk = itopk;
            c.width = width;
            c.max_iter = max_iter;
            c.cand_cap = cand_cap;
            c.n_seeds = std::min<int64_t>(n, std::max<int64_t>(1, (int64_t)nrs * width * g));
            with_metric(metric, [&](auto m) {
                launch<cagra_search_kernel<decltype(m)::value>>(L.grid, kCagraThreads, L.smem, st, c);
            });
            last.launches++;
            KB2_CUDA_CHECK(cudaGetLastError());
        }
        last_engine = 4;
        if (timing) KB2_CUDA_CHECK(cudaEventRecord(ev1, st));
        // rows with fewer than k results although more valid rows exist (k above itopk, or a filtered pool): exact scan
        if (!bf) {
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
                scatter_result_rows_kernel<<<grid1d(ns * k, 256), 256, 0, st>>>(s_bf_ids.p, s_bf_dist.p, s_short.p + 1, ns, k,
                                                                                 d_ids, d_dist);
                KB2_CUDA_CHECK(cudaGetLastError());
                last.flagged = ns;
            }
        }
        unsigned long long* hs = (unsigned long long*)h_counter.p;
        KB2_CUDA_CHECK(cudaMemcpyAsync(hs, d_counter.p, 16, cudaMemcpyDeviceToHost, st));
        results_out(nq, k, out_ids, out_dist, d_ids, d_dist);
        last_ndis = bf ? nq * n_valid : (int64_t)hs[0];
        last_nhops = bf ? 0 : (int64_t)hs[1];
        last.codes = last_ndis;
        last.code_bytes = last_ndis * (int64_t)dim * 4 + last_nhops * (int64_t)g * 4;
        last.pairs = last_nhops;
        if (timing) KB2_CUDA_CHECK(cudaEventElapsedTime(&last_kernel_ms, ev0, ev1));
    }

    // gpu_cuvs_cagra_config.h.  build_algo "NN_DESCENT" (any case) builds the intermediate graph by NN-descent with
    // nn_descent_niter (1..1000, default 20) as its iteration cap; any other build_algo, or none, builds the exact k-NN
    // graph.  build_algo is a build-time key and is not stored.  cache_dataset_on_device and adapt_for_cpu are accepted
    // and have no effect.
    void
    configure(const JsonObj& cfg) override {
        igd = (int)cfg.get_int("intermediate_graph_degree", 128);
        gd = (int)cfg.get_int("graph_degree", 64);
        KB2_REQUIRE(igd >= 1 && igd <= kCagraMaxIgd, KB2_OUT_OF_RANGE_IN_JSON, "intermediate_graph_degree out of range (1..1007)");
        KB2_REQUIRE(gd >= 1 && gd <= kCagraMaxGd && gd <= igd, KB2_OUT_OF_RANGE_IN_JSON,
                    "graph_degree out of range (1..256, and at most intermediate_graph_degree)");
        std::string algo = cfg.get_str("build_algo", "");
        for (char& c : algo) c = (char)toupper((unsigned char)c);
        nn_descent = algo == "NN_DESCENT";
        nnd_niter = (int)cfg.get_int("nn_descent_niter", 20);
        KB2_REQUIRE(!nn_descent || (nnd_niter >= 1 && nnd_niter <= 1000), KB2_OUT_OF_RANGE_IN_JSON,
                    "nn_descent_niter out of range (1..1000)");
    }

    void
    save(BlobWriter& w) override {
        w.put<int32_t>(igd);
        w.put<int32_t>(gd);
        HnswIndex::save(w);
    }
    void
    load(BlobReader& r) override {
        igd = r.get<int32_t>();
        gd = r.get<int32_t>();
        HnswIndex::load(r);
        KB2_REQUIRE(max_level == 0 && h_cum.size() == 2 && !labels.custom, KB2_INVALID_BINARY_SET, "GPU_CAGRA: bad graph in blob");
        for (int64_t i = 0; i < n; i++)
            KB2_REQUIRE(h_offsets[i] == i * h_cum[1], KB2_INVALID_BINARY_SET, "GPU_CAGRA: bad graph in blob");
    }

    // the graph as a one-level HNSW (what the reference's CPU HNSW node loads: build on the GPU, serve on the CPU)
    void
    to_faiss(FaissIndexData& o) override {
        o.kind = "HNSW";
        o.xb = h_vecs;
        o.levels = h_levels;
        o.neighbors = h_neighbors;
        o.offsets.assign(h_offsets.begin(), h_offsets.end());
        o.entry_point = entry_point;
        o.max_level = max_level;
        o.efConstruction = igd;
        o.cum = h_cum;
        o.assign_probas.assign(1, 1.0);
    }

    void
    append_meta(std::string& s) const override {
        s += ", \"intermediate_graph_degree\": " + std::to_string(igd) + ", \"graph_degree\": " + std::to_string(gd) +
             ", \"degree\": " + std::to_string(degree()) + ", \"build_ms\": [" + std::to_string(build_ms[0]) + ", " +
             std::to_string(build_ms[1]) + ", " + std::to_string(build_ms[2]) + "]";
    }

    void
    refuse(Op op) const override {
        KB2_REQUIRE(op != kShard, KB2_NOT_IMPLEMENTED, "GPU_CAGRA: sharding is not implemented");
        KB2_REQUIRE(op != kHnswImport, KB2_NOT_IMPLEMENTED, "GPU_CAGRA builds its own graph: import into an HNSW handle");
        KB2_REQUIRE(op != kRangeSearch, KB2_NOT_IMPLEMENTED, "RangeSearch is not implemented on GPU_CAGRA");
    }
    bool takes_emb_list() const override { return false; }
};

}  // namespace kb2
