// kb2_flat.cuh — dense query x base contraction with fused key epilogue, and key selection.
//
// Replaces the reference's per-query sequential scans (one thread-pool task per query):
//   BruteForce  K/utils/distances.cpp:994 knn_L2sqr -> exhaustive_L2sqr_seq -> fvec_L2sqr_ny_if (:249-322)
//   FLAT index  F/IndexFlat.cpp:29-60 -> F/utils/distances.cpp:834-875, 326-363
//   IVF coarse  F/IndexIVF.cpp:336-342 (quantizer->search)
// with one batched contraction  keys[q][j] = |q|^2 + |x_j|^2 - 2 q.x_j  (L2) / -q.x_j (IP),
// a per-(query,slice) k-selection, and an exact fp32 re-rank of k' > k candidates in
// finalize_kernel so that returned distances are the directly accumulated sum((q-x)^2)
// (self-distance is exactly 0 like fvec_L2sqr, src/simd/distances_ref.cc:31-38).
//
// This file holds the fp32 CUDA-core contraction (bit-for-bit deterministic); the wgmma
// tensor-core contraction lives in kb2_gemm_tc.cuh and produces the same key matrix.
#pragma once
#include "kb2_topk.cuh"

namespace kb2 {

// ---------------------------------------------------------------- row squared norms (warp per row)
__global__ void __launch_bounds__(256)
row_norms_kernel(const float* __restrict__ x, int64_t n, int d, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    const float* r = x + row * d;
    float acc = 0.f;
    for (int j = lane; j < d; j += kWarp) acc = fmaf(r[j], r[j], acc);
    acc = warp_sum(acc);
    if (lane == 0) out[row] = acc;
}

// ---------------------------------------------------------------- fp32 SGEMM-style key kernel
// keys[q][j] for q in [0,nq), j in [0,nb): 128x128 CTA tile, 8x8 register micro-tile, BK=8.
// Q [nq][d], X [nb][d] row-major (both K-contiguous => "NT" GEMM).
constexpr int GK_BM = 128, GK_BN = 128, GK_BK = 8;

template <int METRIC>
__global__ void __launch_bounds__(256)
gemm_keys_kernel(const float* __restrict__ Q, const float* __restrict__ X, const float* __restrict__ qn,
                 const float* __restrict__ xn, int nq, int nb, int d, float* __restrict__ keys, int64_t ldk,
                 const uint8_t* __restrict__ bitset, const int32_t* __restrict__ rows, int64_t row_base) {
    __shared__ float As[2][GK_BK][GK_BM + 4];
    __shared__ float Bs[2][GK_BK][GK_BN + 4];

    const int tid = threadIdx.x;
    const int q0 = blockIdx.y * GK_BM;
    const int j0 = blockIdx.x * GK_BN;
    // loader mapping: 128 rows x 8 k-values = 256 float4 -> one float4 per thread per matrix
    const int lrow = tid >> 1;        // 0..127
    const int lk = (tid & 1) * 4;     // 0 or 4
    const int ty = tid >> 4;          // 0..15 -> 8 query rows each
    const int tx = tid & 15;          // 0..15 -> 8 base rows each

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = 0.f;

    const bool a_ok = (q0 + lrow) < nq;
    const bool b_ok = (j0 + lrow) < nb;
    const float* ap = Q + (int64_t)(q0 + lrow) * d + lk;
    const float* bp = X + (int64_t)(j0 + lrow) * d + lk;

    const bool vec4 = ((d & 3) == 0);
    auto load_tile = [&](int kt, float4& a, float4& b) {
        const int kk = kt * GK_BK + lk;
        a = make_float4(0.f, 0.f, 0.f, 0.f);
        b = a;
        if (vec4 && kk + 3 < d) {
            if (a_ok) a = *reinterpret_cast<const float4*>(ap + kt * GK_BK);
            if (b_ok) b = *reinterpret_cast<const float4*>(bp + kt * GK_BK);
        } else {
            float ta[4] = {0, 0, 0, 0}, tb[4] = {0, 0, 0, 0};
            for (int t = 0; t < 4; t++)
                if (kk + t < d) {
                    if (a_ok) ta[t] = ap[kt * GK_BK + t];
                    if (b_ok) tb[t] = bp[kt * GK_BK + t];
                }
            a = make_float4(ta[0], ta[1], ta[2], ta[3]);
            b = make_float4(tb[0], tb[1], tb[2], tb[3]);
        }
    };
    auto store_tile = [&](int buf, const float4& a, const float4& b) {
        As[buf][lk + 0][lrow] = a.x; As[buf][lk + 1][lrow] = a.y;
        As[buf][lk + 2][lrow] = a.z; As[buf][lk + 3][lrow] = a.w;
        Bs[buf][lk + 0][lrow] = b.x; Bs[buf][lk + 1][lrow] = b.y;
        Bs[buf][lk + 2][lrow] = b.z; Bs[buf][lk + 3][lrow] = b.w;
    };

    const int nkt = (d + GK_BK - 1) / GK_BK;
    float4 ra, rb;
    load_tile(0, ra, rb);
    store_tile(0, ra, rb);
    __syncthreads();
    for (int kt = 0; kt < nkt; kt++) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) load_tile(kt + 1, ra, rb);
#pragma unroll
        for (int kk = 0; kk < GK_BK; kk++) {
            float a[8], b[8];
            // rows {ty*4..+3} U {64+ty*4..+3}: a half-warp reads 16 consecutive float4 (no bank conflict)
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int j = 0; j < 8; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nkt) {
            store_tile(buf ^ 1, ra, rb);
            __syncthreads();
        }
    }

    // epilogue
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int q = q0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (q >= nq) continue;
        const float qq = (METRIC == KB2_METRIC_L2) ? qn[q] : 0.f;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int col = j0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (col >= nb) continue;
            float key;
            if (METRIC == KB2_METRIC_L2) {
                key = qq + xn[col] - 2.f * acc[i][j];
            } else {
                key = -acc[i][j];
            }
            if (bitset) {
                const int64_t row = rows ? (int64_t)rows[row_base + col] : (row_base + col);
                if (bit_is_set(bitset, row)) key = INFINITY;
            }
            keys[(int64_t)q * ldk + col] = key;
        }
    }
}

// ---------------------------------------------------------------- key selection
// grid (nq, nsplit): CTA (q, s) selects the K smallest keys of keys[q][c0..c1) and writes them
// sorted to partial[q][slot_base + s][0..kout).  Position written = pos_base + column.
__global__ void __launch_bounds__(kScanThreads)
select_keys_kernel(const float* __restrict__ keys, int64_t ldk, int ncols, int K, int kout,
                   uint64_t* __restrict__ partial, int slots_per_query, int slot_base, uint32_t pos_base) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* lists = (uint64_t*)smem_raw;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = blockIdx.x;
    const int nsplit = gridDim.y, s = blockIdx.y;
    const int per = (((ncols + nsplit - 1) / nsplit) + 31) / 32 * 32;
    const int c0 = s * per;
    const int c1 = min(ncols, c0 + per);

    WarpTopK tk;
    tk.init(lists + warp * 2 * K, K, lane);
    const float* row = keys + q * ldk;
    for (int base = c0 + warp * kWarp; base < c1; base += kScanWarps * kWarp) {
        const int c = base + lane;
        const bool valid = c < c1;
        const float key = valid ? row[c] : INFINITY;
        // +inf keys are filtered rows: never candidates
        tk.push(pack_kp(key, pos_base + (uint32_t)c), valid && key < INFINITY, lane);
    }
    uint64_t* out = partial + (q * slots_per_query + slot_base + s) * (int64_t)kout;
    tk.finish(lane);
    block_emit_topk(lists, K, out, kout);
}


// ---------------------------------------------------------------- wide key selection by value histogram
// Same contract as select_keys_kernel, for wide selections (IVF coarse: best nprobe+16 of nlist keys).
// One pass builds a 1024-bin histogram of the order-preserving integer image of the keys between the
// slice minimum and maximum; the largest bin prefix holding at most K_cap keys is emitted UNSORTED
// (finalize / reduce sort their input anyway).  It always contains the K_need smallest keys: if the
// prefix would hold fewer than K_need, the next bin is drained in (key, position) order (rare).
// grid (nq, nsplit), block 256, dynamic smem: slice*4 + 4160 bytes.
__global__ void __launch_bounds__(256)
select_keys_hist_kernel(const float* __restrict__ keys, int64_t ldk, int ncols, int K_need, int K_cap,
                        uint64_t* __restrict__ partial, int slots_per_query, int slot_base, uint32_t pos_base) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t* hist = (uint32_t*)smem_raw;          // 1024 bins (+1)
    uint32_t* ctl = hist + 1032;                   // [0] min [1] max [2] out cursor [3] bstar+1 [4] cum(bstar) [5] shift
    uint32_t* ord = ctl + 8;                       // slice
    const int64_t q = blockIdx.x;
    const int nsplit = gridDim.y, s = blockIdx.y;
    const int per = (((ncols + nsplit - 1) / nsplit) + 31) / 32 * 32;
    const int c0 = min(ncols, s * per);
    const int c1 = min(ncols, c0 + per);
    const int n = c1 - c0;
    const float* row = keys + q * ldk + c0;
    uint64_t* out = partial + (q * slots_per_query + slot_base + s) * (int64_t)K_cap;
    const uint32_t kInfOrd = f2ord(INFINITY);      // filtered entries: never emitted
    uint32_t lmin = 0xffffffffu, lmax = 0u;
    // 128-bit loads when the slice allows it (16 keys per thread at the IVF coarse stage: four LDG.128 in flight instead of
    // sixteen LDG.32); thread t then owns the keys {4t .. 4t+3} + 1024 j
    const bool vec = blockDim.x == 256 && (n & 3) == 0 && ((reinterpret_cast<uintptr_t>(row) & 15) == 0);
    if (vec) {
        const float4* row4 = reinterpret_cast<const float4*>(row);
        uint4* ord4 = reinterpret_cast<uint4*>(ord);
        for (int i = threadIdx.x; i < (n >> 2); i += 256) {
            const float4 f = __ldg(row4 + i);
            const uint4 v = make_uint4(f2ord(f.x), f2ord(f.y), f2ord(f.z), f2ord(f.w));
            ord4[i] = v;
            if (v.x < kInfOrd) { lmin = min(lmin, v.x); lmax = max(lmax, v.x); }
            if (v.y < kInfOrd) { lmin = min(lmin, v.y); lmax = max(lmax, v.y); }
            if (v.z < kInfOrd) { lmin = min(lmin, v.z); lmax = max(lmax, v.z); }
            if (v.w < kInfOrd) { lmin = min(lmin, v.w); lmax = max(lmax, v.w); }
        }
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t v = f2ord(row[i]);
            ord[i] = v;
            if (v < kInfOrd) { lmin = min(lmin, v); lmax = max(lmax, v); }
        }
    }
    // Fast path (the IVF coarse stage: best 80 of 4096 keys for each of 10^4 queries).  The keys a thread has just seen form
    // one of 256 disjoint "chunks" of the slice and `lmin` is that chunk's minimum; a value T with at least K_need chunk minima
    // <= T is an upper bound of the K_need-th smallest key (K_need distinct keys are <= T).  T is read off a 256-bin
    // histogram of the chunk minima (256 shared-memory atomics instead of one per key, 8 bins per lane to scan), then every
    // thread emits its keys <= T: about K_need * (1 + K_need / 256) entries.  If more than K_cap qualify (rare: K_cap is the
    // next power of two) the level-wise histogram below redoes the row, so the result is always a superset of the K_need best.
    const bool fast = blockDim.x == 256 && n >= 512 && 2 * K_need <= 256 && K_need <= K_cap;
    const uint32_t cmin = lmin;   // this thread's chunk minimum (0xffffffff: no finite key)
    uint32_t cmax = (cmin != 0xffffffffu) ? cmin : 0u;
    for (int i = threadIdx.x; i < 1032; i += blockDim.x) hist[i] = 0;
    if (threadIdx.x == 0) { ctl[0] = 0xffffffffu; ctl[1] = 0; ctl[2] = 0; ctl[7] = 0; }
    __syncthreads();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lmin = min(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
        lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        cmax = max(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
    }
    if ((threadIdx.x & 31) == 0) { atomicMin(&ctl[0], lmin); atomicMax(&ctl[1], lmax); atomicMax(&ctl[7], cmax); }
    __syncthreads();
    const uint32_t vmin = ctl[0], vmax = ctl[1];
    if (vmin > vmax || n <= K_cap) {
        // nothing selectable, or the whole slice fits: emit every finite key
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            if (ord[i] < kInfOrd) out[atomicAdd(&ctl[2], 1u)] = ((uint64_t)ord[i] << 32) | (pos_base + (uint32_t)(c0 + i));
        __syncthreads();
        for (int i = ctl[2] + threadIdx.x; i < K_cap; i += blockDim.x) out[i] = kEmpty;
        return;
    }
    if (fast) {
        // vmin is the smallest chunk minimum, ctl[7] the largest finite one
        const uint32_t ctop = ctl[7];
        const uint32_t cspan = ctop - vmin;
        const int cshift = cspan < 256u ? 0 : (32 - __clz(cspan)) - 8;   // (cspan >> cshift) <= 255
        if (cmin != 0xffffffffu) atomicAdd(&hist[(cmin - vmin) >> cshift], 1u);
        __syncthreads();
        if (threadIdx.x < 32) {
            const int lane = threadIdx.x;
            uint32_t h[8], sum = 0;
#pragma unroll
            for (int t = 0; t < 8; t++) { h[t] = hist[lane * 8 + t]; sum += h[t]; }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const uint32_t excl = incl - sum;
            const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
            if (lane == 0 && total < (uint32_t)K_need) ctl[6] = 0xffffffffu;   // not enough finite chunks: histogram path
            if (excl < (uint32_t)K_need && incl >= (uint32_t)K_need) {      // exactly one lane when total >= K_need
                uint32_t run = excl;
                int b = lane * 8 + 7;
#pragma unroll
                for (int t = 0; t < 8; t++) {
                    run += h[t];
                    if (run >= (uint32_t)K_need) { b = lane * 8 + t; break; }
                }
                // upper edge of bin b, never above the largest chunk minimum
                const unsigned long long edge = (unsigned long long)vmin + (((unsigned long long)(b + 1)) << cshift) - 1ull;
                ctl[6] = (uint32_t)min(edge, (unsigned long long)ctop);
            }
        }
        __syncthreads();
        const uint32_t T = ctl[6];
        bool done = false;
        if (T < kInfOrd) {   // CTA-uniform
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const uint32_t v = ord[i];
                if (v <= T) {
                    const uint32_t slot = atomicAdd(&ctl[2], 1u);
                    if (slot < (uint32_t)K_cap) out[slot] = ((uint64_t)v << 32) | (pos_base + (uint32_t)(c0 + i));
                }
            }
            __syncthreads();
            done = ctl[2] <= (uint32_t)K_cap;
        }
        if (done) {
            for (int i = ctl[2] + threadIdx.x; i < K_cap; i += blockDim.x) out[i] = kEmpty;
            return;
        }
        __syncthreads();   // everybody has read the counter
        if (threadIdx.x == 0) ctl[2] = 0;
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
    }
    // Level-wise refinement: histogram the keys of the current value range into <= 1024 bins, emit the largest bin prefix
    // that still fits, and if that prefix holds fewer than the keys still needed descend into the crossing bin (its range
    // is 2^shift values: at most 4 levels for 32-bit keys).  Key distributions with outliers (inner products: a few huge
    // values stretch the range so that most keys share one bin) therefore cost one more pass, not a serial drain.
    uint32_t base = vmin, span = vmax - vmin;   // current range [base, base + span]
    uint32_t need = (uint32_t)K_need, cap = (uint32_t)K_cap;
    for (int level = 0; level < 5; level++) {
        const int shift = span < 1024u ? 0 : (32 - __clz(span)) - 10;
        const int nbins = (int)(span >> shift) + 1;   // <= 1024
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t v = ord[i];
            if (v < kInfOrd && v >= base && v - base <= span) atomicAdd(&hist[(v - base) >> shift], 1u);
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            // warp 0: scan 32 bins per lane, find the largest prefix with cumulative count <= cap
            const int lane = threadIdx.x;
            uint32_t sum = 0;
            for (int t = 0; t < 32; t++) sum += hist[lane * 32 + t];
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const uint32_t excl = incl - sum;
            // lane owning the crossing: excl <= cap < incl ; if total <= cap no lane crosses
            const bool crosses = excl <= cap && incl > cap;
            const unsigned who = __ballot_sync(0xffffffffu, crosses);
            const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
            if (who == 0 && lane == 0) { ctl[3] = (uint32_t)nbins; ctl[4] = total; }
            if (crosses) {
                uint32_t run = excl;
                int b = lane * 32;
                for (int t = 0; t < 32; t++) {
                    const uint32_t h = hist[lane * 32 + t];
                    if (run + h > cap) { b = lane * 32 + t; break; }
                    run += h;
                }
                ctl[3] = (uint32_t)b;   // bins [0, b) are taken: cum = run <= cap
                ctl[4] = run;
            }
        }
        __syncthreads();
        const uint32_t btake = ctl[3];
        const uint32_t taken = ctl[4];
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const uint32_t v = ord[i];
            if (v < kInfOrd && v >= base && v - base <= span && ((v - base) >> shift) < btake)
                out[atomicAdd(&ctl[2], 1u)] = ((uint64_t)v << 32) | (pos_base + (uint32_t)(c0 + i));
        }
        __syncthreads();
        if (taken >= need || btake >= (uint32_t)nbins) break;   // enough emitted, or nothing left in this range (CTA-uniform)
        for (int i = threadIdx.x; i < 1032; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        need -= taken;
        cap -= taken;
        if (shift == 0) {
            // the crossing bin is a single key value held by more entries than fit: any `need` of them complete the
            // selection (equal keys); take them in position order
            if (threadIdx.x == 0) {
                const uint32_t v0 = base + btake;
                uint32_t slot = ctl[2];
                for (int i = 0; i < n && need > 0; i++)
                    if (ord[i] == v0) { out[slot++] = ((uint64_t)v0 << 32) | (pos_base + (uint32_t)(c0 + i)); need--; }
                ctl[2] = slot;
            }
            break;
        }
        base += btake << shift;
        span = (1u << shift) - 1u;
    }
    __syncthreads();
    for (int i = ctl[2] + threadIdx.x; i < K_cap; i += blockDim.x) out[i] = kEmpty;
}

// ---------------------------------------------------------------- exact scan of the queries finalize could not certify
// grid (count, nsplit): CTA (i, s) scans row slice s (multiples of 32 rows) of query qlist[i] with the directly accumulated
// sum((q-x)^2) / sum(q*x) -- no norm expansion, so nothing cancels -- and writes its best K keys, sorted, to
// partial[q][s][0..K).  Position = row.  dynamic smem: kScanWarps * 2K entries | query
template <int METRIC>
__global__ void __launch_bounds__(kScanThreads)
flat_exact_scan_kernel(const float* __restrict__ Q, const float* __restrict__ X, int64_t n, int d,
                       const uint8_t* __restrict__ bitset, int64_t bit_base, const uint32_t* __restrict__ qlist, int K,
                       uint64_t* __restrict__ partial) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* lists = (uint64_t*)smem_raw;
    float* s_q = (float*)(lists + kScanWarps * 2 * K);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q = qlist[blockIdx.x];
    const int nsplit = gridDim.y, s = blockIdx.y;
    const int64_t per = ((n + nsplit - 1) / nsplit + 31) / 32 * 32;
    const int64_t r0 = min(n, (int64_t)s * per), r1 = min(n, r0 + per);
    for (int j = threadIdx.x; j < d; j += blockDim.x) s_q[j] = Q[q * d + j];
    WarpTopK tk;
    tk.init(lists + warp * 2 * K, K, lane);
    __syncthreads();
    for (int64_t base = r0 + warp * kWarp; base < r1; base += kScanWarps * kWarp) {
        const int nrows = (int)min((int64_t)kWarp, r1 - base);
        float mykey = INFINITY;
        for (int r = 0; r < nrows; r++) {
            const float* x = X + (base + r) * d;
            float acc = 0.f;
            for (int j = lane; j < d; j += kWarp) {
                if (METRIC == KB2_METRIC_L2) {
                    const float t = s_q[j] - x[j];
                    acc = fmaf(t, t, acc);
                } else {
                    acc = fmaf(s_q[j], x[j], acc);
                }
            }
            acc = warp_sum(acc);
            if (lane == r) mykey = (METRIC == KB2_METRIC_L2) ? acc : -acc;
        }
        bool valid = lane < nrows;
        if (valid && bitset) valid = !bit_is_set(bitset, bit_base + base + lane);
        tk.push(pack_kp(mykey, (uint32_t)(base + lane)), valid, lane);
    }
    uint64_t* out = partial + (q * nsplit + s) * (int64_t)K;
    tk.finish(lane);
    block_emit_topk(lists, K, out, K);
}

}  // namespace kb2
