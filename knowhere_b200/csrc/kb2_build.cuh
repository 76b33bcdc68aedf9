// kb2_build.cuh — device-side index construction: k-means, PQ training/encoding, list layout.
// (SURVEY §8f rank 3 — the step before the search path; kept on the GPU so that a 10M-row
//  Build() finishes in seconds.)  Hyper-parameters:
//   Clustering: niter=25, max_points_per_centroid=256, seed=1234, no renormalisation under IP.  These are faiss's
//               ClusteringParameters defaults (F/Clustering.h:22-80), not what the reference's IVF coarse quantizer
//               runs: Level1Quantizer sets niter=10 (F/IndexIVF.cpp:38-44) and IndexIVF sets spherical=true under
//               inner product (F/IndexIVF.cpp:178-181).  DESIGN §7 lists the difference.
//   PQ        : M independent k-means, ksub=256, <=256*ksub points  F/impl/ProductQuantizer.cpp:130-200
//   encoding  : residual to the assigned centroid, nearest sub-centroid per m (first minimum wins)
//                                                                  F/IndexIVFPQ.cpp:178-200, ProductQuantizer.cpp:220-260
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <random>
#include <vector>

#include "kb2_flat.cuh"
#include "kb2_gemm_tc.cuh"

namespace kb2 {

// keys[nq][ldk] <- contraction of Q[nq][d] with X[cols][d]; returns true if the tensor-core path ran.
// mode: 0 = fp32 CUDA-core contraction, 1 = wgmma (3xTF32) contraction where the shapes allow it.
inline bool
launch_gemm_keys(cudaStream_t st, int mode, int metric, const float* Q, const float* X, const float* qn,
                 const float* xn, int nq, int cols, int d, float* keys, int64_t ldk, const uint8_t* bitset,
                 const int32_t* rows, int64_t row_base) {
    if (mode == 1 && (ldk & 3) == 0) {
        CUtensorMap tq, tx;
        if (tc::make_tmap(&tq, Q, nq, d) && tc::make_tmap(&tx, X, cols, d)) {
            dim3 g((unsigned)((cols + tc::BN - 1) / tc::BN), (unsigned)((nq + tc::BM - 1) / tc::BM));
            with_metric(metric, [&](auto m) {
                constexpr int MM = decltype(m)::value;
                if (d <= tc::SHORT_K)
                    launch<tc::gemm_keys_tc_kernel<MM, 1>, (int)tc::smem_bytes(1)>(g, tc::THREADS, tc::smem_bytes(1), st, tq, tx, qn,
                                                                                   xn, nq, cols, d, keys, ldk, bitset, rows, row_base);
                else
                    launch<tc::gemm_keys_tc_kernel<MM, 3>, (int)tc::smem_bytes(3)>(g, tc::THREADS, tc::smem_bytes(3), st, tq, tx, qn,
                                                                                   xn, nq, cols, d, keys, ldk, bitset, rows, row_base);
            });
            return true;
        }
    }
    dim3 g((unsigned)((cols + GK_BN - 1) / GK_BN), (unsigned)((nq + GK_BM - 1) / GK_BM));
    with_metric(metric, [&](auto m) {
        gemm_keys_kernel<decltype(m)::value><<<g, 256, 0, st>>>(Q, X, qn, xn, nq, cols, d, keys, ldk, bitset, rows, row_base);
    });
    return false;
}



// ---------------------------------------------------------------- small kernels
__global__ void
iota_kernel(int32_t* out, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)i;
}
__global__ void
fill_i32_kernel(int32_t* out, int64_t n, int32_t v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = v;
}
// out[i][:] = x[idx[i]][:]   (warp per row)
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ x, const int32_t* __restrict__ idx, int64_t n, int d, int d_out,
                   float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const int32_t r = idx[i];
    for (int j = lane; j < d_out; j += kWarp) out[i * d_out + j] = (r >= 0 && j < d) ? x[(int64_t)r * d + j] : 0.f;
}
// sub-vector slice: out[i][0..dsub) = x[i][m*dsub .. ) - (cent ? cent[assign[i]][m*dsub..] : 0)
__global__ void
slice_residual_kernel(const float* __restrict__ x, const float* __restrict__ cent, const int32_t* __restrict__ assign,
                      int64_t n, int d, int m, int dsub, float* __restrict__ out) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * dsub) return;
    const int64_t i = t / dsub;
    const int j = (int)(t % dsub);
    float v = x[i * d + m * dsub + j];
    if (cent) v -= cent[(int64_t)assign[i] * d + m * dsub + j];
    out[t] = v;
}
// argmin over a row of keys (warp per row); first minimum wins like the reference's strict '<'
__global__ void __launch_bounds__(256)
argmin_rows_kernel(const float* __restrict__ keys, int64_t ldk, int64_t n, int k, int32_t* __restrict__ out,
                   float* __restrict__ out_val) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const float* row = keys + i * ldk;
    float best = INFINITY;
    int bj = 0x7fffffff;
    for (int j = lane; j < k; j += kWarp) {
        const float v = row[j];
        if (v < best) { best = v; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        if (ov < best || (ov == best && oj < bj)) { best = ov; bj = oj; }
    }
    if (lane == 0) {
        out[i] = (bj == 0x7fffffff) ? 0 : bj;
        if (out_val) out_val[i] = best;
    }
}
// Deterministic centroid update: the points are sorted by (centroid, index) beforehand; one warp per centroid sums its
// points in a fixed order (lane group g takes points g, g+groups, ...; groups are combined by a fixed shuffle tree), so two
// builds of the same data give bit-identical centroids (no float atomics).
__global__ void __launch_bounds__(256)
kmeans_reduce_kernel(const float* __restrict__ x, const int32_t* __restrict__ sorted_idx, const int32_t* __restrict__ seg_off,
                     const int32_t* __restrict__ counts, int k, int d, float* __restrict__ cent) {
    const int lane = threadIdx.x & 31;
    const int c = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (c >= k) return;
    const int cnt = counts[c];
    if (cnt <= 0) return;
    const int32_t* idx = sorted_idx + seg_off[c];
    int dp = 1;
    while (dp < d && dp < 32) dp <<= 1;          // lanes per point (power of two <= 32)
    const int groups = 32 / dp, g = lane / dp, jl = lane % dp;
    const float inv = 1.f / (float)cnt;
    for (int j0 = 0; j0 < d; j0 += dp) {
        const int j = j0 + jl;
        float acc = 0.f;
        if (j < d)
            for (int p = g; p < cnt; p += groups) acc += x[(int64_t)idx[p] * d + j];
        for (int o = dp; o < 32; o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (g == 0 && j < d) cent[(int64_t)c * d + j] = acc * inv;
    }
}
// sequentially applied (ci <- perturbed copy of cj) pairs; faiss split_clusters semantics
__global__ void
kmeans_split_kernel(float* cent, const int32_t* pairs, int npairs, int d) {
    const float eps = 1.f / 1024.f;
    for (int p = 0; p < npairs; p++) {
        const int ci = pairs[2 * p], cj = pairs[2 * p + 1];
        for (int j = threadIdx.x; j < d; j += blockDim.x) {
            const float v = cent[(int64_t)cj * d + j];
            if (j % 2 == 0) {
                cent[(int64_t)ci * d + j] = v * (1 + eps);
                cent[(int64_t)cj * d + j] = v * (1 - eps);
            } else {
                cent[(int64_t)ci * d + j] = v * (1 - eps);
                cent[(int64_t)cj * d + j] = v * (1 + eps);
            }
        }
        __syncthreads();
    }
}

// PQ encode: warp per vector.  codes_flat[i*M + m], residual against cent[assign[i]] when cent != NULL.
__global__ void __launch_bounds__(256)
pq_encode_kernel(const float* __restrict__ x, const float* __restrict__ cent, const int32_t* __restrict__ assign,
                 const float* __restrict__ pqc, int64_t n, int d, int M, int dsub, uint8_t* __restrict__ codes) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const float* xi = x + i * d;
    const float* ci = cent ? cent + (int64_t)assign[i] * d : nullptr;
    for (int m = 0; m < M; m++) {
        float best = INFINITY;
        int bj = 0;
        for (int j = lane; j < 256; j += kWarp) {  // ascending j per lane => first minimum kept
            const float* c = pqc + ((int64_t)m * 256 + j) * dsub;
            float acc = 0.f;
            for (int t = 0; t < dsub; t++) {
                float r = xi[m * dsub + t];
                if (ci) r -= ci[m * dsub + t];
                const float df = r - c[t];
                acc = fmaf(df, df, acc);
            }
            if (acc < best) { best = acc; bj = j; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (ov < best || (ov == best && oj < bj)) { best = ov; bj = oj; }
        }
        if (lane == 0) codes[i * M + m] = (uint8_t)bj;
    }
}

// t1[i] = sum_m ( |c_pq[m][code]|^2 + 2 <cent[assign[i]][m], c_pq[m][code]> )    (warp per vector)
// == sum over m of the reference's precomputed_table[list][m][code] (F/IndexIVFPQ.cpp:462-513)
__global__ void __launch_bounds__(256)
pq_t1_kernel(const uint8_t* __restrict__ codes, const float* __restrict__ cent, const int32_t* __restrict__ assign,
             const float* __restrict__ pqc, int64_t n, int d, int M, int dsub, float* __restrict__ t1) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const float* ci = cent + (int64_t)assign[i] * d;
    float acc = 0.f;
    for (int m = lane; m < M; m += kWarp) {
        const float* c = pqc + ((int64_t)m * 256 + codes[i * M + m]) * dsub;
        float nn = 0.f, ip = 0.f;
        for (int t = 0; t < dsub; t++) {
            nn = fmaf(c[t], c[t], nn);
            ip = fmaf(ci[m * dsub + t], c[t], ip);
        }
        acc += nn + 2.f * ip;
    }
    acc = warp_sum(acc);
    if (lane == 0) t1[i] = acc;
}

__global__ void
histogram_kernel(const int32_t* __restrict__ assign, int64_t n, int32_t* __restrict__ counts) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&counts[assign[i]], 1);
}
// r = rank in the (list, insertion)-sorted order; write rows[pos] for owned lists
__global__ void
place_rows_kernel(const int32_t* __restrict__ sorted_list, const int32_t* __restrict__ sorted_idx, int64_t n,
                  const int64_t* __restrict__ first_rank, const int64_t* __restrict__ list_off,
                  const int32_t* __restrict__ list_len, int32_t* __restrict__ rows, int32_t* __restrict__ pos_of_row) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int l = sorted_list[r];
    if (list_len[l] == 0) {
        if (pos_of_row) pos_of_row[sorted_idx[r]] = -1;
        return;
    }
    const int64_t pos = list_off[l] + (r - first_rank[l]);
    rows[pos] = sorted_idx[r];
    if (pos_of_row) pos_of_row[sorted_idx[r]] = (int32_t)pos;
}
// group-major rotated code layout (see kb2_ivf.cuh header)
__global__ void
layout_codes_kernel(const uint8_t* __restrict__ codes_flat, const int32_t* __restrict__ rows, int64_t npad, int M,
                    int G, uint8_t* __restrict__ out /* [G][npad][16] */) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= npad * G * 16) return;
    const int s = (int)(t & 15);
    const int64_t pos = (t >> 4) % npad;
    const int g = (int)((t >> 4) / npad);
    const int32_t r = rows[pos];
    uint8_t v = 0;
    if (r >= 0) v = codes_flat[(int64_t)r * M + g * 16 + ((s + (int)(pos & 15)) & 15)];
    out[t] = v;
}
__global__ void
layout_codes_plain_kernel(const uint8_t* __restrict__ codes_flat, const int32_t* __restrict__ rows, int64_t npad,
                          int M, uint8_t* __restrict__ out /* [npad][M] */) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= npad * M) return;
    const int64_t pos = t / M;
    const int m = (int)(t % M);
    const int32_t r = rows[pos];
    out[t] = (r >= 0) ? codes_flat[(int64_t)r * M + m] : 0;
}
// inverse of the two layout kernels: codes_flat[row*M + m] from the list-order layout (add() after a search)
__global__ void
unlayout_codes_kernel(const uint8_t* __restrict__ laid, const int32_t* __restrict__ pos_of_row, int64_t n, int64_t npad, int M,
                      int G, uint8_t* __restrict__ codes_flat) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * M) return;
    const int64_t r = t / M;
    const int m = (int)(t % M);
    const int64_t pos = pos_of_row[r];
    uint8_t v = 0;
    if (pos >= 0) {
        if (G > 0) {
            const int g = m >> 4, s = (m - (int)(pos & 15)) & 15;
            v = laid[((int64_t)g * npad + pos) * 16 + s];
        } else {
            v = laid[pos * M + m];
        }
    }
    codes_flat[t] = v;
}
__global__ void
gather_f32_kernel(const float* __restrict__ src, const int32_t* __restrict__ rows, int64_t npad, float* __restrict__ out,
                  float fill) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= npad) return;
    const int32_t r = rows[t];
    out[t] = (r >= 0) ? src[r] : fill;
}

// fp32 -> fp16 (kind 1) / bf16 (kind 2) and back: refine stores of refine_type fp16 / bf16
__global__ void
narrow_kernel(const float* __restrict__ x, int64_t n, int kind, uint16_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = (kind == 1) ? __half_as_ushort(__float2half_rn(x[i])) : __bfloat16_as_ushort(__float2bfloat16_rn(x[i]));
}
__global__ void
widen16_kernel(const uint16_t* __restrict__ x, int64_t n, int kind, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = (kind == 1) ? __half2float(__ushort_as_half(x[i])) : __uint_as_float((uint32_t)x[i] << 16);
}
// out[i] = x[i] / |x[i]|  (rows of norm 0 are copied unchanged), warp per row — COSINE support
__global__ void __launch_bounds__(256)
normalize_rows_kernel(const float* __restrict__ x, int64_t n, int d, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    float acc = 0.f;
    for (int j = lane; j < d; j += kWarp) acc = fmaf(x[i * d + j], x[i * d + j], acc);
    acc = warp_sum(acc);
    const float inv = acc > 0.f ? 1.0f / sqrtf(acc) : 1.0f;
    for (int j = lane; j < d; j += kWarp) out[i * d + j] = x[i * d + j] * inv;
}

// key = nearest list of each query (first entry of its probe row), value = query index
__global__ void
first_probe_kernel(const int64_t* __restrict__ probe_ids, int nprobe, int64_t nq, int32_t* __restrict__ key,
                   int32_t* __restrict__ idx) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const int64_t l = probe_ids[i * nprobe];
    key[i] = l < 0 ? 0 : (int32_t)l;
    idx[i] = (int32_t)i;
}

static inline dim3
grid1d(int64_t n, int block) {
    return dim3((unsigned)((n + block - 1) / block));
}

// ---------------------------------------------------------------- nearest-centroid assignment
// assign[i] = argmin_j key(x_i, c_j)   chunked so that the key matrix stays under ~256 MB
struct AssignScratch {
    DevBuf<float> keys, xn, cn;
};
inline void
assign_nearest(const float* x, int64_t n, int d, const float* cent, int k, int metric, int32_t* assign,
               float* out_val, AssignScratch& sc, cudaStream_t st) {
    if (n == 0) return;
    sc.cn.ensure(k);
    row_norms_kernel<<<grid1d((int64_t)k * 32, 256), 256, 0, st>>>(cent, k, d, sc.cn.p);
    int64_t chunk = std::max<int64_t>(128, std::min<int64_t>(n, (int64_t)(64ll << 20) / std::max(k, 1)));
    chunk = std::min<int64_t>(chunk, 1 << 20);
    // wide codebooks (IVF coarse quantizers): the wgmma 3xTF32 contraction (keys to ~5e-6 relative; the reference's own
    // add()/k-means assignment goes through BLAS sgemm, F/utils/distances.cpp:400-520).  Narrow ones (PQ sub-quantizers,
    // k = 256, d = 2..8) stay on the fp32 CUDA-core kernel.
    const int mode = (k >= 512 && (d & 3) == 0 && n >= 1024) ? 1 : 0;
    const int64_t ldk = (k + 3) & ~3;
    sc.keys.ensure((size_t)chunk * ldk);
    sc.xn.ensure((size_t)chunk);
    for (int64_t i0 = 0; i0 < n; i0 += chunk) {
        const int64_t m = std::min(chunk, n - i0);
        const float* xc = x + i0 * d;
        row_norms_kernel<<<grid1d(m * 32, 256), 256, 0, st>>>(xc, m, d, sc.xn.p);
        launch_gemm_keys(st, mode, metric, xc, cent, sc.xn.p, sc.cn.p, (int)m, k, d, sc.keys.p, ldk, nullptr, nullptr, 0);
        argmin_rows_kernel<<<grid1d(m * 32, 256), 256, 0, st>>>(sc.keys.p, ldk, m, k, assign + i0,
                                                               out_val ? out_val + i0 : nullptr);
    }
    KB2_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------- k-means (device data)
// x: [n][d] device.  centroids: [k][d] device (output).
inline void
kmeans_train(const float* x, int64_t n, int d, int k, int metric, int niter, uint64_t seed, float* centroids,
             cudaStream_t st) {
    KB2_REQUIRE(n >= k, KB2_INVALID_ARGS, "k-means: fewer training points than centroids");
    // subsample to <= 256 points per centroid (F/Clustering.cpp subsample_training_set)
    const int64_t max_pts = (int64_t)256 * k;
    DevBuf<float> sample;
    const float* xt = x;
    int64_t nt = n;
    std::mt19937_64 rng(seed);
    if (n > max_pts) {
        std::vector<int32_t> perm(n);
        for (int64_t i = 0; i < n; i++) perm[i] = (int32_t)i;
        for (int64_t i = 0; i < max_pts; i++) {
            int64_t j = i + (int64_t)(rng() % (uint64_t)(n - i));
            std::swap(perm[i], perm[j]);
        }
        perm.resize(max_pts);
        DevBuf<int32_t> didx;
        didx.ensure(max_pts);
        KB2_CUDA_CHECK(cudaMemcpyAsync(didx.p, perm.data(), max_pts * 4, cudaMemcpyHostToDevice, st));
        sample.ensure((size_t)max_pts * d);
        gather_rows_kernel<<<grid1d(max_pts * 32, 256), 256, 0, st>>>(x, didx.p, max_pts, d, d, sample.p);
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        xt = sample.p;
        nt = max_pts;
    }
    // init: k distinct random training points
    {
        std::vector<int32_t> perm(nt);
        for (int64_t i = 0; i < nt; i++) perm[i] = (int32_t)i;
        for (int64_t i = 0; i < k; i++) {
            int64_t j = i + (int64_t)(rng() % (uint64_t)(nt - i));
            std::swap(perm[i], perm[j]);
        }
        DevBuf<int32_t> didx;
        didx.ensure(k);
        KB2_CUDA_CHECK(cudaMemcpyAsync(didx.p, perm.data(), (size_t)k * 4, cudaMemcpyHostToDevice, st));
        gather_rows_kernel<<<grid1d((int64_t)k * 32, 256), 256, 0, st>>>(xt, didx.p, k, d, d, centroids);
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    DevBuf<int32_t> assign, counts, pairs, idx_in, idx_out, key_out, seg_off;
    DevBuf<uint8_t> sort_tmp;
    assign.ensure(nt);
    counts.ensure(k);
    idx_in.ensure(nt);
    idx_out.ensure(nt);
    key_out.ensure(nt);
    seg_off.ensure(k);
    iota_kernel<<<dim3((unsigned)((nt + 255) / 256)), 256, 0, st>>>(idx_in.p, nt);
    int end_bit = 1;
    while ((1ll << end_bit) < k) end_bit++;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, assign.p, key_out.p, idx_in.p, idx_out.p, (int)nt, 0, end_bit, st);
    sort_tmp.ensure(tmp_bytes);
    AssignScratch sc;
    std::vector<int32_t> hcounts(k), hoff(k);
    for (int it = 0; it < niter; it++) {
        assign_nearest(xt, nt, d, centroids, k, metric, assign.p, nullptr, sc, st);
        KB2_CUDA_CHECK(cudaMemsetAsync(counts.p, 0, (size_t)k * 4, st));
        histogram_kernel<<<dim3((unsigned)((nt + 255) / 256)), 256, 0, st>>>(assign.p, nt, counts.p);
        cub::DeviceRadixSort::SortPairs(sort_tmp.p, tmp_bytes, assign.p, key_out.p, idx_in.p, idx_out.p, (int)nt, 0, end_bit, st);
        KB2_CUDA_CHECK(cudaMemcpyAsync(hcounts.data(), counts.p, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        int32_t run = 0;
        for (int c = 0; c < k; c++) { hoff[c] = run; run += hcounts[c]; }
        KB2_CUDA_CHECK(cudaMemcpyAsync(seg_off.p, hoff.data(), (size_t)k * 4, cudaMemcpyHostToDevice, st));
        kmeans_reduce_kernel<<<dim3((unsigned)(((int64_t)k * 32 + 255) / 256)), 256, 0, st>>>(xt, idx_out.p, seg_off.p, counts.p, k, d,
                                                                                         centroids);
        KB2_CUDA_CHECK(cudaStreamSynchronize(st));   // hoff is reused next iteration
        // empty clusters: split a populated one (probability ~ size), like faiss split_clusters
        std::vector<int32_t> hp;
        for (int ci = 0; ci < k; ci++) {
            if (hcounts[ci] != 0) continue;
            if (nt <= k) break;
            int cj = 0;
            for (cj = 0;; cj = (cj + 1) % k) {
                const double pr = (hcounts[cj] - 1.0) / (double)(nt - k);
                const double r = (double)(rng() >> 11) * (1.0 / 9007199254740992.0);
                if (r < pr) break;
            }
            hp.push_back(ci);
            hp.push_back(cj);
            hcounts[ci] = hcounts[cj] / 2;
            hcounts[cj] -= hcounts[ci];
        }
        if (!hp.empty()) {
            pairs.ensure(hp.size());
            KB2_CUDA_CHECK(cudaMemcpyAsync(pairs.p, hp.data(), hp.size() * 4, cudaMemcpyHostToDevice, st));
            kmeans_split_kernel<<<1, 256, 0, st>>>(centroids, pairs.p, (int)(hp.size() / 2), d);
            KB2_CUDA_CHECK(cudaStreamSynchronize(st));
        }
    }
    KB2_CUDA_CHECK(cudaGetLastError());
}

}  // namespace kb2
