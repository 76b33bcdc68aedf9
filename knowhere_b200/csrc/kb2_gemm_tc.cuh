// kb2_gemm_tc.cuh — the dense query x base contraction on the Hopper tensor cores (wgmma).
//
//   keys[q][j] = |q|^2 + |x_j|^2 - 2 <q, x_j>   (L2)        keys[q][j] = -<q, x_j>   (IP)
//
// Same contract and output as gemm_keys_kernel (kb2_flat.cuh), which stays as the bit-reproducible
// fp32 reference / fallback (d % 4 != 0).  Used by FLAT, BruteForce and the IVF coarse quantizer
// (reference: F/utils/distances.cpp:326-363,834-875; F/IndexIVF.cpp:336-342).
//
// sm_90a mapping
//   * operands: fp32 rows, K-major.  TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B) brings 128 x 32-float
//     boxes (one 128-byte swizzle row per tensor row) of Q and X into a shared-memory ring; warp 8 is the producer.
//   * fp32 fidelity on a tf32 pipe: the two consumer warpgroups split every element into hi = top 19 bits and
//     lo = x - hi (both rounded to tf32), writing hi in place and lo to a twin tile, then issue
//     D += hi*hi + hi*lo + lo*hi  (3 x wgmma m64n128k8 tf32 per k-step, warpgroup w owns rows 64w..64w+63) — error
//     ~2^-21 relative, and the k+16 best candidates are re-ranked exactly afterwards anyway (finalize_kernel).
//   * accumulator: 64 fp32 registers per thread; the split of stage i+1 runs while the wgmmas of stage i are in flight
//     (wgmma.wait_group 1), then the same threads apply the key epilogue (+norms, bitset) straight from registers.
//   * one 128x128 output tile per CTA (K = d is short: 4 k-blocks at d=128, so the kernel is bound by
//     operand/epilogue traffic, not by the tensor pipe).
#pragma once
#include <cuda.h>

#include "kb2_common.cuh"

namespace kb2 {
namespace tc {

constexpr int BM = 128, BN = 128, BK = 32;
constexpr int STAGES = 3;                      // ring depth of the long-K instantiation (1 CTA/SM)
constexpr int TILE_BYTES = 128 * BK * 4;       // 16 KB: a 128-row x 128-byte tile (A or B)
constexpr int STAGE_BYTES = 4 * TILE_BYTES;    // A_hi | B_hi | A_lo | B_lo
constexpr int THREADS = 288;                   // warps 0-7: two consumer warpgroups (split + wgmma + epilogue)   warp 8: TMA
constexpr int CONS_THREADS = 256;
constexpr int PRODUCER_WARP = 8;
constexpr size_t smem_bytes(int nst) { return (size_t)nst * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/; }
constexpr size_t SMEM_BYTES = smem_bytes(STAGES);
// Short contractions (d <= 192: the IVF coarse quantizer, k-means assignment) run a single-stage instantiation with two
// CTAs per SM instead: a 128x128 tile is then a strictly serial TMA -> split -> MMA -> store chain, and a second resident
// CTA overlaps its epilogue store with the other's loads.
constexpr int SHORT_K = 192;                   // largest d served by the single-stage instantiation

__device__ __forceinline__ uint32_t
smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void
mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void
mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void
mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool
mbar_try(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t"
        "}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait (~3 s of SM clocks): a protocol bug must end the launch with an error, never hang the GPU
__device__ __forceinline__ void
mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try(bar, parity)) {
        if (clock64() - t0 > 6000000000ll) __trap();
    }
}
__device__ __forceinline__ void
tma_load_2d(uint32_t dst, const CUtensorMap* tmap, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
        "l"(tmap), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void
fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// ---------------------------------------------------------------- wgmma (sm_90a)
__device__ __forceinline__ void
wgmma_fence() {
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void
wgmma_commit() {
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void
wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of a wgmma accumulator across wgmma issue / wait (the registers are written
// asynchronously between the two)
template <int N>
__device__ __forceinline__ void
fence_operand(float (&acc)[N]) {
#pragma unroll
    for (int i = 0; i < N; i++) asm volatile("" : "+f"(acc[i])::"memory");
}
// wgmma shared-memory descriptor: K-major, SWIZZLE_128B, 8-row groups 1024 B apart (tile base 1024-byte aligned; a K step
// inside the 128-byte swizzle row advances the start address)
__device__ __forceinline__ uint64_t
make_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);   // start address, 16-byte units        bits  0-13
    d |= (uint64_t)1 << 16;                         // leading byte offset (unused here)   bits 16-29
    d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset = 1024 B         bits 32-45
    d |= (uint64_t)1 << 62;                         // layout type SWIZZLE_128B            bits 62-63
    return d;
}
// D (+)= A * B, one warpgroup, A = 64 rows, B = N rows, both K-major in shared memory; D in registers (fragment layout:
// d[4 j + 2 i + c] = row 16 (warp % 4) + lane / 4 + 8 i, column 8 j + 2 (lane % 4) + c)
__device__ __forceinline__ void
wgmma_tf32_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void
wgmma_tf32_n32(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}
// D (+)= A * B with bf16 operands, A = 64 rows, B = N = 16 .. 128 rows (multiple of 16); D in the first N / 2 registers
// of d, in the fragment layout of wgmma_tf32_n128
#define KB2_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define KB2_ACC8 KB2_D8(0)
#define KB2_ACC16 KB2_ACC8, KB2_D8(8)
#define KB2_ACC24 KB2_ACC16, KB2_D8(16)
#define KB2_ACC32 KB2_ACC24, KB2_D8(24)
#define KB2_ACC40 KB2_ACC32, KB2_D8(32)
#define KB2_ACC48 KB2_ACC40, KB2_D8(40)
#define KB2_ACC56 KB2_ACC48, KB2_D8(48)
#define KB2_ACC64 KB2_ACC56, KB2_D8(56)
template <int N, int R>
__device__ __forceinline__ void
wgmma_bf16(float (&d)[R], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    static_assert(N % 16 == 0 && N >= 16 && N <= 128 && N / 2 <= R, "wgmma_bf16: N = 16 .. 128 in steps of 16");
    if constexpr (N == 16) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC8 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
    else if constexpr (N == 32) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC16 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
    else if constexpr (N == 48) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC24 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
    else if constexpr (N == 64) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC32 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
    else if constexpr (N == 80) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC40 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
    else if constexpr (N == 96) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC48 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
    else if constexpr (N == 112) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}, %56, %57, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC56 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
    else if constexpr (N == 128) asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : KB2_ACC64 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}
#undef KB2_ACC8
#undef KB2_ACC16
#undef KB2_ACC24
#undef KB2_ACC32
#undef KB2_ACC40
#undef KB2_ACC48
#undef KB2_ACC56
#undef KB2_ACC64
#undef KB2_D8
// round-to-nearest into the 19-bit tf32 container (low 13 mantissa bits cleared)
__device__ __forceinline__ float
tf32_rn(float x) {
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}

template <int METRIC, int STAGES = 3>
__global__ void __launch_bounds__(THREADS, STAGES == 1 ? 2 : 1)
gemm_keys_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_x,
                    const float* __restrict__ qn, const float* __restrict__ xn, int nq, int nb, int d,
                    float* __restrict__ keys, int64_t ldk, const uint8_t* __restrict__ bitset,
                    const int32_t* __restrict__ rows, int64_t row_base) {
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t raw = smem_u32(smem_dyn);
    const uint32_t base = (raw + 1023u) & ~1023u;          // SWIZZLE_128B tiles need 1024-byte alignment
    unsigned char* base_ptr = smem_dyn + (base - raw);
    const uint32_t bars = base + STAGES * STAGE_BYTES;      // barrier block after the ring
    // barrier layout (8 bytes each): full[S] | empty[S]
    auto bar_full = [&](int s) { return bars + 8u * s; };
    auto bar_empty = [&](int s) { return bars + 8u * (STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.y * BM;
    const int j0 = blockIdx.x * BN;
    const int nkb = (d + BK - 1) / BK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) {
            mbar_init(bar_full(s), 1);
            mbar_init(bar_empty(s), CONS_THREADS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        // ================= TMA producer =================
        if (lane == 0) {
            for (int it = 0; it < nkb; it++) {
                const int s = it % STAGES;
                const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
                mbar_wait(bar_empty(s), ph ^ 1u);
                const uint32_t st = base + (uint32_t)s * STAGE_BYTES;
                mbar_expect_tx(bar_full(s), 2 * TILE_BYTES);
                tma_load_2d(st, &tmap_q, it * BK, q0, bar_full(s));                  // A_hi slot (raw fp32)
                tma_load_2d(st + TILE_BYTES, &tmap_x, it * BK, j0, bar_full(s));     // B_hi slot (raw fp32)
            }
        }
        return;
    }
    // ================= consumers: hi/lo split, wgmma, epilogue =================
    const int t = threadIdx.x;           // 0..255
    const int wg = t >> 7;               // warpgroup: rows 64 wg .. 64 wg + 63 of the tile
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0.f;
    for (int it = 0; it < nkb; it++) {
        const int s = it % STAGES;
        const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
        mbar_wait(bar_full(s), ph);
        float4* hi = reinterpret_cast<float4*>(base_ptr + (size_t)s * STAGE_BYTES);        // A_hi|B_hi contiguous
        float4* lo = reinterpret_cast<float4*>(base_ptr + (size_t)s * STAGE_BYTES + 2 * TILE_BYTES);
#pragma unroll 4
        for (int i = t; i < 2 * TILE_BYTES / 16; i += CONS_THREADS) {
            float4 v = hi[i];
            float4 h, l;
            // hi = x rounded to tf32 (nearest), lo = (x - hi) rounded to tf32: both exactly representable,
            // so the tensor core's own truncation of the low 13 bits changes nothing
            h.x = tf32_rn(v.x); l.x = tf32_rn(v.x - h.x);
            h.y = tf32_rn(v.y); l.y = tf32_rn(v.y - h.y);
            h.z = tf32_rn(v.z); l.z = tf32_rn(v.z - h.z);
            h.w = tf32_rn(v.w); l.w = tf32_rn(v.w - h.w);
            hi[i] = h;
            lo[i] = l;
        }
        fence_proxy_async();            // generic-proxy writes -> visible to the tensor core (async proxy)
        asm volatile("bar.sync 1, 256;" ::: "memory");   // both halves of the stage are split
        const uint32_t st = base + (uint32_t)s * STAGE_BYTES;
        const uint32_t a_off = (uint32_t)wg * 64u * 128u;
        fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / 8; kk++) {
            const uint32_t ko = (uint32_t)kk * 32u;   // 8 tf32 = 32 bytes inside the 128-byte swizzle row
            const uint64_t a_hi = make_desc(st + a_off + ko);
            const uint64_t b_hi = make_desc(st + TILE_BYTES + ko);
            const uint64_t a_lo = make_desc(st + 2 * TILE_BYTES + a_off + ko);
            const uint64_t b_lo = make_desc(st + 3 * TILE_BYTES + ko);
            wgmma_tf32_n128(acc, a_hi, b_hi, (it > 0 || kk > 0) ? 1u : 0u);
            wgmma_tf32_n128(acc, a_hi, b_lo, 1u);
            wgmma_tf32_n128(acc, a_lo, b_hi, 1u);
        }
        wgmma_commit();
        fence_operand(acc);
        if constexpr (STAGES == 1) {
            wgmma_wait<0>();
            mbar_arrive(bar_empty(s));
        } else {
            // the previous stage's wgmmas have retired once at most one group is pending: release its slot
            wgmma_wait<1>();
            if (it > 0) mbar_arrive(bar_empty((it - 1) % STAGES));
        }
    }
    wgmma_wait<0>();
    fence_operand(acc);
    // ---- epilogue: registers -> keys
    const int r0 = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int row = r0 + 8 * i;
        if (row >= nq) continue;
        const float qq = (METRIC == KB2_METRIC_L2) ? qn[row] : 0.f;
        float* out = keys + (int64_t)row * ldk;
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
            const int col0 = j0 + j * 8 + 2 * (lane & 3);
            float o[2];
#pragma unroll
            for (int c = 0; c < 2; c++) {
                const int col = col0 + c;
                const float a = acc[4 * j + 2 * i + c];
                float key = INFINITY;
                if (col < nb) {
                    key = (METRIC == KB2_METRIC_L2) ? (qq + xn[col] - 2.f * a) : -a;
                    if (bitset) {
                        const int64_t rr = rows ? (int64_t)rows[row_base + col] : (row_base + col);
                        if (bit_is_set(bitset, rr)) key = INFINITY;
                    }
                }
                o[c] = key;
            }
            if (col0 + 1 < ldk && (ldk & 1) == 0) {
                *reinterpret_cast<float2*>(out + col0) = make_float2(o[0], o[1]);
            } else {
                for (int c = 0; c < 2; c++)
                    if (col0 + c < ldk) out[col0 + c] = o[c];
            }
        }
    }
}

// ---------------------------------------------------------------- host side: tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled
get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
        cudaGetLastError();
    });
    return fn;
}

// 2-D fp32 row-major [rows][d] -> box of 32 columns x 128 rows, 128-byte swizzle, zero fill out of bounds
inline bool
make_tmap(CUtensorMap* m, const float* ptr, int64_t rows, int d, int box_rows = 128) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) return false;
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (d & 3)) return false;
    cuuint64_t gdim[2] = {(cuuint64_t)d, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)d * 4};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)ptr, gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

}  // namespace tc
}  // namespace kb2
