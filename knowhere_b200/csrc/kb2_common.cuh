// kb2_common.cuh — shared host/device utilities of the H100-native search core.
// (product code; never includes anything under oracle/)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <mutex>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>

#include "../../include/knowhere_b200.h"

namespace kb2 {

// ------------------------------------------------------------------ errors
struct Error : std::runtime_error {
    int status;
    Error(int s, const std::string& m) : std::runtime_error(m), status(s) {}
};

#define KB2_CUDA_CHECK(expr)                                                                       \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            throw ::kb2::Error(KB2_CUDA_RUNTIME_ERROR, std::string(#expr) + ": " +                 \
                                                           cudaGetErrorString(_e) + " @" + __FILE__ + \
                                                           ":" + std::to_string(__LINE__));        \
        }                                                                                          \
    } while (0)

#define KB2_REQUIRE(cond, status, msg)                         \
    do {                                                       \
        if (!(cond)) throw ::kb2::Error((status), (msg));      \
    } while (0)

constexpr int kWarp = 32;
constexpr int kScanThreads = 256;  // 8 warps per scan CTA
constexpr int kScanWarps = kScanThreads / kWarp;
constexpr uint64_t kEmpty = ~0ull; // empty slot of a top-k list (worst possible key)
constexpr uint32_t kNoPos = 0xffffffffu;

// metric handling: internally every kernel minimises a "key":
//   L2 : key = squared L2 distance         IP : key = -inner_product
// (the reference gets the same effect with CMax/CMin heaps and, for HNSW, NegativeDistanceComputer:
//  F/utils/ordered_key_value.h:42-84, F/impl/DistanceComputer.h:77-95)

// ------------------------------------------------------------------ device helpers
// order-preserving float -> uint32 (unsigned compare == float compare, -inf < ... < +inf)
__host__ __device__ __forceinline__ uint32_t
f2ord(float f) {
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float
ord2f(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
// (key, position) packed so that one u64 compare gives the total order (key asc, then pos asc)
__host__ __device__ __forceinline__ uint64_t
pack_kp(float key, uint32_t pos) {
    return ((uint64_t)f2ord(key) << 32) | pos;
}
__host__ __device__ __forceinline__ float
unpack_key(uint64_t p) {
    return ord2f((uint32_t)(p >> 32));
}
__host__ __device__ __forceinline__ uint32_t
unpack_pos(uint64_t p) {
    return (uint32_t)p;
}

__device__ __forceinline__ bool
bit_is_set(const uint8_t* __restrict__ bits, int64_t i) {
    return (bits[i >> 3] >> (i & 7)) & 1;
}

__device__ __forceinline__ float
warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// streaming 128-bit load that does not pollute L1 (codes are read once per CTA)
__device__ __forceinline__ uint4
ldg_stream_u4(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ uint2
ldg_stream_u2(const uint2* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ float4
ldg_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

static inline int
next_pow2(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}
static inline int64_t
round_up(int64_t v, int64_t a) {
    return (v + a - 1) / a * a;
}

// one RangeSearch hit as the device kernels emit it (kb2_range.cuh, kb2_hnsw.cuh)
struct RangeHit {
    int32_t q;
    int32_t probe;   // IVF: rank of the probed list (max_empty_result_buckets); otherwise 0
    uint32_t pos;    // position / internal row
    float dist;
};

// ------------------------------------------------------------------ RAII device buffer
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    bool owned = true;   // false: p is a caller-owned device buffer viewed in place (borrow())
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n), owned(o.owned) { o.p = nullptr; o.n = 0; o.owned = true; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) { release(); p = o.p; n = o.n; owned = o.owned; o.p = nullptr; o.n = 0; o.owned = true; }
        return *this;
    }
    ~DevBuf() { release(); }
    void release() {
        if (p && owned) cudaFree(p);
        p = nullptr;
        n = 0;
        owned = true;
    }
    // view `count` elements of a caller-owned device buffer (never freed, never grown in place)
    void borrow(const T* ptr, size_t count) {
        release();
        p = const_cast<T*>(ptr);
        n = count;
        owned = false;
    }
    // grow-only allocation (contents are NOT preserved)
    void ensure(size_t count) {
        if (count <= n && p && owned) return;
        release();
        if (count == 0) count = 1;
        cudaError_t e = cudaMalloc((void**)&p, count * sizeof(T));
        if (e != cudaSuccess) {
            p = nullptr;
            throw Error(KB2_MALLOC_ERROR, std::string("cudaMalloc(") + std::to_string(count * sizeof(T)) +
                                              "): " + cudaGetErrorString(e));
        }
        n = count;
    }
    void alloc_exact(size_t count) {
        release();
        ensure(count);
    }
    size_t bytes() const { return n * sizeof(T); }
};

// pinned host staging buffer (grow-only)
struct PinnedBuf {
    void* p = nullptr;
    size_t n = 0;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
    void* ensure(size_t bytes) {
        if (bytes <= n && p) return p;
        if (p) cudaFreeHost(p);
        p = nullptr;
        if (bytes == 0) bytes = 1;
        cudaError_t e = cudaMallocHost(&p, bytes);
        if (e != cudaSuccess) {
            p = nullptr; n = 0;
            throw Error(KB2_MALLOC_ERROR, std::string("cudaMallocHost: ") + cudaGetErrorString(e));
        }
        n = bytes;
        return p;
    }
};

// Run `f` once per CUDA device (kernel attributes apply to the current device only; one process may hold
// indexes on several GPUs — the C ABI takes a device ordinal per handle).
struct PerDeviceOnce {
    std::once_flag flags[64];
    template <typename F>
    void run(F&& f) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
        if (dev < 0 || dev >= 64) { f(); return; }
        std::call_once(flags[dev], f);
    }
};

constexpr int kMaxDynSmem = 227 * 1024;   // dynamic shared memory one CTA may use on sm_90

// Launches one kernel instance.  A launch with more than the 48 KB of dynamic shared memory every kernel gets by default
// first raises that instance's limit to MaxSmem, once per device, so no launch depends on a list of instances kept
// elsewhere.  (The default is 48 KB less the kernel's static shared memory; no kernel launched with dynamic shared
// memory here has any.)
template <auto Kernel, int MaxSmem = kMaxDynSmem, typename... Args>
inline void
launch(dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    if (smem > 48 * 1024) {
        static PerDeviceOnce once;
        once.run([] {
            KB2_CUDA_CHECK(cudaFuncSetAttribute((const void*)Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MaxSmem));
        });
    }
    Kernel<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
}

// Calls f(std::integral_constant<int, M>{}) with M the metric as a compile-time constant (COSINE runs as IP).
template <typename F>
inline void
with_metric(int metric, F&& f) {
    if (metric == KB2_METRIC_L2)
        f(std::integral_constant<int, KB2_METRIC_L2>{});
    else
        f(std::integral_constant<int, KB2_METRIC_IP>{});
}

// SM count of the current device (132 on an H100 SXM, 114 on an H100 PCIe): sizes the persistent grids and the per-CTA
// buffers that go with them.  Read once per device.
inline int
num_sms() {
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
    const bool cached = dev >= 0 && dev < 64;
    if (cached) {
        const int v = cache[dev].load(std::memory_order_relaxed);
        if (v > 0) return v;
    }
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
        cudaGetLastError();
        throw Error(KB2_CUDA_RUNTIME_ERROR, "cannot read the SM count of the current device");
    }
    if (cached) cache[dev].store(n, std::memory_order_relaxed);
    return n;
}

inline bool
is_device_ptr(const void* p) {
    if (!p) return false;
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

}  // namespace kb2
