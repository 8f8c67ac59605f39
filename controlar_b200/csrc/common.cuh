// common.cuh — shared device helpers for the ControlAR H100 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <algorithm>
#include <atomic>
#include <string>
#include <cstring>
#include <vector>

#include "../../include/controlar_b200.h"
#include "carve.h"

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------------------------
// host-side error plumbing (no exceptions cross the C ABI)
// ---------------------------------------------------------------------------------------------------------
extern thread_local std::string g_car_err;
extern std::atomic<long long> g_car_launches;

#define CAR_FAIL(code, msg)                                   \
    do {                                                      \
        g_car_err = std::string(__func__) + ": " + (msg);     \
        return (code);                                        \
    } while (0)

#define CAR_CUDA(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            g_car_err = std::string(__func__) + ": " #expr " -> " + cudaGetErrorString(_e);        \
            return CAR_ERR_CUDA;                                                                    \
        }                                                                                           \
    } while (0)

#define CAR_TRY(expr)             \
    do {                          \
        int _r = (expr);          \
        if (_r != CAR_OK) return _r; \
    } while (0)

// per-device once-flags (a process-wide `static bool` would configure the first device only; the Python handles make the
// tensors' device current around every call)
struct DevOnce {
    bool done[64] = {false};
    bool first() { int dev = 0; cudaGetDevice(&dev); if (dev < 0 || dev >= 64) return true; const bool f = !done[dev]; done[dev] = true; return f; }
};

// SM count of the CURRENT device (the Python handles make the tensors' device current around every call)
inline int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (cached[dev] == 0) { int n = 0; cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); cached[dev] = n > 0 ? n : 132; }
    return cached[dev];
}

// grid of a grid-stride loop over `total` elements in blocks of 256 threads: at most 16 CTAs per SM
inline int gsz(long long total) { return (int)std::min<long long>((total + 255) / 256, sm_count() * 16); }

struct Arena {   // grow-only device workspace, re-used across calls (no allocation in steady state)
    // The scratch buffers of one forward.  `list` names them once, as c.take<T>(count) calls; it runs first on a measuring Carve,
    // whose end offset is what the arena grows to, then on the real base — so the size is the sum of the takes by construction.
    template <typename F> int carve(F&& list) {
        Carve measure(nullptr);
        list(measure);
        CAR_TRY(reserve(measure.off));
        Carve c(base);
        list(c);
        return CAR_OK;
    }
    void release() { if (base) cudaFree(base); base = nullptr; cap = 0; }
private:
    char* base = nullptr; size_t cap = 0;
    int reserve(size_t bytes) {
        if (bytes <= cap) return CAR_OK;
        if (base) cudaFree(base);
        base = nullptr; cap = 0;
        CAR_CUDA(cudaMalloc(&base, bytes));
        cap = bytes;
        return CAR_OK;
    }
};

// In front of every launch that writes a scratch buffer shared between stages (sized as the maximum over its uses): refuse, without
// launching, a write of `need` elements into a buffer carved for fewer.  `who` names the writer in the message.
template <typename T> inline int car_fits(const char* who, const Buf<T>& b, size_t need) {
    if (b.fits(need)) return CAR_OK;
    g_car_err = std::string(who) + ": writes " + std::to_string(need) + " elements into a scratch buffer carved for " + std::to_string(b.cap);
    return CAR_ERR_STATE;
}

// Base of every handle: the device memory its create call allocated and its forward workspace, both freed by `delete`.
struct CarOwned {
    std::vector<void*> owned;
    Arena ws;
    // device memory that lives as long as the handle (a zero-byte request still gets its own allocation)
    template <typename T> int alloc(T** p, size_t bytes) {
        CAR_CUDA(cudaMalloc((void**)p, bytes ? bytes : 16));
        owned.push_back((void*)*p);
        return CAR_OK;
    }
    ~CarOwned() {
        for (void* p : owned) cudaFree(p);
        ws.release();
    }
};

// every kernel launch goes through this so that car_launch_count() is an honest count
#define CAR_LAUNCH(kernel, grid, block, smem, stream, ...)                                          \
    do {                                                                                            \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                                 \
        g_car_launches.fetch_add(1, std::memory_order_relaxed);                                     \
        cudaError_t _e = cudaGetLastError();                                                        \
        if (_e != cudaSuccess) {                                                                    \
            g_car_err = std::string(__func__) + ": launch " #kernel " -> " + cudaGetErrorString(_e); \
            return CAR_ERR_CUDA;                                                                    \
        }                                                                                           \
    } while (0)

// Programmatic dependent launch (PDL): the next kernel in the stream is launched while this one still runs; its
// prologue (weight loads / L2 prefetch of immutable data) overlaps our tail, and it blocks in pdl_wait() until
// this grid has completed and its writes are visible.  Rule: nothing mutable may be touched before pdl_wait().
#define CAR_LAUNCH_PDL(kernel, grid_, block_, smem_, strm_, ...)                                      \
    do {                                                                                            \
        cudaLaunchConfig_t _cfg;                                                                    \
        memset(&_cfg, 0, sizeof(_cfg));                                                             \
        _cfg.gridDim = (grid_); _cfg.blockDim = (block_); _cfg.dynamicSmemBytes = (smem_); _cfg.stream = (strm_); \
        cudaLaunchAttribute _at[1];                                                                 \
        _at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                             \
        _at[0].val.programmaticStreamSerializationAllowed = 1;                                      \
        _cfg.attrs = _at; _cfg.numAttrs = 1;                                                        \
        cudaError_t _e = cudaLaunchKernelEx(&_cfg, kernel, __VA_ARGS__);                            \
        g_car_launches.fetch_add(1, std::memory_order_relaxed);                                     \
        if (_e != cudaSuccess) {                                                                    \
            g_car_err = std::string(__func__) + ": launch " #kernel " -> " + cudaGetErrorString(_e); \
            return CAR_ERR_CUDA;                                                                    \
        }                                                                                           \
    } while (0)

__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// mutable data (activations, KV cache, device scalars) is always read through L2 (.cg): with PDL a dependent
// kernel's CTAs are resident before the producer finishes, so an L1 line could otherwise be stale.
__device__ __forceinline__ uint4 ldg_cg128(const void* p) {
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ float ld_cg(const float* p) { return __ldcg(p); }
__device__ __forceinline__ float ld_cg(const bf16* p) {
    unsigned short v;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(v) : "l"(p));
    return __uint_as_float(((uint32_t)v) << 16);
}
__device__ __forceinline__ int ld_cg(const int* p) { return __ldcg(p); }

// ---------------------------------------------------------------------------------------------------------
// storage-type helpers: all arithmetic is fp32; `rnd<T>` marks the points where eager PyTorch would
// materialise a tensor in the model dtype (SURVEY.md §8 a-notes).
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float tof(bf16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float tof(float x) { return x; }
template <typename T> __device__ __forceinline__ T fromf(float x);
template <> __device__ __forceinline__ bf16 fromf<bf16>(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ float fromf<float>(float x) { return x; }
template <typename T> __device__ __forceinline__ float rnd(float x) { return tof(fromf<T>(x)); }

__device__ __forceinline__ float gelu_tanh_f(float x) {
    // nn.GELU(approximate='tanh'), gpt_t2i.py:171
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    float inner = k0 * (x + k1 * x * x * x);
    return 0.5f * x * (1.0f + tanhf(inner));
}
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.7071067811865476f)); }
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---- block reduce helpers (blockDim.x multiple of 32, <= 1024)
// NW: the block's warp count when the kernel fixes it at compile time (the final loop is then unrolled), 0: blockDim.x / 32
template <int NW = 0> __device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    for (int i = 0; i < (NW ? NW : (int)(blockDim.x >> 5)); ++i) s += red[i];
    __syncthreads();
    return s;
}
__device__ __forceinline__ float block_max(float v, float* red) {
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) s = fmaxf(s, red[i]);
    __syncthreads();
    return s;
}

// streaming 128-bit load that does not allocate in L1 (weights / KV are read once per step)
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ void unpack_bf16x2(uint32_t v, float& lo, float& hi) {
    lo = __uint_as_float(v << 16);
    hi = __uint_as_float(v & 0xffff0000u);
}

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
