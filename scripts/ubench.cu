// ubench.cu — dev micro-benchmarks of the primitives the persistent decode kernel is built from (H100, sm_90a):
//   a. grid barrier (release-reduction arrive + acquire-load spin), one CTA per SM x 512 threads
//   b. barrier + all-gather of a 40 KB activation tile through L2 (every CTA writes 1/grid, all read all)
//   c. flag-in-data exchange (16-byte packets {3 x u32 data, seq}) — no fence, no counter
//   d. HBM -> shared-memory weight stream with cp.async.bulk into a ring of slots (one producer thread per CTA)
//   e. HBM stream with plain LDG.128 (L1::no_allocate) for comparison
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/ubench scripts/ubench.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cstring>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); return 1; } } while (0)

constexpr int THREADS = 512;

__device__ __forceinline__ void grid_sync(unsigned int* bar, unsigned int& gen) {
    __syncthreads();
    if (threadIdx.x == 0) {
        gen += gridDim.x;
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
        unsigned int v;
        unsigned int spins = 0;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory"); if (++spins > (1u << 24)) __trap(); } while ((int)(v - gen) < 0);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(THREADS, 1) k_barrier(unsigned int* bar, unsigned int base, int iters) {
    unsigned int gen = base;
    for (int i = 0; i < iters; ++i) grid_sync(bar, gen);
}

// b: tile = 16 rows x 1280 bf16 = 40 KB = 2560 uint4.  CTA c writes uint4 [c*per, (c+1)*per); then everybody reads all.
__global__ void __launch_bounds__(THREADS, 1) k_bar_gather(unsigned int* bar, unsigned int base, int iters, uint4* buf, int n16, unsigned int* sink) {
    unsigned int gen = base;
    unsigned int acc = 0;
    const int per = (n16 + gridDim.x - 1) / gridDim.x;
    for (int i = 0; i < iters; ++i) {
        uint4* b = buf + (size_t)(i & 1) * n16;
        for (int j = threadIdx.x; j < per; j += THREADS) {
            const int idx = blockIdx.x * per + j;
            if (idx < n16) b[idx] = make_uint4(i, idx, acc, 7);
        }
        grid_sync(bar, gen);
        for (int j = threadIdx.x; j < n16; j += THREADS) {
            uint4 v;
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(b + j));
            acc += v.x + v.y + v.w;
        }
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

// c: packets {d0,d1,d2,seq}; n_pk packets per tile; producers write theirs with seq = i+1; consumers poll every packet.
__global__ void __launch_bounds__(THREADS, 1) k_ll(int iters, uint4* buf, int n_pk, unsigned int* sink, unsigned int seq0) {
    unsigned int acc = 0;
    const int per = (n_pk + gridDim.x - 1) / gridDim.x;
    for (int i = 0; i < iters; ++i) {
        uint4* b = buf + (size_t)(i & 1) * n_pk;       // double buffered: a slow reader of i-1 is never overwritten by i+1's
        const unsigned int seq = seq0 + i + 1;         // writer because writers of i+1 first had to read all of i
        for (int j = threadIdx.x; j < per; j += THREADS) {
            const int idx = blockIdx.x * per + j;
            if (idx < n_pk) {
                asm volatile("st.relaxed.gpu.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(b + idx), "r"(acc), "r"(idx), "r"(i), "r"(seq) : "memory");
            }
        }
        for (int j = threadIdx.x; j < n_pk; j += THREADS) {
            uint4 v;
            unsigned int spins = 0;
            do {
                asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(b + j) : "memory");
                if (++spins > (1u << 22)) __trap();
            } while (v.w != seq);
            acc += v.x + v.y;
        }
        __syncthreads();
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

// c2: like c, but a thread issues all its polls first (independent loads), then re-polls only the stale ones
template <int PER_T>
__global__ void __launch_bounds__(THREADS, 1) k_ll2(int iters, uint4* buf, int n_pk, unsigned int* sink, unsigned int seq0) {
    unsigned int acc = 0;
    const int per = (n_pk + gridDim.x - 1) / gridDim.x;
    for (int i = 0; i < iters; ++i) {
        uint4* b = buf + (size_t)(i & 1) * n_pk;
        const unsigned int seq = seq0 + i + 1;
        for (int j = threadIdx.x; j < per; j += THREADS) {
            const int idx = blockIdx.x * per + j;
            if (idx < n_pk) asm volatile("st.relaxed.gpu.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(b + idx), "r"(acc), "r"(idx), "r"(i), "r"(seq) : "memory");
        }
        uint4 v[PER_T];
        bool done = false;
        unsigned int spins = 0;
        while (!done) {
            if (++spins > (1u << 22)) __trap();
#pragma unroll
            for (int u = 0; u < PER_T; ++u) {
                const int j = threadIdx.x + u * THREADS;
                if (j < n_pk) asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w) : "l"(b + j) : "memory");
                else v[u] = make_uint4(0, 0, 0, seq);
            }
            done = true;
#pragma unroll
            for (int u = 0; u < PER_T; ++u) done = done && (v[u].w == seq);
        }
#pragma unroll
        for (int u = 0; u < PER_T; ++u) acc += v[u].x + v[u].y;
        __syncthreads();
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

// d: TMA bulk stream.  Each CTA streams `bytes_per_cta` contiguous bytes in units of `unit` bytes through NSLOT slots.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t ok = 0, spins = 0;
    while (!ok) {
    if (++spins > (1u << 22)) __trap();
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

template <int NSLOT>
__global__ void __launch_bounds__(THREADS, 1) k_tma_stream(const unsigned char* src, size_t bytes_per_cta, int unit, unsigned int* sink, int touch) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t full[NSLOT];
    const unsigned char* my = src + (size_t)blockIdx.x * bytes_per_cta;
    const int n_units = (int)(bytes_per_cta / unit);
    if (threadIdx.x == 0) { for (int s = 0; s < NSLOT; ++s) mbar_init(&full[s], 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int u = 0; u < NSLOT && u < n_units; ++u) { mbar_expect_tx(&full[u], unit); bulk_g2s(smem + (size_t)u * unit, my + (size_t)u * unit, unit, &full[u]); }
    unsigned int acc = 0;
    for (int u = 0; u < n_units; ++u) {
        const int s = u % NSLOT;
        mbar_wait(&full[s], (u / NSLOT) & 1);
        if (touch) {   // consume: every thread reads its share of the slot with LDS.128
            const uint4* p = reinterpret_cast<const uint4*>(smem + (size_t)s * unit);
            for (int j = threadIdx.x; j < unit / 16; j += THREADS) { const uint4 v = p[j]; acc += v.x ^ v.w; }
        }
        __syncthreads();
        if (threadIdx.x == 0 && u + NSLOT < n_units) { mbar_expect_tx(&full[s], unit); bulk_g2s(smem + (size_t)s * unit, my + (size_t)(u + NSLOT) * unit, unit, &full[s]); }
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

// e: LDG stream
__global__ void __launch_bounds__(THREADS, 1) k_ldg_stream(const uint4* src, size_t n16_per_cta, unsigned int* sink) {
    const uint4* my = src + (size_t)blockIdx.x * n16_per_cta;
    unsigned int acc = 0;
    size_t j = threadIdx.x;
    for (; j + 7 * THREADS < n16_per_cta; j += 8 * THREADS) {
        uint4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w) : "l"(my + j + u * THREADS));
#pragma unroll
        for (int u = 0; u < 8; ++u) acc += v[u].x ^ v[u].w;
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

int main(int argc, char** argv) {
    setvbuf(stdout, nullptr, _IONBF, 0);
    const char* which = argc > 1 ? argv[1] : "abcde";
    auto on = [&](char c) { return strchr(which, c) != nullptr; };
    int dev = 0, sms = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    printf("SMs %d\n", sms);
    unsigned int *bar, *sink;
    CK(cudaMalloc(&bar, 256)); CK(cudaMemset(bar, 0, 256));
    CK(cudaMalloc(&sink, 256));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float ms;
    unsigned int base = 0;
    // a
    for (int rep = 0; rep < 3 && on('a'); ++rep) {
        const int iters = 2000;
        void* args[] = {&bar, &base, (void*)&iters};
        cudaEventRecord(e0);
        CK(cudaLaunchCooperativeKernel((void*)k_barrier, dim3(sms), dim3(THREADS), args, 0, 0));
        cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
        base += (unsigned)iters * sms;
        printf("a. grid barrier: %.3f us each\n", ms * 1000.f / iters);
    }
    // b
    for (int n16 : {2560, 7168}) {
        if (!on('b')) break;
        uint4* buf; CK(cudaMalloc(&buf, (size_t)2 * n16 * 16));
        for (int rep = 0; rep < 2; ++rep) {
            const int iters = 2000;
            void* args[] = {&bar, &base, (void*)&iters, &buf, (void*)&n16, &sink};
            cudaEventRecord(e0);
            CK(cudaLaunchCooperativeKernel((void*)k_bar_gather, dim3(sms), dim3(THREADS), args, 0, 0));
            cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
            base += (unsigned)iters * sms;
            printf("b. write + barrier + all-gather %d KB: %.3f us each\n", n16 * 16 / 1024, ms * 1000.f / iters);
        }
        cudaFree(buf);
    }
    // c
    unsigned int seq0 = 0;
    for (int n_pk : {3414, 9558}) {
        if (!on('c')) break;
        uint4* buf; CK(cudaMalloc(&buf, (size_t)2 * n_pk * 16)); CK(cudaMemset(buf, 0, (size_t)2 * n_pk * 16));
        for (int rep = 0; rep < 2; ++rep) {
            const int iters = 2000;
            void* args[] = {(void*)&iters, &buf, (void*)&n_pk, &sink, &seq0};
            cudaEventRecord(e0);
            CK(cudaLaunchCooperativeKernel((void*)k_ll, dim3(sms), dim3(THREADS), args, 0, 0));
            cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
            seq0 += iters;
            printf("c. flag-in-data exchange %d packets (%d KB payload): %.3f us each\n", n_pk, n_pk * 12 / 1024, ms * 1000.f / iters);
        }
        for (int rep = 0; rep < 2; ++rep) {
            const int iters = 2000;
            void* args[] = {(void*)&iters, &buf, (void*)&n_pk, &sink, &seq0};
            cudaEventRecord(e0);
            if (n_pk <= 7 * THREADS) CK(cudaLaunchCooperativeKernel((void*)k_ll2<7>, dim3(sms), dim3(THREADS), args, 0, 0));
            else CK(cudaLaunchCooperativeKernel((void*)k_ll2<19>, dim3(sms), dim3(THREADS), args, 0, 0));
            cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
            seq0 += iters;
            printf("c2. flag-in-data, batched polls %d packets: %.3f us each\n", n_pk, ms * 1000.f / iters);
        }
        cudaFree(buf);
    }
    // d / e
    const size_t per_cta = (size_t)20 << 20;    // 20 MB per CTA -> 2.96 GB total (>> L2)
    unsigned char* src; CK(cudaMalloc(&src, per_cta * sms)); CK(cudaMemset(src, 1, per_cta * sms));
    CK(cudaFuncSetAttribute(k_tma_stream<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(k_tma_stream<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(k_tma_stream<14>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    for (int touch = 0; touch < 2 && on('d'); ++touch)
        for (int cfg = 0; cfg < 4; ++cfg) {
            const int unit = cfg == 0 ? 28672 : (cfg == 1 ? 20480 : (cfg == 2 ? 40960 : 8192));
            const size_t bytes = per_cta / unit * unit;
            for (int rep = 0; rep < 2; ++rep) {
                cudaEventRecord(e0);
                if (cfg == 2) k_tma_stream<4><<<sms, THREADS, 4 * unit>>>(src, bytes, unit, sink, touch);
                else if (cfg == 3) k_tma_stream<14><<<sms, THREADS, 14 * unit>>>(src, bytes, unit, sink, touch);
                else k_tma_stream<7><<<sms, THREADS, 7 * unit>>>(src, bytes, unit, sink, touch);
                cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
                CK(cudaGetLastError());
            }
            printf("d. bulk-copy stream unit %d B x %d slots, touch=%d: %.1f GB/s\n", unit, cfg == 2 ? 4 : (cfg == 3 ? 14 : 7), touch, bytes * sms / (ms * 1e6));
        }
    for (int rep = 0; rep < 2 && on('e'); ++rep) {
        cudaEventRecord(e0);
        k_ldg_stream<<<sms, THREADS>>>((const uint4*)src, per_cta / 16, sink);
        cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); cudaEventElapsedTime(&ms, e0, e1);
        printf("e. LDG.128 stream: %.1f GB/s\n", per_cta * sms / (ms * 1e6));
    }
    return 0;
}
