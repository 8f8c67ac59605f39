// misc.cuh — weight packing and the small gather / element-wise kernels around the GEMMs.
#pragma once
#include "common.cuh"
#include "misc.h"

// Pack nn.Linear weight W[N][K] (bf16, row-major) into the fragment-streaming layout of gemm_skinny.cuh:
// chunk (nb, s) = 8 rows x 32 k, stored as 32 lanes x 16 B with lane (g = l>>2, t = l&3) holding
// W[nb*8 + g][s*32 + 8t .. 8t+7].   dst index (in uint4) = (nb*(K/32) + s)*32 + lane.
// `row_map`: 0 = identity; 1 = SwiGLU interleave: packed block 2j <- W1 rows [8j,8j+8), 2j+1 <- W3 rows.
__global__ void pack_weight_bf16_kernel(const bf16* __restrict__ w1, const bf16* __restrict__ w3, uint4* __restrict__ dst,
                                        int nblk, int K, int interleave) {
    const int ksteps = K >> 5;
    const long long total = (long long)nblk * ksteps * 32;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int lane = (int)(i & 31);
        const long long c = i >> 5;
        const int s = (int)(c % ksteps);
        const int nb = (int)(c / ksteps);
        const int g = lane >> 2, t = lane & 3;
        const bf16* src;
        if (interleave) src = ((nb & 1) ? w3 : w1) + ((size_t)(nb >> 1) * 8 + g) * K;
        else src = w1 + ((size_t)nb * 8 + g) * K;
        dst[i] = *reinterpret_cast<const uint4*>(src + s * 32 + t * 8);
    }
}

// fp32 SwiGLU interleave: dst rows alternate 8 rows of w1 / 8 rows of w3
__global__ void interleave_rows_f32_kernel(const float* __restrict__ w1, const float* __restrict__ w3,
                                           float* __restrict__ dst, int F, int K) {
    const long long total = (long long)2 * F * K;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % K);
        const int r = (int)(i / K);
        const int blk = r >> 3, g = r & 7;
        const float* src = (blk & 1) ? w3 : w1;
        dst[i] = src[((size_t)(blk >> 1) * 8 + g) * K + k];
    }
}

// h[r] = table[idx[r]] (+ cs[r] * ctrl[r][p]) — tok_embeddings / LabelEmbedder gather, gpt_t2i.py:445,89-97,466
template <typename T>
__global__ void gather_rows_kernel(const T* __restrict__ table, const int* __restrict__ idx, T* __restrict__ out,
                                   int d, const T* __restrict__ ctrl, int n_img, int p, const float* __restrict__ cs) {
    const int r = blockIdx.x;
    const T* src = table + (size_t)idx[r] * d;
    const T* c = (ctrl && p >= 0 && p < n_img) ? ctrl + ((size_t)r * n_img + p) * d : nullptr;
    const float s = c ? cs[r] : 0.f;
    for (int k = threadIdx.x; k < d; k += blockDim.x) {
        float v = tof(src[k]);
        if (c) v = rnd<T>(v + rnd<T>(s * tof(c[k])));
        out[(size_t)r * d + k] = fromf<T>(v);
    }
}

// prefill control add: h[b][T-1][:] += cs[b] * ctrl[b][0][:]     gpt_t2i.py:463
template <typename T>
__global__ void prefill_ctrl_add_kernel(T* __restrict__ h, const T* __restrict__ ctrl, int Tq, int n_img, int d, const float* __restrict__ cs) {
    const int b = blockIdx.x;
    T* hp = h + ((size_t)b * Tq + (Tq - 1)) * d;
    const T* c = ctrl + (size_t)b * n_img * d;
    const float s = cs[b];
    for (int k = threadIdx.x; k < d; k += blockDim.x)
        hp[k] = fromf<T>(rnd<T>(tof(hp[k]) + rnd<T>(s * tof(c[k]))));
}

// copy row T-1 of every batch element: [B][Tq][d] -> [B][d]
template <typename T>
__global__ void take_last_row_kernel(const T* __restrict__ src, T* __restrict__ dst, int Tq, int d) {
    const int b = blockIdx.x;
    for (int k = threadIdx.x; k < d; k += blockDim.x) dst[(size_t)b * d + k] = src[((size_t)b * Tq + Tq - 1) * d + k];
}

template <typename T>
__global__ void rmsnorm_rows_kernel(const T* __restrict__ x, const T* __restrict__ w, T* __restrict__ y, int K, float eps) {
    // RMSNorm.forward gpt_t2i.py:193-198 (stand-alone form, unit tests)
    __shared__ float red[32];
    const int r = blockIdx.x;
    float ss = 0.f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) { const float a = tof(x[(size_t)r * K + k]); ss += a * a; }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    ss = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) ss += red[i];
    const float rstd = rsqrtf(ss / (float)K + eps);
    for (int k = threadIdx.x; k < K; k += blockDim.x)
        y[(size_t)r * K + k] = fromf<T>(rnd<T>(tof(x[(size_t)r * K + k]) * rstd) * tof(w[k]));
}

__global__ void set_int_kernel(int* p, int v) { *p = v; }

// ---- prefill helpers of the dense (M = B_eff * T rows) path ------------------------------------------------
// qkv [rows][3d] (bf16 GEMM output) -> q [rows][d] with RoPE, K/V cache rows (RoPE on K) — gpt_t2i.py:264-271,227-235.
// row = b * Tq + t, sequence position = t.  rope null: no rotation (the plain head split of the control encoder).
__global__ void rope_kv_write_kernel(const bf16* __restrict__ qkv, const float* __restrict__ rope, bf16* __restrict__ q,
                                     bf16* __restrict__ kc, bf16* __restrict__ vc, int rows, int Tq, int d, int H, int S) {
    const long long total = (long long)rows * (3 * d / 2);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / (3 * d / 2));
        const int n = (int)(i % (3 * d / 2)) * 2;
        const int sec = n / d, w = n - sec * d, head = w >> 6, e = w & 63;
        const int b = r / Tq, t = r - b * Tq;
        float v0 = tof(qkv[(size_t)r * 3 * d + n]), v1 = tof(qkv[(size_t)r * 3 * d + n + 1]);
        if (sec < 2 && rope) {
            const float2 cs2 = *reinterpret_cast<const float2*>(rope + ((size_t)t * 32 + (e >> 1)) * 2);
            const float x0 = v0 * cs2.x - v1 * cs2.y, x1 = v1 * cs2.x + v0 * cs2.y;
            v0 = x0; v1 = x1;
        }
        bf16* dst = sec == 0 ? q + (size_t)r * d + w : (sec == 1 ? kc : vc) + (((size_t)b * H + head) * S + t) * 64 + e;
        dst[0] = fromf<bf16>(v0); dst[1] = fromf<bf16>(v1);
    }
}
// act = bf16(bf16(silu(g)) * u)   FeedForward.forward gpt_t2i.py:217
__global__ void swiglu_kernel(const bf16* __restrict__ g, const bf16* __restrict__ u, bf16* __restrict__ out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = fromf<bf16>(rnd<bf16>(silu_f(tof(g[i]))) * tof(u[i]));
}
