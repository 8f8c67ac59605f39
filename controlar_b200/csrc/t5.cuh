// t5.cuh — small kernels of the T5 text encoder forward (SURVEY.md §8 row f3): language/t5.py:58-79 calls HF
// T5EncoderModel(input_ids, attention_mask).last_hidden_state in bf16 (transformers 5.5.0, models/t5/modeling_t5.py, un-pinned third
// party).  The GEMMs run on the dense wgmma kernel (gemm_wgmma.cuh); everything here mirrors the bf16 rounding points of the eager
// HF modules: every elementwise PyTorch op on a bf16 tensor computes in fp32 and rounds its output to bf16.
#pragma once
#include "common.cuh"

__device__ __forceinline__ float t5r(float v) { return rnd<bf16>(v); }

// embed_tokens(input_ids)  (T5Stack: shared embedding)
__global__ void t5_embed_kernel(const int* __restrict__ ids, const bf16* __restrict__ table, bf16* __restrict__ out, int rows, int d) {
    const int r = blockIdx.x;
    const uint4* src = reinterpret_cast<const uint4*>(table + (size_t)ids[r] * d);
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)r * d);
    for (int k = threadIdx.x; k < d / 8; k += blockDim.x) dst[k] = src[k];
}

// T5Attention._relative_position_bucket (modeling_t5.py:189-234), bidirectional
__device__ __forceinline__ int t5_bucket(int rel, int num_buckets, int max_distance) {
    const int nb = num_buckets / 2;
    int ret = rel > 0 ? nb : 0;
    const int n = abs(rel);
    const int max_exact = nb / 2;
    if (n < max_exact) return ret + n;
    int v = max_exact + (int)(logf((float)n / (float)max_exact) / logf((float)max_distance / (float)max_exact) * (float)(nb - max_exact));
    return ret + min(v, nb - 1);
}

// T5Attention.forward (modeling_t5.py:253-340), encoder self-attention: scores = q k^T (bf16), + position_bias (bf16 table lookup;
// masked keys get the dtype's most negative value added => probability 0), soft-max in fp32 cast to bf16, times v (bf16).  No
// 1/sqrt(d) scaling (T5).  One warp per (b, h, query); q / k / v [rows][H*64] (GEMM outputs), out the same layout.
constexpr int T5A_WARPS = 4;
__global__ void __launch_bounds__(T5A_WARPS * 32)
t5_attention_kernel(const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v, const bf16* __restrict__ rel_bias /*[nb][H]*/,
                    const int* __restrict__ mask /*[B][L]*/, int B, int H, int L, int num_buckets, int max_distance, bf16* __restrict__ out) {
    extern __shared__ float t5_sc[];                           // [T5A_WARPS][L]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * T5A_WARPS + warp;
    if (item >= (long long)B * H * L) return;                  // (whole warp)
    const int i = (int)(item % L);
    const int hd = (int)((item / L) % H);
    const int b = (int)(item / ((long long)L * H));
    const int inner = H * 64;
    float* sc = t5_sc + (size_t)warp * L;
    const bf16* qp = q + ((size_t)b * L + i) * inner + hd * 64;
    float qf[64];
#pragma unroll
    for (int e = 0; e < 64; e += 2) unpack_bf16x2(*reinterpret_cast<const uint32_t*>(qp + e), qf[e], qf[e + 1]);
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) {
        float s = -INFINITY;
        if (mask[(size_t)b * L + j] != 0) {
            const uint4* kr = reinterpret_cast<const uint4*>(k + ((size_t)b * L + j) * inner + hd * 64);
            float d = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 kk = kr[c];
                float k0, k1;
                unpack_bf16x2(kk.x, k0, k1); d = fmaf(qf[c * 8 + 0], k0, d); d = fmaf(qf[c * 8 + 1], k1, d);
                unpack_bf16x2(kk.y, k0, k1); d = fmaf(qf[c * 8 + 2], k0, d); d = fmaf(qf[c * 8 + 3], k1, d);
                unpack_bf16x2(kk.z, k0, k1); d = fmaf(qf[c * 8 + 4], k0, d); d = fmaf(qf[c * 8 + 5], k1, d);
                unpack_bf16x2(kk.w, k0, k1); d = fmaf(qf[c * 8 + 6], k0, d); d = fmaf(qf[c * 8 + 7], k1, d);
            }
            const float pb = tof(rel_bias[(size_t)t5_bucket(j - i, num_buckets, max_distance) * H + hd]);
            s = t5r(t5r(d) + pb);                               // matmul output in bf16, `scores += position_bias` in bf16
        }
        sc[j] = s;
        mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) {
        const float p = (sc[j] == -INFINITY) ? 0.f : expf(sc[j] - mx);
        sc[j] = p;
        sum += p;
    }
    sum = warp_sum(sum);
    __syncwarp();
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j < L; ++j) {
        const float p = t5r(sc[j] / sum);                       // soft-max(fp32).type_as(scores)
        if (p != 0.f) {
            float v0, v1;
            unpack_bf16x2(*reinterpret_cast<const uint32_t*>(v + ((size_t)b * L + j) * inner + hd * 64 + 2 * lane), v0, v1);
            o0 = fmaf(p, v0, o0); o1 = fmaf(p, v1, o1);
        }
    }
    __nv_bfloat162 o = __floats2bfloat162_rn(o0, o1);
    *reinterpret_cast<__nv_bfloat162*>(out + ((size_t)b * L + i) * inner + hd * 64 + 2 * lane) = o;
}

// T5DenseGatedActDense (modeling_t5.py:115-118) with dense_act_fn = "gelu_new" (NewGELUActivation):
//   0.5 * x * (1.0 + tanh(sqrt(2 / pi) * (x + 0.044715 * pow(x, 3.0))))  evaluated op by op on bf16 tensors, then * hidden_linear
__global__ void t5_geglu_kernel(const bf16* __restrict__ g, const bf16* __restrict__ u, bf16* __restrict__ out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float x = tof(g[i]);
        const float p3 = t5r(x * x * x);                        // torch.pow(input, 3.0)
        const float t2 = t5r(0.044715f * p3);
        const float t3 = t5r(x + t2);
        const float t4 = t5r(0.7978845608028654f * t3);
        const float t5v = t5r(tanhf(t4));
        const float t6 = t5r(1.0f + t5v);
        const float t7 = t5r(0.5f * x);
        const float ge = t5r(t7 * t6);
        out[i] = fromf<bf16>(t5r(ge * tof(u[i])));
    }
}
