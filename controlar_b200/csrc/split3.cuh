// split3.cuh — the split-bf16 ("x3") operand format of the fp32-grade networks (the VQ encoder, HED, LineArt, DPT-Large and MiDaS
// DPT-Hybrid), and the kernels every one of them uses to write it.
// These networks run in fp32 in the reference, and a bf16 network cannot match them: the VQ encoder's latent would carry ~1e-2
// relative noise and 6-7 % of its arg-min indices would flip (SURVEY.md §8 a18: index work is bit-exact).  Here every fp32 value x
// travels as the pair hi = bf16(x), lo = bf16(x - hi) (x = hi + lo to 2^-17) and a product x·w is evaluated as
// hi·w_hi + lo·w_hi + hi·w_lo on the bf16 tensor cores with fp32 accumulation, by tripling the GEMM's K dimension:
//   activations "S3" : 3C bf16 per pixel or row   [ hi(C) | lo(C) | hi(C) ]   (A side)
//   weights     "W3" : [Cout][tap][3 Cin_pad]      [ w_hi  | w_hi  | w_lo  ]   (B side)
// so the bf16 GEMM kernels (gemm.h) run unchanged, with fp32 output, fp32 bias and fp32 residual.
#pragma once
#include "common.cuh"

__device__ __forceinline__ void x3_split(float v, bf16& hi, bf16& lo) {
    hi = __float2bfloat16_rn(v);
    lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
// S3 element: o[0] = hi, o[C] = lo, o[2C] = hi
__device__ __forceinline__ void x3_put_s3(bf16* o, int C, float v) {
    bf16 hi, lo;
    x3_split(v, hi, lo);
    o[0] = hi; o[C] = lo; o[2 * C] = hi;
}
// W3 element: o[0] = hi, o[C] = hi, o[2C] = lo
__device__ __forceinline__ void x3_put_w3(bf16* o, int C, float v) {
    bf16 hi, lo;
    x3_split(v, hi, lo);
    o[0] = hi; o[C] = hi; o[2 * C] = lo;
}

// fp32 rows x [M][N] -> rows [M][3N]: S3 (the A side), S3 through exact GELU, or W3 (the B side)
enum { X3_ROWS_A = 0, X3_ROWS_A_GELU = 1, X3_ROWS_B = 2 };
__global__ void split3_rows_kernel(const float* __restrict__ x, bf16* __restrict__ y, long long M, int N, int mode) {
    const long long total = M * N;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / N;
        const int n = (int)(i - r * N);
        const float v = x[i];
        bf16* o = y + r * 3 * N + n;
        if (mode == X3_ROWS_B) x3_put_w3(o, N, v);
        else x3_put_s3(o, N, mode == X3_ROWS_A_GELU ? gelu_erf_f(v) : v);
    }
}

// image fp32 NCHW [B][C][H][W] (minus sub[c] when sub is given) -> S3 NHWC [B][pt+H+pb][pl+W+pr][3 Cpad] with the image at (pt, pl),
// reflection or zero padding around it and zero channels from C to Cpad
struct X3Image { int B, C, H, W, Cpad, pt, pl, pb, pr, reflect; };
__global__ void image_split3_kernel(const float* __restrict__ x, const float* __restrict__ sub, bf16* __restrict__ y, X3Image q) {
    const int Hp = q.pt + q.H + q.pb, Wp = q.pl + q.W + q.pr;
    const long long total = (long long)q.B * Hp * Wp * q.Cpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % q.Cpad);
        const long long bp = i / q.Cpad;
        const int px = (int)(bp % Wp);
        const long long r = bp / Wp;
        const int py = (int)(r % Hp), b = (int)(r / Hp);
        int sy = py - q.pt, sx = px - q.pl;
        if (q.reflect) {
            sy = sy < 0 ? -sy : (sy >= q.H ? 2 * q.H - 2 - sy : sy);
            sx = sx < 0 ? -sx : (sx >= q.W ? 2 * q.W - 2 - sx : sx);
        }
        float v = 0.f;
        if (c < q.C && sy >= 0 && sy < q.H && sx >= 0 && sx < q.W) {
            v = x[(((size_t)b * q.C + c) * q.H + sy) * q.W + sx];
            if (sub) v -= sub[c];
        }
        x3_put_s3(y + bp * 3 * q.Cpad + c, q.Cpad, v);
    }
}
