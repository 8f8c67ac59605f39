// midas.cuh — the ResNet-50 trunk of MiDaS DPT-Hybrid (reference condition/midas/midas/vit.py, timm ResNetV2 with preact=False and
// stem_type "same"), fp32 in the reference => fp32-grade here.  The convolutions run on the split-bf16 ("x3", split3.cuh) GEMMs of
// car_vision.cu, the stem's input written by image_split3_kernel with TF "SAME" padding of the 7x7/2 stem (2 before, 3 after; the
// sides are even); the kernels below are the rest of the glue:
//   weight standardisation  per output channel (w - mean) / sqrt(biased var + 1e-8), statistics in fp64, once at create time
//   group norm              GroupNorm(32, eps 1e-5) statistics in two deterministic passes (group mean, then centred squares) over
//                           NHWC fp32, reduced in an order that depends on the map size only, never on the batch; one apply kernel
//                           fuses the affine, the residual (optionally group-normalised itself: the downsample shortcut), ReLU, the
//                           stem's 3x3/2 max-pool and the padded S3 write of the next convolution's operand
// The ViT, reassemble, fusion and head stages are the DPT kernels (dpt.cuh).
#pragma once
#include "split3.cuh"

constexpr int MD_GROUPS = 32;
constexpr int MD_THREADS = 256;

// fp32 weight [n][K] -> standardised fp32 weight [n][K]; one block per output channel, fp64 statistics in a fixed order
__global__ void __launch_bounds__(MD_THREADS) midas_ws_kernel(const float* __restrict__ w, float* __restrict__ y, int K, double eps) {
    __shared__ double red[MD_THREADS];
    const float* x = w + (size_t)blockIdx.x * K;
    double s = 0.0;
    for (int k = threadIdx.x; k < K; k += MD_THREADS) s += (double)x[k];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = MD_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    const double mean = red[0] / K;
    __syncthreads();
    double q = 0.0;
    for (int k = threadIdx.x; k < K; k += MD_THREADS) { const double d = (double)x[k] - mean; q += d * d; }
    red[threadIdx.x] = q;
    __syncthreads();
    for (int o = MD_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    const double inv = 1.0 / sqrt(red[0] / K + eps);
    for (int k = threadIdx.x; k < K; k += MD_THREADS) y[(size_t)blockIdx.x * K + k] = (float)(((double)x[k] - mean) * inv);
}

// ---- group-norm statistics over NHWC fp32 [B][HW][C], 32 groups of cpg = C / 32 channels.  grid (32, B, nch), 256 threads; pixel
// chunk j of nch covers [j*per, (j+1)*per); element e of a chunk is (pixel p0 + e / cpg, channel g*cpg + e % cpg).  Every sum has a
// fixed order that depends on (HW, C) only.
__device__ __forceinline__ float md_chunk_sum(const float* __restrict__ xb, int HW, int C, int g, int nch, int j, float mean, bool centred,
                                              float* red) {
    const int cpg = C / MD_GROUPS, per = (HW + nch - 1) / nch;
    const int p0 = j * per, p1 = min(HW, p0 + per);
    const int n = max(0, p1 - p0) * cpg;
    const float* base = xb + (size_t)p0 * C + g * cpg;
    float s = 0.f;
    for (int e = threadIdx.x; e < n; e += MD_THREADS) {
        const int p = e / cpg, k = e - p * cpg;
        const float v = base[(size_t)p * C + k];
        if (centred) { const float d = v - mean; s = fmaf(d, d, s); } else s += v;
    }
    return block_sum<MD_THREADS / 32>(s, red);
}
__device__ __forceinline__ float md_mean(const float* __restrict__ part_s, int b, int nch, int g, int HW, int C) {
    float s = 0.f;
    for (int j = 0; j < nch; ++j) s += part_s[((size_t)b * nch + j) * MD_GROUPS + g];
    return s / ((float)HW * (float)(C / MD_GROUPS));
}
__global__ void __launch_bounds__(MD_THREADS) midas_gn_sum_kernel(const float* __restrict__ x, float* __restrict__ part_s /*[B][nch][32]*/, int HW, int C) {
    __shared__ float red[MD_THREADS / 32];
    const int g = blockIdx.x, b = blockIdx.y, j = blockIdx.z, nch = gridDim.z;
    const float t = md_chunk_sum(x + (size_t)b * HW * C, HW, C, g, nch, j, 0.f, false, red);
    if (threadIdx.x == 0) part_s[((size_t)b * nch + j) * MD_GROUPS + g] = t;
}
__global__ void __launch_bounds__(MD_THREADS) midas_gn_sq_kernel(const float* __restrict__ x, const float* __restrict__ part_s, float* __restrict__ part_q,
                                                                int HW, int C) {
    __shared__ float red[MD_THREADS / 32];
    const int g = blockIdx.x, b = blockIdx.y, j = blockIdx.z, nch = gridDim.z;
    const float mean = md_mean(part_s, b, nch, g, HW, C);
    const float t = md_chunk_sum(x + (size_t)b * HW * C, HW, C, g, nch, j, mean, true, red);
    if (threadIdx.x == 0) part_q[((size_t)b * nch + j) * MD_GROUPS + g] = t;
}
// stats [B][32][2] = (mean, 1 / sqrt(biased variance + 1e-5))
__global__ void midas_gn_finish_kernel(const float* __restrict__ part_s, const float* __restrict__ part_q, float* __restrict__ stats, int B, int HW,
                                       int C, int nch) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * MD_GROUPS) return;
    const int b = i / MD_GROUPS, g = i - b * MD_GROUPS;
    float q = 0.f;
    for (int j = 0; j < nch; ++j) q += part_q[((size_t)b * nch + j) * MD_GROUPS + g];
    stats[2 * i] = md_mean(part_s, b, nch, g, HW, C);
    stats[2 * i + 1] = 1.0f / sqrtf(q / ((float)HW * (float)(C / MD_GROUPS)) + 1e-5f);
}

// v = GN(x) (+ r) (ReLU) with r = resid, or GN_r(resid) when rstats is given; with pool, the 3x3 / stride 2 max-pool (TF "SAME":
// no padding before, one after) of that over an even H x W map.  The Ho x Wo result (Ho = H / 2 with pool, else H) is written as
// S3 (3C bf16 per pixel) into a zero-filled frame [B][Hp][Wp] at (pt, pl), and, when carrier is given, as fp32 [B][Ho][Wo][C].
struct GnApply { int pt, pl, Hp, Wp, relu, pool; };
struct GnAffine { const float* stats; const float* w; const float* b; };
__device__ __forceinline__ float md_gn(const GnAffine& a, float v, int b, int c, int cpg) {
    const float* st = a.stats + ((size_t)b * MD_GROUPS + c / cpg) * 2;
    return (v - st[0]) * st[1] * a.w[c] + a.b[c];
}
__global__ void midas_gn_apply_kernel(const float* __restrict__ x, GnAffine n, const float* __restrict__ resid, GnAffine rn,
                                      float* __restrict__ carrier, bf16* __restrict__ y, int B, int H, int W, int C, GnApply a) {
    const int cpg = C / MD_GROUPS, Ho = a.pool ? H / 2 : H, Wo = a.pool ? W / 2 : W;
    const long long total = (long long)B * a.Hp * a.Wp * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long bp = i / C;
        const int px = (int)(bp % a.Wp);
        const long long r = bp / a.Wp;
        const int py = (int)(r % a.Hp), b = (int)(r / a.Hp);
        const int oy = py - a.pt, ox = px - a.pl;
        float v = 0.f;
        if (oy >= 0 && oy < Ho && ox >= 0 && ox < Wo) {
            if (a.pool) {                                // post-ReLU values are >= 0: the window's max over in-range taps
                for (int ky = 0; ky < 3; ++ky)
                    for (int kx = 0; kx < 3; ++kx) {
                        const int iy = 2 * oy + ky, ix = 2 * ox + kx;
                        if (iy < H && ix < W) v = fmaxf(v, fmaxf(md_gn(n, x[(((size_t)b * H + iy) * W + ix) * C + c], b, c, cpg), 0.f));
                    }
            } else {
                const size_t src = (((size_t)b * H + oy) * W + ox) * C + c;
                v = md_gn(n, x[src], b, c, cpg);
                if (resid) v += rn.stats ? md_gn(rn, resid[src], b, c, cpg) : resid[src];
                if (a.relu) v = fmaxf(v, 0.f);
            }
            if (carrier) carrier[(((size_t)b * Ho + oy) * Wo + ox) * C + c] = v;
        }
        x3_put_s3(y + bp * 3 * C + c, C, v);
    }
}
