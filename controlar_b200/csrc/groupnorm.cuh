// groupnorm.cuh — fp32 normalisation of the fp32-grade networks: GroupNorm statistics over NHWC fp32 maps, shared by the VQ
// encoder's and MiDaS's GroupNorm(32) (cpg = C / 32 channels per group) and LineArt's InstanceNorm (cpg = 1), and the GroupNorm
// apply that writes the next convolution's split-bf16 ("x3", split3.cuh) operand.  LineArt's InstanceNorm apply, the only one with
// reflection padding and fp32 output, stays in lineart.cuh and reads these statistics.
//   statistics  two passes, mean then centred squares, three launches: gn_partial_kernel<false> writes per-channel sums of each
//               pixel chunk, gn_partial_kernel<true> per-channel sums of squared deviations from the group mean, gn_finish_kernel
//               folds them into stats [B][C/cpg][2] = (mean, 1 / sqrtf(biased variance + eps)).  A block covers 32 channels x 8
//               pixel rows, reading 32 consecutive floats per pixel; pixel chunk j of nch = gn_nch(HW) covers [j*per, (j+1)*per).
//               Every sum has a fixed order that depends on (HW, C, cpg) only, never on B, so a sample's statistics do not depend on
//               the batch: a chunk's 8 rows are added in row order, a channel's chunks in chunk order, a group's channels in
//               channel order.  Needs C % 32 == 0 and cpg dividing 32.
#pragma once
#include "split3.cuh"

constexpr int GN_THREADS = 256;                     // 32 channels x 8 pixel rows
constexpr int GN_MAX_CHUNKS = 64;
// pixel chunks per image: about 2048 pixels each, at most GN_MAX_CHUNKS
inline int gn_nch(int HW) { return std::max(1, std::min(GN_MAX_CHUNKS, (HW + 2047) / 2048)); }

// channel c's total over the nch chunk partials part [B][nch][C] of image b
__device__ __forceinline__ float gn_chan(const float* __restrict__ part, int b, int nch, int C, int c) {
    float s = 0.f;
    for (int j = 0; j < nch; ++j) s += part[((size_t)b * nch + j) * C + c];
    return s;
}
// a group's total from its cpg channel totals t[0 .. cpg)
__device__ __forceinline__ float gn_group(const float* t, int cpg) {
    float s = t[0];
    for (int k = 1; k < cpg; ++k) s += t[k];
    return s;
}

// grid (C/32, B, nch): part [B][nch][C] = sum over chunk j of x (CENTRED: of (x - group mean)^2, the mean from part_s)
template <bool CENTRED>
__global__ void __launch_bounds__(GN_THREADS) gn_partial_kernel(const float* __restrict__ x, const float* __restrict__ part_s,
                                                                 float* __restrict__ part, int HW, int C, int cpg) {
    __shared__ float red[GN_THREADS / 32][32];
    const int lane = threadIdx.x & 31, row = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane, b = blockIdx.y, j = blockIdx.z, nch = gridDim.z;
    float mean = 0.f;
    if (CENTRED) {
        __shared__ float tot[32];
        if (row == 0) tot[lane] = gn_chan(part_s, b, nch, C, c);
        __syncthreads();
        mean = gn_group(tot + lane / cpg * cpg, cpg) / ((float)HW * (float)cpg);
    }
    const int per = (HW + nch - 1) / nch;
    const int p0 = j * per, p1 = min(HW, p0 + per);
    const float* xb = x + (size_t)b * HW * C + c;
    float s = 0.f;
    for (int p = p0 + row; p < p1; p += GN_THREADS / 32) {
        const float v = xb[(size_t)p * C];
        if (CENTRED) { const float d = v - mean; s = fmaf(d, d, s); } else s += v;
    }
    red[row][lane] = s;
    __syncthreads();
    if (row == 0) {
        float t = 0.f;
        for (int k = 0; k < GN_THREADS / 32; ++k) t += red[k][lane];
        part[((size_t)b * nch + j) * C + c] = t;
    }
}
// grid (C/32, B), 32 threads: stats [B][C/cpg][2] = (mean, 1 / sqrtf(biased variance + eps))
__global__ void __launch_bounds__(32) gn_finish_kernel(const float* __restrict__ part_s, const float* __restrict__ part_q,
                                                       float* __restrict__ stats, int HW, int C, int cpg, int nch, float eps) {
    __shared__ float ts[32], tq[32];
    const int lane = threadIdx.x, c = blockIdx.x * 32 + lane, b = blockIdx.y;
    ts[lane] = gn_chan(part_s, b, nch, C, c);
    tq[lane] = gn_chan(part_q, b, nch, C, c);
    __syncwarp();
    if (lane % cpg) return;
    const float n = (float)HW * (float)cpg;
    float* o = stats + ((size_t)b * (C / cpg) + c / cpg) * 2;
    o[0] = gn_group(ts + lane, cpg) / n;
    o[1] = 1.0f / sqrtf(gn_group(tq + lane, cpg) / n + eps);
}

// ---- GroupNorm(32) apply: v = GN(x) (+ r) (act) with r = resid, or GN_r(resid) when rn.stats is given; with pool (ReLU only), the
// 3x3 / stride 2 max-pool (TF "SAME": no padding before, one after) of that over an even H x W map.  The Ho x Wo result (Ho = H / 2
// with pool, else H) is written as S3 (3C bf16 per pixel) into a zero-filled frame [B][Hp][Wp] at (pt, pl), and, when carrier is
// given, as fp32 [B][Ho][Wo][C].
constexpr int GN_GROUPS = 32;
enum { GN_ACT_NONE = 0, GN_ACT_RELU = 1, GN_ACT_SWISH = 2 };
struct GnApply { int pt, pl, Hp, Wp, act, pool; };
struct GnAffine { const float* stats; const float* w; const float* b; };
__device__ __forceinline__ float gn_affine(const GnAffine& a, float v, int b, int c, int cpg) {
    const float* st = a.stats + ((size_t)b * GN_GROUPS + c / cpg) * 2;
    return (v - st[0]) * st[1] * a.w[c] + a.b[c];
}
__global__ void gn_apply_s3_kernel(const float* __restrict__ x, GnAffine n, const float* __restrict__ resid, GnAffine rn,
                                   float* __restrict__ carrier, bf16* __restrict__ y, int B, int H, int W, int C, GnApply a) {
    const int cpg = C / GN_GROUPS, Ho = a.pool ? H / 2 : H, Wo = a.pool ? W / 2 : W;
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
                        if (iy < H && ix < W) v = fmaxf(v, fmaxf(gn_affine(n, x[(((size_t)b * H + iy) * W + ix) * C + c], b, c, cpg), 0.f));
                    }
            } else {
                const size_t src = (((size_t)b * H + oy) * W + ox) * C + c;
                v = gn_affine(n, x[src], b, c, cpg);
                if (resid) v += rn.stats ? gn_affine(rn, resid[src], b, c, cpg) : resid[src];
                if (a.act == GN_ACT_RELU) v = fmaxf(v, 0.f);
                else if (a.act == GN_ACT_SWISH) v = v / (1.0f + expf(-v));      // nonlinearity(x) = x * sigmoid(x), vq_model.py:355-357
            }
            if (carrier) carrier[(((size_t)b * Ho + oy) * Wo + ox) * C + c] = v;
        }
        x3_put_s3(y + bp * 3 * C + c, C, v);
    }
}
