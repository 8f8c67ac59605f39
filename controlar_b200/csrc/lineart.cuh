// lineart.cuh — the LineArt control-map detector (reference condition/lineart.py:8-86), fp32 in the reference => fp32-grade here.
// Every wide convolution is one A_WIN launch of the split-bf16 ("x3", split3.cuh) implicit GEMM over an S3 source whose padding was
// written by the kernel that produced it (the stem's input: image_split3_kernel, reflect-pad 3, 8 channels per part); the kernels
// below are the rest of that glue:
//   instance norm  InstanceNorm2d defaults (affine=False, eps 1e-5, biased variance per (sample, channel)): the statistics are
//                  groupnorm.cuh's with one channel per group; the apply kernel here adds the residual, applies ReLU and writes the
//                  next convolution's padded input (reflect or zero, S3 or fp32) plus, where asked, the fp32 carrier
//   transposed     ConvTranspose2d(3, stride 2, pad 1, output_padding 1) as four sub-pixel stride-1 convolutions (parity class
//   convolution    (a, b) of the output): along an axis even outputs 2i take tap 1 of input i, odd outputs 2i+1 take tap 2 of input
//                  i and tap 0 of input i+1 (a zero row / column is appended at the bottom / right) -> windows of 1x1, 1x2, 2x1, 2x2
//   head           7x7 convolution to one channel + bias + sigmoid, direct fp32
#pragma once
#include "split3.cuh"

// ConvTranspose2d weight fp32 [Cin][Cout][3][3] -> W3 of the four parity classes back to back, class (a, b) in the order (0,0) (0,1)
// (1,0) (1,1), each [Cout][ty < 1+a][tx < 1+b][3 Cin_pad] = [ w_hi | w_hi | w_lo ]; window tap t of an odd class reads kernel tap 2 - 2t
__global__ void convT_weight_pack_x3_kernel(const float* __restrict__ w, bf16* __restrict__ y, int Cin, int Cout, int Cin_pad) {
    const long long per_tap = (long long)Cout * Cin_pad;
    const long long total = 9 * per_tap;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        long long r = i;
        int cls = 0, nt = 1;
        for (; cls < 4; ++cls) {                         // taps per class: 1, 2, 2, 4
            nt = (1 + (cls >> 1)) * (1 + (cls & 1));
            if (r < nt * per_tap) break;
            r -= nt * per_tap;
        }
        const int a = cls >> 1, bb = cls & 1, ntx = 1 + bb;
        const int c = (int)(r % Cin_pad);
        long long q = r / Cin_pad;
        const int tap = (int)(q % nt), o = (int)(q / nt);
        const int ty = tap / ntx, tx = tap - ty * ntx;
        const int ky = a ? 2 - 2 * ty : 1, kx = bb ? 2 - 2 * tx : 1;
        const float v = c < Cin ? w[(((size_t)c * Cout + o) * 3 + ky) * 3 + kx] : 0.f;
        x3_put_w3(y + (i - c) * 3 + c, Cin_pad, v);     // (i - c) = index of this (class, o, tap) row times Cin_pad
    }
}

// v = IN(x) (+ resid) (ReLU), in fp32, written as the next convolution's padded input y [B][H+pt+pb][W+pl+pr][C] (S3: 3C bf16 per
// pixel, else fp32), padding by reflection or zeros; carrier (optional) receives v at every unpadded pixel [B][H][W][C]
struct InApply { int pt, pl, pb, pr, reflect, s3, relu; };
__global__ void instnorm_apply_pad_kernel(const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ resid,
                                          float* __restrict__ carrier, void* __restrict__ y, int B, int H, int W, int C, InApply a) {
    const int Hp = H + a.pt + a.pb, Wp = W + a.pl + a.pr;
    const long long total = (long long)B * Hp * Wp * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long bp = i / C;
        const int px = (int)(bp % Wp);
        const long long r = bp / Wp;
        const int py = (int)(r % Hp), b = (int)(r / Hp);
        int sy = py - a.pt, sx = px - a.pl;
        const bool inside = sy >= 0 && sy < H && sx >= 0 && sx < W;
        float v = 0.f;
        if (inside || a.reflect) {
            sy = sy < 0 ? -sy : (sy >= H ? 2 * H - 2 - sy : sy);
            sx = sx < 0 ? -sx : (sx >= W ? 2 * W - 2 - sx : sx);
            const size_t src = (((size_t)b * H + sy) * W + sx) * C + c;
            const float* st = stats + ((size_t)b * C + c) * 2;
            v = (x[src] - st[0]) * st[1];
            if (resid) v += resid[src];
            if (a.relu) v = fmaxf(v, 0.f);
            if (carrier && inside) carrier[src] = v;
        }
        if (a.s3) x3_put_s3((bf16*)y + bp * 3 * C + c, C, v);
        else ((float*)y)[i] = v;
    }
}

// model4 (lineart.py:67-70): 7x7 convolution C -> 1 over the reflect-padded fp32 map [B][Ho+6][Wo+6][C] (C == 64), bias, sigmoid ->
// out [B][1][Ho][Wo].  One warp per output pixel: lane l holds channels 2l, 2l+1; taps in fixed order, then a fixed shuffle tree.
constexpr int LA_HEAD_C = 64;
__global__ void __launch_bounds__(256) lineart_head_kernel(const float* __restrict__ x, const float* __restrict__ w /*[C][7][7]*/, const float* __restrict__ bias,
                                                           float* __restrict__ out, int B, int Ho, int Wo) {
    __shared__ float2 sw[49][LA_HEAD_C / 2];
    for (int i = threadIdx.x; i < 49 * LA_HEAD_C; i += blockDim.x) {
        const int c = i / 49, t = i - c * 49;
        reinterpret_cast<float*>(&sw[t][0])[c] = w[i];
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, Wp = Wo + 6;
    const long long npix = (long long)B * Ho * Wo;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pix < npix; pix += warps) {
        const int ox = (int)(pix % Wo);
        const long long r = pix / Wo;
        const int oy = (int)(r % Ho), b = (int)(r / Ho);
        const float* base = x + (((size_t)b * (Ho + 6) + oy) * Wp + ox) * LA_HEAD_C + 2 * lane;
        float s = 0.f;
        for (int ky = 0; ky < 7; ++ky)
#pragma unroll
            for (int kx = 0; kx < 7; ++kx) {
                const float2 v = *reinterpret_cast<const float2*>(base + ((size_t)ky * Wp + kx) * LA_HEAD_C);
                const float2 q = sw[ky * 7 + kx][lane];
                s = fmaf(v.x, q.x, s); s = fmaf(v.y, q.y, s);
            }
        s = warp_sum(s);
        if (lane == 0) out[pix] = 1.0f / (1.0f + expf(-(s + bias[0])));
    }
}
