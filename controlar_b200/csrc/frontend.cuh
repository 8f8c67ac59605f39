// frontend.cuh — control-map / prompt front-end kernels (SURVEY.md §8 row f3): what runs right before generate().
//   Canny edges      condition/canny.py:14 (cv2.Canny, OpenCV 4.x, aperture 3, L1 gradient) — integer arithmetic, bit-exact
//   left-padding     autoregressive/sample/sample_t2i.py:146-156 (valid caption tokens rotated to the end, mask flipped)
// The Canny map is uint8 work: every stage below is integer and reproduces cv::Canny exactly (oracle/canny_oracle.py).
#pragma once
#include "common.cuh"

// per pixel: Sobel 3x3 (BORDER_REPLICATE) on every channel, norm = |dx| + |dy|, the FIRST channel with the largest norm wins.
// img uint8 [H][W][C] -> mag uint16, xs / ys int16 [H][W]
__global__ void canny_grad_kernel(const unsigned char* __restrict__ img, int H, int W, int C, unsigned short* __restrict__ mag,
                                  short* __restrict__ xs, short* __restrict__ ys) {
    const long long total = (long long)H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i / W), x = (int)(i - (long long)y * W);
        const int y0 = max(y - 1, 0), y2 = min(y + 1, H - 1), x0 = max(x - 1, 0), x2 = min(x + 1, W - 1);
        int best = -1, bdx = 0, bdy = 0;
        for (int c = 0; c < C; ++c) {
            auto px = [&](int yy, int xx) { return (int)img[((size_t)yy * W + xx) * C + c]; };
            const int p00 = px(y0, x0), p01 = px(y0, x), p02 = px(y0, x2);
            const int p10 = px(y, x0), p12 = px(y, x2);
            const int p20 = px(y2, x0), p21 = px(y2, x), p22 = px(y2, x2);
            const int dx = (p02 + 2 * p12 + p22) - (p00 + 2 * p10 + p20);
            const int dy = (p20 + 2 * p21 + p22) - (p00 + 2 * p01 + p02);
            const int n = abs(dx) + abs(dy);
            if (n > best) { best = n; bdx = dx; bdy = dy; }
        }
        mag[i] = (unsigned short)best; xs[i] = (short)bdx; ys[i] = (short)bdy;
    }
}

// non-maximum suppression + double threshold -> map: 0 none, 1 weak (kept, mag <= high), 2 edge (kept, mag > high)
__global__ void canny_nms_kernel(const unsigned short* __restrict__ mag, const short* __restrict__ xs, const short* __restrict__ ys, int H, int W,
                                 int low, int high, unsigned char* __restrict__ map) {
    const long long total = (long long)H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i / W), x = (int)(i - (long long)y * W);
        auto M = [&](int yy, int xx) { return (yy < 0 || yy >= H || xx < 0 || xx >= W) ? 0 : (int)mag[(size_t)yy * W + xx]; };   // zero border
        const int m = mag[i];
        unsigned char r = 0;
        if (m > low) {
            const int sx = xs[i], sy = ys[i];
            const int ax = abs(sx), ay = abs(sy) << 15;
            const int tg22x = ax * 13573;                                  // round(tan(22.5 deg) * 2^15)
            bool keep;
            if (ay < tg22x) keep = m > M(y, x - 1) && m >= M(y, x + 1);
            else {
                const int tg67x = tg22x + (ax << 16);
                if (ay > tg67x) keep = m > M(y - 1, x) && m >= M(y + 1, x);
                else {
                    const int s = ((sx ^ sy) < 0) ? -1 : 1;                // same sign: up-left / down-right
                    keep = m > M(y - 1, x - s) && m > M(y + 1, x + s);
                }
            }
            if (keep) r = m > high ? 2 : 1;
        }
        map[i] = r;
    }
}

// one hysteresis sweep: every 32 x 32 tile (+ 1 halo) is grown to its local fixed point in shared memory; *changed is set when any
// pixel of the image turned into an edge during this sweep (the caller repeats sweeps until a sweep changes nothing)
constexpr int CH_T = 32;
__global__ void __launch_bounds__(CH_T * CH_T / 4) canny_hyst_kernel(unsigned char* __restrict__ map, int H, int W, int* __restrict__ changed) {
    __shared__ unsigned char t[CH_T + 2][CH_T + 2];
    const int tx0 = blockIdx.x * CH_T, ty0 = blockIdx.y * CH_T;
    const int tid = threadIdx.x, nthr = blockDim.x;
    for (int i = tid; i < (CH_T + 2) * (CH_T + 2); i += nthr) {
        const int ly = i / (CH_T + 2), lx = i - ly * (CH_T + 2);
        const int y = ty0 + ly - 1, x = tx0 + lx - 1;
        t[ly][lx] = (y >= 0 && y < H && x >= 0 && x < W) ? map[(size_t)y * W + x] : 0;
    }
    __syncthreads();
    bool any = false;
    for (int it = 0; it < CH_T * CH_T; ++it) {       // (a chain inside a tile is at most this long; normally a handful of rounds)
        bool ch = false;
        for (int i = tid; i < CH_T * CH_T; i += nthr) {
            const int ly = i / CH_T + 1, lx = i % CH_T + 1;
            if (t[ly][lx] == 1) {
                const bool nb = t[ly - 1][lx - 1] == 2 || t[ly - 1][lx] == 2 || t[ly - 1][lx + 1] == 2 || t[ly][lx - 1] == 2 || t[ly][lx + 1] == 2 ||
                                t[ly + 1][lx - 1] == 2 || t[ly + 1][lx] == 2 || t[ly + 1][lx + 1] == 2;
                if (nb) { t[ly][lx] = 2; ch = true; }            // (monotone 1 -> 2: racing readers see 1 or 2, both fine)
            }
        }
        if (!__syncthreads_or(ch)) break;
        any = true;
    }
    if (any) {
        for (int i = tid; i < CH_T * CH_T; i += nthr) {
            const int ly = i / CH_T + 1, lx = i % CH_T + 1;
            const int y = ty0 + ly - 1, x = tx0 + lx - 1;
            if (y < H && x < W && t[ly][lx] == 2) map[(size_t)y * W + x] = 2;
        }
        if (tid == 0) *changed = 1;
    }
}
// edges uint8 [H][W]: 255 where the map says edge
__global__ void canny_finish_kernel(const unsigned char* __restrict__ map, unsigned char* __restrict__ out, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        out[i] = map[i] == 2 ? 255 : 0;
}

// left-padding of the caption embeddings (sample_t2i.py:146-156): out[b][i] = in[b][(i + valid_b) % L], valid_b = sum(mask_in[b]);
// mask_out[b][i] = mask_in[b][L - 1 - i].  Rows are copied as 16-byte words (row_bytes % 16 == 0).  One block per (b, i).
__global__ void left_pad_pack_kernel(const uint4* __restrict__ in, const long long* __restrict__ mask_in, uint4* __restrict__ out,
                                     long long* __restrict__ mask_out, int L, int row_words) {
    __shared__ int s_valid;
    const int b = blockIdx.x / L, i = blockIdx.x - b * L;
    if (threadIdx.x == 0) {
        int v = 0;
        for (int k = 0; k < L; ++k) v += mask_in[(size_t)b * L + k] != 0 ? 1 : 0;
        s_valid = v;
        mask_out[(size_t)b * L + i] = mask_in[(size_t)b * L + (L - 1 - i)];
    }
    __syncthreads();
    const int src = (i + s_valid) % L;
    const uint4* s = in + ((size_t)b * L + src) * row_words;
    uint4* d = out + ((size_t)b * L + i) * row_words;
    for (int k = threadIdx.x; k < row_words; k += blockDim.x) d[k] = s[k];
}

// ---- HED soft-edge detector (condition/hed.py:17-84), fp32 in the reference: the convolutions run on the fp32-grade split-bf16
// path ("x3", split3.cuh; the input minus the per-channel `norm` of ControlNetHED_Apache2.__call__ :47 is written by
// image_split3_kernel); the kernels below are the glue around them ----
// F.max_pool2d(kernel 2, stride 2) on NHWC fp32 (floor: odd trailing rows / columns are dropped), :29-30
__global__ void maxpool2_nhwc_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
    const int Ho = H / 2, Wo = W / 2;
    const long long total = (long long)B * Ho * Wo * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        long long r = i / C;
        const int xo = (int)(r % Wo); r /= Wo;
        const int yo = (int)(r % Ho);
        const int b = (int)(r / Ho);
        const float* p = x + (((size_t)b * H + 2 * yo) * W + 2 * xo) * C + c;
        y[i] = fmaxf(fmaxf(p[0], p[C]), fmaxf(p[(size_t)W * C], p[(size_t)W * C + C]));
    }
}
// DoubleConvBlock.projection (1x1 convolution to ONE channel, :25,34): one warp per pixel, fp32
__global__ void hed_proj_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ out,
                                long long npix, int C) {
    const long long pix = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pix >= npix) return;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(x[pix * C + c], w[c], s);
    s = warp_sum(s);
    if (lane == 0) out[pix] = s + b[0];
}
// HEDdetector.__call__ :75-78: the five projections resized to (H, W) with F.interpolate(mode='bilinear', align_corners=False),
// averaged, sigmoid, * 255, clamped.  maps[k]: [B][hk][wk] fp32.
struct HedMaps { const float* p[5]; int h[5], w[5]; };
__global__ void hed_merge_kernel(HedMaps m, int B, int H, int W, float* __restrict__ out) {
    const long long total = (long long)B * H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        const long long r = i / W;
        const int y = (int)(r % H), b = (int)(r / H);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const int hk = m.h[k], wk = m.w[k];
            const float* src = m.p[k] + (size_t)b * hk * wk;
            float v;
            if (hk == H && wk == W) v = src[(size_t)y * W + x];
            else {   // ATen upsample_bilinear2d: src = max(0, scale * (dst + 0.5) - 0.5), scale = in / out
                const float sy = fmaxf(((float)hk / (float)H) * ((float)y + 0.5f) - 0.5f, 0.f);
                const float sx = fmaxf(((float)wk / (float)W) * ((float)x + 0.5f) - 0.5f, 0.f);
                const int y0 = (int)sy, x0 = (int)sx;
                const int y1 = y0 + (y0 < hk - 1 ? 1 : 0), x1 = x0 + (x0 < wk - 1 ? 1 : 0);
                const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
                v = hy * (hx * src[(size_t)y0 * wk + x0] + lx * src[(size_t)y0 * wk + x1]) + ly * (hx * src[(size_t)y1 * wk + x0] + lx * src[(size_t)y1 * wk + x1]);
            }
            acc += v;
        }
        const float mean = acc / 5.0f;
        const float e = 1.0f / (1.0f + expf(-mean));
        out[i] = fminf(fmaxf(e * 255.0f, 0.f), 255.f);
    }
}
