// dpt.cuh — the DPT depth detector (HF transformers DPTForDepthEstimation, non-hybrid ViT backbone), fp32 in the reference =>
// fp32-grade here.  Every GEMM and 3x3 stride-1 convolution runs on the fp32-output wgmma instantiation (gemm_wgmma.cuh) over
// split-bf16 "x3" operands (split3.cuh): activations S3 = [ hi | lo | hi ], weights W3 = [ w_hi | w_hi | w_lo ].  The kernels below
// are the fp32 glue that writes each S3 operand, plus the fused attention and the 1x1 output head (fp32 rows, optionally through
// exact GELU, go through split3_rows_kernel):
//   patchify       image NCHW -> S3 rows of the 16x16/16 patch convolution, K index c * 256 + ky * 16 + kx (the weight's order)
//   assemble       [CLS] + patch tokens + position embeddings bilinearly resized (align_corners=False) from the stored grid
//   layernorm      two-pass fp32 row statistics (mean, then centred squares) -> S3 row
//   readout        S3 of cat(token, [CLS]) per patch token (readout_type "project")
//   image          fp32 NHWC (or the GEMM output of a k = s ConvTranspose2d, pixel shuffle folded in) -> S3 NHWC image, optionally
//                  + a second map (the fusion add, also written back in fp32), ReLU, or a x2 bilinear upsample (align_corners=True);
//                  written into a zero-filled frame of [Hp][Wp] pixels at offset (pt, pl) (padding for the window convolution, or
//                  the minimum box of the TMA convolution)
//   attention      fused multi-head attention for 64-dim heads: scores and probabilities stay in registers (online soft-max)
//   head           ReLU -> 1x1 convolution to one channel + bias -> ReLU, direct fp32
#pragma once
#include "split3.cuh"

// ConvTranspose2d(k = s = f) weight fp32 [Cin][Cout][f][f] -> W3 [(ky f + kx) Cout + o][3 Cin]: the transposed convolution is one
// GEMM whose output row is an input pixel and whose column is (ky, kx, o) of its f x f output block
__global__ void dpt_convT_pack_kernel(const float* __restrict__ w, bf16* __restrict__ y, int Cin, int Cout, int f) {
    const long long total = (long long)f * f * Cout * Cin;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cin);
        const long long n = i / Cin;
        const int o = (int)(n % Cout), tap = (int)(n / Cout), ky = tap / f, kx = tap - ky * f;
        x3_put_w3(y + n * 3 * Cin + c, Cin, w[(((size_t)c * Cout + o) * f + ky) * f + kx]);
    }
}

// pixel_values fp32 NCHW [B][3][16 h][16 h] -> S3 rows [B h^2][3 * 768]
__global__ void dpt_patchify_kernel(const float* __restrict__ x, bf16* __restrict__ y, int B, int h) {
    const int K = 3 * 256, H = 16 * h;
    const long long total = (long long)B * h * h * K;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % K);
        const long long row = i / K;
        const int p = (int)(row % (h * h)), b = (int)(row / (h * h));
        const int c = k >> 8, ky = (k >> 4) & 15, kx = k & 15, py = p / h, px = p - py * h;
        x3_put_s3(y + row * 3 * K + k, K, x[(((size_t)b * 3 + c) * H + 16 * py + ky) * H + 16 * px + kx]);
    }
}

// X [B][1 + h w][C]: row 0 = cls + pos[0], row 1 + p = patch[b, p] + bilinear(pos grid g x g -> h x w, align_corners=False)[p]
__global__ void dpt_assemble_kernel(const float* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos, float* __restrict__ X,
                                    int B, int h, int w, int g, int C) {
    const int T = 1 + h * w;
    const long long total = (long long)B * T * C;
    const float scale_y = (float)g / (float)h, scale_x = (float)g / (float)w;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long r = i / C;
        const int t = (int)(r % T), b = (int)(r / T);
        if (t == 0) { X[i] = cls[c] + pos[c]; continue; }
        const int p = t - 1, oy = p / w, ox = p - oy * w;
        // torch upsample_bilinear2d, align_corners=False: src = max(scale * (dst + 0.5) - 0.5, 0)
        const float sy = fmaxf(scale_y * (oy + 0.5f) - 0.5f, 0.f), sx = fmaxf(scale_x * (ox + 0.5f) - 0.5f, 0.f);
        const int y0 = (int)sy, x0 = (int)sx, y1 = y0 + (y0 < g - 1), x1 = x0 + (x0 < g - 1);
        const float ly = sy - y0, lx = sx - x0;
        const float* P = pos + C + c;
        const float v00 = P[(size_t)(y0 * g + x0) * C], v01 = P[(size_t)(y0 * g + x1) * C];
        const float v10 = P[(size_t)(y1 * g + x0) * C], v11 = P[(size_t)(y1 * g + x1) * C];
        const float pe = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
        X[i] = patch[((size_t)b * h * w + p) * C + c] + pe;
    }
}

// LayerNorm (biased variance, eps) of each row of X [M][C] -> S3 rows [M][3C]; one block per row, fixed reduction order
constexpr int DPT_LN_THREADS = 256;
__global__ void __launch_bounds__(DPT_LN_THREADS) dpt_layernorm_split_kernel(const float* __restrict__ X, const float* __restrict__ w,
                                                                            const float* __restrict__ bias, bf16* __restrict__ y, int C, float eps) {
    __shared__ float red[DPT_LN_THREADS / 32];
    const float* x = X + (size_t)blockIdx.x * C;
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += DPT_LN_THREADS) s += x[c];
    const float mean = block_sum<DPT_LN_THREADS / 32>(s, red) / (float)C;
    float q = 0.f;
    for (int c = threadIdx.x; c < C; c += DPT_LN_THREADS) { const float d = x[c] - mean; q = fmaf(d, d, q); }
    const float rstd = 1.0f / sqrtf(block_sum<DPT_LN_THREADS / 32>(q, red) / (float)C + eps);
    bf16* o = y + (size_t)blockIdx.x * 3 * C;
    for (int c = threadIdx.x; c < C; c += DPT_LN_THREADS) x3_put_s3(o + c, C, (x[c] - mean) * rstd * w[c] + bias[c]);
}

// readout "project": S3 rows [B h^2][3 * 2C] of cat(X[b, 1 + p], X[b, 0])
__global__ void dpt_readout_split_kernel(const float* __restrict__ X, bf16* __restrict__ y, int B, int hh, int C) {
    const int T = 1 + hh, K = 2 * C;
    const long long total = (long long)B * hh * K;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % K);
        const long long row = i / K;
        const int p = (int)(row % hh), b = (int)(row / hh);
        const float v = k < C ? X[((size_t)b * T + 1 + p) * C + k] : X[(size_t)b * T * C + (k - C)];
        x3_put_s3(y + row * 3 * K + k, K, v);
    }
}

// S3 NHWC image y [B][Hp][Wp][3C] of an Ho x Wo map placed at (pt, pl), zeros elsewhere.  Source a:
//   shuf == 0, up == 0 : fp32 NHWC [B][Ho][Wo][C] (+ b of the same shape; the sum is also written to sum_out when given)
//   shuf == f          : ConvTranspose2d(k = s = f) GEMM output [B][Ho/f][Wo/f][f][f][C] (pixel shuffle)
//   up == 1            : fp32 NHWC [B][Ho/2][Wo/2][C], x2 bilinear upsample with align_corners=True
// then ReLU when asked
struct DptImg { int B, Ho, Wo, C, Hp, Wp, pt, pl, shuf, up, relu; };
__global__ void dpt_image_split_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ sum_out, bf16* __restrict__ y,
                                       DptImg q) {
    const long long total = (long long)q.B * q.Hp * q.Wp * q.C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % q.C);
        const long long bp = i / q.C;
        const int px = (int)(bp % q.Wp);
        const long long r = bp / q.Wp;
        const int py = (int)(r % q.Hp), n = (int)(r / q.Hp);
        const int oy = py - q.pt, ox = px - q.pl;
        float v = 0.f;
        if (oy >= 0 && oy < q.Ho && ox >= 0 && ox < q.Wo) {
            if (q.shuf) {
                const int f = q.shuf, hs = q.Ho / f, ws = q.Wo / f;
                v = a[((((size_t)n * hs + oy / f) * ws + ox / f) * f * f + (oy % f) * f + ox % f) * q.C + c];
            } else if (q.up) {
                const int hs = q.Ho / 2, ws = q.Wo / 2;
                const float ry = q.Ho > 1 ? (float)(hs - 1) / (float)(q.Ho - 1) : 0.f, rx = q.Wo > 1 ? (float)(ws - 1) / (float)(q.Wo - 1) : 0.f;
                const float sy = ry * oy, sx = rx * ox;
                const int y0 = (int)sy, x0 = (int)sx, y1 = y0 + (y0 < hs - 1), x1 = x0 + (x0 < ws - 1);
                const float ly = sy - y0, lx = sx - x0;
                const float* A = a + (size_t)n * hs * ws * q.C + c;
                const float v00 = A[(size_t)(y0 * ws + x0) * q.C], v01 = A[(size_t)(y0 * ws + x1) * q.C];
                const float v10 = A[(size_t)(y1 * ws + x0) * q.C], v11 = A[(size_t)(y1 * ws + x1) * q.C];
                v = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
            } else {
                const size_t src = (((size_t)n * q.Ho + oy) * q.Wo + ox) * q.C + c;
                v = a[src];
                if (b) v += b[src];
                if (sum_out) sum_out[src] = v;
            }
            if (q.relu) v = fmaxf(v, 0.f);
        }
        x3_put_s3(y + bp * 3 * q.C + c, q.C, v);
    }
}

// ---- fused multi-head attention, 64-dim heads, fp32 grade.  qkv fp32 [B][T][3C] (q | k | v, head h at columns 64 h ..), out S3
// rows [B][T][3C] of the context (the output projection's A operand).  grid (ceil(T / 64), heads, B), 4 warps x 16 query rows.
// Every product is hi·hi + lo·hi + hi·lo on mma.sync m16n8k16 with fp32 accumulation; q is scaled by 1/8 (exact) before the split.
// Key blocks of 64 run in a fixed order and the soft-max is online in fp32, so results do not depend on the batch or the launch.
constexpr int DPT_AT_B = 64, DPT_AT_LD = 72;            // keys per block, shared row pitch (bf16; 36 words: conflict-free)
__device__ __forceinline__ uint32_t dpt_pack(bf16 a, bf16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
__device__ __forceinline__ void dpt_split2(float x, float y, uint32_t& hi, uint32_t& lo) {
    bf16 xh, xl, yh, yl;
    x3_split(x, xh, xl); x3_split(y, yh, yl);
    hi = dpt_pack(xh, yh); lo = dpt_pack(xl, yl);
}
__device__ __forceinline__ void dpt_mma3(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint32_t bh0, uint32_t bh1, uint32_t bl0,
                                         uint32_t bl1) {
    mma_bf16_16816(c, ah[0], ah[1], ah[2], ah[3], bh0, bh1);
    mma_bf16_16816(c, al[0], al[1], al[2], al[3], bh0, bh1);
    mma_bf16_16816(c, ah[0], ah[1], ah[2], ah[3], bl0, bl1);
}
__global__ void __launch_bounds__(128) dpt_attention_kernel(const float* __restrict__ qkv, bf16* __restrict__ out, int T, int C) {
    __shared__ __align__(16) bf16 sk[2][DPT_AT_B][DPT_AT_LD];     // K hi / lo   [key][dim]
    __shared__ __align__(16) bf16 sv[2][64][DPT_AT_LD];           // V^T hi / lo [dim][key]
    const int h = blockIdx.y, bz = blockIdx.z, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const size_t ld = 3 * (size_t)C;
    const float* base = qkv + (size_t)bz * T * ld + h * 64;
    const int r0 = blockIdx.x * 64 + warp * 16 + g, r1 = r0 + 8;

    uint32_t qh[4][4], ql[4][4];                                  // A fragments of q / 8, per k16 step of the head dimension
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int row = (i & 1) ? r1 : r0, col = kk * 16 + 2 * t + ((i >> 1) << 3);
            float2 v = make_float2(0.f, 0.f);
            if (row < T) v = *reinterpret_cast<const float2*>(base + (size_t)row * ld + col);
            dpt_split2(v.x * 0.125f, v.y * 0.125f, qh[kk][i], ql[kk][i]);
        }
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;       // running max / partial sums of rows r0, r1

    const int nkb = (T + DPT_AT_B - 1) / DPT_AT_B;
    for (int kb = 0; kb < nkb; ++kb) {
        __syncthreads();
#pragma unroll
        for (int it = 0; it < 8; ++it) {                           // 64 keys x 16 float4 of k and of v
            const int idx = tid + it * 128, key = idx >> 4, d = (idx & 15) * 4, kg = kb * DPT_AT_B + key;
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (kg < T) {
                kv = *reinterpret_cast<const float4*>(base + (size_t)kg * ld + C + d);
                vv = *reinterpret_cast<const float4*>(base + (size_t)kg * ld + 2 * C + d);
            }
            const float ke[4] = {kv.x, kv.y, kv.z, kv.w}, ve[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                x3_split(ke[e], sk[0][key][d + e], sk[1][key][d + e]);
                x3_split(ve[e], sv[0][d + e][key], sv[1][d + e][key]);
            }
        }
        __syncthreads();

        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const int key = j * 8 + g, c0 = kk * 16 + 2 * t;
                dpt_mma3(s[j], qh[kk], ql[kk], *reinterpret_cast<const uint32_t*>(&sk[0][key][c0]), *reinterpret_cast<const uint32_t*>(&sk[0][key][c0 + 8]),
                         *reinterpret_cast<const uint32_t*>(&sk[1][key][c0]), *reinterpret_cast<const uint32_t*>(&sk[1][key][c0 + 8]));
            }
        }
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (kb * DPT_AT_B + j * 8 + 2 * t + e >= T) { s[j][e] = -INFINITY; s[j][2 + e] = -INFINITY; }
                mx0 = fmaxf(mx0, s[j][e]); mx1 = fmaxf(mx1, s[j][2 + e]);
            }
#pragma unroll
        for (int off = 1; off < 4; off <<= 1) {
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
        }
        const float a0 = expf(m0 - mx0), a1 = expf(m1 - mx1);     // block 0 always holds a valid key: mx is finite
        m0 = mx0; m1 = mx1;
        l0 *= a0; l1 *= a1;
#pragma unroll
        for (int j = 0; j < 8; ++j) { o[j][0] *= a0; o[j][1] *= a0; o[j][2] *= a1; o[j][3] *= a1; }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = expf(s[j][0] - m0); s[j][1] = expf(s[j][1] - m0); s[j][2] = expf(s[j][2] - m1); s[j][3] = expf(s[j][3] - m1);
            l0 += s[j][0] + s[j][1]; l1 += s[j][2] + s[j][3];
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {                           // P (accumulator layout) is the A fragment of P·V directly
            uint32_t ph[4], pl[4];
            dpt_split2(s[2 * kk][0], s[2 * kk][1], ph[0], pl[0]);
            dpt_split2(s[2 * kk][2], s[2 * kk][3], ph[1], pl[1]);
            dpt_split2(s[2 * kk + 1][0], s[2 * kk + 1][1], ph[2], pl[2]);
            dpt_split2(s[2 * kk + 1][2], s[2 * kk + 1][3], ph[3], pl[3]);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int dim = j * 8 + g, c0 = kk * 16 + 2 * t;
                dpt_mma3(o[j], ph, pl, *reinterpret_cast<const uint32_t*>(&sv[0][dim][c0]), *reinterpret_cast<const uint32_t*>(&sv[0][dim][c0 + 8]),
                         *reinterpret_cast<const uint32_t*>(&sv[1][dim][c0]), *reinterpret_cast<const uint32_t*>(&sv[1][dim][c0 + 8]));
            }
        }
    }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, off);
        l1 += __shfl_xor_sync(0xffffffffu, l1, off);
    }
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int row = hh ? r1 : r0;
        if (row >= T) continue;
        const float inv = hh ? i1 : i0;
        bf16* dst = out + ((size_t)bz * T + row) * ld + h * 64;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            uint32_t hi, lo;
            dpt_split2(o[j][2 * hh] * inv, o[j][2 * hh + 1] * inv, hi, lo);
            const int col = j * 8 + 2 * t;
            *reinterpret_cast<uint32_t*>(dst + col) = hi;
            *reinterpret_cast<uint32_t*>(dst + C + col) = lo;
            *reinterpret_cast<uint32_t*>(dst + 2 * C + col) = hi;
        }
    }
}

// head.head.3-5: ReLU -> Conv2d(32, 1, 1) + bias -> ReLU over fp32 NHWC [npix][32] -> depth [npix]; one warp per pixel, lane = channel
__global__ void __launch_bounds__(256) dpt_head_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                       float* __restrict__ out, long long npix) {
    const int lane = threadIdx.x & 31;
    const float wl = w[lane];
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < npix; p += warps) {
        const float s = warp_sum(fmaxf(x[p * 32 + lane], 0.f) * wl);
        if (lane == 0) out[p] = fmaxf(s + bias[0], 0.f);
    }
}
