// vision.cuh — normalisation / resampling / soft-max / quantiser kernels around the dense GEMM for the control
// encoder (HF Dinov2Model as used by autoregressive/models/dinov2_adapter.py) and the VQGAN tokenizer
// (tokenizer/tokenizer_image/vq_model.py).  The fp32-grade encoder's GroupNorm is groupnorm.cuh's.
#pragma once
#include "common.cuh"
#include "patch_embed.cuh"
#include "split3.cuh"

// nn.LayerNorm over the last dim (fp32 statistics, eps inside the sqrt), bf16 in/out.  one block per row.
__global__ void layernorm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, const bf16* __restrict__ b,
                                 bf16* __restrict__ y, int C, float eps, long long in_stride, long long out_stride) {
    __shared__ float red[32];
    const bf16* xr = x + (size_t)blockIdx.x * in_stride;
    bf16* yr = y + (size_t)blockIdx.x * out_stride;
    float s = 0.f;
    for (int i = threadIdx.x; i < C; i += blockDim.x) s += tof(xr[i]);
    const float mean = block_sum(s, red) / C;
    float v = 0.f;
    for (int i = threadIdx.x; i < C; i += blockDim.x) { const float d = tof(xr[i]) - mean; v += d * d; }
    const float rstd = rsqrtf(block_sum(v, red) / C + eps);
    for (int i = threadIdx.x; i < C; i += blockDim.x)
        yr[i] = fromf<bf16>((tof(xr[i]) - mean) * rstd * tof(w[i]) + tof(b[i]));
}

// row soft-max: fp32 scores [rows, ld_in] (first n valid) -> bf16 probabilities [rows, ld_out], zero padded
__global__ void softmax_rows_kernel(const float* __restrict__ s, bf16* __restrict__ p, int n, int ld_in, int ld_out) {
    __shared__ float red[32];
    const float* sr = s + (size_t)blockIdx.x * ld_in;
    bf16* pr = p + (size_t)blockIdx.x * ld_out;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, sr[i]);
    mx = block_max(mx, red);
    float sum = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) sum += expf(sr[i] - mx);
    sum = block_sum(sum, red);
    for (int i = threadIdx.x; i < ld_out; i += blockDim.x)
        pr[i] = fromf<bf16>(i < n ? expf(sr[i] - mx) / sum : 0.f);
}

// GroupNorm(32 groups, eps 1e-6, affine) statistics over NHWC bf16: one block per (b, group)
__global__ void groupnorm_stats_kernel(const bf16* __restrict__ x, float* __restrict__ stats /*[B*G][2]*/, int HW, int C, int G) {
    __shared__ float red[32];
    const int b = blockIdx.x / G, g = blockIdx.x % G, cg = C / G;
    const bf16* xb = x + (size_t)b * HW * C + g * cg;
    const long long n = (long long)HW * cg;
    float s = 0.f, ss = 0.f;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = tof(xb[(i / cg) * C + (i % cg)]);
        s += v; ss += v * v;
    }
    s = block_sum(s, red); ss = block_sum(ss, red);
    if (threadIdx.x == 0) {
        const float mean = s / n;
        stats[blockIdx.x * 2] = mean;
        stats[blockIdx.x * 2 + 1] = rsqrtf(fmaxf(ss / n - mean * mean, 0.f) + 1e-6f);
    }
}
// y = GN(x) (*swish): nonlinearity(x) = x*sigmoid(x), vq_model.py:355-357
__global__ void groupnorm_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ stats, const bf16* __restrict__ w,
                                       const bf16* __restrict__ bsh, bf16* __restrict__ y, long long total, int HW, int C, int G, int swish) {
    const int cg = C / G;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int b = (int)(i / ((long long)HW * C));
        const float* st = stats + ((size_t)b * G + c / cg) * 2;
        float v = (tof(x[i]) - st[0]) * st[1] * tof(w[c]) + tof(bsh[c]);
        if (swish) v = v / (1.0f + expf(-v));
        y[i] = fromf<bf16>(v);
    }
}

// ---- fused multi-head attention of the control encoders (Dinov2SelfAttention / ViTSelfAttention, head dim 64): one CTA = 64
// queries of one (image, head), 4 warps x 16 queries; key tiles of 64 stream through shared memory; S = q k^T * scale in fp32
// (mma.sync m16n8k16), online soft-max in fp32, probabilities rounded to bf16, ctx += P V (fp32 accumulate), bf16 out.
// Replaces the per-head S GEMM -> soft-max -> P V GEMM chain (fp32 S and bf16 P round trips through HBM: ~10 of DINOv2-small's 17 ms).
//   qk  [B*Tn][2C]: q at column hd*64, k at column C + hd*64 (bias included)      vT [B][C][Tp]: V^T per image, row = channel
//   ctx [B*Tn][C]
constexpr int FA_PITCH = 72;                                  // bf16 per shared-memory row (64 + 8: conflict-free 4-byte fragment loads)
__global__ void __launch_bounds__(128) vit_attention_kernel(const bf16* __restrict__ qk, const bf16* __restrict__ vT, bf16* __restrict__ ctx,
                                                             int Tn, int Tp, int C, float scale) {
    __shared__ __align__(16) bf16 sK[64 * FA_PITCH];          // [key][dim]
    __shared__ __align__(16) bf16 sV[64 * FA_PITCH];          // [dim][key]
    const int b = blockIdx.z, hd = blockIdx.y, q0 = blockIdx.x * 64;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const size_t ldq = (size_t)2 * C;
    // Q fragments of this warp's 16 rows (rows past Tn read row Tn - 1; their output is never stored)
    const int r_lo = min(q0 + warp * 16 + g, Tn - 1), r_hi = min(q0 + warp * 16 + g + 8, Tn - 1);
    const bf16* qlo = qk + ((size_t)b * Tn + r_lo) * ldq + hd * 64;
    const bf16* qhi = qk + ((size_t)b * Tn + r_hi) * ldq + hd * 64;
    uint32_t qa[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        qa[ks][0] = *reinterpret_cast<const uint32_t*>(qlo + ks * 16 + 2 * t);
        qa[ks][1] = *reinterpret_cast<const uint32_t*>(qhi + ks * 16 + 2 * t);
        qa[ks][2] = *reinterpret_cast<const uint32_t*>(qlo + ks * 16 + 8 + 2 * t);
        qa[ks][3] = *reinterpret_cast<const uint32_t*>(qhi + ks * 16 + 8 + 2 * t);
    }
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
    float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
    const bf16* kbase = qk + (size_t)b * Tn * ldq + C + hd * 64;
    const bf16* vbase = vT + ((size_t)b * C + hd * 64) * Tp;
    for (int k0 = 0; k0 < Tn; k0 += 64) {
        __syncthreads();                                       // previous tile consumed
        for (int i = tid; i < 64 * 8; i += 128) {              // 64 rows x 8 chunks of 16 bytes, both tiles
            const int r = i >> 3, c = i & 7;
            const int key = min(k0 + r, Tn - 1);               // keys past Tn are masked below
            *reinterpret_cast<uint4*>(sK + r * FA_PITCH + c * 8) = *reinterpret_cast<const uint4*>(kbase + (size_t)key * ldq + c * 8);
            const int kc = k0 + c * 8;                         // vT rows are padded to Tp (>= Tn, multiple of 32) and zero past Tn
            uint4 vv = make_uint4(0u, 0u, 0u, 0u);
            if (kc < Tp) vv = *reinterpret_cast<const uint4*>(vbase + (size_t)r * Tp + kc);
            *reinterpret_cast<uint4*>(sV + r * FA_PITCH + c * 8) = vv;
        }
        __syncthreads();
        // S tile 16 x 64
        float sacc[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sK + (j * 8 + g) * FA_PITCH + ks * 16 + 2 * t);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sK + (j * 8 + g) * FA_PITCH + ks * 16 + 8 + 2 * t);
                mma_bf16_16816(sacc[j], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
            }
        }
        // scale, mask the keys past Tn, running max
        float mx_lo = m_lo, mx_hi = m_hi;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = k0 + j * 8 + 2 * t + (e & 1);
                const float v = key < Tn ? sacc[j][e] * scale : -INFINITY;
                sacc[j][e] = v;
                if (e < 2) mx_lo = fmaxf(mx_lo, v); else mx_hi = fmaxf(mx_hi, v);
            }
        }
        mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1)); mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
        mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1)); mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
        const float c_lo = __expf(m_lo - mx_lo), c_hi = __expf(m_hi - mx_hi);     // exp(-inf) = 0 on the first tile
        m_lo = mx_lo; m_hi = mx_hi;
        l_lo *= c_lo; l_hi *= c_hi;
#pragma unroll
        for (int j = 0; j < 8; ++j) { o[j][0] *= c_lo; o[j][1] *= c_lo; o[j][2] *= c_hi; o[j][3] *= c_hi; }
        // probabilities -> bf16 A fragments (two adjacent 8-key blocks = one k16 step), row sums of the ROUNDED values
        uint32_t pa[4][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float p0 = rnd<bf16>(__expf(sacc[j][0] - m_lo)), p1 = rnd<bf16>(__expf(sacc[j][1] - m_lo));
            const float p2 = rnd<bf16>(__expf(sacc[j][2] - m_hi)), p3 = rnd<bf16>(__expf(sacc[j][3] - m_hi));
            l_lo += p0 + p1; l_hi += p2 + p3;
            __nv_bfloat162 lo2 = __floats2bfloat162_rn(p0, p1), hi2 = __floats2bfloat162_rn(p2, p3);
            pa[j >> 1][(j & 1) * 2 + 0] = *reinterpret_cast<uint32_t*>(&lo2);
            pa[j >> 1][(j & 1) * 2 + 1] = *reinterpret_cast<uint32_t*>(&hi2);
        }
        // ctx += P V : B fragments from V^T [dim][key]
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sV + (j * 8 + g) * FA_PITCH + ks * 16 + 2 * t);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sV + (j * 8 + g) * FA_PITCH + ks * 16 + 8 + 2 * t);
                mma_bf16_16816(o[j], pa[ks][0], pa[ks][1], pa[ks][2], pa[ks][3], b0, b1);
            }
        }
    }
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1); l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1); l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const int row_lo = q0 + warp * 16 + g, row_hi = row_lo + 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (row_lo < Tn) {
            __nv_bfloat162 v = __floats2bfloat162_rn(o[j][0] / l_lo, o[j][1] / l_lo);
            *reinterpret_cast<__nv_bfloat162*>(ctx + ((size_t)b * Tn + row_lo) * C + hd * 64 + j * 8 + 2 * t) = v;
        }
        if (row_hi < Tn) {
            __nv_bfloat162 v = __floats2bfloat162_rn(o[j][2] / l_hi, o[j][3] / l_hi);
            *reinterpret_cast<__nv_bfloat162*>(ctx + ((size_t)b * Tn + row_hi) * C + hd * 64 + j * 8 + 2 * t) = v;
        }
    }
}

// ---- GroupNorm(32), coalesced two-stage form (r2).  The one-block-per-(image, group) kernel above reads 8-byte pieces at a stride of
// C * 2 bytes (a quarter of every 32-byte sector) and wrote / read bf16 one element per thread: 19 ms per 8-image VQ decode.  Here
// every block streams a contiguous run of pixels with 16-byte loads, a thread keeps sums for the (at most two) groups its fixed
// 8-channel slot belongs to, partial sums are combined in a fixed order (deterministic), and a tiny second kernel folds the chunks.
constexpr int GN_CHUNKS = 64;                 // partial-sum chunks per image
__global__ void __launch_bounds__(256) groupnorm_partial_kernel(const bf16* __restrict__ x, float* __restrict__ part /*[B][GN_CHUNKS][32][2]*/, int HW, int C) {
    __shared__ float sh[256][4];
    const int b = blockIdx.y, chunk = blockIdx.x;
    const int C8 = C >> 3, cg = C >> 5;                      // 16-byte slots per pixel, channels per group (4, 8, 16, ...)
    const int ppi = 256 / C8;                                // pixels per block iteration (C8 divides 256: C in {128, 256, 512})
    const int slot = threadIdx.x % C8, prow = threadIdx.x / C8;
    const long long p0 = (long long)HW * chunk / GN_CHUNKS, p1 = (long long)HW * (chunk + 1) / GN_CHUNKS;
    float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;           // first / second half of the slot's 8 channels
    const uint4* base = reinterpret_cast<const uint4*>(x + (size_t)b * HW * C);
    for (long long pix = p0 + prow; pix < p1; pix += ppi) {
        const uint4 v = base[pix * C8 + slot];
        float a, c;
        unpack_bf16x2(v.x, a, c); s0 += a + c; q0 += a * a + c * c;
        unpack_bf16x2(v.y, a, c); s0 += a + c; q0 += a * a + c * c;
        unpack_bf16x2(v.z, a, c); s1 += a + c; q1 += a * a + c * c;
        unpack_bf16x2(v.w, a, c); s1 += a + c; q1 += a * a + c * c;
    }
    sh[threadIdx.x][0] = s0; sh[threadIdx.x][1] = q0; sh[threadIdx.x][2] = s1; sh[threadIdx.x][3] = q1;
    __syncthreads();
    if (threadIdx.x < 32) {                                   // thread g folds the partials of group g in a fixed order
        const int g = threadIdx.x;
        float s = 0.f, q = 0.f;
        for (int t = 0; t < 256; ++t) {
            const int sl = t % C8;
            const int c_lo = sl * 8, c_hi = sl * 8 + 4;       // first channels of the slot's two halves
            if (c_lo / cg == g) { s += sh[t][0]; q += sh[t][1]; }
            if (c_hi / cg == g) { s += sh[t][2]; q += sh[t][3]; }
        }
        float* o = part + (((size_t)b * GN_CHUNKS + chunk) * 32 + g) * 2;
        o[0] = s; o[1] = q;
    }
}
__global__ void groupnorm_finish_kernel(const float* __restrict__ part, float* __restrict__ stats /*[B*32][2]*/, int HW, int C) {
    const int bg = blockIdx.x * blockDim.x + threadIdx.x;     // b * 32 + g
    if (bg >= (int)gridDim.x * (int)blockDim.x) return;
    const int b = bg >> 5, g = bg & 31;
    float s = 0.f, q = 0.f;
    for (int c = 0; c < GN_CHUNKS; ++c) { const float* p = part + (((size_t)b * GN_CHUNKS + c) * 32 + g) * 2; s += p[0]; q += p[1]; }
    const float n = (float)HW * (float)(C >> 5);
    const float mean = s / n;
    stats[bg * 2] = mean;
    stats[bg * 2 + 1] = rsqrtf(fmaxf(q / n - mean * mean, 0.f) + 1e-6f);
}
// y = GN(x) (* swish), 8 channels (16 bytes) per thread
__global__ void groupnorm_apply8_kernel(const bf16* __restrict__ x, const float* __restrict__ stats, const bf16* __restrict__ w,
                                        const bf16* __restrict__ bsh, bf16* __restrict__ y, long long total8, int HW, int C, int swish) {
    const int C8 = C >> 3, cg = C >> 5;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total8; i += (long long)gridDim.x * blockDim.x) {
        const int slot = (int)(i % C8);
        const int b = (int)(i / ((long long)HW * C8));
        const uint4 v = reinterpret_cast<const uint4*>(x)[i];
        const uint4 wv = reinterpret_cast<const uint4*>(w)[slot], bv = reinterpret_cast<const uint4*>(bsh)[slot];
        const uint32_t vi[4] = {v.x, v.y, v.z, v.w}, wi[4] = {wv.x, wv.y, wv.z, wv.w}, bi[4] = {bv.x, bv.y, bv.z, bv.w};
        uint32_t oi[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int c = slot * 8 + 2 * k;
            const float* st = stats + ((size_t)b * 32 + c / cg) * 2;       // (both channels of a pair lie in one group: cg is even)
            float a0, a1, w0, w1, b0, b1;
            unpack_bf16x2(vi[k], a0, a1); unpack_bf16x2(wi[k], w0, w1); unpack_bf16x2(bi[k], b0, b1);
            float r0 = (a0 - st[0]) * st[1] * w0 + b0, r1 = (a1 - st[0]) * st[1] * w1 + b1;
            if (swish) { r0 = r0 / (1.0f + expf(-r0)); r1 = r1 / (1.0f + expf(-r1)); }
            __nv_bfloat162 o = __floats2bfloat162_rn(r0, r1);
            oi[k] = *reinterpret_cast<uint32_t*>(&o);
        }
        reinterpret_cast<uint4*>(y)[i] = make_uint4(oi[0], oi[1], oi[2], oi[3]);
    }
}
// last decoder convolution (conv_out, vq_model.py:193: 3x3, C -> 3 channels, fp32 NCHW image out).  An implicit GEMM would compute
// a 128-wide tile for 3 output channels; here one thread owns one pixel: 9 taps x C channels by 16-byte loads, weights in shared memory.
__global__ void __launch_bounds__(256) conv3x3_to3_kernel(const bf16* __restrict__ x /*NHWC*/, const bf16* __restrict__ w /*[3][9][C]*/,
                                                           const bf16* __restrict__ bias, float* __restrict__ out /*[B][3][H][W]*/, int B, int H, int W, int C) {
    extern __shared__ bf16 c3_w[];                             // [3][9][C]
    for (int i = threadIdx.x; i < 27 * C; i += blockDim.x) c3_w[i] = w[i];
    __syncthreads();
    const long long total = (long long)B * H * W;
    const int C8 = C >> 3;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int xx = (int)(i % W);
        const long long r = i / W;
        const int yy = (int)(r % H), b = (int)(r / H);
        float acc[3] = {0.f, 0.f, 0.f};
        for (int tap = 0; tap < 9; ++tap) {
            const int sy = yy + tap / 3 - 1, sx = xx + tap % 3 - 1;
            if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
            const uint4* px = reinterpret_cast<const uint4*>(x + (((size_t)b * H + sy) * W + sx) * C);
            for (int c8 = 0; c8 < C8; ++c8) {
                const uint4 v = px[c8];
                const uint32_t vi[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int o = 0; o < 3; ++o) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(c3_w + ((size_t)o * 9 + tap) * C + c8 * 8);
                    const uint32_t wi[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float a0, a1, w0, w1;
                        unpack_bf16x2(vi[k], a0, a1); unpack_bf16x2(wi[k], w0, w1);
                        acc[o] = fmaf(a0, w0, acc[o]); acc[o] = fmaf(a1, w1, acc[o]);
                    }
                }
            }
        }
#pragma unroll
        for (int o = 0; o < 3; ++o) out[(((size_t)b * 3 + o) * H + yy) * W + xx] = acc[o] + tof(bias[o]);
    }
}

// ---- layout / dtype conversions
template <typename TI>
__global__ void nchw_to_nhwc_bf16_kernel(const TI* __restrict__ x, bf16* __restrict__ y, int B, int C, int HW, int Cpad) {
    const long long total = (long long)B * HW * Cpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cpad);
        const long long bp = i / Cpad;
        const int pix = (int)(bp % HW), b = (int)(bp / HW);
        y[i] = c < C ? fromf<bf16>(tof(x[((size_t)b * C + c) * HW + pix])) : fromf<bf16>(0.f);
    }
}
// conv weight [Cout][Cin][kh][kw] (fp32 or bf16) -> bf16 [Cout][kh][kw][Cin_pad]
template <typename TI>
__global__ void conv_weight_pack_kernel(const TI* __restrict__ w, bf16* __restrict__ y, int Cout, int Cin, int KH, int KW, int Cin_pad) {
    const long long total = (long long)Cout * KH * KW * Cin_pad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cin_pad);
        long long r = i / Cin_pad;
        const int kx = (int)(r % KW); r /= KW;
        const int ky = (int)(r % KH);
        const int o = (int)(r / KH);
        y[i] = c < Cin ? fromf<bf16>(tof(w[(((size_t)o * Cin + c) * KH + ky) * KW + kx])) : fromf<bf16>(0.f);
    }
}
template <typename TI>
__global__ void cast_to_bf16_kernel(const TI* __restrict__ x, bf16* __restrict__ y, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        y[i] = fromf<bf16>(tof(x[i]));
}

// nearest-neighbour x2 up-sampling of an NHWC bf16 tensor (Upsample, vq_model.py:368-379), 16 bytes per thread; C % 8 == 0
__global__ void upsample2x_nhwc_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int B, int H, int W, int C) {
    const int C8 = C >> 3;
    const long long total = (long long)B * (2 * H) * (2 * W) * C8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        long long r = i / C8;
        const int X = (int)(r % (2 * W)); r /= 2 * W;
        const int Y = (int)(r % (2 * H));
        const int b = (int)(r / (2 * H));
        reinterpret_cast<uint4*>(y)[i] = reinterpret_cast<const uint4*>(x)[(((size_t)b * H + (Y >> 1)) * W + (X >> 1)) * C8 + c8];
    }
}

// ---- fp32-grade path of the VQGAN encoder (split-bf16 "x3" operands, split3.cuh).  VQModel.encode runs in fp32 in the reference
// (vq_model.py:41-46; sample / extract scripts keep the tokenizer in fp32) and its arg-min indices must come out the same.
// conv weight fp32 [Cout][Cin][kh][kw] -> W3 bf16 [Cout][kh][kw][3 Cin_pad] = [ w_hi | w_hi | w_lo ] per tap
__global__ void conv_weight_pack_x3_kernel(const float* __restrict__ w, bf16* __restrict__ y, int Cout, int Cin, int KH, int KW, int Cin_pad) {
    const long long total = (long long)Cout * KH * KW * Cin_pad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cin_pad);
        long long r = i / Cin_pad;
        const long long tapidx = r;                     // (o * KH + ky) * KW + kx
        const int kx = (int)(r % KW); r /= KW;
        const int ky = (int)(r % KH);
        const int o = (int)(r / KH);
        const float v = c < Cin ? w[(((size_t)o * Cin + c) * KH + ky) * KW + kx] : 0.f;
        x3_put_w3(y + tapidx * 3 * Cin_pad + c, Cin_pad, v);
    }
}
// soft-max over rows of fp32 scores, fp32 out (columns >= n of the padded row are zeroed)
__global__ void softmax_rows_f32_kernel(const float* __restrict__ s, float* __restrict__ p, int n, int ld) {
    __shared__ float red[32];
    const float* sr = s + (size_t)blockIdx.x * ld;
    float* pr = p + (size_t)blockIdx.x * ld;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, sr[i]);
    mx = block_max(mx, red);
    float sum = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) sum += expf(sr[i] - mx);
    sum = block_sum(sum, red);
    for (int i = threadIdx.x; i < ld; i += blockDim.x) pr[i] = i < n ? expf(sr[i] - mx) / sum : 0.f;
}
// v fp32 [B][hw][C] -> V^T as a B-side split operand [B][C][3 hwp]  ( hi | hi | lo over the hw dimension, zero padded to hwp )
__global__ void transpose_split3b_kernel(const float* __restrict__ v, bf16* __restrict__ y, int B, int hw, int hwp, int C) {
    const long long total = (long long)B * C * hwp;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % hwp);
        const long long bc = i / hwp;
        const int c = (int)(bc % C), b = (int)(bc / C);
        const float x = t < hw ? v[((size_t)b * hw + t) * C + c] : 0.f;
        x3_put_w3(y + bc * 3 * hwp + t, hwp, x);
    }
}

// x[b][0] = cls + pos[0];  x[b][1+i] = patch[b][i] + pos_i   (bf16 adds, modeling_dinov2.py Dinov2Embeddings.forward)
template <typename TI>
__global__ void dino_assemble_kernel(const bf16* __restrict__ patch, const TI* __restrict__ cls, const TI* __restrict__ pos0,
                                     const bf16* __restrict__ pos_i, bf16* __restrict__ x, int B, int hw, int C) {
    const long long total = (long long)B * (hw + 1) * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int t = (int)((i / C) % (hw + 1)), b = (int)(i / ((long long)C * (hw + 1)));
        float v;
        if (t == 0) v = rnd<bf16>(tof(cls[c])) + rnd<bf16>(tof(pos0[c]));
        else v = tof(patch[((size_t)b * hw + t - 1) * C + c]) + tof(pos_i[(size_t)(t - 1) * C + c]);
        x[i] = fromf<bf16>(v);
    }
}

// ---- VQ codebook: F.normalize(embedding, p=2, dim=-1) (eps 1e-12) in fp32; lookup -> NHWC bf16 padded to Kpad ch
__global__ void codebook_normalize_kernel(const float* __restrict__ e, float* __restrict__ en, int n, int d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float ss = 0.f;
    for (int k = 0; k < d; ++k) ss += e[(size_t)i * d + k] * e[(size_t)i * d + k];
    const float nrm = fmaxf(sqrtf(ss), 1e-12f);
    for (int k = 0; k < d; ++k) en[(size_t)i * d + k] = e[(size_t)i * d + k] / nrm;
}
__global__ void codebook_lookup_kernel(const float* __restrict__ en, const int* __restrict__ codes, bf16* __restrict__ out,
                                       long long npix, int d, int Kpad, int n_codes) {
    const long long total = npix * Kpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % Kpad);
        const long long pix = i / Kpad;
        int code = codes[pix];
        code = min(max(code, 0), n_codes - 1);
        out[i] = fromf<bf16>(k < d ? en[(size_t)code * d + k] : 0.f);
    }
}
// VectorQuantizer.forward (vq_model.py:216-236): z (fp32 [npix][d]) l2-normalised; d_j = |z|^2 + |e_j|^2 - 2 z.e_j;
// arg-min over j (lowest index on ties).  One thread per pixel, codebook broadcast through L1.
__global__ void vq_argmin_kernel(const float* __restrict__ z, const float* __restrict__ en, int* __restrict__ idx,
                                 float* __restrict__ zq /*[npix][d] or null*/, long long npix, int d, int n_codes) {
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    float zz[8];
    float ss = 0.f;
    for (int k = 0; k < 8; ++k) { zz[k] = k < d ? z[pix * d + k] : 0.f; ss += zz[k] * zz[k]; }
    const float nrm = fmaxf(sqrtf(ss), 1e-12f);
    float z2 = 0.f;
    for (int k = 0; k < 8; ++k) { zz[k] /= nrm; z2 += zz[k] * zz[k]; }
    float best = INFINITY; int bi = 0;
    for (int j = 0; j < n_codes; ++j) {
        float e2 = 0.f, dot = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) { const float ev = k < d ? __ldg(en + (size_t)j * d + k) : 0.f; e2 += ev * ev; dot += zz[k] * ev; }
        const float dist = (z2 + e2) - 2.f * dot;
        if (dist < best) { best = dist; bi = j; }
    }
    idx[pix] = bi;
    if (zq) for (int k = 0; k < d; ++k) zq[pix * d + k] = en[(size_t)bi * d + k];
}
// [npix][C] bf16 (NHWC) -> fp32 [npix][d] taking the first d channels
__global__ void take_channels_f32_kernel(const bf16* __restrict__ x, float* __restrict__ y, long long npix, int C, int d) {
    const long long total = npix * d;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        y[i] = tof(x[(i / d) * C + (i % d)]);
}
// zq [B*h*w][d] fp32 -> NCHW fp32 [B][d][h][w]
__global__ void nhwc_to_nchw_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int HW, int d) {
    const long long total = (long long)B * HW * d;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int pix = (int)(i % HW);
        const int k = (int)((i / HW) % d), b = (int)(i / ((long long)HW * d));
        y[i] = x[((size_t)b * HW + pix) * d + k];
    }
}

// ---------------------------------------------------------------------------------------------------------
// Antialiased bilinear resize along ONE axis (SURVEY.md §8 row f2): F.interpolate(x, size, mode='bilinear', align_corners=False,
// antialias=True) of the multi-resolution training scripts (autoregressive/train/train_t2i_depth_multiscale.py:44-56) is two of
// these passes, width then height.  Third-party arithmetic (ATen _upsample_bilinear2d_aa, HelperInterpBase::
// _compute_indices_min_size_weights_aa; restated in oracle/resize_oracle.py): triangle filter stretched by the down-scale factor,
// every weight computed in fp32 exactly as ATen does — scale = in / out, support = max(scale, 1), centre = scale (i + 0.5),
// taps [max(int(c - support + 0.5), 0), min(int(c + support + 0.5), in)), w_j = max(0, 1 - |(j - c + 0.5) / max(scale, 1)|) / sum.
// Tensor viewed as [outer][n_in][inner] -> [outer][n_out][inner] (inner = 1: width pass; inner = W_out: height pass).
// HBM-bound gather: consecutive threads take consecutive `inner` (height pass) or consecutive outputs of a row (width pass).
// ---------------------------------------------------------------------------------------------------------
__global__ void resize_aa_axis_kernel(const float* __restrict__ in, float* __restrict__ out, long long outer, int n_in, int n_out, int inner) {
    const float scale = (float)n_in / (float)n_out;
    const float support = scale >= 1.f ? scale : 1.f;
    const float inv = scale >= 1.f ? 1.f / scale : 1.f;
    const long long total = outer * n_out * inner;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(i % inner);
        const long long t = i / inner;
        const int o = (int)(t % n_out);
        const long long r = t / n_out;
        const float c = scale * ((float)o + 0.5f);
        const int lo = max((int)(c - support + 0.5f), 0);
        const int hi = min((int)(c + support + 0.5f), n_in);
        float tot = 0.f;
        for (int j = lo; j < hi; ++j) tot += fmaxf(0.f, 1.f - fabsf(((float)j - c + 0.5f) * inv));
        const float* src = in + (r * n_in) * inner + q;
        float acc = 0.f;
        for (int j = lo; j < hi; ++j) {
            const float w = fmaxf(0.f, 1.f - fabsf(((float)j - c + 0.5f) * inv)) / tot;
            acc += w * src[(size_t)j * inner];
        }
        out[i] = acc;
    }
}
