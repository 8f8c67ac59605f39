// train_bwd.cuh — kernels of the BACKWARD of the teacher-forced training forward (SURVEY.md §8 row f1).  In the reference the
// backward is autograd's (autoregressive/train/train_c2i_canny.py:200-211 `scaler.scale(loss).backward()`) over
// Transformer.forward (autoregressive/models/gpt_t2i.py:420-431,451-484) under bf16 autocast; here every step is written out
// (formulas validated on CPU against autograd: oracle/train_backward_manual.py, tests/test_train_backward_cpu.py):
// gradients are bf16 wherever autograd produces bf16 ones (operands / results of nn.Linear, SDPA, GELU, SiLU) and fp32 on the
// residual stream, RMSNorm and the loss.  First correct path: the GEMMs (dgrad = dY W, wgrad = dY^T X) run on the dense
// tensor-core kernels through explicit transposes, attention is two plain one-warp-per-row kernels; fusing is future work.
#pragma once
#include "common.cuh"
#include "dropout.cuh"
#include "train.cuh"

// dst[c][r] = src[r][c] for r < rows, 0 for rows <= r < ldp: the K-major operand the [N][K] x [M][K]^T GEMM kernels want,
// with the reduction extent padded to a whole number of 64-element K tiles.  block (32, 8), grid (ceil(ldp/32), ceil(cols/32)).
__global__ void tr_transpose_pad_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int rows, int cols, int ldp) {
    __shared__ bf16 tile[32][33];
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int r = r0 + j, c = c0 + threadIdx.x;
        tile[j][threadIdx.x] = (r < rows && c < cols) ? src[(size_t)r * cols + c] : __float2bfloat16_rn(0.f);
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int c = c0 + j, r = r0 + threadIdx.x;
        if (c < cols && r < ldp) dst[(size_t)c * ldp + r] = tile[threadIdx.x][j];
    }
}

// the cast at the end of a weight-gradient GEMM: autograd's bf16 gradient of the autocast copy -> fp32 .grad of the master.
// dst [rows][cols] fp32 = src [rows][lds] bf16 (columns >= cols of src are padding, dropped)
__global__ void tr_bf16_to_f32_2d_kernel(const bf16* __restrict__ src, int lds, float* __restrict__ dst, int rows, int cols) {
    const long long total = (long long)rows * cols;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        dst[i] = __bfloat162float(src[(i / cols) * lds + i % cols]);
}

// out[b][j][:] = bf16(dh[b][row0 + j][:]) — the bf16 gradient a bf16 branch receives from the fp32 stream (fp32 + bf16 add) —
// through the branch's drop path and dropout, as autograd orders them: out = bf16(bf16(bf16(dh) * path) * m * scale), every step
// skipped when its site is off.  Token site (the prefix rows of the caption MLP): out = bf16(dh * m * scale), fp32 product first.
// Four columns per thread (one generator call); d % 4 == 0.
__global__ void tr_take_rows_bf16_kernel(const float* __restrict__ dh, bf16* __restrict__ out, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = tr_drop_seed(dr);
    const int d4 = d / 4;
    const long long total = (long long)B * nrows * d4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % d4);
        const long long rj = i / d4;
        const int j = (int)(rj % nrows), b = (int)(rj / nrows);
        const uint4 r = tr_drop_words(dr, seed, b, row0 + j, c4);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
        const float pm = tr_path_mult(dr, seed, b);
        const float* src = dh + ((size_t)b * S + row0 + j) * d + 4 * c4;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float g = src[e];
            if (dr.site == CAR_DROP_TOKEN) {
                if (dr.keep < 1.f) g = g * car_keep_bit(rr[e], dr.keep) * dr.scale;
            } else {
                g = rnd<bf16>(g);
                if (dr.path_keep < 1.f) g = rnd<bf16>(g * pm);
                if (dr.keep < 1.f) g = g * car_keep_bit(rr[e], dr.keep) * dr.scale;
            }
            out[(size_t)rj * d + 4 * c4 + e] = __float2bfloat16_rn(g);
        }
    }
}

// ConditionEmbedder.token_drop (gpt_t2i.py:110-120): rows of dropped samples become uncond_embedding[j][:] (a buffer, all zero in
// the released checkpoints; kept general because a state dict carries it)
__global__ void tr_select_uncond_kernel(bf16* __restrict__ c, const float* __restrict__ uncond, const unsigned char* __restrict__ drop, int B,
                                        long long per_sample) {
    const long long total = (long long)B * per_sample;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        if (drop[i / per_sample]) c[i] = __float2bfloat16_rn(uncond ? uncond[i % per_sample] : 0.f);
}

__device__ __forceinline__ float tr_block_sum(float v, float* red) {        // red: >= 32 floats of shared memory; all threads get the sum
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    return t;
}

// d loss / d logits of F.cross_entropy (gpt_t2i.py:474-481) folded with the `valid` weighting, as the bf16 tensor autograd hands
// to the output projection: dlg[r][k] = bf16((softmax(lg[r])[k] - [k == target[r]]) * w_r / den), w_r = valid[b] (or 1),
// den = max(sum_r w_r, 1) (or the row count), times the incoming d / d loss (*loss_grad, 1 when NULL).  One CTA per row.
__global__ void tr_ce_grad_kernel(const bf16* __restrict__ lg, const int* __restrict__ targets, const float* __restrict__ valid,
                                  const float* __restrict__ loss_grad, int B, int n_img, bf16* __restrict__ dlg, int V) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const bf16* row = lg + (size_t)r * V;
    float mx = -INFINITY;
    for (int k = threadIdx.x; k < V; k += blockDim.x) mx = fmaxf(mx, __bfloat162float(row[k]));
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
    float sum = 0.f;
    for (int k = threadIdx.x; k < V; k += blockDim.x) sum += expf(__bfloat162float(row[k]) - mx);
    sum = tr_block_sum(sum, red);
    float w = 1.f, den = (float)(B * n_img);
    if (valid) {
        den = 0.f;
        for (int b = 0; b < B; ++b) den += valid[b] * (float)n_img;
        den = fmaxf(den, 1.f);
        w = valid[r / n_img];
    }
    const float scale = (w / den) * (loss_grad ? loss_grad[0] : 1.f), inv = 1.f / sum;
    const int tg = targets[r];
    for (int k = threadIdx.x; k < V; k += blockDim.x) {
        const float p = expf(__bfloat162float(row[k]) - mx) * inv;
        dlg[(size_t)r * V + k] = __float2bfloat16_rn((p - (k == tg ? 1.f : 0.f)) * scale);
    }
}

// RMSNorm backward on the fp32 stream (forward: y = bf16((x * rstd) * w), gpt_t2i.py:193-198).  dy: bf16 [rows][K] (gradient of
// the bf16 cast); stream row of output row r: (r / nrows) * S + row0 + r % nrows.  dh[row] += rstd * (dn - n * mean(dn * n)) with
// n = x * rstd, dn = dy * w; scr[r][k] = dy * n (summed over rows into the weight gradient by tr_colsum_*).  One CTA per row.
__global__ void tr_rmsnorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const bf16* __restrict__ dy, float* __restrict__ dh,
                                      float* __restrict__ scr, int K, float eps, int nrows, int S, int row0) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const int b = r / nrows, j = r - b * nrows;
    const size_t off = ((size_t)b * S + row0 + j) * K;
    const float* xr = x + off;
    float ss = 0.f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) { const float a = xr[k]; ss += a * a; }
    ss = tr_block_sum(ss, red);
    const float rstd = rsqrtf(ss / (float)K + eps);
    float acc = 0.f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const float n = xr[k] * rstd, d = __bfloat162float(dy[(size_t)r * K + k]);
        scr[(size_t)r * K + k] = d * n;
        acc += (d * w[k]) * n;
    }
    acc = tr_block_sum(acc, red);
    const float m = acc / (float)K;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        const float n = xr[k] * rstd, dn = __bfloat162float(dy[(size_t)r * K + k]) * w[k];
        dh[off + k] += rstd * (dn - n * m);
    }
}

// column sums of src [rows][K] (fp32 or bf16, summed in fp32) in two deterministic passes: part[c][k] = sum of the rows of chunk c
// (fixed order), then dst[k] = sum_c part[c][k].  block (32, 8); grid (ceil(K/32), TR_COLSUM_CHUNKS).
constexpr int TR_COLSUM_CHUNKS = 32;
template <typename T>
__global__ void tr_colsum_part_kernel(const T* __restrict__ src, float* __restrict__ part, int rows, int K) {
    __shared__ float red[8][32];
    const int k = blockIdx.x * 32 + threadIdx.x;
    const int per = (rows + TR_COLSUM_CHUNKS - 1) / TR_COLSUM_CHUNKS;
    const int lo = blockIdx.y * per, hi = min(rows, lo + per);
    float a = 0.f;
    if (k < K) for (int r = lo + threadIdx.y; r < hi; r += 8) a += tof(src[(size_t)r * K + k]);
    red[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.y == 0 && k < K) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
        part[(size_t)blockIdx.y * K + k] = t;
    }
}
__global__ void tr_colsum_final_kernel(const float* __restrict__ part, float* __restrict__ dst, int K) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    float t = 0.f;
    for (int c = 0; c < TR_COLSUM_CHUNKS; ++c) t += part[(size_t)c * K + k];
    dst[k] = t;
}

// backward of act = bf16(bf16(silu(g)) * u) (FeedForward.forward gpt_t2i.py:217), every intermediate gradient rounded to bf16
// like autograd's: d_s = bf16(dact * u), du = bf16(dact * s), dg = bf16(d_s * silu'(g)), silu'(g) = sig (1 + g (1 - sig))
__global__ void tr_swiglu_bwd_kernel(const bf16* __restrict__ g, const bf16* __restrict__ u, const bf16* __restrict__ dact, bf16* __restrict__ dg,
                                     bf16* __restrict__ du, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gf = tof(g[i]), uf = tof(u[i]), da = tof(dact[i]);
        const float s = rnd<bf16>(silu_f(gf));
        const float ds = rnd<bf16>(da * uf);
        const float sig = 1.f / (1.f + expf(-gf));
        du[i] = fromf<bf16>(da * s);
        dg[i] = fromf<bf16>(ds * (sig * (1.f + gf * (1.f - sig))));
    }
}

// MLP's nn.GELU(approximate='tanh') (gpt_t2i.py:171) on the bf16 tensor fc1 returned, and its backward
__global__ void tr_gelu_kernel(const bf16* __restrict__ t, bf16* __restrict__ a, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        a[i] = fromf<bf16>(gelu_tanh_f(tof(t[i])));
}
__global__ void tr_gelu_bwd_kernel(const bf16* __restrict__ t, const bf16* __restrict__ da, bf16* __restrict__ dt, long long n) {
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float x = tof(t[i]);
        const float th = tanhf(k0 * (x + k1 * x * x * x));
        const float dgelu = 0.5f * (1.f + th) + 0.5f * x * (1.f - th * th) * k0 * (1.f + 3.f * k1 * x * x);
        dt[i] = fromf<bf16>(tof(da[i]) * dgelu);
    }
}

// ---- scaled-dot-product attention backward (forward: tr_attention_kernel, gpt_t2i.py:282-286) ---------------------------------
// P = softmax(Q K^T / 8 + mask), O = P V.  dV = P^T dO, dP = dO V^T, dS = P o (dP - rowsum(dP o P)), dQ = dS K / 8, dK = dS^T Q / 8.
// Pass 1, one warp per (b, h, query i): recomputes the row of P, writes lse = max + log(sum), D = rowsum(dP o P) and dQ.
// q / dout / dq: [B*S][H*64]; k / v: [B][H][S][64]; mask / causal as in tr_attention_kernel.  Shared memory: TRA_WARPS * (2 S + 128) floats.
__global__ void __launch_bounds__(TRA_WARPS * 32)
tr_attn_bwd_q_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kc, const bf16* __restrict__ vc, const unsigned char* __restrict__ mask,
                     const bf16* __restrict__ dout, int B, int H, int S, float* __restrict__ lse, float* __restrict__ dsum, bf16* __restrict__ dq,
                     int causal) {
    extern __shared__ float trb_sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * TRA_WARPS + warp;
    if (item >= (long long)B * H * S) return;                // (whole warp)
    const int i = (int)(item % S);
    const int hd = (int)((item / S) % H);
    const int b = (int)(item / ((long long)S * H));
    float* sc = trb_sm + (size_t)warp * (2 * S + 128);       // p, then dS
    float* dp = sc + S;
    float* qs = dp + S;
    float* gs = qs + 64;
    const size_t qoff = ((size_t)b * S + i) * H * 64 + hd * 64;
    const bf16* kb = kc + (((size_t)b * H + hd) * S) * 64;
    const bf16* vb = vc + (((size_t)b * H + hd) * S) * 64;
    unpack_bf16x2(*reinterpret_cast<const uint32_t*>(q + qoff + 2 * lane), qs[2 * lane], qs[2 * lane + 1]);
    unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + qoff + 2 * lane), gs[2 * lane], gs[2 * lane + 1]);
    __syncwarp();
    const unsigned char* mrow = mask ? mask + ((size_t)b * S + i) * S : nullptr;
    const int s_end = (mask || !causal) ? S : i + 1;
    float mx = -INFINITY;
    for (int s = lane; s < s_end; s += 32) {
        float v = -INFINITY;
        if (mrow == nullptr || mrow[s] != 0) {
            float d = 0.f;
            const uint4* kr = reinterpret_cast<const uint4*>(kb + (size_t)s * 64);
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 kk = kr[c];
                float k0, k1;
                unpack_bf16x2(kk.x, k0, k1); d = fmaf(qs[c * 8 + 0], k0, d); d = fmaf(qs[c * 8 + 1], k1, d);
                unpack_bf16x2(kk.y, k0, k1); d = fmaf(qs[c * 8 + 2], k0, d); d = fmaf(qs[c * 8 + 3], k1, d);
                unpack_bf16x2(kk.z, k0, k1); d = fmaf(qs[c * 8 + 4], k0, d); d = fmaf(qs[c * 8 + 5], k1, d);
                unpack_bf16x2(kk.w, k0, k1); d = fmaf(qs[c * 8 + 6], k0, d); d = fmaf(qs[c * 8 + 7], k1, d);
            }
            v = d * 0.125f;
        }
        sc[s] = v;
        mx = fmaxf(mx, v);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int s = lane; s < s_end; s += 32) {
        const float p = (sc[s] == -INFINITY) ? 0.f : expf(sc[s] - mx);
        sc[s] = p;
        sum += p;
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    float D = 0.f;
    for (int s = lane; s < s_end; s += 32) {
        const float p = sc[s] * inv;
        float d = 0.f;
        if (p != 0.f) {
            const uint4* vr = reinterpret_cast<const uint4*>(vb + (size_t)s * 64);
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 vv = vr[c];
                float v0, v1;
                unpack_bf16x2(vv.x, v0, v1); d = fmaf(gs[c * 8 + 0], v0, d); d = fmaf(gs[c * 8 + 1], v1, d);
                unpack_bf16x2(vv.y, v0, v1); d = fmaf(gs[c * 8 + 2], v0, d); d = fmaf(gs[c * 8 + 3], v1, d);
                unpack_bf16x2(vv.z, v0, v1); d = fmaf(gs[c * 8 + 4], v0, d); d = fmaf(gs[c * 8 + 5], v1, d);
                unpack_bf16x2(vv.w, v0, v1); d = fmaf(gs[c * 8 + 6], v0, d); d = fmaf(gs[c * 8 + 7], v1, d);
            }
        }
        sc[s] = p;
        dp[s] = d;
        D = fmaf(p, d, D);
    }
    D = warp_sum(D);
    for (int s = lane; s < s_end; s += 32) sc[s] = sc[s] * (dp[s] - D);      // dS
    __syncwarp();
    float a0 = 0.f, a1 = 0.f;
    for (int s = 0; s < s_end; ++s) {
        const float w = sc[s];                                // (broadcast read)
        if (w != 0.f) {
            float k0, k1;
            unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kb + (size_t)s * 64 + 2 * lane), k0, k1);
            a0 = fmaf(w, k0, a0); a1 = fmaf(w, k1, a1);
        }
    }
    *reinterpret_cast<__nv_bfloat162*>(dq + qoff + 2 * lane) = __floats2bfloat162_rn(a0 * 0.125f, a1 * 0.125f);
    if (lane == 0) { lse[item] = mx + logf(sum); dsum[item] = D; }
}

// Pass 2, one warp per (b, h, key s): p_i = exp(q_i k_s / 8 - lse_i) and dS_i = p_i (dO_i v_s - D_i) for every query i that
// attends s, then dV_s = sum_i p_i dO_i and dK_s = sum_i dS_i q_i / 8.  dk / dv: [B][H][S][64].  Shared memory as in pass 1.
__global__ void __launch_bounds__(TRA_WARPS * 32)
tr_attn_bwd_kv_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kc, const bf16* __restrict__ vc, const unsigned char* __restrict__ mask,
                      const bf16* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ dsum, int B, int H, int S,
                      bf16* __restrict__ dk, bf16* __restrict__ dv, int causal) {
    extern __shared__ float trb_sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * TRA_WARPS + warp;
    if (item >= (long long)B * H * S) return;                // (whole warp)
    const int s = (int)(item % S);
    const int hd = (int)((item / S) % H);
    const int b = (int)(item / ((long long)S * H));
    float* pp = trb_sm + (size_t)warp * (2 * S + 128);
    float* dd = pp + S;
    float* ks = dd + S;
    float* vs = ks + 64;
    const size_t kvoff = (((size_t)b * H + hd) * S + s) * 64;
    unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kc + kvoff + 2 * lane), ks[2 * lane], ks[2 * lane + 1]);
    unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vc + kvoff + 2 * lane), vs[2 * lane], vs[2 * lane + 1]);
    __syncwarp();
    const int i_begin = (mask || !causal) ? 0 : s;            // causal: queries i >= s
    const float* lrow = lse + ((size_t)b * H + hd) * S;
    const float* drow = dsum + ((size_t)b * H + hd) * S;
    for (int i = i_begin + lane; i < S; i += 32) {
        float p = 0.f, dS = 0.f;
        if (mask == nullptr || mask[((size_t)b * S + i) * S + s] != 0) {
            const size_t qoff = ((size_t)b * S + i) * H * 64 + hd * 64;
            const uint4* qr = reinterpret_cast<const uint4*>(q + qoff);
            const uint4* gr = reinterpret_cast<const uint4*>(dout + qoff);
            float d = 0.f, e = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const uint4 qq = qr[c], gg = gr[c];
                float x0, x1;
                unpack_bf16x2(qq.x, x0, x1); d = fmaf(x0, ks[c * 8 + 0], d); d = fmaf(x1, ks[c * 8 + 1], d);
                unpack_bf16x2(qq.y, x0, x1); d = fmaf(x0, ks[c * 8 + 2], d); d = fmaf(x1, ks[c * 8 + 3], d);
                unpack_bf16x2(qq.z, x0, x1); d = fmaf(x0, ks[c * 8 + 4], d); d = fmaf(x1, ks[c * 8 + 5], d);
                unpack_bf16x2(qq.w, x0, x1); d = fmaf(x0, ks[c * 8 + 6], d); d = fmaf(x1, ks[c * 8 + 7], d);
                unpack_bf16x2(gg.x, x0, x1); e = fmaf(x0, vs[c * 8 + 0], e); e = fmaf(x1, vs[c * 8 + 1], e);
                unpack_bf16x2(gg.y, x0, x1); e = fmaf(x0, vs[c * 8 + 2], e); e = fmaf(x1, vs[c * 8 + 3], e);
                unpack_bf16x2(gg.z, x0, x1); e = fmaf(x0, vs[c * 8 + 4], e); e = fmaf(x1, vs[c * 8 + 5], e);
                unpack_bf16x2(gg.w, x0, x1); e = fmaf(x0, vs[c * 8 + 6], e); e = fmaf(x1, vs[c * 8 + 7], e);
            }
            p = expf(d * 0.125f - lrow[i]);
            dS = p * (e - drow[i]);
        }
        pp[i] = p;
        dd[i] = dS;
    }
    __syncwarp();
    float v0 = 0.f, v1 = 0.f, k0 = 0.f, k1 = 0.f;
    for (int i = i_begin; i < S; ++i) {
        const float p = pp[i], dS = dd[i];                    // (broadcast reads)
        if (p != 0.f || dS != 0.f) {
            const size_t qoff = ((size_t)b * S + i) * H * 64 + hd * 64 + 2 * lane;
            float g0, g1, q0, q1;
            unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dout + qoff), g0, g1);
            unpack_bf16x2(*reinterpret_cast<const uint32_t*>(q + qoff), q0, q1);
            v0 = fmaf(p, g0, v0); v1 = fmaf(p, g1, v1);
            k0 = fmaf(dS, q0, k0); k1 = fmaf(dS, q1, k1);
        }
    }
    *reinterpret_cast<__nv_bfloat162*>(dv + kvoff + 2 * lane) = __floats2bfloat162_rn(v0, v1);
    *reinterpret_cast<__nv_bfloat162*>(dk + kvoff + 2 * lane) = __floats2bfloat162_rn(k0 * 0.125f, k1 * 0.125f);
}

// backward of rope_kv_write_kernel (apply_rotary_emb gpt_t2i.py:522-532 + the head split): dq [rows][d], dk / dv [B][H][S][64]
// -> dqkv [rows][3d]; the rotation of a pair by (cos, sin) is undone on the gradient by the transposed rotation (no rotation when
// rope is null: the plain head merge of the control encoder).
__global__ void tr_rope_bwd_kernel(const bf16* __restrict__ dq, const bf16* __restrict__ dk, const bf16* __restrict__ dv, const float* __restrict__ rope,
                                   bf16* __restrict__ dqkv, int rows, int Tq, int d, int H, int S) {
    const long long total = (long long)rows * (3 * d / 2);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / (3 * d / 2));
        const int n = (int)(i % (3 * d / 2)) * 2;
        const int sec = n / d, w = n - sec * d, head = w >> 6, e = w & 63;
        const int b = r / Tq, t = r - b * Tq;
        const bf16* src = sec == 0 ? dq + (size_t)r * d + w : (sec == 1 ? dk : dv) + (((size_t)b * H + head) * S + t) * 64 + e;
        float g0 = tof(src[0]), g1 = tof(src[1]);
        if (sec < 2 && rope) {
            const float2 cs2 = *reinterpret_cast<const float2*>(rope + ((size_t)t * 32 + (e >> 1)) * 2);
            const float x0 = g0 * cs2.x + g1 * cs2.y, x1 = g1 * cs2.x - g0 * cs2.y;
            g0 = x0; g1 = x1;
        }
        dqkv[(size_t)r * 3 * d + n] = fromf<bf16>(g0);
        dqkv[(size_t)r * 3 * d + n + 1] = fromf<bf16>(g1);
    }
}

// embedding-table gradients (tok_embeddings gpt_t2i.py:423, LabelEmbedder :78-97) through the token dropout:
// grad[index(b, j)][:] += dh[b][row0 + j][:] * m * scale (fp32 atomics: rows that repeat an index accumulate in arrival order).
// One CTA per row, four columns per thread; d % 4 == 0.
__global__ void tr_embed_grad_kernel(const float* __restrict__ dh, const int* __restrict__ idx, int ld, const unsigned char* __restrict__ drop,
                                     int drop_to, float* __restrict__ grad, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = tr_drop_seed(dr);
    const int bj = blockIdx.x;
    const int b = bj / nrows, j = bj - b * nrows;
    int id = idx[(size_t)b * ld + j];
    if (drop != nullptr && drop[b]) id = drop_to;
    const float* src = dh + ((size_t)b * S + row0 + j) * d;
    float* dst = grad + (size_t)id * d;
    for (int c4 = threadIdx.x; c4 < d / 4; c4 += blockDim.x) {
        const uint4 r = tr_drop_words(dr, seed, b, row0 + j, c4);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float v = src[4 * c4 + e];
            if (dr.keep < 1.f) v = v * car_keep_bit(rr[e], dr.keep) * dr.scale;
            atomicAdd(dst + 4 * c4 + e, v);
        }
    }
}
