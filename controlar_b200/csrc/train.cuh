// train.cuh — small kernels of the teacher-forced TRAINING forward (SURVEY.md §8 row f1): Transformer.forward with idx and
// cond_idx, module in train mode, fp32 parameters under bf16 autocast (autoregressive/models/gpt_t2i.py:420-431,451-484;
// autoregressive/train/train_t2i_canny.py:166-167).  Autocast numerics (oracle/train_oracle.py): the residual stream, the
// embeddings and the RMSNorm stay fp32; every nn.Linear takes bf16 operands (cast of the fp32 tensor) and returns bf16;
// fp32 + bf16 adds promote to fp32; GELU / SiLU / the SwiGLU product run on the bf16 tensors; cross-entropy is fp32.
// First correct path: the GEMMs are the dense tensor-core kernels of the prefill (gemm_wgmma.cuh / gemm_dense.cuh), everything
// here is bandwidth-trivial glue plus a plain attention kernel; fusing them is the next step of this row.  The row passes that
// write the fp32 stream take a TrDrop (dropout.cuh): token, residual and feed-forward dropout and drop path apply as they write.
#pragma once
#include "common.cuh"
#include "dropout.cuh"

// dst[i] = bf16(src[i]) — autocast's per-forward cast of an fp32 weight (or activation) to the GEMM operand type
__global__ void tr_cast_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dst[i] = __float2bfloat16_rn(src[i]);
}

// CaptionEmbedder.token_drop + the cast in front of cap_proj.fc1 (gpt_t2i.py:145-152,158): out[b][t][:] = bf16(drop[b] ? uncond[t][:] : cap[b][t][:])
__global__ void tr_caption_select_kernel(const float* __restrict__ cap, const float* __restrict__ uncond, const unsigned char* __restrict__ drop,
                                         bf16* __restrict__ out, int B, int T, int C) {
    const long long total = (long long)B * T * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / ((long long)T * C));
        const long long r = i - (long long)b * T * C;
        out[i] = __float2bfloat16_rn(drop[b] ? uncond[r] : cap[i]);
    }
}

// h[b][row0 + j][:] = float(src[b][j][:]) * m * scale, j < nrows — the cls_embedding rows of torch.cat (gpt_t2i.py:428) through
// tok_dropout (:430, after the cat that promotes to fp32); also the fp32 copy of the logits (TrDrop{}).  Four columns per thread
// (one generator call); d % 4 == 0.
__global__ void tr_put_rows_bf16_kernel(const bf16* __restrict__ src, float* __restrict__ h, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = tr_drop_seed(dr);
    const int d4 = d / 4;
    const long long total = (long long)B * nrows * d4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % d4);
        const long long rj = i / d4;
        const int j = (int)(rj % nrows), b = (int)(rj / nrows);
        const uint4 r = tr_drop_words(dr, seed, b, row0 + j, c4);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float v = __bfloat162float(src[(size_t)rj * d + 4 * c4 + e]);
            if (dr.keep < 1.f) v = v * car_keep_bit(rr[e], dr.keep) * dr.scale;
            h[((size_t)b * S + row0 + j) * d + 4 * c4 + e] = v;
        }
    }
}

// h[b][row0 + j][:] = table[index(b, j)][:] * m * scale (fp32 gather through tok_dropout): tok_embeddings(idx) (gpt_t2i.py:423,
// ld = n tokens) and LabelEmbedder (gpt_t2i.py:78-97: index = drop ? num_classes : label; nrows = 1, drop / drop_to given).
// One CTA per row, four columns per thread; d % 4 == 0.
__global__ void tr_embed_rows_kernel(const float* __restrict__ table, const int* __restrict__ idx, int ld, const unsigned char* __restrict__ drop,
                                     int drop_to, float* __restrict__ h, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = tr_drop_seed(dr);
    const int bj = blockIdx.x;
    const int b = bj / nrows, j = bj - b * nrows;
    int id = idx[(size_t)b * ld + j];
    if (drop != nullptr && drop[b]) id = drop_to;
    const float* src = table + (size_t)id * d;
    float* dst = h + ((size_t)b * S + row0 + j) * d;
    for (int c4 = threadIdx.x; c4 < d / 4; c4 += blockDim.x) {
        const uint4 r = tr_drop_words(dr, seed, b, row0 + j, c4);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float v = src[4 * c4 + e];
            if (dr.keep < 1.f) v = v * car_keep_bit(rr[e], dr.keep) * dr.scale;
            dst[4 * c4 + e] = v;
        }
    }
}

// ConditionEmbedder.token_drop (gpt_t2i.py:110-120): rows of dropped samples become the all-zero uncond_embedding
__global__ void tr_zero_dropped_kernel(bf16* __restrict__ c, const unsigned char* __restrict__ drop, int B, long long per_sample) {
    const long long total = (long long)B * per_sample;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        if (drop[i / per_sample]) c[i] = __float2bfloat16_rn(0.f);
}

// h[b][row0 + j][:] += float(bf16(bf16(o * m * scale) * path)), o = add[b][j][:] bf16 (fp32 += bf16, every step skipped when its
// site is off): the residual adds of the wo / w2 outputs through their dropout and drop path (gpt_t2i.py:305-306; row0 = 0,
// nrows = S) and the control add h[:, T-1:] += condition_layers[i](condition_token) (gpt_t2i.py:458-460; row0 = T - 1,
// nrows = n_img, TrDrop{}).  Four columns per thread (one generator call); d % 4 == 0.
__global__ void tr_add_rows_kernel(float* __restrict__ h, const bf16* __restrict__ add, int B, int nrows, int S, int row0, int d, TrDrop dr) {
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
        const size_t o = ((size_t)b * S + row0 + j) * d + 4 * c4;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float v = __bfloat162float(add[(size_t)rj * d + 4 * c4 + e]);
            if (dr.keep < 1.f) v = rnd<bf16>(v * car_keep_bit(rr[e], dr.keep) * dr.scale);
            if (dr.path_keep < 1.f) v = rnd<bf16>(v * pm);
            h[o + e] = h[o + e] + v;
        }
    }
}

// RMSNorm.forward on the fp32 stream (gpt_t2i.py:193-198): y = bf16((x * rsqrt(mean(x^2) + eps)) * w), w fp32 — the bf16
// rounding is the cast in front of the following nn.Linear.  Optional row map: output row r reads x row (r / nrows) * S + row0 + r % nrows.
__global__ void tr_rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ w, bf16* __restrict__ y, int K, float eps,
                                  int nrows, int S, int row0) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const int b = r / nrows, j = r - b * nrows;
    const float* xr = x + ((size_t)b * S + row0 + j) * K;
    float ss = 0.f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) { const float a = xr[k]; ss += a * a; }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    ss = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) ss += red[i];
    const float rstd = rsqrtf(ss / (float)K + eps);
    for (int k = threadIdx.x; k < K; k += blockDim.x) y[(size_t)r * K + k] = __float2bfloat16_rn((xr[k] * rstd) * w[k]);
}

// F.scaled_dot_product_attention over full sequences (gpt_t2i.py:282-286), math semantics: fp32 scores, fp32 soft-max over
// the allowed keys, fp32 probability-weighted sum, one rounding to bf16.  One warp per (b, h, query i); the row of scores
// lives in shared memory (S floats per warp).  mask: uint8 [B][S][S] (1 = attend); without one, causal != 0 attends keys 0 .. i and
// causal == 0 every key (the bidirectional attention of the control encoder, Dinov2SelfAttention).
// q [B*S][H*64] (RoPE applied), k / v [B][H][S][64] bf16 (RoPE applied to k), out [B*S][H*64].
constexpr int TRA_WARPS = 4;
__global__ void __launch_bounds__(TRA_WARPS * 32)
tr_attention_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kc, const bf16* __restrict__ vc, const unsigned char* __restrict__ mask,
                    int B, int H, int S, bf16* __restrict__ out, int causal) {
    extern __shared__ float tra_sc[];                         // [TRA_WARPS][S]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * TRA_WARPS + warp;
    if (item >= (long long)B * H * S) return;                // (whole warp)
    const int i = (int)(item % S);
    const int hd = (int)((item / S) % H);
    const int b = (int)(item / ((long long)S * H));
    float* sc = tra_sc + (size_t)warp * S;
    const bf16* qp = q + ((size_t)b * S + i) * H * 64 + hd * 64;
    const bf16* kb = kc + (((size_t)b * H + hd) * S) * 64;
    const bf16* vb = vc + (((size_t)b * H + hd) * S) * 64;
    const unsigned char* mrow = mask ? mask + ((size_t)b * S + i) * S : nullptr;
    const int s_end = (mask || !causal) ? S : i + 1;          // causal: keys 0 .. i
    float qf[64];
#pragma unroll
    for (int e = 0; e < 64; e += 2) unpack_bf16x2(*reinterpret_cast<const uint32_t*>(qp + e), qf[e], qf[e + 1]);
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
                unpack_bf16x2(kk.x, k0, k1); d = fmaf(qf[c * 8 + 0], k0, d); d = fmaf(qf[c * 8 + 1], k1, d);
                unpack_bf16x2(kk.y, k0, k1); d = fmaf(qf[c * 8 + 2], k0, d); d = fmaf(qf[c * 8 + 3], k1, d);
                unpack_bf16x2(kk.z, k0, k1); d = fmaf(qf[c * 8 + 4], k0, d); d = fmaf(qf[c * 8 + 5], k1, d);
                unpack_bf16x2(kk.w, k0, k1); d = fmaf(qf[c * 8 + 6], k0, d); d = fmaf(qf[c * 8 + 7], k1, d);
            }
            v = d * 0.125f;                                   // 1 / sqrt(head_dim = 64)
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
    __syncwarp();
    float o0 = 0.f, o1 = 0.f;
    for (int s = 0; s < s_end; ++s) {
        const float p = sc[s];                                // (broadcast read)
        if (p != 0.f) {
            float v0, v1;
            unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vb + (size_t)s * 64 + 2 * lane), v0, v1);
            o0 = fmaf(p, v0, o0); o1 = fmaf(p, v1, o1);
        }
    }
    __nv_bfloat162 o = __floats2bfloat162_rn(o0 / sum, o1 / sum);
    *reinterpret_cast<__nv_bfloat162*>(out + ((size_t)b * S + i) * H * 64 + hd * 64 + 2 * lane) = o;
}

// logits = output(norm(h)).float()[:, T-1:] (gpt_t2i.py:469-473) then F.cross_entropy (:476-481), one CTA per (b, j) row:
// copies the bf16 logits to fp32 (when logits_out is given) and writes nll[row] = logsumexp(row) - row[target].
__global__ void tr_ce_rows_kernel(const bf16* __restrict__ lg, const int* __restrict__ targets, float* __restrict__ logits_out,
                                  float* __restrict__ nll, int V) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const bf16* row = lg + (size_t)r * V;
    float mx = -INFINITY;
    for (int k = threadIdx.x; k < V; k += blockDim.x) {
        const float v = __bfloat162float(row[k]);
        if (logits_out) logits_out[(size_t)r * V + k] = v;
        mx = fmaxf(mx, v);
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
    __syncthreads();
    float sum = 0.f;
    for (int k = threadIdx.x; k < V; k += blockDim.x) sum += expf(__bfloat162float(row[k]) - mx);
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
        nll[r] = (mx + logf(t)) - __bfloat162float(row[targets[r]]);
    }
}

// loss = sum(nll * valid_row) / max(sum(valid_row), 1)  (valid given, gpt_t2i.py:476-479) or mean(nll) (:480-481); one CTA,
// fixed summation order (deterministic)
__global__ void tr_ce_reduce_kernel(const float* __restrict__ nll, const float* __restrict__ valid, int B, int n_img, float* __restrict__ loss) {
    __shared__ float red_a[32], red_b[32];
    float a = 0.f, c = 0.f;
    const int rows = B * n_img;
    for (int r = threadIdx.x; r < rows; r += blockDim.x) {
        const float w = valid ? valid[r / n_img] : 1.f;
        a += nll[r] * w; c += w;
    }
    a = warp_sum(a); c = warp_sum(c);
    if ((threadIdx.x & 31) == 0) { red_a[threadIdx.x >> 5] = a; red_b[threadIdx.x >> 5] = c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float ta = 0.f, tc = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { ta += red_a[i]; tc += red_b[i]; }
        loss[0] = valid ? ta / fmaxf(tc, 1.f) : ta / (float)rows;
    }
}

// ---- fused multi-tensor AdamW (row f1: the optimiser step of autoregressive/train/train_c2i.py:28-50, torch.optim.AdamW(fused=True)) ----
// One launch for every parameter of the model: chunk c of the chunk list covers up to ADAMW_CHUNK elements of tensor `t`.
// Arithmetic = ATen's fused kernel in fp32: decoupled weight decay, exp_avg = lerp(exp_avg, grad, 1 - beta1),
// exp_avg_sq = beta2 * exp_avg_sq + (1 - beta2) * grad^2, param -= (lr / bc1) * exp_avg / (sqrt(exp_avg_sq) / sqrt(bc2) + eps).
struct CarAdamWTensorDev { float* p; const float* g; float* m; float* v; long long n; float weight_decay; int pad_; };
constexpr int ADAMW_CHUNK = 65536;
__global__ void __launch_bounds__(256) adamw_multi_kernel(const CarAdamWTensorDev* __restrict__ tensors, const int2* __restrict__ chunks,
                                                          float lr, float beta1, float beta2, float eps, float bc1, float bc2_sqrt) {
    const int2 ck = chunks[blockIdx.x];                        // {tensor index, chunk index inside the tensor}
    const CarAdamWTensorDev T = tensors[ck.x];
    const long long lo = (long long)ck.y * ADAMW_CHUNK, hi = min(T.n, lo + ADAMW_CHUNK);
    const float step_size = lr / bc1, decay = lr * T.weight_decay;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const float g = T.g[i];
        float p = T.p[i], m = T.m[i], v = T.v[i];
        if (T.weight_decay != 0.f) p -= decay * p;
        m = m + (g - m) * (1.f - beta1);
        v = beta2 * v + (1.f - beta2) * g * g;
        const float denom = sqrtf(v) / bc2_sqrt + eps;
        p -= step_size * m / denom;
        T.p[i] = p; T.m[i] = m; T.v[i] = v;
    }
}
