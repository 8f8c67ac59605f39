// dino_train.cuh — kernels of the TRAINABLE control encoder: Dinov2_Adapter.forward (autoregressive/models/dinov2_adapter.py:16-29,
// HF modeling_dinov2.py 5.5.0) or ViT_Adapter.forward (vit_adapter.py:13-15, HF modeling_vit.py) with fp32 parameters under the
// train loop's bf16 autocast (train_t2i_canny.py:166-167), and its backward (oracle/train_encoder_oracle.py writes the numerics out):
// the residual stream, the position embeddings, the CLS row, LayerNorm and LayerScale are fp32; the patch projection and every
// nn.Linear take bf16 operands and return bf16; attention and GELU-erf run on bf16 tensors.  The inference encoder of
// car_dino_forward keeps a bf16 stream instead and is a different arithmetic.
// The GEMMs, the attention kernels, the head split / merge, the transposes and the column sums are the transformer training
// path's (train.cuh, train_bwd.cuh, misc.h); what is here is the encoder-only glue.  dt_cubic_t_kernel takes the bicubic weights
// cubic1 / cubic2 of patch_embed.cuh, which car_train.cu includes first.
#pragma once
#include "common.cuh"

// nn.LayerNorm on the fp32 stream (fp32 statistics, eps inside the sqrt, fp32 affine).  Output row r reads stream row
// (r / nrows) * S + row0 + r % nrows; writes yb = bf16(y) (the cast in front of the next nn.Linear) or, when yb is null, yf = y.
// One CTA per output row.
__global__ void dt_layernorm_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b, bf16* __restrict__ yb,
                                    float* __restrict__ yf, int C, float eps, int nrows, int S, int row0) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const float* xr = x + ((size_t)(r / nrows) * S + row0 + r % nrows) * C;
    float s = 0.f;
    for (int k = threadIdx.x; k < C; k += blockDim.x) s += xr[k];
    const float mean = block_sum(s, red) / C;
    float v = 0.f;
    for (int k = threadIdx.x; k < C; k += blockDim.x) { const float d = xr[k] - mean; v += d * d; }
    const float rstd = rsqrtf(block_sum(v, red) / C + eps);
    for (int k = threadIdx.x; k < C; k += blockDim.x) {
        const float y = (xr[k] - mean) * rstd * w[k] + b[k];
        if (yb) yb[(size_t)r * C + k] = __float2bfloat16_rn(y);
        else yf[(size_t)r * C + k] = y;
    }
}

// LayerNorm backward (row map as above), with dy the gradient of the LayerNorm output (fp32 for the final norm, the bf16 gradient
// of the cast for the block norms): dx[row] += rstd (g - mean(g) - n mean(g n)), g = dy w, n = (x - mean) rstd; scr[r][k] = dy n
// (column-summed into the weight gradient; the bias gradient is the column sum of dy itself).  One CTA per output row.
template <typename TD>
__global__ void dt_layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const TD* __restrict__ dy, float* __restrict__ dx,
                                        float* __restrict__ scr, int C, float eps, int nrows, int S, int row0) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const size_t off = ((size_t)(r / nrows) * S + row0 + r % nrows) * C;
    const float* xr = x + off;
    const TD* dr = dy + (size_t)r * C;
    float s = 0.f;
    for (int k = threadIdx.x; k < C; k += blockDim.x) s += xr[k];
    const float mean = block_sum(s, red) / C;
    float v = 0.f;
    for (int k = threadIdx.x; k < C; k += blockDim.x) { const float d = xr[k] - mean; v += d * d; }
    const float rstd = rsqrtf(block_sum(v, red) / C + eps);
    float sg = 0.f, sgn = 0.f;
    for (int k = threadIdx.x; k < C; k += blockDim.x) {
        const float n = (xr[k] - mean) * rstd, d = tof(dr[k]), g = d * w[k];
        scr[(size_t)r * C + k] = d * n;
        sg += g; sgn += g * n;
    }
    sg = block_sum(sg, red) / C;
    sgn = block_sum(sgn, red) / C;
    for (int k = threadIdx.x; k < C; k += blockDim.x) {
        const float n = (xr[k] - mean) * rstd, g = tof(dr[k]) * w[k];
        dx[off + k] += rstd * (g - sg - n * sgn);
    }
}

// nn.GELU() (erf form) on the bf16 tensor fc1 returned, and its backward: dt = bf16(da (Phi(x) + x phi(x))).  dt may alias da.
__global__ void dt_gelu_erf_kernel(const bf16* __restrict__ t, bf16* __restrict__ a, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        a[i] = fromf<bf16>(gelu_erf_f(tof(t[i])));
}
__global__ void dt_gelu_erf_bwd_kernel(const bf16* __restrict__ t, const bf16* da, bf16* dt, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float x = tof(t[i]);
        const float cdf = 0.5f * (1.f + erff(x * 0.7071067811865476f)), pdf = 0.3989422804014327f * expf(-0.5f * x * x);
        dt[i] = fromf<bf16>(tof(da[i]) * (cdf + x * pdf));
    }
}

// residual add of a branch: x += y * ls (Dinov2LayerScale: bf16 x fp32 -> fp32) or x += y (ViT, ls null); x fp32, y bf16 [rows][C]
__global__ void dt_layerscale_add_kernel(float* __restrict__ x, const bf16* __restrict__ y, const float* __restrict__ ls, long long n, int C) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        x[i] = (ls ? tof(y[i]) * ls[i % C] : tof(y[i])) + x[i];
}
// its backward from the stream gradient dx: dy = bf16(dx * ls) (bf16(dx) without LayerScale); scr = dx * y (column-summed into
// d lambda, fp32) when scr is given
__global__ void dt_layerscale_bwd_kernel(const float* __restrict__ dx, const bf16* __restrict__ y, const float* __restrict__ ls, bf16* __restrict__ dy,
                                         float* __restrict__ scr, long long n, int C) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float g = dx[i];
        dy[i] = fromf<bf16>(ls ? g * ls[i % C] : g);
        if (scr) scr[i] = g * tof(y[i]);
    }
}

// Dinov2Embeddings.forward / ViTEmbeddings.forward: x[b][0] = cls + pos[0], x[b][1 + i] = float(ptok[b][i]) + pos_i[i] (fp32 stream;
// torch.cat of the fp32 CLS row and the bf16 patch tokens promotes to fp32)
__global__ void dt_assemble_kernel(const bf16* __restrict__ ptok, const float* __restrict__ cls, const float* __restrict__ pos,
                                   const float* __restrict__ posi, float* __restrict__ x, int B, int hw, int C) {
    const long long total = (long long)B * (hw + 1) * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int t = (int)((i / C) % (hw + 1)), b = (int)(i / ((long long)C * (hw + 1)));
        x[i] = t == 0 ? cls[c] + pos[c] : tof(ptok[((size_t)b * hw + t - 1) * C + c]) + posi[(size_t)(t - 1) * C + c];
    }
}
// its backward for the fp32 inputs: s[t][c] = sum_b dx[b][t][c] (batch order); row 0 -> d cls_token and d position_embeddings[0]
// (each when given), rows 1.. -> d pos_i
__global__ void dt_embed_bwd_kernel(const float* __restrict__ dx, float* __restrict__ dcls, float* __restrict__ dpos0, float* __restrict__ dposi,
                                    int B, int Tn, int C) {
    const long long total = (long long)Tn * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int b = 0; b < B; ++b) s += dx[(size_t)b * total + i];
        if (i < C) {
            if (dcls) dcls[i] = s;
            if (dpos0) dpos0[i] = s;
        } else if (dposi) {
            dposi[i - C] = s;
        }
    }
}

// Transposed 1-D bicubic stencil of pos_embed_interp_kernel (align_corners=False, A = -0.75, border taps clamped) along one axis:
// out[o][g][k] = sum_{i < n_in} W(i, g) in[o][i][k], W(i, g) = sum of the tap weights of target cell i whose clamped source index
// is g.  A gather over target cells in fixed order (deterministic); applied along y then x it turns d pos_i [h][w][C] into
// d position_embeddings[1:] [G][G][C].
__global__ void dt_cubic_t_kernel(const float* __restrict__ in, float* __restrict__ out, int G, int n_in, int outer, int inner) {
    const long long total = (long long)outer * G * inner;
    const float scale = (float)G / n_in;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % inner);
        const int g = (int)((i / inner) % G), o = (int)(i / ((long long)inner * G));
        const float* src = in + (size_t)o * n_in * inner + k;
        float acc = 0.f;
        for (int j = 0; j < n_in; ++j) {
            const float f = (j + 0.5f) * scale - 0.5f;
            const int i0 = (int)floorf(f);
            if (g < i0 - 1 && g != 0) continue;              // every tap of j lies past g (g is not the clamped border)
            if (g > i0 + 2 && g != G - 1) continue;
            const float t = f - i0;
            const float wt[4] = {cubic2(t + 1.f), cubic1(t), cubic1(1.f - t), cubic2(2.f - t)};
            float wsum = 0.f;
#pragma unroll
            for (int a = 0; a < 4; ++a)
                if (min(max(i0 - 1 + a, 0), G - 1) == g) wsum += wt[a];
            if (wsum != 0.f) acc += wsum * src[(size_t)j * inner];
        }
        out[i] = acc;
    }
}

// autocast's bf16 copy of an fp32 weight [rows][cols] into a [rows][ld] operand, zero padded (the patch projection's k tiles)
__global__ void dt_cast_pad_kernel(const float* __restrict__ src, bf16* __restrict__ dst, int rows, int cols, int ld) {
    const long long total = (long long)rows * ld;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % ld);
        const long long r = i / ld;
        dst[i] = __float2bfloat16_rn(c < cols ? src[r * cols + c] : 0.f);
    }
}
// dst = float(bf16(src)): the bias gradient of an nn.Linear under autocast is the bf16 column sum of its bf16 output gradient
__global__ void dt_round_bf16_kernel(const float* __restrict__ src, float* __restrict__ dst, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __bfloat162float(__float2bfloat16_rn(src[i]));
}
