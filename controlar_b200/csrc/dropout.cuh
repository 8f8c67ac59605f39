// dropout.cuh — the keep decisions of the training path's dropout layers (reference gpt_t2i.py:217,290,430 nn.Dropout and the
// stochastic depth of utils/drop_path.py, TransformerBlock gpt_t2i.py:305-306) and the kernels that fuse them into the existing
// passes of the training forward / backward.
//
// Generator: Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011), stateless and counter based.
// Key = the 64-bit seed, counter = (column / 4, row, sample, site << 16 | layer); the four output words are the decisions of the
// four columns 4 (column / 4) + 0..3.  A decision is a pure function of (seed, site, layer, sample, row, column), so the
// backward's recompute and its gradient kernels regenerate the forward's masks: nothing is stored.  Keep test on word r:
// (r >> 8) * 2^-24 < keep, keep an fp32 value fixed on the host.  Drop path draws word 0 of (column 0, row 0) of its own site.
// oracle/dropout_masks.py restates this bit for bit.
#pragma once
#include "common.cuh"

enum CarDropSite { CAR_DROP_TOKEN = 0, CAR_DROP_RESID = 1, CAR_DROP_FFN = 2, CAR_DROP_PATH_ATTN = 3, CAR_DROP_PATH_FFN = 4 };

__host__ __device__ __forceinline__ void car_philox_round(uint32_t c[4], uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#ifdef __CUDA_ARCH__
    const uint32_t hi0 = __umulhi(M0, c[0]), hi1 = __umulhi(M1, c[2]);
#else
    const uint32_t hi0 = (uint32_t)(((uint64_t)M0 * c[0]) >> 32), hi1 = (uint32_t)(((uint64_t)M1 * c[2]) >> 32);
#endif
    const uint32_t lo0 = M0 * c[0], lo1 = M1 * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}

// the one generator every dropout site uses: four 32-bit words for columns 4 col4 .. 4 col4 + 3 of (site, layer, sample, row)
__device__ __forceinline__ uint4 car_dropout_bits(uint64_t seed, int site, int layer, int sample, int row, int col4) {
    uint32_t c[4] = {(uint32_t)col4, (uint32_t)row, (uint32_t)sample, ((uint32_t)site << 16) | (uint32_t)layer};
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        if (i) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        car_philox_round(c, k0, k1);
    }
    return make_uint4(c[0], c[1], c[2], c[3]);
}

__device__ __forceinline__ float car_keep_bit(uint32_t r, float keep) { return (float)(r >> 8) * 0x1p-24f < keep ? 1.f : 0.f; }

// What one fused pass applies.  Element dropout (nn.Dropout on CUDA): x * mask * scale in fp32, scale = fp32(1 / keep), one
// rounding to the tensor's dtype; off when keep >= 1.  Drop path: x * bf16(bernoulli(keep) / keep) on the bf16 branch, one draw
// per sample; off when path_keep >= 1.  seed == nullptr: both off.
struct TrDrop {
    const uint64_t* seed;
    int site, layer;
    float keep, scale;
    int path_site;
    float path_keep, path_mult;
};

__device__ __forceinline__ float tr_path_mult(const TrDrop& dr, uint64_t seed, int b) {
    if (dr.path_keep >= 1.f) return 1.f;
    return car_keep_bit(car_dropout_bits(seed, dr.path_site, dr.layer, b, 0, 0).x, dr.path_keep) * dr.path_mult;
}

// forward of a residual branch: h[b][s][:] += float(bf16(bf16(o * m * scale) * path)), o = add[b][s][:] bf16 (the wo / w2 output),
// every step skipped when its site is off.  Four columns per thread (one generator call); d % 4 == 0.
__global__ void tr_add_rows_drop_kernel(float* __restrict__ h, const bf16* __restrict__ add, int B, int S, int d, TrDrop dr) {
    const uint64_t seed = *dr.seed;
    const int d4 = d / 4;
    const long long total = (long long)B * S * d4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % d4);
        const long long rs = i / d4;
        const int s = (int)(rs % S), b = (int)(rs / S);
        const uint4 r = dr.keep < 1.f ? car_dropout_bits(seed, dr.site, dr.layer, b, s, c4) : make_uint4(0, 0, 0, 0);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
        const float pm = tr_path_mult(dr, seed, b);
        const size_t o = (size_t)rs * d + 4 * c4;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float v = __bfloat162float(add[o + e]);
            if (dr.keep < 1.f) v = rnd<bf16>(v * car_keep_bit(rr[e], dr.keep) * dr.scale);
            if (dr.path_keep < 1.f) v = rnd<bf16>(v * pm);
            h[o + e] = h[o + e] + v;
        }
    }
}

// backward of the same branch, as autograd orders it: out = bf16(bf16(bf16(dh) * path) * m * scale) — the bf16 gradient the
// wo / w2 output receives from the fp32 stream through drop path and then dropout.
// Token site (the prefix rows of the caption MLP): out[b][j][:] = bf16(dh[b][row0 + j][:] * m * scale), fp32 product first.
__global__ void tr_take_rows_drop_kernel(const float* __restrict__ dh, bf16* __restrict__ out, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = *dr.seed;
    const int d4 = d / 4;
    const long long total = (long long)B * nrows * d4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % d4);
        const long long rj = i / d4;
        const int j = (int)(rj % nrows), b = (int)(rj / nrows);
        const int s = row0 + j;
        const uint4 r = dr.keep < 1.f ? car_dropout_bits(seed, dr.site, dr.layer, b, s, c4) : make_uint4(0, 0, 0, 0);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
        const float pm = tr_path_mult(dr, seed, b);
        const float* src = dh + ((size_t)b * S + s) * d + 4 * c4;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float g = src[e];
            if (dr.site == CAR_DROP_TOKEN) {
                g = g * car_keep_bit(rr[e], dr.keep) * dr.scale;
            } else {
                g = rnd<bf16>(g);
                if (dr.path_keep < 1.f) g = rnd<bf16>(g * pm);
                if (dr.keep < 1.f) g = g * car_keep_bit(rr[e], dr.keep) * dr.scale;
            }
            out[(size_t)rj * d + 4 * c4 + e] = __float2bfloat16_rn(g);
        }
    }
}

// token dropout on the fp32 rows the embedding gathers write (tok_dropout gpt_t2i.py:430, after the cat that promotes to fp32):
// h[b][row0 + j][:] = table[index(b, j)][:] * m * scale — tr_embed_rows_kernel with the mask fused.  One CTA per row.
__global__ void tr_embed_rows_drop_kernel(const float* __restrict__ table, const int* __restrict__ idx, int ld, const unsigned char* __restrict__ drop,
                                          int drop_to, float* __restrict__ h, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = *dr.seed;
    const int bj = blockIdx.x;
    const int b = bj / nrows, j = bj - b * nrows;
    int id = idx[(size_t)b * ld + j];
    if (drop != nullptr && drop[b]) id = drop_to;
    const float* src = table + (size_t)id * d;
    float* dst = h + ((size_t)b * S + row0 + j) * d;
    for (int c4 = threadIdx.x; c4 < d / 4; c4 += blockDim.x) {
        const uint4 r = car_dropout_bits(seed, dr.site, dr.layer, b, row0 + j, c4);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) dst[4 * c4 + e] = src[4 * c4 + e] * car_keep_bit(rr[e], dr.keep) * dr.scale;
    }
}

// the same on the caption MLP's bf16 prefix rows: h[b][row0 + j][:] = float(src[b][j][:]) * m * scale (tr_put_rows_bf16_kernel + mask)
__global__ void tr_put_rows_drop_kernel(const bf16* __restrict__ src, float* __restrict__ h, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = *dr.seed;
    const int d4 = d / 4;
    const long long total = (long long)B * nrows * d4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % d4);
        const long long rj = i / d4;
        const int j = (int)(rj % nrows), b = (int)(rj / nrows);
        const uint4 r = car_dropout_bits(seed, dr.site, dr.layer, b, row0 + j, c4);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int e = 0; e < 4; ++e)
            h[((size_t)b * S + row0 + j) * d + 4 * c4 + e] = __bfloat162float(src[(size_t)rj * d + 4 * c4 + e]) * car_keep_bit(rr[e], dr.keep) * dr.scale;
    }
}

// embedding-table gradient through the token dropout: grad[index(b, j)][:] += dh[b][row0 + j][:] * m * scale (tr_embed_grad_kernel + mask)
__global__ void tr_embed_grad_drop_kernel(const float* __restrict__ dh, const int* __restrict__ idx, int ld, const unsigned char* __restrict__ drop,
                                          int drop_to, float* __restrict__ grad, int B, int nrows, int S, int row0, int d, TrDrop dr) {
    const uint64_t seed = *dr.seed;
    const int bj = blockIdx.x;
    const int b = bj / nrows, j = bj - b * nrows;
    int id = idx[(size_t)b * ld + j];
    if (drop != nullptr && drop[b]) id = drop_to;
    const float* src = dh + ((size_t)b * S + row0 + j) * d;
    float* dst = grad + (size_t)id * d;
    for (int c4 = threadIdx.x; c4 < d / 4; c4 += blockDim.x) {
        const uint4 r = car_dropout_bits(seed, dr.site, dr.layer, b, row0 + j, c4);
        const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) atomicAdd(dst + 4 * c4 + e, src[4 * c4 + e] * car_keep_bit(rr[e], dr.keep) * dr.scale);
    }
}

// conformance view of the generator: out[b][r][c] = keep decision of (site, layer, b, r, c); drop-path sites give every (r, c) of a
// sample that sample's decision
__global__ void car_dropout_mask_kernel(const uint64_t* __restrict__ seed_p, int site, int layer, int B, int rows, int cols, float keep,
                                        uint8_t* __restrict__ out) {
    const uint64_t seed = *seed_p;
    const bool path = site == CAR_DROP_PATH_ATTN || site == CAR_DROP_PATH_FFN;
    const long long total = (long long)B * rows * cols;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % cols);
        const long long br = i / cols;
        const int r = (int)(br % rows), b = (int)(br / rows);
        const uint4 w = path ? car_dropout_bits(seed, site, layer, b, 0, 0) : car_dropout_bits(seed, site, layer, b, r, c >> 2);
        const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
        out[i] = car_keep_bit(ww[path ? 0 : (c & 3)], keep) != 0.f ? 1 : 0;
    }
}
