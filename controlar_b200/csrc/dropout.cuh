// dropout.cuh — the keep decisions of the training path's dropout layers (reference gpt_t2i.py:217,290,430 nn.Dropout and the
// stochastic depth of utils/drop_path.py, TransformerBlock gpt_t2i.py:305-306).  The row passes of the training forward / backward
// (train.cuh, train_bwd.cuh) take a TrDrop and apply the masks as they write; a site that is off skips its mask steps.
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

// What one row pass applies.  Element dropout (nn.Dropout on CUDA): x * mask * scale in fp32, scale = fp32(1 / keep), one
// rounding to the tensor's dtype; off when keep >= 1.  Drop path: x * bf16(bernoulli(keep) / keep) on the bf16 branch, one draw
// per sample; off when path_keep >= 1.  TrDrop{} is both off; seed is read only when one of them is on.
struct TrDrop {
    const uint64_t* seed = nullptr;
    int site = CAR_DROP_TOKEN, layer = 0;
    float keep = 1.f, scale = 1.f;
    int path_site = 0;
    float path_keep = 1.f, path_mult = 1.f;
};

__device__ __forceinline__ uint64_t tr_drop_seed(const TrDrop& dr) { return dr.keep < 1.f || dr.path_keep < 1.f ? *dr.seed : 0; }

// the keep words of columns 4 c4 .. 4 c4 + 3 of (sample b, row); zeros when element dropout is off (then nothing reads them)
__device__ __forceinline__ uint4 tr_drop_words(const TrDrop& dr, uint64_t seed, int b, int row, int c4) {
    return dr.keep < 1.f ? car_dropout_bits(seed, dr.site, dr.layer, b, row, c4) : make_uint4(0, 0, 0, 0);
}

__device__ __forceinline__ float tr_path_mult(const TrDrop& dr, uint64_t seed, int b) {
    if (dr.path_keep >= 1.f) return 1.f;
    return car_keep_bit(car_dropout_bits(seed, dr.path_site, dr.layer, b, 0, 0).x, dr.path_keep) * dr.path_mult;
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
