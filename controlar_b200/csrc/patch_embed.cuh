// patch_embed.cuh — the control encoders' patch embedding front end: the control-map resize fused with the patch im2col and the
// bicubic interpolation of the position embeddings.  Templates and device functions only, so that the inference encoder
// (car_vision.cu) and the trainable one (car_train.cu) can both instantiate them.
#pragma once
#include "common.cuh"

// ---- control-map resize to multiples of the patch size P (dinov2_adapter.py:16-24) fused with the PxP patch im2col:
// out[b*hw + py*w + px][c*P*P + ky*P + kx] (Kpad columns, zero padded) = resized[b][c][py*P+ky][px*P+kx]
// mode 0: F.interpolate(mode='nearest')  src = floor(dst * in/out)
// mode 1: bicubic, align_corners=True (A = -0.75), computed in fp32 and rounded to the model dtype like
//         upsample_bicubic2d on a bf16 tensor (opmath float, output cast)
__device__ __forceinline__ float cubic1(float x) { const float A = -0.75f; return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x) { const float A = -0.75f; return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
template <typename TI>
__global__ void resize_patchify_kernel(const TI* __restrict__ img, bf16* __restrict__ out, int B, int H, int W, int h, int w,
                                       int Kpad, int mode, int P) {
    // P = patch size: 14 (DINOv2: the map is first resized to (h*14, w*14)) or 16 (ViT-S/16 of the legacy c2i class,
    // vit_adapter.py:13-15: no resize — with nh == H the nearest mode below is the identity)
    const int nh = h * P, nw = w * P, PP = P * P;
    const long long total = (long long)B * h * w * Kpad;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % Kpad);
        const long long row = i / Kpad;
        float v = 0.f;
        if (k < 3 * PP) {
            const int c = k / PP, r = k % PP, ky = r / P, kx = r % P;
            const int px = (int)(row % w), py = (int)((row / w) % h), b = (int)(row / ((long long)w * h));
            const int oy = py * P + ky, ox = px * P + kx;
            const TI* src = img + ((size_t)b * 3 + c) * H * W;
            if (mode == 0) {
                const int sy = min((int)floorf(oy * ((float)H / nh)), H - 1);
                const int sx = min((int)floorf(ox * ((float)W / nw)), W - 1);
                v = tof(src[(size_t)sy * W + sx]);
            } else {
                const float fy = nh > 1 ? oy * ((float)(H - 1) / (nh - 1)) : 0.f;
                const float fx = nw > 1 ? ox * ((float)(W - 1) / (nw - 1)) : 0.f;
                const int iy = (int)floorf(fy), ix = (int)floorf(fx);
                const float ty = fy - iy, tx = fx - ix;
                const float wy[4] = {cubic2(ty + 1.f), cubic1(ty), cubic1(1.f - ty), cubic2(2.f - ty)};
                const float wx[4] = {cubic2(tx + 1.f), cubic1(tx), cubic1(1.f - tx), cubic2(2.f - tx)};
                float acc = 0.f;
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    const int yy = min(max(iy - 1 + a, 0), H - 1);
                    float rowv = 0.f;
#pragma unroll
                    for (int bb = 0; bb < 4; ++bb) {
                        const int xx = min(max(ix - 1 + bb, 0), W - 1);
                        rowv += tof(src[(size_t)yy * W + xx]) * wx[bb];
                    }
                    acc += rowv * wy[a];
                }
                v = acc;
            }
        }
        out[i] = fromf<bf16>(v);
    }
}

// position embeddings: bicubic (align_corners=False, A=-0.75, fp32) resize of the [G,G,C] grid to [h,w,C], cast to
// the model dtype (modeling_dinov2.py interpolate_pos_encoding); pos: [1 + G*G, C].  TO = float: the fp32 table of training.
template <typename TI, typename TO = bf16>
__global__ void pos_embed_interp_kernel(const TI* __restrict__ pos, TO* __restrict__ out /*[h*w][C]*/, int G, int h, int w, int C) {
    const long long total = (long long)h * w * C;
    const float sy = (float)G / h, sx = (float)G / w;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int ox = (int)((i / C) % w), oy = (int)(i / ((long long)C * w));
        const float fy = (oy + 0.5f) * sy - 0.5f, fx = (ox + 0.5f) * sx - 0.5f;
        const int iy = (int)floorf(fy), ix = (int)floorf(fx);
        const float ty = fy - iy, tx = fx - ix;
        const float wy[4] = {cubic2(ty + 1.f), cubic1(ty), cubic1(1.f - ty), cubic2(2.f - ty)};
        const float wx[4] = {cubic2(tx + 1.f), cubic1(tx), cubic1(1.f - tx), cubic2(2.f - tx)};
        float acc = 0.f;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int yy = min(max(iy - 1 + a, 0), G - 1);
            float rowv = 0.f;
#pragma unroll
            for (int bb = 0; bb < 4; ++bb) {
                const int xx = min(max(ix - 1 + bb, 0), G - 1);
                rowv += tof(pos[(size_t)(1 + yy * G + xx) * C + c]) * wx[bb];
            }
            acc += rowv * wy[a];
        }
        out[i] = fromf<TO>(acc);
    }
}
