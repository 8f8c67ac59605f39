// midas.cuh — the ResNet-50 trunk of MiDaS DPT-Hybrid (reference condition/midas/midas/vit.py, timm ResNetV2 with preact=False and
// stem_type "same"), fp32 in the reference => fp32-grade here.  The convolutions run on the split-bf16 ("x3", split3.cuh) GEMMs of
// car_vision.cu, the stem's input written by image_split3_kernel with TF "SAME" padding of the 7x7/2 stem (2 before, 3 after; the
// sides are even).  The kernel below standardises the weights: per output channel (w - mean) / sqrt(biased var + 1e-8),
// statistics in fp64, once at create time.  GroupNorm(32, eps 1e-5) is groupnorm.cuh's: the shared fp32 statistics, then gn_apply_s3_kernel fusing the affine, the residual
// (optionally group-normalised itself: the downsample shortcut), ReLU, the stem's 3x3/2 max-pool and the padded S3 write of the next
// convolution's operand.  The ViT, reassemble, fusion and head stages are the DPT kernels (dpt.cuh).
#pragma once
#include "split3.cuh"

constexpr int MD_THREADS = 256;

// fp32 weight [n][K] -> standardised fp32 weight [n][K]; one block per output channel, fp64 statistics in a fixed order
__global__ void __launch_bounds__(MD_THREADS) midas_ws_kernel(const float* __restrict__ w, float* __restrict__ y, int K, double eps) {
    __shared__ double red[MD_THREADS];
    const float* x = w + (size_t)blockIdx.x * K;
    double s = 0.0;
    for (int k = threadIdx.x; k < K; k += MD_THREADS) s += (double)x[k];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = MD_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    const double mean = red[0] / K;
    __syncthreads();
    double q = 0.0;
    for (int k = threadIdx.x; k < K; k += MD_THREADS) { const double d = (double)x[k] - mean; q += d * d; }
    red[threadIdx.x] = q;
    __syncthreads();
    for (int o = MD_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    const double inv = 1.0 / sqrt(red[0] / K + eps);
    for (int k = threadIdx.x; k < K; k += MD_THREADS) y[(size_t)blockIdx.x * K + k] = (float)(((double)x[k] - mean) * inv);
}
