// gemm.h — host interface of the dense bf16 tensor-core GEMMs (gemm.cu).  Callers describe a GEMM; gemm.cu chooses the kernel
// (the wgmma kernel of gemm_wgmma.cuh or the mma.sync kernels of gemm_dense.cuh), builds its tensor maps and sizes its grid.
#pragma once
#include "common.cuh"

//   A operand addressing modes
//     A_PLAIN   : row-major [M, lda]
//     A_CONV3x3 : implicit im2col of an NHWC tensor for a 3x3 / pad 1 / stride 1 convolution, optionally reading a
//                 nearest-2x up-sampled view of the source (Upsample, tokenizer/tokenizer_image/vq_model.py:368-379);
//                 K index = tap*Cin + c, tap = ky*3+kx; row m = (b*Ho + y)*Wo + x
//     A_CONV3x3S2: 3x3 / stride 2 on an input padded (0,1,0,1) (Downsample, vq_model.py:382-397)
//     A_WIN      : kh x kw window, stride s, over an already padded NHWC source [B][Hs][Ws][Cin] (no bounds checks in the
//                  window): row m = (b*Ho + oy)*Wo + ox reads pixels (s*oy + ky, s*ox + kx), K index = (ky*kw + kx)*Cin + c.
//                  fp32 output through a pixel map: row (b, oy, ox) is stored at pixel (osy*oy + oay, osx*ox + oax) of an
//                  [B][oH][oW][ldc] tensor.  Own instantiation (dense_win_gemm_kernel); dense_gemm_kernel does not take it.
//   B operand: row-major [N, K] (nn.Linear / flattened conv weight [Cout, 9*Cin] in (ky,kx,c) order)
//   batched via blockIdx.z with element strides.
enum { A_PLAIN = 0, A_CONV3x3 = 1, A_CONV3x3S2 = 2, A_WIN = 3 };
enum { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_GELU_ERF = 2, ACT_RELU = 3 };

struct DenseP {
    const bf16* A; const bf16* B;
    int M, N, K;
    int lda, ldb;
    long long sA, sB, sC, sR;          // batch strides (elements) for A, B, C, resid
    int amode; int Hs, Ws, Cin, Ho, Wo, ups;   // conv source dims (before up-sampling), output dims
    // epilogue: v = acc*alpha (+bias[n] | bias[m]); v = rnd(v); act; (*scale[n]); (+resid); store
    float alpha;
    const bf16* bias; int bias_along_m;
    const float* bias_f;               // fp32 bias (per n), fp32-output modes
    const float* resid_f;              // fp32 residual [M, ldr] (+ z * sR), fp32-output modes: added without rounding
    int act;
    const bf16* scale;                 // LayerScale lambda (per n), applied after rounding: r(r(v)*scale)
    const bf16* resid; int ldr;        // residual added last: r(v + resid)
    void* C; int ldc;
    int out_mode;                      // 0: bf16 [M, ldc]; 1: fp32 [M, ldc]; 2: fp32 NCHW image: C[(b*N + n)*Ho*Wo + pix]
    int kh, kw, ws;                    // A_WIN: window and stride
    int osy, osx, oay, oax, oH, oW;    // A_WIN: output pixel map
};

inline DenseP dp_plain(const bf16* A, int lda, const bf16* B, int ldb, int M, int N, int K, void* C, int ldc) {
    DenseP p;
    memset(&p, 0, sizeof(p));
    p.A = A; p.B = B; p.M = M; p.N = N; p.K = K; p.lda = lda; p.ldb = ldb; p.C = C; p.ldc = ldc; p.alpha = 1.f;
    return p;
}

// A wgmma convolution tile is WG_TW x WG_TH output pixels of one image by one WG_CBLK-channel block of the NHWC source.
constexpr int WG_TW = 16, WG_TH = 8, WG_CBLK = 64;

// C = epi(A · B^T) over `batch` GEMMs.  Runs on the wgmma kernel when its epilogue implements every field set in p and the
// operands fit its tensor maps, otherwise on the mma.sync kernel (A_WIN: always its window instantiation).  alpha == 0 means 1.
int gemm(cudaStream_t st, const DenseP& p, int batch = 1);

// fp32-output wgmma GEMMs over split-bf16 ("x3") operands: out fp32 [M][ldc] = A [M][K] · B [N][K]^T + bias (+ resid [M][ldc]),
// no rounding; bias and resid may be null.  N % 8 == 0, K % 8 == 0, 16-byte aligned operands.
int gemm_f32(cudaStream_t st, const bf16* A, const bf16* B, int M, int N, int K, const float* bias, const float* resid, float* out, int ldc);
// 3x3 / pad 1 / stride 1 convolution: src NHWC frame [nimg][fh][fw][cin] (fh >= H, fw >= W, zero outside the H x W map; cin a
// multiple of WG_CBLK), B [N][9 cin] in (ky, kx, c) order -> out fp32 NHWC [nimg][H][W][N] = conv + bias (+ resid, same shape).
int gemm_f32_conv3(cudaStream_t st, const bf16* src, int fh, int fw, const bf16* B, int nimg, int H, int W, int cin, int N, const float* bias,
                   const float* resid, float* out);
