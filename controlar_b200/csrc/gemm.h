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
    // epilogue: v = acc*alpha (+bias[n] | bias[m]) (+bias_f[n]) (+resid_f); v = rnd(v) (out_mode 0 only); act (GELU: r(gelu(v)));
    // (*scale[n]); (+resid); store.  fp32 sums in this order; rnd = round to bf16 (nearest even).
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

// The contract gemm() checks before any launch (gemm_route).  Every descriptor outside it is refused with CAR_ERR_ARG and a message
// naming the field; no field is ever ignored.
//   all modes : A, B, C non-null; M, N >= 0 (M == 0 or N == 0 launches nothing); K > 0; 1 <= batch <= 65535; amode, act and
//               out_mode known; alpha == 0 means 1.  The mma.sync loader moves 16-byte chunks, so K, ldb (and lda, Cin) are
//               multiples of 8, ldb >= K, and A and B are 16-byte aligned; with batch > 1, sA and sB are multiples of 8 (0 broadcasts).
//               bias_along_m needs a bf16 bias; resid and resid_f need ldr >= N.
//   bf16-only : scale, resid and GELU round to bf16, so they need out_mode 0.
//   out_mode  : 0 and 1 need ldc >= N (C advances by sC per batch).  2 (NCHW) writes image b = m / (Ho Wo): it needs batch == 1,
//               ldc == 0 and M a multiple of Ho Wo.
//   A_PLAIN   : lda >= K, lda % 8 == 0.
//   A_CONV3x3, A_CONV3x3S2: Hs, Ws, Ho, Wo > 0, M a multiple of Ho Wo, K == 9 Cin; ups (0 or 1) only with A_CONV3x3.
//   A_WIN     : its epilogue is acc + bias_f[n] stored as fp32 through the pixel map, so it needs bias_f, out_mode 1, ldc >= N and
//               batch == 1, and refuses alpha != 1, bias, act, scale, resid and resid_f.  kh, kw, ws >= 1, K == kh kw Cin, every
//               window inside the Hs x Ws source, M a multiple of Ho Wo, osy, osx >= 1, oay, oax >= 0 and every mapped pixel inside oH x oW.
// Routes: the wgmma kernel takes A_PLAIN and exact-fit A_CONV3x3 (no ups, Cin % 64 == 0, Ho == Hs >= 8, Wo == Ws >= 16) when the
// epilogue is its own (batch 1, out_mode 0, alpha 1, bias along n, act none or GELU, no bias_f / resid_f) and C, resid fit its
// paired stores (N, ldc, ldr multiples of 8, 16-byte aligned); A_WIN takes the window kernel; everything else the mma.sync kernel.
enum { GEMM_WGMMA = 0, GEMM_WGMMA_CONV3 = 1, GEMM_MMA = 2, GEMM_MMA_WIN = 3 };
// the route gemm() takes for (p, batch), or CAR_ERR_ARG (message in car_last_error) when the descriptor is outside the contract;
// host only, never touches the device
int gemm_route(const DenseP& p, int batch = 1);

// C = epi(A · B^T) over `batch` GEMMs, on the kernel gemm_route(p, batch) names.
int gemm(cudaStream_t st, const DenseP& p, int batch = 1);

// fp32-output wgmma GEMMs over split-bf16 ("x3") operands: out fp32 [M][ldc] = A [M][K] · B [N][K]^T + bias (+ resid [M][ldc]),
// no rounding; bias and resid may be null.  M >= 0, N > 0 and N % 8 == 0, K > 0 and K % 8 == 0, ldc >= N and even; A and B
// 16-byte aligned, out and resid 8-byte aligned.  Checked before any launch (CAR_ERR_ARG).
int gemm_f32(cudaStream_t st, const bf16* A, const bf16* B, int M, int N, int K, const float* bias, const float* resid, float* out, int ldc);
// Decode-step GEMM for 1 <= M <= 64 rows (the wide decode route, car_api.cu): A bf16 [M][lda] (one m64 wgmma tile) times the
// weights B bf16 [N][K] (nn.Linear layout, read in place), fp32 accumulate, then the decode epilogue `ep` (EpiParams,
// gemm_skinny.cuh: QKV + RoPE + KV append, residual (+ control add), SwiGLU, logits).  B3: the w3 weights of the SwiGLU epilogue
// (given exactly when ep.kind == EPI_SWIGLU), over the same N columns as B = w1.  K is split over CTAs as gemm_wide_plan says;
// with more than one split the fp32 partials go to `part` (part_bytes >= plan.part_bytes) and `tickets` (n_tickets >= plan.tiles,
// zero before the first launch, left zero by every launch), and they are summed in split order: results do not depend on timing
// and a row's result does not depend on the other rows.  N, K multiples of 8, lda >= K and a multiple of 8, A, B, B3 16-byte
// aligned.  Checked before any launch (CAR_ERR_ARG).
struct EpiParams;
struct WidePlan { int tiles, splits, kper; size_t part_bytes; };
WidePlan gemm_wide_plan(int M, int N, int K, bool dual);
int gemm_wide(cudaStream_t st, const bf16* A, int lda, const bf16* B, const bf16* B3, int M, int N, int K, const EpiParams& ep, float* part,
              size_t part_bytes, int* tickets, int n_tickets);
// 3x3 / pad 1 / stride 1 convolution: src NHWC frame [nimg][fh][fw][cin] (fh >= max(H, 8), fw >= max(W, 16), zero outside the
// H x W map; cin a positive multiple of WG_CBLK), B [N][9 cin] in (ky, kx, c) order -> out fp32 NHWC [nimg][H][W][N] = conv + bias
// (+ resid, same shape).  nimg, H, W > 0, N > 0 and N % 8 == 0; src and B 16-byte aligned, out and resid 8-byte aligned.  Checked
// before any launch (CAR_ERR_ARG).
int gemm_f32_conv3(cudaStream_t st, const bf16* src, int fh, int fw, const bf16* B, int nimg, int H, int W, int cin, int N, const float* bias,
                   const float* resid, float* out);
