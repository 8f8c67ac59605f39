// gemm.cu — the one place a dense tensor-core GEMM picks its kernel, gets its TMA tensor maps, shared-memory opt-in and grid.
#include "gemm.h"
#include "gemm_dense.cuh"
#include "gemm_wgmma.cuh"

static_assert(ACT_GELU_TANH == 1 && ACT_GELU_ERF == 2, "WgP::act takes the ACT_* codes of the activations the wgmma epilogue implements");

// ---- TMA tensor maps (driver entry point fetched through the runtime: the library does not link libcuda) ----
typedef CUresult (*wg_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static wg_encode_fn wg_encoder() {
    static wg_encode_fn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
        return (wg_encode_fn)f;
    }();
    return fn;
}
// bf16 tensor of `rank` dimensions (innermost first, byte strides of the outer ones), 128-byte swizzle, zero fill out of bounds
static int wg_encode(CUtensorMap* map, cuuint32_t rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box) {
    const wg_encode_fn enc = wg_encoder();
    if (!enc) CAR_FAIL(CAR_ERR_UNSUPPORTED, "the wgmma GEMM needs the driver's TMA tensor-map encoder (cuTensorMapEncodeTiled)");
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    if (enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        CAR_FAIL(CAR_ERR_CUDA, "cuTensorMapEncodeTiled failed");
    return CAR_OK;
}
// row-major bf16 matrix [rows][cols] with row pitch ld elements; box = 64 columns x box_rows rows
static int wg_make_map(CUtensorMap* map, const void* base, int rows, int cols, int ld, int box_rows = WG_BM) {
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    const cuuint32_t box[2] = {WG_BK, (cuuint32_t)box_rows};
    return wg_encode(map, 2, base, dims, strides, box);
}
// NHWC bf16 tensor [N][H][W][C] as a 4-D map {C, W, H, N}; box = {64 channels, 16 x, 8 y, 1 image}
static int wg_make_map_nhwc(CUtensorMap* map, const void* base, int N, int H, int W, int C) {
    const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    const cuuint32_t box[4] = {WG_BK, WG_TW, WG_TH, 1};
    return wg_encode(map, 4, base, dims, strides, box);
}

// ---- launchers: one shared-memory opt-in and one grid rule per kernel ----
// wgmma: persistent, at most one CTA per SM over the tiles_m x n-tiles schedule
template <bool F32>
static int wg_launch(cudaStream_t st, const CUtensorMap& mapA, const CUtensorMap& mapB, const WgP& q, int tiles_m) {
    static DevOnce once;
    const auto kernel = F32 ? gemm_wgmma_f32_kernel : gemm_wgmma_kernel;
    if (once.first()) CAR_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM));
    const int ntiles = tiles_m * ((q.N + WG_BN - 1) / WG_BN);
    CAR_LAUNCH(kernel, std::min(ntiles, sm_count()), WG_THREADS, WG_SMEM, st, mapA, mapB, q);
    return CAR_OK;
}
// wgmma plain GEMM: q holds M, N, K and the epilogue; A [M][lda], B [N][ldb]
template <bool F32>
static int wg_plain(cudaStream_t st, const WgP& q, const bf16* A, int lda, const bf16* B, int ldb) {
    alignas(64) CUtensorMap mapA, mapB;
    CAR_TRY(wg_make_map(&mapA, A, q.M, q.K, lda));
    CAR_TRY(wg_make_map(&mapB, B, q.N, q.K, ldb));
    return wg_launch<F32>(st, mapA, mapB, q, (q.M + WG_BM - 1) / WG_BM);
}
// wgmma 3x3 / pad 1 convolution (one 4-D TMA box per (tap, 64-channel block), padding by TMA zero fill): q holds M = nimg H W, N,
// K = 9 cin and the epilogue; src NHWC frame [nimg][fh][fw][cin] around the H x W map, B [N][ldb]
template <bool F32>
static int wg_conv3(cudaStream_t st, WgP q, const bf16* src, int nimg, int fh, int fw, int cin, int H, int W, const bf16* B, int ldb) {
    alignas(64) CUtensorMap mapA, mapB;
    CAR_TRY(wg_make_map_nhwc(&mapA, src, nimg, fh, fw, cin));
    CAR_TRY(wg_make_map(&mapB, B, q.N, q.K, ldb));
    q.conv = 1; q.H = H; q.W = W; q.tiles_x = (W + WG_TW - 1) / WG_TW; q.tiles_y = (H + WG_TH - 1) / WG_TH; q.cblks = cin / WG_BK;
    return wg_launch<F32>(st, mapA, mapB, q, nimg * q.tiles_x * q.tiles_y);
}
// mma.sync: one CTA per 128 x 128 output tile, blockIdx.z over the batch
template <bool WIN>
static int dg_launch(cudaStream_t st, const DenseP& p, int batch) {
    static DevOnce once;
    const auto kernel = WIN ? dense_win_gemm_kernel : dense_gemm_kernel;
    if (once.first()) CAR_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DG_SMEM));
    CAR_LAUNCH(kernel, dim3((p.N + DG_BN - 1) / DG_BN, (p.M + DG_BM - 1) / DG_BM, batch), DG_THREADS, DG_SMEM, st, p);
    return CAR_OK;
}

static bool aligned(const void* p, int bytes) { return ((uintptr_t)p % bytes) == 0; }
static bool aligned16(const void* p) { return aligned(p, 16); }

// the contract of gemm.h, field by field, then the route
int gemm_route(const DenseP& p, int batch) {
    if (!p.A || !p.B || !p.C) CAR_FAIL(CAR_ERR_ARG, "A, B and C must be non-null");
    if (p.M < 0 || p.N < 0) CAR_FAIL(CAR_ERR_ARG, "M and N must be >= 0");
    if (p.K <= 0) CAR_FAIL(CAR_ERR_ARG, "K must be > 0");
    if (batch < 1 || batch > 65535) CAR_FAIL(CAR_ERR_ARG, "batch must be in [1, 65535]");
    if (p.amode < A_PLAIN || p.amode > A_WIN) CAR_FAIL(CAR_ERR_ARG, "unknown amode");
    if (p.act < ACT_NONE || p.act > ACT_RELU) CAR_FAIL(CAR_ERR_ARG, "unknown act");
    if (p.out_mode < 0 || p.out_mode > 2) CAR_FAIL(CAR_ERR_ARG, "out_mode must be 0, 1 or 2");
    // the mma.sync loader: 16-byte cp.async chunks along K
    if (p.K % 8 || p.ldb % 8) CAR_FAIL(CAR_ERR_ARG, "K and ldb must be multiples of 8");
    if (p.ldb < p.K) CAR_FAIL(CAR_ERR_ARG, "ldb must be >= K");
    if (!aligned16(p.A) || !aligned16(p.B)) CAR_FAIL(CAR_ERR_ARG, "A and B must be 16-byte aligned");
    if (batch > 1 && (p.sA % 8 || p.sB % 8)) CAR_FAIL(CAR_ERR_ARG, "sA and sB must be multiples of 8");
    if (p.bias_along_m && !p.bias) CAR_FAIL(CAR_ERR_ARG, "bias_along_m needs a bf16 bias");
    if ((p.resid || p.resid_f) && p.ldr < p.N) CAR_FAIL(CAR_ERR_ARG, "ldr must be >= N");
    const bool gelu = p.act == ACT_GELU_TANH || p.act == ACT_GELU_ERF;
    if (p.out_mode != 0 && (p.scale || p.resid || gelu)) CAR_FAIL(CAR_ERR_ARG, "scale, resid and GELU round to bf16: they need out_mode 0");
    if (p.out_mode == 2) {
        if (batch != 1) CAR_FAIL(CAR_ERR_ARG, "out_mode 2 (NCHW) needs batch 1");
        if (p.ldc != 0) CAR_FAIL(CAR_ERR_ARG, "out_mode 2 (NCHW) has no ldc: it must be 0");
        if (p.Ho <= 0 || p.Wo <= 0 || p.M % (p.Ho * p.Wo)) CAR_FAIL(CAR_ERR_ARG, "out_mode 2 (NCHW) needs Ho, Wo > 0 and M a multiple of Ho Wo");
    } else if (p.ldc < p.N) {
        CAR_FAIL(CAR_ERR_ARG, "ldc must be >= N");
    }
    if (p.amode == A_PLAIN) {
        if (p.lda < p.K || p.lda % 8) CAR_FAIL(CAR_ERR_ARG, "lda must be >= K and a multiple of 8");
    } else {
        if (p.Cin <= 0 || p.Cin % 8) CAR_FAIL(CAR_ERR_ARG, "Cin must be a positive multiple of 8");
        if (p.Hs <= 0 || p.Ws <= 0 || p.Ho <= 0 || p.Wo <= 0) CAR_FAIL(CAR_ERR_ARG, "Hs, Ws, Ho and Wo must be > 0");
        if (p.M % (p.Ho * p.Wo)) CAR_FAIL(CAR_ERR_ARG, "M must be a multiple of Ho Wo");
        if (p.ups != 0 && !(p.ups == 1 && p.amode == A_CONV3x3)) CAR_FAIL(CAR_ERR_ARG, "ups must be 0, or 1 with A_CONV3x3");
    }
    if (p.amode == A_CONV3x3 || p.amode == A_CONV3x3S2) {
        if (p.K != 9 * p.Cin) CAR_FAIL(CAR_ERR_ARG, "a 3x3 convolution needs K == 9 Cin");
    }
    if (p.amode == A_WIN) {
        if (!p.bias_f) CAR_FAIL(CAR_ERR_ARG, "A_WIN needs bias_f");
        if (p.out_mode != 1) CAR_FAIL(CAR_ERR_ARG, "A_WIN stores fp32: out_mode must be 1");
        if (batch != 1) CAR_FAIL(CAR_ERR_ARG, "A_WIN needs batch 1");
        if ((p.alpha != 0.f && p.alpha != 1.f) || p.bias || p.act != ACT_NONE || p.resid_f)
            CAR_FAIL(CAR_ERR_ARG, "A_WIN does not apply alpha, bias, act or resid_f");
        if (p.kh < 1 || p.kw < 1 || p.ws < 1) CAR_FAIL(CAR_ERR_ARG, "kh, kw and ws must be >= 1");
        if (p.K != p.kh * p.kw * p.Cin) CAR_FAIL(CAR_ERR_ARG, "A_WIN needs K == kh kw Cin");
        if ((long long)p.ws * (p.Ho - 1) + p.kh > p.Hs || (long long)p.ws * (p.Wo - 1) + p.kw > p.Ws)
            CAR_FAIL(CAR_ERR_ARG, "A_WIN windows must lie inside the Hs x Ws source");
        if (p.osy < 1 || p.osx < 1 || p.oay < 0 || p.oax < 0) CAR_FAIL(CAR_ERR_ARG, "A_WIN needs osy, osx >= 1 and oay, oax >= 0");
        if ((long long)p.osy * (p.Ho - 1) + p.oay >= p.oH || (long long)p.osx * (p.Wo - 1) + p.oax >= p.oW)
            CAR_FAIL(CAR_ERR_ARG, "A_WIN pixel map must land inside oH x oW");
        return GEMM_MMA_WIN;
    }
    // the wgmma epilogue: bf16 bias along n, bf16 rounding, GELU (tanh or erf), LayerScale, bf16 residual, one bf16 [M][ldc] output
    const bool wg_epi = batch == 1 && p.out_mode == 0 && (p.alpha == 0.f || p.alpha == 1.f) && !p.bias_along_m && !p.bias_f && !p.resid_f &&
                        (p.act == ACT_NONE || gelu);
    // its paired stores: 16-byte row pitches and base pointers, whole 8-column groups (A and B are checked above)
    const bool wg_ok = wg_epi && p.N % 8 == 0 && p.ldc % 8 == 0 && aligned16(p.C) && (!p.resid || (p.ldr % 8 == 0 && aligned16(p.resid)));
    // the convolution walks whole 64-channel blocks of 16 x 8 pixel boxes over an unscaled map
    const bool wg_conv = p.amode == A_CONV3x3 && !p.ups && p.Cin % WG_BK == 0 && p.Ho == p.Hs && p.Wo == p.Ws && p.Hs >= WG_TH && p.Ws >= WG_TW;
    if (wg_ok && p.amode == A_PLAIN) return GEMM_WGMMA;
    if (wg_ok && wg_conv) return GEMM_WGMMA_CONV3;
    return GEMM_MMA;
}

int gemm(cudaStream_t st, const DenseP& dp, int batch) {
    const int route = gemm_route(dp, batch);
    if (route < 0) return route;
    if (dp.M == 0 || dp.N == 0) return CAR_OK;
    DenseP p = dp;
    if (p.alpha == 0.f) p.alpha = 1.f;
    if (route == GEMM_MMA_WIN) return dg_launch<true>(st, p, batch);
    if (route == GEMM_MMA) return dg_launch<false>(st, p, batch);
    WgP q;
    memset(&q, 0, sizeof(q));
    q.M = p.M; q.N = p.N; q.K = p.K; q.resid = p.resid; q.ldr = p.ldr; q.C = (bf16*)p.C; q.ldc = p.ldc;
    q.act = p.act; q.bias = p.bias; q.scale = p.scale;
    if (route == GEMM_WGMMA) return wg_plain<false>(st, q, p.A, p.lda, p.B, p.ldb);
    return wg_conv3<false>(st, q, p.A, p.M / (p.Hs * p.Ws), p.Hs, p.Ws, p.Cin, p.Hs, p.Ws, p.B, p.ldb);
}

int gemm_f32(cudaStream_t st, const bf16* A, const bf16* B, int M, int N, int K, const float* bias, const float* resid, float* out, int ldc) {
    if (!A || !B) CAR_FAIL(CAR_ERR_ARG, "A and B must be non-null");
    if (!out) CAR_FAIL(CAR_ERR_ARG, "out must be non-null");
    // the fp32 epilogue's paired float2 stores and loads
    if (!aligned(out, 8) || (resid && !aligned(resid, 8))) CAR_FAIL(CAR_ERR_ARG, "out and resid must be 8-byte aligned");
    if (M < 0) CAR_FAIL(CAR_ERR_ARG, "M must be >= 0");
    if (N <= 0 || N % 8) CAR_FAIL(CAR_ERR_ARG, "N must be a positive multiple of 8");
    if (K <= 0 || K % 8) CAR_FAIL(CAR_ERR_ARG, "K must be a positive multiple of 8");
    if (ldc < N || ldc % 2) CAR_FAIL(CAR_ERR_ARG, "ldc must be >= N and even");
    if (!aligned16(A) || !aligned16(B)) CAR_FAIL(CAR_ERR_ARG, "A and B must be 16-byte aligned");
    if (M == 0) return CAR_OK;
    WgP q;
    memset(&q, 0, sizeof(q));
    q.M = M; q.N = N; q.K = K; q.bias_f = bias; q.resid_f = resid; q.ldr = ldc; q.C32 = out; q.ldc = ldc;
    return wg_plain<true>(st, q, A, K, B, K);
}

// one CTA per 64-column tile and K split; the fewest splits that give every SM a CTA (fewer fp32 partials to sum), each split
// a whole number of k-blocks.  Depends on the SM count only, so a given card always reduces in the same order.
WidePlan gemm_wide_plan(int M, int N, int K, bool dual) {
    WidePlan w;
    w.tiles = (N + WD_BN - 1) / WD_BN;
    const int nkb = (K + WG_BK - 1) / WG_BK;
    const int want = std::max(1, std::min(nkb, (sm_count() + w.tiles - 1) / w.tiles));
    w.kper = (nkb + want - 1) / want;
    w.splits = (nkb + w.kper - 1) / w.kper;
    w.part_bytes = w.splits > 1 ? (size_t)w.tiles * w.splits * M * (dual ? 2 : 1) * WD_BN * 4 : 0;
    return w;
}

int gemm_wide(cudaStream_t st, const bf16* A, int lda, const bf16* B, const bf16* B3, int M, int N, int K, const EpiParams& ep, float* part,
              size_t part_bytes, int* tickets, int n_tickets) {
    if (!A || !B) CAR_FAIL(CAR_ERR_ARG, "A and B must be non-null");
    if (M < 1 || M > 64) CAR_FAIL(CAR_ERR_ARG, "M must be in [1, 64]");
    if (N <= 0 || N % 8) CAR_FAIL(CAR_ERR_ARG, "N must be a positive multiple of 8");
    if (K <= 0 || K % 8) CAR_FAIL(CAR_ERR_ARG, "K must be a positive multiple of 8");
    if (lda < K || lda % 8) CAR_FAIL(CAR_ERR_ARG, "lda must be >= K and a multiple of 8");
    if (!aligned16(A) || !aligned16(B) || (B3 && !aligned16(B3))) CAR_FAIL(CAR_ERR_ARG, "A, B and B3 must be 16-byte aligned");
    if ((B3 != nullptr) != (ep.kind == EPI_SWIGLU)) CAR_FAIL(CAR_ERR_ARG, "B3 (w3) is given exactly for the SwiGLU epilogue");
    const bool dual = B3 != nullptr;
    const WidePlan w = gemm_wide_plan(M, N, K, dual);
    if (w.splits > 1 && (!part || part_bytes < w.part_bytes || !tickets || n_tickets < w.tiles))
        CAR_FAIL(CAR_ERR_ARG, "split-K workspace or tickets smaller than gemm_wide_plan asks");
    alignas(64) CUtensorMap mapA, mapB, mapB3;
    CAR_TRY(wg_make_map(&mapA, A, M, K, lda, 64));
    CAR_TRY(wg_make_map(&mapB, B, N, K, K, WD_BN));
    CAR_TRY(wg_make_map(&mapB3, dual ? B3 : B, N, K, K, WD_BN));
    WdP q;
    memset(&q, 0, sizeof(q));
    q.M = M; q.N = N; q.K = K; q.splits = w.splits; q.kper = w.kper; q.part = part; q.tickets = tickets; q.ep = ep; q.ep.M = M;
    static DevOnce once;
    if (once.first()) {
        CAR_CUDA(cudaFuncSetAttribute(gemm_wide_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, wd_smem(false)));
        CAR_CUDA(cudaFuncSetAttribute(gemm_wide_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, wd_smem(true)));
    }
    if (dual) CAR_LAUNCH_PDL(gemm_wide_kernel<true>, dim3(w.tiles * w.splits), dim3(WD_THREADS), wd_smem(true), st, mapA, mapB, mapB3, q);
    else CAR_LAUNCH_PDL(gemm_wide_kernel<false>, dim3(w.tiles * w.splits), dim3(WD_THREADS), wd_smem(false), st, mapA, mapB, mapB3, q);
    return CAR_OK;
}

int gemm_f32_conv3(cudaStream_t st, const bf16* src, int fh, int fw, const bf16* B, int nimg, int H, int W, int cin, int N, const float* bias,
                   const float* resid, float* out) {
    if (!src || !B) CAR_FAIL(CAR_ERR_ARG, "src and B must be non-null");
    if (!out) CAR_FAIL(CAR_ERR_ARG, "out must be non-null");
    // the fp32 epilogue's paired float2 stores and loads
    if (!aligned(out, 8) || (resid && !aligned(resid, 8))) CAR_FAIL(CAR_ERR_ARG, "out and resid must be 8-byte aligned");
    if (nimg <= 0 || H <= 0 || W <= 0) CAR_FAIL(CAR_ERR_ARG, "nimg, H and W must be > 0");
    if (cin <= 0 || cin % WG_CBLK) CAR_FAIL(CAR_ERR_ARG, "cin must be a positive multiple of 64");
    if (N <= 0 || N % 8) CAR_FAIL(CAR_ERR_ARG, "N must be a positive multiple of 8");
    if (fh < H || fw < W || fh < WG_TH || fw < WG_TW) CAR_FAIL(CAR_ERR_ARG, "the frame must hold the H x W map and one 16 x 8 pixel box");
    if (!aligned16(src) || !aligned16(B)) CAR_FAIL(CAR_ERR_ARG, "src and B must be 16-byte aligned");
    WgP q;
    memset(&q, 0, sizeof(q));
    q.M = nimg * H * W; q.N = N; q.K = 9 * cin; q.bias_f = bias; q.resid_f = resid; q.ldr = N; q.C32 = out; q.ldc = N;
    return wg_conv3<true>(st, q, src, nimg, fh, fw, cin, H, W, B, q.K);
}
