// gemm_dense.cuh — tiled bf16 tensor-core GEMM for the dense (M >= 128) stages: DINOv2 linears/attention, VQGAN
// convolutions as implicit GEMM (NHWC), VQGAN attention.  C[M,N] = epi(A[M,K] · B[N,K]^T), fp32 accumulate.
// A operand addressing modes and the DenseP fields: gemm.h.
//
// Round-1 implementation note: mma.sync m16n8k16 + cp.async 3-stage pipeline + ldmatrix (the robust legacy tensor
// path).  gemm() (gemm.cu) sends the plain GEMMs and 3x3 convolutions that fit the TMA tile walk to gemm_wgmma.cuh
// instead; this kernel takes the batched, strided, up-sampling and fp32-output cases.
#pragma once
#include "gemm.h"

constexpr int DG_BM = 128, DG_BN = 128, DG_BK = 32, DG_STAGES = 3, DG_THREADS = 256;
constexpr int DG_SMEM = DG_STAGES * (DG_BM + DG_BN) * DG_BK * 2;   // 48 KB

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gsrc, bool valid) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gsrc), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// smem tile layout: rows of 32 bf16 (64 B = 4 chunks of 16 B); chunk index XOR-swizzled with (row>>1)&3 so that
// ldmatrix (8 rows x 16 B) and the 16-B cp.async stores are bank-conflict free.
__device__ __forceinline__ int dg_off(int row, int chunk) { return row * DG_BK + ((chunk ^ ((row >> 1) & 3)) << 3); }

template <bool WIN>
__device__ __forceinline__ void dense_gemm_body(const DenseP& p) {
    extern __shared__ __align__(128) unsigned char dg_smem[];
    bf16* sA = reinterpret_cast<bf16*>(dg_smem);
    bf16* sB = sA + DG_STAGES * DG_BM * DG_BK;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 2, wn = warp & 3;            // 2 x 4 warps -> warp tile 64 x 32
    const int m0 = blockIdx.y * DG_BM, n0 = blockIdx.x * DG_BN;
    const int z = blockIdx.z;
    const bf16* A = p.A + (size_t)z * p.sA;
    const bf16* B = p.B + (size_t)z * p.sB;
    const int ktiles = (p.K + DG_BK - 1) / DG_BK;

    // each thread copies 2 A chunks and 2 B chunks per k-tile: chunk id c = tid + i*256 -> row = c>>2, kc = c&3
    int a_row[2], a_kc[2];
    // conv decode of the two A rows this thread loads
    int cb[2], cy[2], cx[2];
    bool a_ok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c = tid + i * DG_THREADS;
        a_row[i] = c >> 2; a_kc[i] = c & 3;
        const int m = m0 + a_row[i];
        a_ok[i] = m < p.M;
        if (p.amode != A_PLAIN) {
            const int hw = p.Ho * p.Wo;
            const int mm = a_ok[i] ? m : 0;
            cb[i] = mm / hw; const int r = mm - cb[i] * hw; cy[i] = r / p.Wo; cx[i] = r - cy[i] * p.Wo;
        }
    }
    auto load_tile = [&](int stage, int kt) {
        bf16* a_s = sA + stage * DG_BM * DG_BK;
        bf16* b_s = sB + stage * DG_BN * DG_BK;
        const int kbase = kt * DG_BK;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int k = kbase + a_kc[i] * 8;
            const bf16* src = A;
            bool ok = a_ok[i] && k < p.K;
            if (p.amode == A_PLAIN) {
                src = A + (size_t)(m0 + a_row[i]) * p.lda + k;
            } else {
                const int tap = k / p.Cin, c = k - tap * p.Cin;
                if constexpr (WIN) {
                    const int ky = tap / p.kw, kx = tap - ky * p.kw;
                    src = A + (((size_t)cb[i] * p.Hs + cy[i] * p.ws + ky) * p.Ws + cx[i] * p.ws + kx) * p.Cin + c;
                    cp_async16_zfill(a_s + dg_off(a_row[i], a_kc[i]), ok ? src : A, ok);
                    continue;
                }
                const int ky = tap / 3, kx = tap - ky * 3;
                int yy, xx;
                if (p.amode == A_CONV3x3) { yy = cy[i] + ky - 1; xx = cx[i] + kx - 1; }
                else { yy = cy[i] * 2 + ky; xx = cx[i] * 2 + kx; }            // pad (0,1,0,1): only bottom/right OOB
                const int Hv = p.Hs << p.ups, Wv = p.Ws << p.ups;            // virtual (up-sampled) source dims
                ok = ok && yy >= 0 && yy < Hv && xx >= 0 && xx < Wv;
                if (ok) src = A + (((size_t)cb[i] * p.Hs + (yy >> p.ups)) * p.Ws + (xx >> p.ups)) * p.Cin + c;
            }
            cp_async16_zfill(a_s + dg_off(a_row[i], a_kc[i]), ok ? src : A, ok);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int c = tid + i * DG_THREADS;
            const int row = c >> 2, kc = c & 3;
            const int k = kbase + kc * 8;
            const bool ok = (n0 + row) < p.N && k < p.K;
            cp_async16_zfill(b_s + dg_off(row, kc), ok ? B + (size_t)(n0 + row) * p.ldb + k : B, ok);
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f; }

#pragma unroll
    for (int s = 0; s < DG_STAGES - 1; ++s) {
        if (s < ktiles) load_tile(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < ktiles; ++kt) {
        cp_async_wait<DG_STAGES - 2>();
        __syncthreads();
        const int nk = kt + DG_STAGES - 1;
        if (nk < ktiles) load_tile(nk % DG_STAGES, nk);
        cp_async_commit();
        const bf16* a_s = sA + (kt % DG_STAGES) * DG_BM * DG_BK;
        const bf16* b_s = sB + (kt % DG_STAGES) * DG_BN * DG_BK;
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {                 // two k16 steps per k-tile
            uint32_t af[4][4], bfm[4][2];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = wm * 64 + i * 16 + (lane & 15);
                const int chunk = kk * 2 + (lane >> 4);
                ldmatrix_x4(af[i][0], af[i][1], af[i][2], af[i][3], a_s + dg_off(row, chunk));
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {                // each x4 covers two n8 blocks
                const int row = wn * 32 + j * 16 + (lane & 7) + ((lane >> 4) << 3);
                const int chunk = kk * 2 + ((lane >> 3) & 1);
                uint32_t r0, r1, r2, r3;
                ldmatrix_x4(r0, r1, r2, r3, b_s + dg_off(row, chunk));
                bfm[j * 2][0] = r0; bfm[j * 2][1] = r1; bfm[j * 2 + 1][0] = r2; bfm[j * 2 + 1][1] = r3;
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_bf16_16816(acc[i][j], af[i][0], af[i][1], af[i][2], af[i][3], bfm[j][0], bfm[j][1]);
        }
    }
    cp_async_wait<0>();

    // ---- epilogue
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int m = m0 + wm * 64 + i * 16 + g + hh * 8;
            if (m >= p.M) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = n0 + wn * 32 + j * 8 + 2 * t + e;
                    if (n >= p.N) continue;
                    if constexpr (WIN) {   // fp32 bias, pixel-mapped fp32 store
                        const int hw = p.Ho * p.Wo;
                        const int b = m / hw, r = m - b * hw, oy = r / p.Wo, ox = r - oy * p.Wo;
                        const size_t pix = ((size_t)b * p.oH + p.osy * oy + p.oay) * p.oW + p.osx * ox + p.oax;
                        ((float*)p.C)[pix * p.ldc + n] = acc[i][j][hh * 2 + e] + p.bias_f[n];
                        continue;
                    }
                    float v = acc[i][j][hh * 2 + e] * p.alpha;
                    if (p.bias) v += tof(p.bias[p.bias_along_m ? m : n]);
                    if (p.bias_f) v += p.bias_f[n];
                    if (p.resid_f) v += p.resid_f[(size_t)z * p.sR + (size_t)m * p.ldr + n];
                    if (p.out_mode == 0) v = rnd<bf16>(v);
                    if (p.act == ACT_GELU_TANH) v = rnd<bf16>(gelu_tanh_f(v));
                    else if (p.act == ACT_GELU_ERF) v = rnd<bf16>(gelu_erf_f(v));
                    else if (p.act == ACT_RELU) v = fmaxf(v, 0.f);
                    if (p.scale) v = rnd<bf16>(v * tof(p.scale[n]));
                    if (p.resid) v = rnd<bf16>(v + tof(p.resid[(size_t)z * p.sR + (size_t)m * p.ldr + n]));
                    if (p.out_mode == 0) ((bf16*)p.C)[(size_t)z * p.sC + (size_t)m * p.ldc + n] = fromf<bf16>(v);
                    else if (p.out_mode == 1) ((float*)p.C)[(size_t)z * p.sC + (size_t)m * p.ldc + n] = v;
                    else {
                        const int hw = p.Ho * p.Wo;
                        const int b = m / hw, pix = m - b * hw;
                        ((float*)p.C)[((size_t)b * p.N + n) * hw + pix] = v;
                    }
                }
            }
        }
    }
}
__global__ void __launch_bounds__(DG_THREADS) dense_gemm_kernel(DenseP p) { dense_gemm_body<false>(p); }
__global__ void __launch_bounds__(DG_THREADS) dense_win_gemm_kernel(DenseP p) { dense_gemm_body<true>(p); }
