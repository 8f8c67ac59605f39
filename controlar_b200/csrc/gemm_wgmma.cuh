// gemm_wgmma.cuh — dense bf16 GEMM on the Hopper tensor cores: TMA tensor-map loads (128-byte swizzle) into an mbarrier ring ->
// wgmma.mma_async from shared-memory descriptors, fp32 accumulators in registers -> register epilogue, warp-specialised and
// persistent.  C[M,N] = epi(A[M,K] · B[N,K]^T), fp32 accumulate.
// Used by the prefill (autoregressive/models/gpt_t2i.py:433-470: wqkv / wo / w1 / w3 / w2 over B_eff·T rows) and the control-token
// MLPs (gpt_t2i.py:165-181 over B_eff·N rows).  lda, ldb % 8 == 0 (16-byte row pitch for the tensor map); M, N, K tails are
// zero-filled by TMA on load and masked on store (N % 8 == 0).
//
// Roles (384 threads = 3 warpgroups, one CTA per SM, static tile schedule t = blockIdx.x + i · gridDim.x over 128 x 128 tiles):
//   warpgroup 0, one lane : TMA producer — per 64-wide k-block two cp.async.bulk.tensor (A 128 x 64, B 128 x 64, SWIZZLE_128B)
//                           into a 6-stage ring (32 KB per stage), completion on full[stage] (expect_tx), slot reuse on empty[stage].
//                           It runs ahead into the next tile while the consumers are in their epilogue.
//   warpgroups 1, 2       : consumers — warpgroup g owns output rows [64 (g - 1), +64) of the tile: per k-block four
//                           wgmma.m64n128k16 (A rows of its half, all 128 B rows), one commit group per k-block with one group
//                           left in flight; the stage of the previous k-block is released (empty, one arrive per warp) once
//                           wgmma.wait_group 1 has retired it.  The epilogue applies bf16 round / GELU / LayerScale / residual (same
//                           rounding points as gemm_dense.cuh) straight from the accumulator registers.
// Two instantiations of one body: gemm_wgmma_kernel (the bf16 epilogue above) and gemm_wgmma_f32_kernel (acc + fp32 bias
// (+ fp32 residual) stored as fp32, no rounding: the split-bf16 "x3" GEMMs and 3x3 convolutions of the DPT depth detector).
// Shared-memory descriptors (sm_90 layout): start >> 4 | LBO (unused for swizzled K-major, 1) << 16 | SBO 1024 >> 4 << 32 |
// layout 1 (128-byte swizzle) << 62; the k16 step inside a 128-byte swizzle atom advances the start address by 32 bytes.
#pragma once
#include "gemm.h"
#include "gemm_skinny.cuh"
#include <cuda.h>

constexpr int WG_BM = 128, WG_BN = 128, WG_BK = WG_CBLK, WG_STAGES = 6, WG_THREADS = 384, WG_CONSUMERS = 2;
constexpr int WG_TILE_BYTES = WG_BM * WG_BK * 2;                               // 16 KB per operand and stage
constexpr int WG_STAGE_BYTES = 2 * WG_TILE_BYTES;
constexpr int WG_SMEM = WG_STAGES * WG_STAGE_BYTES + 1024;                     // + 1024-byte alignment slack (swizzle atoms)

struct WgP {
    int M, N, K;
    const bf16* resid; int ldr;
    bf16* C; int ldc;
    int act;            // 0 none, 1 GELU-tanh, 2 exact (erf) GELU
    const bf16* bias;   // per output column, added to the fp32 accumulator before the bf16 rounding (nn.Linear / Conv2d bias)
    const bf16* scale;  // per output column, applied after the activation: r(r(v) * scale) (DINOv2 LayerScale)
    // 3x3 / pad 1 / stride 1 convolution over an NHWC tensor as an implicit GEMM (conv = 1): the A tile of output-pixel block
    // (image n, rows 8 ty .., columns 16 tx ..) and k-block (tap, 64-channel block) is ONE 4-D TMA box {64 ch, 16 x, 8 y, 1 n} at
    // (c0, 16 tx + kx - 1, 8 ty + ky - 1, n): out-of-bounds pixels (the padding) are zero-filled by TMA, and the box lands in shared
    // memory as 128 rows x 128 bytes — exactly the K-major SWIZZLE_128B operand tile of the plain GEMM.
    int conv, H, W, tiles_x, tiles_y, cblks;
    // fp32-output instantiation (gemm_wgmma_f32_kernel, the split-bf16 "x3" path of vision.cuh): C32[row, n] = acc + bias_f[n]
    // (+ resid_f[row, n]) stored as fp32 with no rounding; resid_f has row pitch ldr, C32 row pitch ldc.  The fields above that
    // round to bf16 (resid, C, act, bias, scale) are not read there.
    const float* bias_f; const float* resid_f; float* C32;
};
static_assert(WG_TW * WG_TH == WG_BM, "a conv tile's output-pixel block is one 128-row A tile");

__device__ __forceinline__ uint32_t wg_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void wg_mbar_init(uint32_t bar, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void wg_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0, spins = 0;
    while (!ok) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (!ok && ++spins > (1u << 24)) __trap();            // never hang the box
    }
}
__device__ __forceinline__ void wg_mbar_expect(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void wg_mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void wg_tma_2d(uint32_t sdst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(sdst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
__device__ __forceinline__ void wg_tma_4d(uint32_t sdst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(sdst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}
// K-major operand tile [rows][64 bf16] written by TMA with SWIZZLE_128B: 8-row groups are 1024-byte atoms
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// d[64 rows x 128 cols] (+)= A[64 x 16] · B[128 x 16]^T, both operands K-major in shared memory; scale_d = 0 overwrites d
__device__ __forceinline__ void wg_mma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
        "%26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, "
        "%51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
          "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),
          "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
          "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d)
        : "memory");
}

// epilogue of one row and one pair of adjacent columns n, n + 1 (n even, n + 1 < N)
__device__ __forceinline__ void wg_store_pair(const WgP& p, int row, int n, float a0, float a1) {
    float f[2] = {a0, a1};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        if (p.bias) f[j] += tof(p.bias[n + j]);
        f[j] = rnd<bf16>(f[j]);
        if (p.act == 1) f[j] = rnd<bf16>(gelu_tanh_f(f[j]));
        else if (p.act == 2) f[j] = rnd<bf16>(gelu_erf_f(f[j]));
        if (p.scale) f[j] = rnd<bf16>(f[j] * tof(p.scale[n + j]));
    }
    if (p.resid) {
        float x, y;
        unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.resid + (size_t)row * p.ldr + n), x, y);
        f[0] = rnd<bf16>(f[0] + x); f[1] = rnd<bf16>(f[1] + y);
    }
    *reinterpret_cast<__nv_bfloat162*>(p.C + (size_t)row * p.ldc + n) = __floats2bfloat162_rn(f[0], f[1]);
}

// fp32 epilogue of one row and one pair of adjacent columns n, n + 1: the order of nn.Linear / Conv2d (bias) then `+ residual`
__device__ __forceinline__ void wg_store_pair_f32(const WgP& p, int row, int n, float a0, float a1) {
    float2 f = make_float2(a0, a1);
    if (p.bias_f) { f.x += p.bias_f[n]; f.y += p.bias_f[n + 1]; }
    if (p.resid_f) {
        const float2 r = *reinterpret_cast<const float2*>(p.resid_f + (size_t)row * p.ldr + n);
        f.x += r.x; f.y += r.y;
    }
    *reinterpret_cast<float2*>(p.C32 + (size_t)row * p.ldc + n) = f;
}

template <bool F32>
__device__ __forceinline__ void gemm_wgmma_body(const CUtensorMap& mapA, const CUtensorMap& mapB, const WgP& p) {
    extern __shared__ unsigned char wg_raw[];
    __shared__ __align__(8) uint64_t bar_full[WG_STAGES], bar_empty[WG_STAGES];
    const uint32_t smem0 = (wg_smem(wg_raw) + 1023u) & ~1023u;                 // stage s: A at smem0 + s * 32 KB, B 16 KB after
    const int tid = threadIdx.x, wgi = tid >> 7, warp = tid >> 5, lane = tid & 31;
    const int tiles_xy = p.tiles_x * p.tiles_y;                                 // (conv) pixel blocks per image
    const int tiles_m = p.conv ? (p.M / (p.H * p.W)) * tiles_xy : (p.M + WG_BM - 1) / WG_BM, tiles_n = (p.N + WG_BN - 1) / WG_BN;
    const int ntiles = tiles_m * tiles_n;
    const int nkb = (p.K + WG_BK - 1) / WG_BK;

    if (tid == 0) {
        for (int s = 0; s < WG_STAGES; ++s) { wg_mbar_init(wg_smem(&bar_full[s]), 1); wg_mbar_init(wg_smem(&bar_empty[s]), 4 * WG_CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
    }
    __syncthreads();

    // tile t -> (m-tile, n-tile): plain n-major walk keeps the B (weight) tile hot in L2 for the CTAs that run the same n-tile
    // at the same time
    if (wgi == 0) {
        if (tid == 0) {
            // ===== TMA producer =====
            uint32_t it = 0;
            for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
                const int tm = t % tiles_m, tn = t / tiles_m;
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const uint32_t s = it % WG_STAGES, use = it / WG_STAGES;
                    if (use > 0) wg_mbar_wait(wg_smem(&bar_empty[s]), (use - 1) & 1);
                    const uint32_t sA = smem0 + s * WG_STAGE_BYTES, sB = sA + WG_TILE_BYTES, fb = wg_smem(&bar_full[s]);
                    wg_mbar_expect(fb, WG_STAGE_BYTES);
                    if (p.conv) {
                        const int n_img = tm / tiles_xy, r = tm - n_img * tiles_xy, ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                        const int tap = kb / p.cblks, cb = kb - tap * p.cblks, ky = tap / 3, kx = tap - 3 * ky;
                        wg_tma_4d(sA, &mapA, cb * WG_BK, tx * WG_TW + kx - 1, ty * WG_TH + ky - 1, n_img, fb);
                    } else {
                        wg_tma_2d(sA, &mapA, kb * WG_BK, tm * WG_BM, fb);
                    }
                    wg_tma_2d(sB, &mapB, kb * WG_BK, tn * WG_BN, fb);
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wgi owns tile rows [64 (wgi - 1), +64) =====
    const int half = wgi - 1, wq = warp & 3;
    uint32_t it = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int tm = t % tiles_m, tn = t / tiles_m;
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
            const uint32_t s = it % WG_STAGES, use = it / WG_STAGES;
            wg_mbar_wait(wg_smem(&bar_full[s]), use & 1);
            const uint32_t sA = smem0 + s * WG_STAGE_BYTES + half * (64 * WG_BK * 2), sB = smem0 + s * WG_STAGE_BYTES + WG_TILE_BYTES;
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int kk = 0; kk < WG_BK / 16; ++kk)
                wg_mma_m64n128k16(acc, wg_desc_sw128(sA + kk * 32), wg_desc_sw128(sB + kk * 32), (kb > 0 || kk > 0) ? 1u : 0u);
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
            if (kb > 0) {                                   // the previous k-block's group has retired: its stage is free
                __syncwarp();
                if (lane == 0) wg_mbar_arrive(wg_smem(&bar_empty[(it - 1) % WG_STAGES]));
            }
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        __syncwarp();
        if (lane == 0) wg_mbar_arrive(wg_smem(&bar_empty[(it - 1) % WG_STAGES]));

        // accumulator fragment of m64nNk16: acc[4 j + 2 h + c] is row 16 wq + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + c
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int rr = half * 64 + wq * 16 + (lane >> 2) + 8 * h;          // row inside the 128-row tile
            int row = tm * WG_BM + rr;                                          // output row (plain) / NHWC pixel index (conv)
            bool row_ok = row < p.M;
            if (p.conv) {
                const int n_img = tm / tiles_xy, r = tm - n_img * tiles_xy, ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                const int py = ty * WG_TH + (rr >> 4), px = tx * WG_TW + (rr & 15);
                row_ok = py < p.H && px < p.W;
                row = (n_img * p.H + py) * p.W + px;
            }
            if (!row_ok) continue;
#pragma unroll
            for (int j = 0; j < WG_BN / 8; ++j) {
                const int n8 = tn * WG_BN + j * 8;
                if (n8 < p.N) {                                                 // N % 8 == 0 (host-checked): whole 8-column groups
                    if constexpr (F32) wg_store_pair_f32(p, row, n8 + 2 * (lane & 3), acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                    else wg_store_pair(p, row, n8 + 2 * (lane & 3), acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                }
            }
        }
    }
}
__global__ void __launch_bounds__(WG_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                                                                   const WgP p) {
    gemm_wgmma_body<false>(mapA, mapB, p);
}
__global__ void __launch_bounds__(WG_THREADS, 1) gemm_wgmma_f32_kernel(const __grid_constant__ CUtensorMap mapA,
                                                                       const __grid_constant__ CUtensorMap mapB, const WgP p) {
    gemm_wgmma_body<true>(mapA, mapB, p);
}

// ---------------------------------------------------------------------------------------------------------
// Wide decode GEMM (gemm_wide, gemm.h): one decode step's M <= 64 rows times the borrowed [N][K] weights, every weight read once
// per step.  A is one m64 tile (rows M..63 zero-filled by TMA); CTA c = tile · splits + split owns 64 output columns and the
// k-blocks [split · kper, +kper).  The fp32 partials of a column tile go to a workspace; the CTA that takes the last ticket of the
// tile sums them in split order (the same order whichever CTA finishes last, so two runs give identical bits and every row is
// reduced the same way), then runs the decode epilogue of gemm_skinny.cuh (run_epilogue<bf16>) on 16-row slabs.  One split: the
// accumulators go to the epilogue directly.  DUAL (SwiGLU): a second weight map (w3) over the same columns, a second accumulator.
// Roles: warps 0-3 (one warpgroup) issue wgmma.m64n64k16, warp 4 lane 0 is the TMA producer, all 8 warps reduce and store.
// ---------------------------------------------------------------------------------------------------------
constexpr int WD_BN = 64, WD_STAGES = 4, WD_THREADS = 256;
constexpr int WD_A_BYTES = 64 * WG_BK * 2, WD_B_BYTES = WD_BN * WG_BK * 2;
__host__ __device__ constexpr int wd_stage_bytes(bool dual) { return WD_A_BYTES + (dual ? 2 : 1) * WD_B_BYTES; }
__host__ __device__ constexpr int wd_smem(bool dual) { return WD_STAGES * wd_stage_bytes(dual) + 1024; }
static_assert(64 * 2 * WD_BN * 4 <= WD_STAGES * WD_A_BYTES, "the reduced [64][2 x 64] fp32 tile fits in the drained ring");

struct WdP {
    int M, N, K;
    int splits, kper;     // K splits per column tile, k-blocks per split
    float* part;          // [tiles · splits][M][(DUAL ? 2 : 1) · 64] fp32 partials (splits > 1)
    int* tickets;         // [tiles], zero between launches: the last CTA of a tile resets its ticket
    EpiParams ep;
};

// d[64 rows x 64 cols] (+)= A[64 x 16] · B[64 x 16]^T, both operands K-major in shared memory; scale_d = 0 overwrites d
__device__ __forceinline__ void wg_mma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, "
        "%26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
          "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d)
        : "memory");
}

// column c of the tile (w3 columns at 64 + c when DUAL) -> its place in the epilogue tile: run_epilogue's SwiGLU reads 8 w1
// columns then the same 8 w3 columns (the packed interleave of the skinny kernel)
template <bool DUAL>
__device__ __forceinline__ int wd_tile_col(int c) {
    if (!DUAL) return c;
    const int u = c >> 6, cc = c & 63;
    return (cc >> 3) * 16 + u * 8 + (cc & 7);
}

template <bool DUAL>
__global__ void __launch_bounds__(WD_THREADS) gemm_wide_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                                                               const __grid_constant__ CUtensorMap mapB3, const WdP p) {
    constexpr int STAGE = wd_stage_bytes(DUAL), W = (DUAL ? 2 : 1) * WD_BN;     // W: fp32 columns per row of a partial
    extern __shared__ unsigned char wg_raw[];
    __shared__ __align__(8) uint64_t bar_full[WD_STAGES], bar_empty[WD_STAGES];
    __shared__ int s_last;
    const uint32_t smem0 = (wg_smem(wg_raw) + 1023u) & ~1023u;
    float* tileS = reinterpret_cast<float*>(wg_raw + (smem0 - wg_smem(wg_raw)));      // [64][W], over the drained ring
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.x / p.splits, split = blockIdx.x - tile * p.splits;
    const int n0 = tile * WD_BN, kb0 = split * p.kper;
    const int nk = min(p.kper, (p.K + WG_BK - 1) / WG_BK - kb0);

    if (tid == 0) {
        for (int s = 0; s < WD_STAGES; ++s) { wg_mbar_init(wg_smem(&bar_full[s]), 1); wg_mbar_init(wg_smem(&bar_empty[s]), 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
        if (DUAL) asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB3) : "memory");
    }
    __syncthreads();
    pdl_launch_dependents();

    float acc[32], acc3[DUAL ? 32 : 1];
    if (warp == 4) {
        if (lane == 0) {
            // ===== TMA producer: the first stages' weights are immutable and go in flight before the previous kernel has finished
            const int pre = min(nk, WD_STAGES);
            for (int i = 0; i < pre; ++i) {
                const uint32_t sA = smem0 + i * STAGE, fb = wg_smem(&bar_full[i]);
                wg_mbar_expect(fb, STAGE);
                wg_tma_2d(sA + WD_A_BYTES, &mapB, (kb0 + i) * WG_BK, n0, fb);
                if (DUAL) wg_tma_2d(sA + WD_A_BYTES + WD_B_BYTES, &mapB3, (kb0 + i) * WG_BK, n0, fb);
            }
            pdl_wait();
            for (int i = 0; i < pre; ++i) wg_tma_2d(smem0 + i * STAGE, &mapA, (kb0 + i) * WG_BK, 0, wg_smem(&bar_full[i]));
            for (int i = pre; i < nk; ++i) {
                const uint32_t s = i % WD_STAGES, use = i / WD_STAGES;
                wg_mbar_wait(wg_smem(&bar_empty[s]), (use - 1) & 1);
                const uint32_t sA = smem0 + s * STAGE, fb = wg_smem(&bar_full[s]);
                wg_mbar_expect(fb, STAGE);
                wg_tma_2d(sA, &mapA, (kb0 + i) * WG_BK, 0, fb);
                wg_tma_2d(sA + WD_A_BYTES, &mapB, (kb0 + i) * WG_BK, n0, fb);
                if (DUAL) wg_tma_2d(sA + WD_A_BYTES + WD_B_BYTES, &mapB3, (kb0 + i) * WG_BK, n0, fb);
            }
        }
        __syncwarp();
    }
    pdl_wait();
    if (warp < 4) {
        // ===== consumers: the warpgroup owns all 64 rows
        for (int i = 0; i < nk; ++i) {
            const uint32_t s = i % WD_STAGES, use = i / WD_STAGES;
            wg_mbar_wait(wg_smem(&bar_full[s]), use & 1);
            const uint32_t sA = smem0 + s * STAGE, sB = sA + WD_A_BYTES;
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int kk = 0; kk < WG_BK / 16; ++kk) {
                const uint32_t sc = (i > 0 || kk > 0) ? 1u : 0u;
                wg_mma_m64n64k16(acc, wg_desc_sw128(sA + kk * 32), wg_desc_sw128(sB + kk * 32), sc);
                if constexpr (DUAL) wg_mma_m64n64k16(acc3, wg_desc_sw128(sA + kk * 32), wg_desc_sw128(sB + WD_B_BYTES + kk * 32), sc);
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
            if (i > 0) {                                    // the previous k-block's group has retired: its stage is free
                __syncwarp();
                if (lane == 0) wg_mbar_arrive(wg_smem(&bar_empty[(i - 1) % WD_STAGES]));
            }
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    }
    // accumulator fragment of m64nNk16: acc[4 j + 2 h + c] is row 16 warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + c
    auto for_each_pair = [&](auto&& f) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = warp * 16 + (lane >> 2) + 8 * h;
#pragma unroll
            for (int j = 0; j < WD_BN / 8; ++j) {
                const int c = 8 * j + 2 * (lane & 3);
                f(row, c, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                if constexpr (DUAL) f(row, WD_BN + c, acc3[4 * j + 2 * h], acc3[4 * j + 2 * h + 1]);
            }
        }
    };
    if (p.splits == 1) {
        __syncthreads();                                    // every stage consumed: the ring becomes the epilogue tile
        if (warp < 4)
            for_each_pair([&](int row, int c, float a0, float a1) {
                *reinterpret_cast<float2*>(tileS + row * W + wd_tile_col<DUAL>(c)) = make_float2(a0, a1);
            });
    } else {
        float* part = p.part + (size_t)blockIdx.x * p.M * W;
        if (warp < 4)
            for_each_pair([&](int row, int c, float a0, float a1) {
                if (row < p.M) __stcg(reinterpret_cast<float2*>(part + (size_t)row * W + c), make_float2(a0, a1));
            });
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const int old = atomicAdd(p.tickets + tile, 1);
            s_last = old == p.splits - 1;
            if (s_last) p.tickets[tile] = 0;                // every split has arrived: ready for the next launch
        }
        __syncthreads();
        if (!s_last) return;
        __threadfence();
        // the last CTA of the tile: sum the splits in index order, four columns per thread
        const float* base = p.part + (size_t)tile * p.splits * p.M * W;
        for (int idx = tid; idx < p.M * (W / 4); idx += WD_THREADS) {
            const int row = idx / (W / 4), c = (idx - row * (W / 4)) * 4;
            float4 s = __ldcg(reinterpret_cast<const float4*>(base + (size_t)row * W + c));
#pragma unroll 4
            for (int sp = 1; sp < p.splits; ++sp) {
                const float4 v = __ldcg(reinterpret_cast<const float4*>(base + ((size_t)sp * p.M + row) * W + c));
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            }
            *reinterpret_cast<float4*>(tileS + row * W + wd_tile_col<DUAL>(c)) = s;
        }
    }
    __syncthreads();
    const int ncols = min(WD_BN, p.N - n0) * (DUAL ? 2 : 1);
    for (int m0 = 0; m0 < p.M; m0 += 16)
        run_epilogue<bf16>(p.ep, tileS + m0 * W, W, m0, (DUAL ? 2 : 1) * (n0 >> 3), ncols, tid, WD_THREADS);
}
