// gemm_skinny.cuh — weight-streaming GEMMs for M <= 16 rows per tile (the decode-step shape, B_eff rows), with
// the fused prologues/epilogues of the LlamaGen block.  Replaces, per decode step (reference file:line):
//   RMSNorm            autoregressive/models/gpt_t2i.py:193-198   (prologue, NORM=true)
//   wqkv + RoPE + KV   gpt_t2i.py:264,270-271,227-235,522-532     (EPI_QKV)
//   wo / w2 + residual gpt_t2i.py:290,305-306 (+ control add :466) (EPI_RESID)
//   w1,w3 + SwiGLU     gpt_t2i.py:216-217                          (EPI_SWIGLU)
//   output head        gpt_t2i.py:469-470                          (EPI_LOGITS)
//   MLP fc1/fc2        gpt_t2i.py:165-181                          (EPI_STORE, act)
//
// bf16 path: HBM-bound.  Weights are pre-packed (pack.cuh) so that one warp-wide LDG.128 fetches, for one
// 8-column block, a contiguous 512 B chunk that is *already* the B fragment of two mma.m16n8k16 — no shared
// memory round trip for weights; the 16-row activation tile is staged once per CTA in shared memory (with the
// RMSNorm applied on the way in) and read back with conflict-free LDS.128.  K is split across the 8 warps of
// the CTA and reduced in a fixed order (deterministic).
#pragma once
#include "common.cuh"

enum { EPI_STORE = 0, EPI_QKV = 1, EPI_RESID = 2, EPI_SWIGLU = 3, EPI_LOGITS = 4 };

struct EpiParams {
    int kind;
    int M;                // valid rows
    int rpb;              // rows per batch element: T in prefill, 1 in decode
    const int* pos_ptr;   // decode: device scalar with the sequence position; null => pos = row % rpb
    int pos_fixed_p1;     // persistent decode kernel: position + 1 passed by value (0 = unused)
    // EPI_STORE
    void* out; int ldo; int act; const void* bias;
    int out_reps; long long out_rep_stride;   // EPI_SWIGLU: extra replicas of the output (persistent kernel)
    // EPI_RESID (+ optional control add for the *next* layer group)
    void* h; int ldh;
    const void* ctrl; int n_img; int T; const float* cs;   // cs: control strength per batch element
    // EPI_QKV
    const float* rope; void* kc; void* vc; void* q; int S; int H; int d;
    // EPI_LOGITS
    float* logits; long long ldl;
};

// tile: [16][ldt] fp32 accumulators for columns [nb0*8, nb0*8 + ncols) of rows [m0, m0+16)
template <typename T>
__device__ __forceinline__ void run_epilogue(const EpiParams& ep, const float* tile, int ldt, int m0, int nb0,
                                             int ncols, int tid, int nthreads) {
    const int half = ncols >> 1;
    for (int idx = tid; idx < 16 * half; idx += nthreads) {
        const int m = idx / half, cp = idx - m * half;
        const int r = m0 + m;
        if (r >= ep.M) continue;
        if (ep.kind == EPI_SWIGLU) {
            // packed rows alternate 8 rows of w1 / 8 rows of w3 (pack.cuh: pack_w13)
            const int jj = cp >> 3, ci = cp & 7;
            const float g = rnd<T>(tile[m * ldt + jj * 16 + ci]);
            const float u = rnd<T>(tile[m * ldt + jj * 16 + 8 + ci]);
            const float s = rnd<T>(silu_f(g));
            const int col = ((nb0 >> 1) + jj) * 8 + ci;
            const T ov = fromf<T>(s * u);
            ((T*)ep.out)[(size_t)r * ep.ldo + col] = ov;
            for (int rep = 1; rep < ep.out_reps; ++rep) ((T*)ep.out)[(size_t)rep * ep.out_rep_stride + (size_t)r * ep.ldo + col] = ov;
            continue;
        }
        const int c = cp * 2;
        const int n = nb0 * 8 + c;
        float v0 = tile[m * ldt + c], v1 = tile[m * ldt + c + 1];
        const int b = r / ep.rpb;
        const int pos = ep.pos_fixed_p1 ? ep.pos_fixed_p1 - 1 : (ep.pos_ptr ? ld_cg(ep.pos_ptr) : (r - b * ep.rpb));
        switch (ep.kind) {
            case EPI_STORE: {
                if (ep.bias) { v0 += tof(((const T*)ep.bias)[n]); v1 += tof(((const T*)ep.bias)[n + 1]); }
                v0 = rnd<T>(v0); v1 = rnd<T>(v1);
                if (ep.act == 1) { v0 = gelu_tanh_f(v0); v1 = gelu_tanh_f(v1); }
                else if (ep.act == 2) { v0 = gelu_erf_f(v0); v1 = gelu_erf_f(v1); }
                T* o = (T*)ep.out + (size_t)r * ep.ldo + n;
                o[0] = fromf<T>(v0); o[1] = fromf<T>(v1);
            } break;
            case EPI_RESID: {
                T* hp = (T*)ep.h + (size_t)r * ep.ldh + n;
                float o0 = rnd<T>(ld_cg(hp) + rnd<T>(v0));
                float o1 = rnd<T>(ld_cg(hp + 1) + rnd<T>(v1));
                if (ep.ctrl) {   // gpt_t2i.py:466 — h += cs * ctrl[:, pos - T + 1] ahead of the next layer group
                    const int p = pos - ep.T + 1;
                    if (p >= 0 && p < ep.n_img) {
                        const T* cp_ = (const T*)ep.ctrl + ((size_t)b * ep.n_img + p) * ep.ldh + n;
                        const float s = __ldg(ep.cs + b);
                        o0 = rnd<T>(o0 + rnd<T>(s * tof(cp_[0])));
                        o1 = rnd<T>(o1 + rnd<T>(s * tof(cp_[1])));
                    }
                }
                hp[0] = fromf<T>(o0); hp[1] = fromf<T>(o1);
            } break;
            case EPI_QKV: {
                v0 = rnd<T>(v0); v1 = rnd<T>(v1);
                const int sec = n / ep.d, w = n - sec * ep.d;
                const int head = w >> 6, e = w & 63;
                if (sec < 2) {   // apply_rotary_emb gpt_t2i.py:522-532 (interleaved pairs, fp32, then cast)
                    const float2 cs2 = *(const float2*)(ep.rope + ((size_t)pos * 32 + (e >> 1)) * 2);
                    const float x0 = v0 * cs2.x - v1 * cs2.y;
                    const float x1 = v1 * cs2.x + v0 * cs2.y;
                    v0 = x0; v1 = x1;
                }
                T* dst;
                if (sec == 0) dst = (T*)ep.q + (size_t)r * ep.d + w;
                else {
                    T* base = (T*)(sec == 1 ? ep.kc : ep.vc);
                    dst = base + (((size_t)b * ep.H + head) * ep.S + pos) * 64 + e;   // KVCache.update :227-235
                }
                dst[0] = fromf<T>(v0); dst[1] = fromf<T>(v1);
            } break;
            case EPI_LOGITS: {
                float* o = ep.logits + (size_t)r * ep.ldl + n;
                o[0] = rnd<T>(v0); o[1] = rnd<T>(v1);   // .float() of the model-dtype head output, :470
            } break;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// bf16 tensor-core path
// ---------------------------------------------------------------------------------------------------------
constexpr int SK_WARPS = 8;
constexpr int SK_THREADS = SK_WARPS * 32;

static inline size_t skinny_smem_bytes(int K, int NB) {
    return (size_t)16 * (K + 32) * 2 + (size_t)SK_WARPS * NB * 128 * 4 + (size_t)16 * NB * 8 * 4;
}

// grid = (ceil(nblk/NB), ceil(M/16)); Wp: packed weights, chunk (nb, s) at ((nb*(K/32)+s)*32 + lane) uint4
template <int NB, int U, bool NORM>
__global__ void __launch_bounds__(SK_THREADS)
skinny_gemm_bf16(const bf16* __restrict__ A, int lda, const uint4* __restrict__ Wp, const bf16* __restrict__ nw,
                 float eps, int K, int nblk, EpiParams ep) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int KS = K + 32;                                  // bf16 elements per smem row (+64 B: conflict-free)
    bf16* As = reinterpret_cast<bf16*>(smem_raw);
    float* red = reinterpret_cast<float*>(smem_raw + (size_t)16 * KS * 2);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int m0 = blockIdx.y * 16;
    const int mrows = min(16, ep.M - m0);
    int nb0 = blockIdx.x * NB;
    const int ksteps = K >> 5;
    const int nsteps = (ksteps - warp + SK_WARPS - 1) / SK_WARPS;   // k32-steps owned by this warp: warp, warp+8, ..

    // ---- 1. first batch of weight fragments in flight before anything that depends on the previous kernel
    uint4 wf[U][NB];
    auto load_batch = [&](int i0) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int s = warp + (i0 + u) * SK_WARPS;
#pragma unroll
            for (int j = 0; j < NB; ++j) {
                if (i0 + u < nsteps && nb0 + j < nblk)
                    wf[u][j] = ldg_stream(Wp + ((size_t)(nb0 + j) * ksteps + s) * 32 + lane);
                else
                    wf[u][j] = make_uint4(0, 0, 0, 0);
            }
        }
    };
    pdl_launch_dependents();
    load_batch(0);
    // the rest of this warp's weight stream goes to L2 now, so the post-dependency loop never waits on HBM (fire-and-forget
    // prefetches: unrolling the loop only adds code in front of pdl_wait())
#pragma unroll 1
    for (int i = U; i < nsteps; ++i) {
        const int s = warp + i * SK_WARPS;
#pragma unroll
        for (int j = 0; j < NB; ++j)
            if (nb0 + j < nblk && (lane & 7) == 0)
                prefetch_l2(Wp + ((size_t)(nb0 + j) * ksteps + s) * 32 + lane);
    }
    pdl_wait();   // ---- everything below may read what the previous kernel wrote

    // ---- 2. stage the 16-row activation tile (RMSNorm fused when NORM): one pass over global memory
    const int chunks = K >> 3;   // 16-byte chunks per row
    if (NORM) {
        constexpr int MAXC = 8;                       // register-held chunks per lane (K <= 2048)
        for (int rr = warp; rr < 16; rr += SK_WARPS) {
            bf16* dst = As + (size_t)rr * KS;
            if (rr >= mrows) {
                for (int c = lane; c < chunks; c += 32) *reinterpret_cast<uint4*>(dst + c * 8) = make_uint4(0, 0, 0, 0);
                continue;
            }
            const bf16* src = A + (size_t)(m0 + rr) * lda;
            uint4 held[MAXC];
            float ss = 0.f;
            auto sq = [&](const uint4& v) {
                float a, b;
                unpack_bf16x2(v.x, a, b); ss += a * a + b * b;
                unpack_bf16x2(v.y, a, b); ss += a * a + b * b;
                unpack_bf16x2(v.z, a, b); ss += a * a + b * b;
                unpack_bf16x2(v.w, a, b); ss += a * a + b * b;
            };
#pragma unroll
            for (int ci = 0; ci < MAXC; ++ci) {
                const int c = lane + 32 * ci;
                held[ci] = c < chunks ? ldg_cg128(src + c * 8) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int ci = 0; ci < MAXC; ++ci) sq(held[ci]);
            for (int c = lane + 32 * MAXC; c < chunks; c += 32) sq(ldg_cg128(src + c * 8));   // K > 2048 tail
            ss = warp_sum(ss);
            const float rstd = rsqrtf(ss / (float)K + eps);
            auto norm_store = [&](const uint4& v, int c) {
                const uint4 wv = *reinterpret_cast<const uint4*>(nw + c * 8);
                const uint32_t xi[4] = {v.x, v.y, v.z, v.w};
                const uint32_t wi[4] = {wv.x, wv.y, wv.z, wv.w};
                uint32_t o[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float a, b, wa, wb;
                    unpack_bf16x2(xi[q], a, b);
                    unpack_bf16x2(wi[q], wa, wb);
                    // RMSNorm.forward: _norm(x.float()).type_as(x) * weight  (two roundings)
                    const float na = rnd<bf16>(a * rstd) * wa;
                    const float nb_ = rnd<bf16>(b * rstd) * wb;
                    __nv_bfloat162 pk = __floats2bfloat162_rn(na, nb_);
                    o[q] = *reinterpret_cast<uint32_t*>(&pk);
                }
                *reinterpret_cast<uint4*>(dst + c * 8) = make_uint4(o[0], o[1], o[2], o[3]);
            };
#pragma unroll
            for (int ci = 0; ci < MAXC; ++ci) {
                const int c = lane + 32 * ci;
                if (c < chunks) norm_store(held[ci], c);
            }
            for (int c = lane + 32 * MAXC; c < chunks; c += 32) norm_store(ldg_cg128(src + c * 8), c);
        }
    } else {
        for (int idx = tid; idx < 16 * chunks; idx += SK_THREADS) {
            const int rr = idx / chunks, c = idx - rr * chunks;
            bf16* dst = As + (size_t)rr * KS + c * 8;
            if (rr < mrows) cp_async16(dst, A + (size_t)(m0 + rr) * lda + c * 8);
            else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
        }
        cp_async_wait_all();
    }
    __syncthreads();

    // ---- 3. main loop: this warp's k-steps, all NB column blocks; the CTA then strides to its next column group
    // (grid.x is capped at one wave, the staged activation tile is reused)
    float* tile = reinterpret_cast<float*>(smem_raw + (size_t)16 * KS * 2 + (size_t)SK_WARPS * NB * 128 * 4);   // [16][NB*8]
  for (bool first = true; nb0 < nblk; nb0 += gridDim.x * NB, first = false) {
    if (!first) load_batch(0);
    float acc[NB][4];
#pragma unroll
    for (int j = 0; j < NB; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
    const bf16* a_lo_base = As + (size_t)g * KS + t * 8;
    const bf16* a_hi_base = As + (size_t)(g + 8) * KS + t * 8;
    for (int i0 = 0; i0 < nsteps; i0 += U) {
        if (i0 > 0) load_batch(i0);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (i0 + u < nsteps) {
                const int s = warp + (i0 + u) * SK_WARPS;
                const uint4 lo = *reinterpret_cast<const uint4*>(a_lo_base + s * 32);
                const uint4 hi = *reinterpret_cast<const uint4*>(a_hi_base + s * 32);
#pragma unroll
                for (int j = 0; j < NB; ++j) {
                    mma_bf16_16816(acc[j], lo.x, hi.x, lo.y, hi.y, wf[u][j].x, wf[u][j].y);
                    mma_bf16_16816(acc[j], lo.z, hi.z, lo.w, hi.w, wf[u][j].z, wf[u][j].w);
                }
            }
        }
    }

    // ---- 4. cross-warp K reduction in fixed order, then the fused epilogue
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        float* rp = red + ((size_t)warp * NB + j) * 128;
        rp[g * 8 + 2 * t] = acc[j][0];
        rp[g * 8 + 2 * t + 1] = acc[j][1];
        rp[(g + 8) * 8 + 2 * t] = acc[j][2];
        rp[(g + 8) * 8 + 2 * t + 1] = acc[j][3];
    }
    __syncthreads();
    for (int idx = tid; idx < NB * 128; idx += SK_THREADS) {
        const int j = idx >> 7, e = idx & 127;
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < SK_WARPS; ++w) s += red[((size_t)w * NB + j) * 128 + e];
        tile[(e >> 3) * (NB * 8) + j * 8 + (e & 7)] = s;
    }
    __syncthreads();
    const int ncols = min(NB, nblk - nb0) * 8;
    run_epilogue<bf16>(ep, tile, NB * 8, m0, nb0, ncols, tid, SK_THREADS);
  }
}

// ---------------------------------------------------------------------------------------------------------
// fp32 reference-precision path (CUDA-core FMA; used for fp32 checkpoints, where greedy parity is bit-exact)
// W plain [N][K] fp32; one CTA = 16 columns (two 8-blocks), warp w owns columns w and w+8.
// ---------------------------------------------------------------------------------------------------------
template <bool NORM>
__global__ void __launch_bounds__(SK_THREADS)
skinny_gemm_f32(const float* __restrict__ A, int lda, const float* __restrict__ W, const float* __restrict__ nw,
                float eps, int K, int nblk, EpiParams ep) {
    __shared__ float rstd_s[16];
    __shared__ float tile[16 * 16];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * 16;
    const int mrows = min(16, ep.M - m0);
    const int nb0 = blockIdx.x * 2;
    if (NORM) {
        for (int rr = warp; rr < 16; rr += SK_WARPS) {
            float ss = 0.f;
            if (rr < mrows)
                for (int k = lane; k < K; k += 32) { const float a = A[(size_t)(m0 + rr) * lda + k]; ss += a * a; }
            ss = warp_sum(ss);
            if (lane == 0) rstd_s[rr] = rsqrtf(ss / (float)K + eps);
        }
        __syncthreads();
    }
#pragma unroll 1
    for (int cc = 0; cc < 2; ++cc) {
        const int col = cc * 8 + warp;              // local column 0..15
        const int n = nb0 * 8 + col;
        float acc[16];
#pragma unroll
        for (int m = 0; m < 16; ++m) acc[m] = 0.f;
        if (nb0 + cc < nblk) {
            const float* wrow = W + (size_t)n * K;
            for (int k = lane; k < K; k += 32) {
                const float wv = wrow[k];
                const float nv = NORM ? nw[k] : 1.f;
#pragma unroll
                for (int m = 0; m < 16; ++m) {
                    if (m < mrows) {
                        float a = A[(size_t)(m0 + m) * lda + k];
                        if (NORM) a = (a * rstd_s[m]) * nv;
                        acc[m] = fmaf(a, wv, acc[m]);
                    }
                }
            }
        }
#pragma unroll
        for (int m = 0; m < 16; ++m) {
            const float s = warp_sum(acc[m]);
            if (lane == 0) tile[m * 16 + col] = s;
        }
    }
    __syncthreads();
    const int ncols = min(2, nblk - nb0) * 8;
    run_epilogue<float>(ep, tile, 16, m0, nb0, ncols, tid, SK_THREADS);
}
