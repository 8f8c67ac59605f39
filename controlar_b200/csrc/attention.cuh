// attention.cuh — KV-cache attention of the LlamaGen block.
//   attn_decode : one query row per (sequence, head) against the cache [0, pos]  — the HBM-bound part of a
//                 decode step.  Replaces F.scaled_dot_product_attention with the math backend forced
//                 (autoregressive/models/generate.py:120, gpt_t2i.py:282-286) and the bool mask
//                 causal_mask[:, None, input_pos] edited by generate.py:184-193.
//   attn_prefill: the T prefix rows (causal + emb_mask columns + forced diagonal), gpt_t2i.py:448,282-286.
// Cache layout is the reference's KVCache: [B_eff, H, S, 64] (gpt_t2i.py:220-235).
// The reference soft-maxes over all S slots with -inf on masked ones; skipping masked slots is identical.
#pragma once
#include "common.cuh"

constexpr int AD_WARPS = 4;
constexpr int AD_THREADS = AD_WARPS * 32;
constexpr int AD_PART = 68;   // m, l, pad, pad, acc[64]

template <typename T> struct RowLanes;                 // lanes that share one 64-element row with 16-byte loads
template <> struct RowLanes<bf16> { static constexpr int LPR = 8, EPL = 8; };
template <> struct RowLanes<float> { static constexpr int LPR = 16, EPL = 4; };

template <typename T> __device__ __forceinline__ void load_row_frag(const T* p, float (&f)[RowLanes<T>::EPL]);
template <> __device__ __forceinline__ void load_row_frag<bf16>(const bf16* p, float (&f)[8]) {
    const uint4 v = ldg_cg128(p);
    unpack_bf16x2(v.x, f[0], f[1]); unpack_bf16x2(v.y, f[2], f[3]);
    unpack_bf16x2(v.z, f[4], f[5]); unpack_bf16x2(v.w, f[6], f[7]);
}
template <> __device__ __forceinline__ void load_row_frag<float>(const float* p, float (&f)[4]) {
    const uint4 v = ldg_cg128(p);
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y); f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
}

// grid = (B_eff*H, nsplit), block = 128.  Split s handles keys [s*chunk, min(n,(s+1)*chunk)), n = pos+1.
// The last CTA to finish a (b,h) combines the nsplit partials in index order (deterministic) and writes
// out[b][h*64 + e] rounded to T (the SDPA output cast).
template <typename T>
__global__ void __launch_bounds__(AD_THREADS, 6)
attn_decode_kernel(const T* __restrict__ q, const T* __restrict__ kc, const T* __restrict__ vc,
                   const int* __restrict__ emb_mask, int mask_ld, const int* __restrict__ pos_ptr, int H, int S,
                   int Tpre, int nsplit, float* __restrict__ part, int* __restrict__ tickets, T* __restrict__ out) {
    constexpr int LPR = RowLanes<T>::LPR, EPL = RowLanes<T>::EPL, RPW = 32 / LPR;
    constexpr int UNR = 4;
    __shared__ float sm_m[AD_WARPS * RPW], sm_l[AD_WARPS * RPW];
    __shared__ float sm_acc[AD_WARPS * RPW][64];
    __shared__ int sm_last;

    const int bh = blockIdx.x, b = bh / H, hd = bh - b * H;
    const int split = blockIdx.y;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int sub = lane / LPR, cl = lane % LPR;          // row slot within the warp, column chunk
    // `pos` is only ever advanced by the sampler, which never triggers its dependents early, so it is stable for
    // every kernel of the step — including before pdl_wait().
    pdl_launch_dependents();
    const int pos = ld_cg(pos_ptr), n = pos + 1;
    int chunk = (n + nsplit - 1) / nsplit;
    chunk = (chunk + 7) & ~7;
    const int k0 = split * chunk, k1 = min(n, k0 + chunk);
    // pull this CTA's slice of the cache towards L2 while the QKV GEMM is still running (rows < pos are final)
    {
        const char* kb = reinterpret_cast<const char*>(kc + ((size_t)bh * S + k0) * 64);
        const char* vb = reinterpret_cast<const char*>(vc + ((size_t)bh * S + k0) * 64);
        const int lines = max(0, min(k1, pos) - k0) * 64 * (int)sizeof(T) / 128;
        for (int i = tid; i < lines; i += AD_THREADS) { prefetch_l2(kb + (size_t)i * 128); prefetch_l2(vb + (size_t)i * 128); }
    }
    pdl_wait();

    float qf[EPL];
    {
        const T* qp = q + (size_t)b * H * 64 + hd * 64 + cl * EPL;
#pragma unroll
        for (int e = 0; e < EPL; ++e) qf[e] = ld_cg(qp + e);
    }
    const T* kbase = kc + ((size_t)bh * S) * 64 + cl * EPL;
    const T* vbase = vc + ((size_t)bh * S) * 64 + cl * EPL;
    const int* mrow = emb_mask ? emb_mask + (size_t)b * mask_ld : nullptr;

    float m_run = -INFINITY, l_run = 0.f, acc[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) acc[e] = 0.f;

    const int stride = AD_WARPS * RPW;                    // rows per CTA sweep
    for (int rb = k0 + warp * RPW; rb < k1; rb += stride * UNR) {      // warp-uniform trip count (full-mask shuffles)
        const int r0 = rb + sub;
        float kf[UNR][EPL], vf[UNR][EPL];
        bool ok[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            const int r = r0 + u * stride;
            ok[u] = r < k1 && (r >= Tpre || mrow == nullptr || mrow[r] != 0);
            if (ok[u]) { load_row_frag<T>(kbase + (size_t)r * 64, kf[u]); load_row_frag<T>(vbase + (size_t)r * 64, vf[u]); }
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
            float s = 0.f;
            if (ok[u]) {
#pragma unroll
                for (int e = 0; e < EPL; ++e) s = fmaf(qf[e], kf[u][e], s);
            }
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (ok[u]) {
                s *= 0.125f;                              // 1/sqrt(head_dim=64)
                const float m_new = fmaxf(m_run, s);
                const float corr = __expf(m_run - m_new);  // exp(-inf) = 0 on the first row
                const float p = __expf(s - m_new);
                l_run = l_run * corr + p;
#pragma unroll
                for (int e = 0; e < EPL; ++e) acc[e] = fmaf(p, vf[u][e], acc[e] * corr);
                m_run = m_new;
            }
        }
    }
    // ---- merge the AD_WARPS*RPW row slots of this CTA
    const int slot = warp * RPW + sub;
    if (cl == 0) { sm_m[slot] = m_run; sm_l[slot] = l_run; }
#pragma unroll
    for (int e = 0; e < EPL; ++e) sm_acc[slot][cl * EPL + e] = acc[e];
    __syncthreads();
    float* my_part = part + ((size_t)bh * nsplit + split) * AD_PART;
    if (tid < 64) {
        float M = -INFINITY;
        for (int s = 0; s < AD_WARPS * RPW; ++s) M = fmaxf(M, sm_m[s]);
        float L = 0.f, a = 0.f;
        for (int s = 0; s < AD_WARPS * RPW; ++s) {
            const float w = (sm_m[s] == -INFINITY) ? 0.f : __expf(sm_m[s] - M);
            L += sm_l[s] * w;
            a += sm_acc[s][tid] * w;
        }
        if (tid == 0) { my_part[0] = M; my_part[1] = L; }
        my_part[4 + tid] = a;
    }
    // ---- last-arriving split combines
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const int old = atomicAdd(&tickets[bh], 1);
        sm_last = (old == nsplit - 1);
    }
    __syncthreads();
    if (!sm_last) return;
    __threadfence();
    if (tid < 64) {
        const float* pp = part + (size_t)bh * nsplit * AD_PART;
        float M = -INFINITY;
        for (int s = 0; s < nsplit; ++s) M = fmaxf(M, __ldcg(pp + s * AD_PART));
        float L = 0.f, a = 0.f;
        for (int s = 0; s < nsplit; ++s) {
            const float ms = __ldcg(pp + s * AD_PART);
            const float w = (ms == -INFINITY) ? 0.f : __expf(ms - M);
            L += __ldcg(pp + s * AD_PART + 1) * w;
            a += __ldcg(pp + s * AD_PART + 4 + tid) * w;
        }
        out[(size_t)b * H * 64 + hd * 64 + tid] = fromf<T>(a / L);
    }
    if (tid == 0) tickets[bh] = 0;
}

// ---------------------------------------------------------------------------------------------------------
// prefill attention: one warp per (b, h, query row i); keys [0, i] from the cache; Tq <= 256.
// mask(i, s) = s <= i and (s >= Tpre or emb_mask[b][s]) or s == i   (generate.py:184-193)
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128)
attn_prefill_kernel(const T* __restrict__ q /*[B*Tq][H*64]*/, const T* __restrict__ kc, const T* __restrict__ vc,
                    const int* __restrict__ emb_mask, int mask_ld, int B, int H, int S, int Tq, int Tpre,
                    T* __restrict__ out /*[B*Tq][H*64]*/) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * 4 + warp;
    if (item >= (long long)B * H * Tq) return;
    const int i = (int)(item % Tq);
    const int hd = (int)((item / Tq) % H);
    const int b = (int)(item / ((long long)Tq * H));
    const T* qp = q + ((size_t)b * Tq + i) * H * 64 + hd * 64;
    const T* kb = kc + (((size_t)b * H + hd) * S) * 64;
    const T* vb = vc + (((size_t)b * H + hd) * S) * 64;
    const int* mrow = emb_mask ? emb_mask + (size_t)b * mask_ld : nullptr;
    float sc[8];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int s = lane + 32 * j;
        sc[j] = -INFINITY;
        if (s <= i && (s == i || s >= Tpre || mrow == nullptr || mrow[s] != 0)) {
            float d = 0.f;
            for (int e = 0; e < 64; ++e) d = fmaf(tof(qp[e]), tof(kb[(size_t)s * 64 + e]), d);
            sc[j] = d * 0.125f;
            mx = fmaxf(mx, sc[j]);
        }
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sc[j] = (sc[j] == -INFINITY) ? 0.f : expf(sc[j] - mx);
        sum += sc[j];
    }
    sum = warp_sum(sum);
    float o0 = 0.f, o1 = 0.f;
    for (int s = 0; s <= i; ++s) {
        const float p = __shfl_sync(0xffffffffu, sc[s >> 5], s & 31);
        if (p != 0.f) {
            o0 = fmaf(p, tof(vb[(size_t)s * 64 + 2 * lane]), o0);
            o1 = fmaf(p, tof(vb[(size_t)s * 64 + 2 * lane + 1]), o1);
        }
    }
    T* op = out + ((size_t)b * Tq + i) * H * 64 + hd * 64 + 2 * lane;
    op[0] = fromf<T>(o0 / sum);
    op[1] = fromf<T>(o1 / sum);
}

// ---------------------------------------------------------------------------------------------------------
// prefill attention on the tensor cores (bf16 checkpoints): same mask as above, one CTA = 64 query rows of one (b, h), 4 warps x 16
// rows; key tiles of 64 from the cache through shared memory; S = q k^T / 8 in fp32 (mma.sync m16n8k16), online soft-max in fp32,
// probabilities rounded to bf16 (the reference's SDPA math path casts the soft-max to the model dtype before the value product),
// fp32 accumulate, bf16 out.  The scalar kernel above spent 0.2 ms per layer on 2-byte loads (7.4 ms of a 32 ms prefill).
// ---------------------------------------------------------------------------------------------------------
constexpr int PFA_PITCH = 72;
__global__ void __launch_bounds__(128)
attn_prefill_mma_kernel(const bf16* __restrict__ q /*[B*Tq][H*64]*/, const bf16* __restrict__ kc, const bf16* __restrict__ vc,
                        const int* __restrict__ emb_mask, int mask_ld, int H, int S, int Tq, int Tpre, bf16* __restrict__ out) {
    __shared__ __align__(16) bf16 sK[64 * PFA_PITCH];          // [key][dim]
    __shared__ __align__(16) bf16 sV[64 * PFA_PITCH];          // [dim][key]
    __shared__ int s_m[64];                                     // emb_mask of the tile's keys (1 = attend)
    const int b = blockIdx.z, hd = blockIdx.y, q0 = blockIdx.x * 64;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const size_t ldq = (size_t)H * 64;
    const int i_lo = q0 + warp * 16 + g, i_hi = i_lo + 8;       // this thread's two query rows
    const bf16* qlo = q + ((size_t)b * Tq + min(i_lo, Tq - 1)) * ldq + hd * 64;
    const bf16* qhi = q + ((size_t)b * Tq + min(i_hi, Tq - 1)) * ldq + hd * 64;
    uint32_t qa[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        qa[ks][0] = *reinterpret_cast<const uint32_t*>(qlo + ks * 16 + 2 * t);
        qa[ks][1] = *reinterpret_cast<const uint32_t*>(qhi + ks * 16 + 2 * t);
        qa[ks][2] = *reinterpret_cast<const uint32_t*>(qlo + ks * 16 + 8 + 2 * t);
        qa[ks][3] = *reinterpret_cast<const uint32_t*>(qhi + ks * 16 + 8 + 2 * t);
    }
    float o[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
    float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
    const bf16* kb = kc + (((size_t)b * H + hd) * S) * 64;
    const bf16* vb = vc + (((size_t)b * H + hd) * S) * 64;
    const int k_end = min(q0 + 64, Tq);                         // causal: keys beyond the tile's last query are never needed
    for (int k0 = 0; k0 < k_end; k0 += 64) {
        __syncthreads();
        for (int i = tid; i < 64 * 8; i += 128) {
            const int r = i >> 3, c = i & 7;
            const int key = min(k0 + r, Tq - 1);
            *reinterpret_cast<uint4*>(sK + r * PFA_PITCH + c * 8) = *reinterpret_cast<const uint4*>(kb + (size_t)key * 64 + c * 8);
            const uint4 vv = *reinterpret_cast<const uint4*>(vb + (size_t)key * 64 + c * 8);
            const bf16* ve = reinterpret_cast<const bf16*>(&vv);
#pragma unroll
            for (int e = 0; e < 8; ++e) sV[(c * 8 + e) * PFA_PITCH + r] = ve[e];      // transposed: [dim][key]
        }
        if (tid < 64) { const int s = k0 + tid; s_m[tid] = (s >= Tpre || emb_mask == nullptr || s >= mask_ld) ? 1 : (emb_mask[(size_t)b * mask_ld + s] != 0); }
        __syncthreads();
        float sacc[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sK + (j * 8 + g) * PFA_PITCH + ks * 16 + 2 * t);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sK + (j * 8 + g) * PFA_PITCH + ks * 16 + 8 + 2 * t);
                mma_bf16_16816(sacc[j], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3], b0, b1);
            }
        }
        float mx_lo = m_lo, mx_hi = m_hi;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int kl = j * 8 + 2 * t + (e & 1), s = k0 + kl;
                const int i = e < 2 ? i_lo : i_hi;
                const bool ok = s <= i && s < Tq && (s == i || s_m[kl] != 0);     // generate.py:184-193: causal, gated text columns, forced diagonal
                const float v = ok ? sacc[j][e] * 0.125f : -INFINITY;
                sacc[j][e] = v;
                if (e < 2) mx_lo = fmaxf(mx_lo, v); else mx_hi = fmaxf(mx_hi, v);
            }
        }
        mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1)); mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
        mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1)); mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
        // (a row whose keys are all masked so far keeps m = -inf: exp(-inf - (-inf)) must not produce NaN)
        const float c_lo = m_lo == -INFINITY ? 0.f : __expf(m_lo - mx_lo), c_hi = m_hi == -INFINITY ? 0.f : __expf(m_hi - mx_hi);
        m_lo = mx_lo; m_hi = mx_hi;
        l_lo *= c_lo; l_hi *= c_hi;
#pragma unroll
        for (int j = 0; j < 8; ++j) { o[j][0] *= c_lo; o[j][1] *= c_lo; o[j][2] *= c_hi; o[j][3] *= c_hi; }
        uint32_t pa[4][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float p0 = sacc[j][0] == -INFINITY ? 0.f : rnd<bf16>(__expf(sacc[j][0] - m_lo)), p1 = sacc[j][1] == -INFINITY ? 0.f : rnd<bf16>(__expf(sacc[j][1] - m_lo));
            const float p2 = sacc[j][2] == -INFINITY ? 0.f : rnd<bf16>(__expf(sacc[j][2] - m_hi)), p3 = sacc[j][3] == -INFINITY ? 0.f : rnd<bf16>(__expf(sacc[j][3] - m_hi));
            l_lo += p0 + p1; l_hi += p2 + p3;
            __nv_bfloat162 lo2 = __floats2bfloat162_rn(p0, p1), hi2 = __floats2bfloat162_rn(p2, p3);
            pa[j >> 1][(j & 1) * 2 + 0] = *reinterpret_cast<uint32_t*>(&lo2);
            pa[j >> 1][(j & 1) * 2 + 1] = *reinterpret_cast<uint32_t*>(&hi2);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sV + (j * 8 + g) * PFA_PITCH + ks * 16 + 2 * t);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sV + (j * 8 + g) * PFA_PITCH + ks * 16 + 8 + 2 * t);
                mma_bf16_16816(o[j], pa[ks][0], pa[ks][1], pa[ks][2], pa[ks][3], b0, b1);
            }
        }
    }
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1); l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1); l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (i_lo < Tq) {
            __nv_bfloat162 v = __floats2bfloat162_rn(o[j][0] / l_lo, o[j][1] / l_lo);
            *reinterpret_cast<__nv_bfloat162*>(out + ((size_t)b * Tq + i_lo) * ldq + hd * 64 + j * 8 + 2 * t) = v;
        }
        if (i_hi < Tq) {
            __nv_bfloat162 v = __floats2bfloat162_rn(o[j][2] / l_hi, o[j][3] / l_hi);
            *reinterpret_cast<__nv_bfloat162*>(out + ((size_t)b * Tq + i_hi) * ldq + hd * 64 + j * 8 + 2 * t) = v;
        }
    }
}
