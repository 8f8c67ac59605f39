// sampler.cuh — CFG combine + temperature + top-k/top-p + soft-max + multinomial/arg-max in ONE kernel,
// plus the embedding gather (+ layer-0 control add) of the *next* decode step.
// Replaces (reference file:line):
//   CFG combine                 autoregressive/models/generate.py:89-90,103-107
//   sample()                    generate.py:59-74
//   top_k_top_p_filtering()     generate.py:17-56
//   tok_embeddings(idx)         gpt_t2i.py:445     } fused tail: h for the next position
//   h += cs*ctrl[0][:, p+1]     gpt_t2i.py:466     }
// torch.multinomial(p, 1) == argmax(p / q), q ~ Exp(1) (SURVEY.md §7 hard-part 4).  q comes either from a
// caller-provided buffer (parity tests) or from Philox4x32-10 keyed by (seed; step, noise_row, index).
// Every image of a launch has its own temperature, top-k, top-p, greedy flag, Philox key and counter word (SmpRow); the scalar
// entry points fill all rows alike.  The CFG combine pairs row b with row b + B and is the only cross-row arithmetic.
#pragma once
#include "common.cuh"

constexpr int SMP_THREADS = 1024;

__device__ __forceinline__ uint32_t float_order_key(float f) {   // larger float -> larger key; -0.0 and +0.0 share one key
    uint32_t u = __float_as_uint(f);                               // (-0 == +0 in the reference's comparisons: a top-k threshold
    u = u == 0x80000000u ? 0u : u;                                 //  of +0 keeps every -0 entry)
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ void philox4x32_10(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2,
                                              uint32_t c3, uint32_t (&out)[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ float exp1_from_bits(uint32_t x);
// Exp(1) draw of element i at token `step` of the stream with counter word `row` (kept out of line: it sits in a fully unrolled loop)
__device__ __noinline__ float exp1_noise(uint32_t seed_lo, uint32_t seed_hi, int i, uint32_t row, int step) {
    uint32_t r[4];
    philox4x32_10(seed_lo, seed_hi, (uint32_t)(i >> 2), row, (uint32_t)step, 0x43415231u, r);
    return exp1_from_bits(r[i & 3]);
}
__device__ __forceinline__ float exp1_from_bits(uint32_t x) {
    // u in (0,1]: (x + 1) * 2^-32 ;  q = -log(u) ~ Exp(1)
    const float u = ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f);
    return -logf(u);
}

// sampling parameters of one image (32 bytes, read as two 16-byte loads)
struct __align__(16) SmpRow {
    float inv_temp; int top_k; float top_p; int sample_logits;
    uint32_t seed_lo, seed_hi;  // Philox key
    uint32_t noise_row;         // Philox counter word 1: the image's index under one seed per launch, 0 under a seed per image
    uint32_t pad;
};

struct SampleArgs {
    const float* logits;    // [b_eff, V]
    int V; int B;           // B images; b_eff = 2B when cfg
    int use_cfg; int cfg_on; float cfg_scale;
    const SmpRow* rows;     // [B] (device)
    const float* noise;     // [B, V] (or [steps, B, V] when noise_per_step) or null
    int noise_per_step;
    int step;               // Philox sub-stream = index of the token being produced
    int cfg_interval;       // device-side cfg_flag: off when step-1 > cfg_interval >= 0  (generate.py:121-122)
    int* idx_out;           // [B] (or tokens_out + step when tokens_ld > 0)
    int tokens_ld;
    float* probs_out;       // [B, V] or null
    unsigned char* kept_out; // [B, V] or null: 1 where the token survives top-k and top-p (also when its probability underflows to 0)
    // fused next-step embedding (decode loop only; null => skip)
    void* h_out; const void* tok_emb; const void* ctrl0; int d; int n_img; int T; const float* cs; int dtype;   // cs: [b_eff] strengths
    int* tok_buf;           // [b_eff] int32 tokens consumed by teacher-free decode
    int* pos_ptr;           // device scalar: position of the token being produced is *pos_ptr + 1
    int* done_ctr;          // ticket: the last block to finish advances *pos_ptr
    int pos_val;            // position when pos_ptr is null (persistent decode kernel)
    float* ssq_rows;        // optional [16]: sum of squares of the written h rows (index = row), else null
    int h_reps; long long h_rep_stride;
    long long* dbg_ts;      // dev (PK_TRACE builds): globaltimer stamps of the sampler's stages, written by thread 0   // extra replicas of h_out (persistent kernel), 0/1 = none
};

template <typename T>
__device__ __forceinline__ void write_next_h(const SampleArgs& a, int b_row, int tok, int pos_next, float* red32) {
    // h = tok_embeddings[tok] (+ cs[b] * ctrl0[b][pos_next - T + 1])    gpt_t2i.py:445,466
    const T* e = (const T*)a.tok_emb + (size_t)tok * a.d;
    T* h = (T*)a.h_out + (size_t)b_row * a.d;
    const int p = pos_next - a.T + 1;
    const T* c = (a.ctrl0 && p >= 0 && p < a.n_img) ? (const T*)a.ctrl0 + ((size_t)b_row * a.n_img + p) * a.d : nullptr;
    const float s = c ? __ldg(a.cs + b_row) : 0.f;
    float ss = 0.f;
    for (int k = threadIdx.x; k < a.d; k += blockDim.x) {
        float v = tof(e[k]);
        if (c) v = rnd<T>(v + rnd<T>(s * tof(c[k])));
        const T hv = fromf<T>(v);
        h[k] = hv;
        for (int rep = 1; rep < a.h_reps; ++rep) h[(size_t)rep * a.h_rep_stride + k] = hv;
        ss += v * v;
    }
    if (a.ssq_rows) {     // deterministic block reduction (fixed thread->element map, fixed tree)
        ss = warp_sum(ss);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) red32[threadIdx.x >> 5] = ss;
        __syncthreads();
        if (threadIdx.x == 0) {
            float t = 0.f;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red32[w];
            a.ssq_rows[b_row] = t;
        }
    }
}

// Block-wide reductions; `red` holds THREADS/32 slots.  max / count are order-independent; the soft-max mass is accumulated in
// 64-bit fixed point (2^-40 units), which is associative — so the result does not depend on the order in which the kept elements
// were compacted, and two runs give identical tokens.
template <int THREADS> __device__ __forceinline__ float smp_block_max(float v, float* red) {
    v = warp_max(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = red[0];
#pragma unroll
    for (int w = 1; w < THREADS / 32; ++w) s = fmaxf(s, red[w]);
    return s;
}
template <int THREADS> __device__ __forceinline__ unsigned long long smp_block_sum64(unsigned long long v, unsigned long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned long long s = 0ull;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) s += red[w];
    return s;
}
template <int THREADS> __device__ __forceinline__ void smp_block_count3(unsigned& c1, unsigned& c2, unsigned& c3, unsigned (*red)[3]) {
    c1 = __reduce_add_sync(0xffffffffu, c1); c2 = __reduce_add_sync(0xffffffffu, c2); c3 = __reduce_add_sync(0xffffffffu, c3);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = c1; red[threadIdx.x >> 5][1] = c2; red[threadIdx.x >> 5][2] = c3; }
    __syncthreads();
    c1 = c2 = c3 = 0u;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) { c1 += red[w][0]; c2 += red[w][1]; c3 += red[w][2]; }
}

// shared scratch of sample_body: selection histogram | boundary-bin candidates (index, value) | compacted kept list (index, value)
constexpr int SMP_NBIN = 2048, SMP_NCAND = 1024, SMP_CAP = 2304;        // CAP: top_k <= 2000 plus ties at the threshold
constexpr int SMP_SCRATCH = SMP_NBIN * 4 + SMP_NCAND * 8 + SMP_CAP * 8;
constexpr float SMP_FIX = 1099511627776.0f;                              // 2^40: fixed-point unit of the soft-max mass

// four consecutive elements of the CFG-combined, temperature-scaled row (generate.py:103-107, :60); separate sub / mul / add like
// the eager reference (no FMA contraction), identical bits in every pass over the row
__device__ __forceinline__ float4 smp_z4(const SampleArgs& a, float inv_temp, const float* lc, const float* lu, int i4, bool cfg) {
    float4 v = __ldcg(reinterpret_cast<const float4*>(lc) + i4);
    if (cfg) {
        const float4 u = __ldcg(reinterpret_cast<const float4*>(lu) + i4);
        v.x = __fadd_rn(u.x, __fmul_rn(__fsub_rn(v.x, u.x), a.cfg_scale)); v.y = __fadd_rn(u.y, __fmul_rn(__fsub_rn(v.y, u.y), a.cfg_scale));
        v.z = __fadd_rn(u.z, __fmul_rn(__fsub_rn(v.z, u.z), a.cfg_scale)); v.w = __fadd_rn(u.w, __fmul_rn(__fsub_rn(v.w, u.w), a.cfg_scale));
    }
    v.x = __fmul_rn(v.x, inv_temp); v.y = __fmul_rn(v.y, inv_temp); v.z = __fmul_rn(v.z, inv_temp); v.w = __fmul_rn(v.w, inv_temp);
    return v;
}

// One CTA per image (b).  Nothing of the row is kept in registers: every stage is a short rolled loop, either over the row itself
// (re-read from L2 and re-combined: 2 x 64 KB per pass) or over the compacted list of kept elements in shared memory.  (The
// register-resident version was 8 K fully unrolled instructions executed once per token — in the persistent decode kernel that
// is 130 KB of cold instruction fetch per token, and its per-element shared-memory atomics serialised: 49 us per token.)
//   top-k : exact k-th largest by a two-level selection — a 2048-bin histogram over a monotone linear map of the value range, then
//           exact ranks of the few candidates of the boundary bin on the order-preserving integer keys; ties at the threshold are
//           kept (generate.py:37).  Crowded boundary bin (degenerate rows): bit-wise bisection over the row, two bits per pass.
//   kept  : elements above the boundary bin + the candidates at or above the threshold, compacted into shared memory (<= SMP_CAP
//           entries; larger kept sets — top_k = 0 or huge — run the same stages as passes over the row instead).
//   soft-max / nucleus / exponential race touch the kept elements only; Philox is evaluated per kept element.
#ifdef PK_TRACE
#define SMP_STAMP(k) do { if (a.dbg_ts != nullptr && threadIdx.x == 0) { long long t_; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t_)); a.dbg_ts[k] = t_; } } while (0)
#else
#define SMP_STAMP(k) do { } while (0)
#endif

// visit every kept element (index, value): the compacted list, or the whole row filtered by the threshold key
template <int THREADS, typename F>
__device__ __forceinline__ void smp_for_kept(const SampleArgs& a, float inv_temp, const float* lc, const float* lu, bool cfg, bool use_list, const int* ki,
                                             const float* kz, unsigned nk, bool has_thr, unsigned thr, F f) {
    if (use_list) {
        for (unsigned c = threadIdx.x; c < nk; c += THREADS) f(ki[c], kz[c]);
    } else {
        const int V4 = a.V >> 2;
#pragma unroll 1
        for (int i4 = threadIdx.x; i4 < V4; i4 += THREADS) {   // (rare path: kept small, not fast)
            const float4 z = smp_z4(a, inv_temp, lc, lu, i4, cfg);
            const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll 1
            for (int q = 0; q < 4; ++q)
                if (!has_thr || float_order_key(zz[q]) >= thr) f(4 * i4 + q, zz[q]);
        }
    }
}

template <int THREADS>
__device__ __forceinline__ void sample_body(const SampleArgs& a, const int b, unsigned char* scratch) {
    constexpr int NW = THREADS / 32;
    __shared__ float red_f[NW];
    __shared__ unsigned long long red_q[NW];
    __shared__ unsigned red_u[NW];
    __shared__ unsigned red_c[NW][3];
    __shared__ int red_i[NW];
    __shared__ int s_tok;
    __shared__ unsigned s_cnt, s_nk, s_bin, s_krem, s_thr, s_over;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int V = a.V, V4 = V >> 2;                        // (host-checked: V % 4 == 0)
    // the image's parameters in two 16-byte loads, issued together before the first pass over the row
    const uint4 r0 = __ldg(reinterpret_cast<const uint4*>(a.rows + b)), r1 = __ldg(reinterpret_cast<const uint4*>(a.rows + b) + 1);
    const float inv_temp = __uint_as_float(r0.x), top_p = __uint_as_float(r0.z);
    const int top_k = (int)r0.y;
    const bool sample_logits = r0.w != 0u;
    const uint32_t seed_lo = r1.x, seed_hi = r1.y, noise_row = r1.z;
    const int pos = a.pos_ptr ? ld_cg(a.pos_ptr) : a.pos_val;
    const int step = a.pos_ptr ? (pos - a.T + 1) : a.step;   // index of the token being produced
    bool cfg_on = a.cfg_on != 0;
    if (a.cfg_interval > -1 && step - 1 > a.cfg_interval) cfg_on = false;
    const bool cfg = a.use_cfg && cfg_on;
    const float* lc = a.logits + (size_t)b * V;
    const float* lu = a.logits + (size_t)(b + a.B) * V;
    unsigned* const s_hist = reinterpret_cast<unsigned*>(scratch);
    int* const s_ci = reinterpret_cast<int*>(scratch + SMP_NBIN * 4);
    float* const s_cz = reinterpret_cast<float*>(scratch + SMP_NBIN * 4 + SMP_NCAND * 4);
    int* const s_ki = reinterpret_cast<int*>(scratch + SMP_NBIN * 4 + SMP_NCAND * 8);
    float* const s_kz = reinterpret_cast<float*>(scratch + SMP_NBIN * 4 + SMP_NCAND * 8 + SMP_CAP * 4);

    SMP_STAMP(0);
    const bool has_thr = top_k > 0 && top_k < V;
    bool use_list = has_thr && top_k + 64 <= SMP_CAP;   // room for ties at the threshold; else the stages run over the row
    unsigned thr = 0u, nk = 0u;
    if (has_thr) {
        // ---- level 1: value range, histogram, boundary bin
        float lo = INFINITY, hi = -INFINITY;
#pragma unroll 2
        for (int i4 = tid; i4 < V4; i4 += THREADS) {
            const float4 z = smp_z4(a, inv_temp, lc, lu, i4, cfg);
            lo = fminf(fminf(lo, z.x), fminf(z.y, fminf(z.z, z.w)));
            hi = fmaxf(fmaxf(hi, z.x), fmaxf(z.y, fmaxf(z.z, z.w)));
        }
        hi = smp_block_max<THREADS>(hi, red_f);
        lo = -smp_block_max<THREADS>(-lo, red_f);
        const float scale = (hi > lo && lo > -INFINITY) ? (float)(SMP_NBIN - 1) / (hi - lo) : 0.f;
        for (int i = tid; i < SMP_NBIN; i += THREADS) s_hist[i] = 0u;
        if (tid == 0) { s_cnt = 0u; s_nk = 0u; s_thr = 0u; s_over = 0u; s_bin = 0u; s_krem = (unsigned)top_k; }
        __syncthreads();
        SMP_STAMP(1);
#pragma unroll 2
        for (int i4 = tid; i4 < V4; i4 += THREADS) {
            const float4 z = smp_z4(a, inv_temp, lc, lu, i4, cfg);
            const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) atomicAdd(&s_hist[min(max((int)((zz[q] - lo) * scale), 0), SMP_NBIN - 1)], 1u);
        }
        __syncthreads();
        SMP_STAMP(5);
        {   // bin (from the top) in which the cumulative count reaches k: thread t owns bins [t BPT, (t + 1) BPT)
            constexpr int BPT = (SMP_NBIN + THREADS - 1) / THREADS;
            unsigned loc[BPT], mine = 0u;
#pragma unroll
            for (int i = 0; i < BPT; ++i) { const int bi = tid * BPT + i; loc[i] = bi < SMP_NBIN ? s_hist[bi] : 0u; mine += loc[i]; }
            unsigned incl = mine;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_down_sync(0xffffffffu, incl, o); if (lane + o < 32) incl += v; }
            if (lane == 0) red_u[warp] = incl;
            __syncthreads();
            unsigned above = incl - mine;
            for (int w = warp + 1; w < NW; ++w) above += red_u[w];
            const unsigned kk = (unsigned)top_k;
#pragma unroll
            for (int i = BPT - 1; i >= 0; --i) {
                if (above < kk && kk <= above + loc[i]) { s_bin = (unsigned)(tid * BPT + i); s_krem = kk - above; }
                above += loc[i];
            }
        }
        __syncthreads();
        SMP_STAMP(6);
        const int bsel = (int)s_bin;
        const unsigned krem = s_krem;
        // ---- level 2: one pass collects the elements above the boundary bin (kept for sure) and the boundary bin's candidates
#pragma unroll 2
        for (int i0 = 0; i0 < V4; i0 += THREADS) {         // (warp-uniform trip count: the allocation below uses warp collectives)
            const int i4 = i0 + tid;
            const bool valid = i4 < V4;
            const float4 z = smp_z4(a, inv_temp, lc, lu, valid ? i4 : 0, cfg);
            const float zz[4] = {z.x, z.y, z.z, z.w};
            int bin[4];
            unsigned mykeep = 0u;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                bin[q] = valid ? min(max((int)((zz[q] - lo) * scale), 0), SMP_NBIN - 1) : -1;
                mykeep += bin[q] > bsel ? 1u : 0u;
                if (bin[q] == bsel) {
                    const unsigned pc = atomicAdd(&s_cnt, 1u);
                    if (pc < (unsigned)SMP_NCAND) { s_ci[pc] = 4 * i4 + q; s_cz[pc] = zz[q]; }
                }
            }
            if (use_list) {                                // warp-aggregated allocation: one shared-memory atomic per warp and iteration
                unsigned incl = mykeep;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
                const unsigned tot = __shfl_sync(0xffffffffu, incl, 31);
                unsigned base = 0u;
                if (tot != 0u) {
                    if (lane == 31) base = atomicAdd(&s_nk, tot);
                    base = __shfl_sync(0xffffffffu, base, 31);
                    unsigned at = base + incl - mykeep;
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        if (bin[q] > bsel) { if (at < (unsigned)SMP_CAP) { s_ki[at] = 4 * i4 + q; s_kz[at] = zz[q]; } ++at; }
                }
            }
        }
        __syncthreads();
        SMP_STAMP(7);
        const unsigned ncand = s_cnt;
        if (ncand <= (unsigned)SMP_NCAND) {
            // exact rank inside the bin: the k_rem-th largest candidate (duplicates counted) is the one with
            // #{greater} < k_rem <= #{greater or equal}
            for (unsigned c = tid; c < ncand; c += THREADS) {
                const unsigned key = float_order_key(s_cz[c]);
                unsigned gt = 0u, ge = 0u;
                for (unsigned q = 0; q < ncand; ++q) { const unsigned kq = float_order_key(s_cz[q]); gt += kq > key ? 1u : 0u; ge += kq >= key ? 1u : 0u; }
                if (gt < krem && krem <= ge) s_thr = key;                  // (ties write the same value)
            }
            __syncthreads();
            thr = s_thr;
            if (use_list) {                                // candidates at or above the threshold join the kept list
                for (unsigned c = tid; c < ncand; c += THREADS)
                    if (float_order_key(s_cz[c]) >= thr) {
                        const unsigned at = atomicAdd(&s_nk, 1u);
                        if (at < (unsigned)SMP_CAP) { s_ki[at] = s_ci[c]; s_kz[at] = s_cz[c]; }
                    }
                __syncthreads();
            }
        } else {
            // crowded bin: bit-wise bisection on the integer keys of the whole row, two bits per pass
#pragma unroll 1
            for (int shift = 30; shift >= 0; shift -= 2) {
                const unsigned t1 = thr | (1u << shift), t2 = thr | (2u << shift), t3 = thr | (3u << shift);
                unsigned c1 = 0, c2 = 0, c3 = 0;
                for (int i4 = tid; i4 < V4; i4 += THREADS) {
                    const float4 z = smp_z4(a, inv_temp, lc, lu, i4, cfg);
                    const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) { const unsigned k = float_order_key(zz[q]); c1 += k >= t1 ? 1u : 0u; c2 += k >= t2 ? 1u : 0u; c3 += k >= t3 ? 1u : 0u; }
                }
                smp_block_count3<THREADS>(c1, c2, c3, red_c);
                const unsigned kk = (unsigned)top_k;                 // counts are non-increasing in the threshold
                thr = c3 >= kk ? t3 : (c2 >= kk ? t2 : (c1 >= kk ? t1 : thr));
            }
            use_list = false;                              // (the list holds only the bins above; this rare path runs over the row)
        }
        nk = s_nk;
        if (nk > (unsigned)SMP_CAP) use_list = false;      // (CTA-uniform) more ties than the list holds
    }
    SMP_STAMP(2);
    auto for_kept = [&](auto f) { smp_for_kept<THREADS>(a, inv_temp, lc, lu, cfg, use_list, s_ki, s_kz, nk, has_thr, thr, f); };

    // ---- soft-max over the kept elements
    float mx = -INFINITY;
    for_kept([&](int, float z) { mx = fmaxf(mx, z); });
    mx = smp_block_max<THREADS>(mx, red_f);
    unsigned long long mass = 0ull;
    for_kept([&](int, float z) { mass += __float2ull_rn(expf(z - mx) * SMP_FIX); });
    mass = smp_block_sum64<THREADS>(mass, red_q);
    float sum = (float)mass * (1.0f / SMP_FIX);
    // ---- nucleus (top-p), generate.py:40-55: in descending order a token is removed iff the cumulative probability of the tokens
    // strictly before it exceeds top_p (first always kept).  Equivalently token x is kept iff f(p_x) <= top_p with f(v) = mass of the
    // tokens with probability > v; f is a non-increasing step function, so the kept set is {p >= tau*} with tau* the SMALLEST
    // probability that satisfies it.  tau* is found exactly by a 32-step binary search over the order-preserving integer keys of the
    // probabilities (ADVICE r1: a bisection on the value with a fixed step count kept tokens within 2^-30 of the boundary), the masses
    // compared in 64-bit fixed point.  (torch.sort's order among exactly tied probabilities is unspecified; ties are kept together.)
    const float sum_pre = sum;                             // normaliser of the pre-nucleus probabilities
    unsigned p_key = 0u;                                   // elements whose pre-nucleus probability key is below p_key are dropped
    if (top_p < 1.0f) {
        const double budget = (double)top_p * (double)mass;
        unsigned long long lo = 0ull, hi = 0xFFFFFFFFull;  // predicate(k): mass{key(p) > k} <= budget; true at hi, monotone in k
        while (lo < hi) {                                  // (CTA-uniform: every thread sees the same block sums)
            const unsigned mid = (unsigned)((lo + hi) >> 1);
            unsigned long long ma = 0ull;
            for_kept([&](int, float z) { const float e = expf(z - mx); if (float_order_key(e / sum_pre) > mid) ma += __float2ull_rn(e * SMP_FIX); });
            ma = smp_block_sum64<THREADS>(ma, red_q);
            if ((double)ma <= budget) hi = mid; else lo = (unsigned long long)mid + 1ull;
        }
        p_key = (unsigned)hi;
        unsigned long long m2 = 0ull;
        for_kept([&](int, float z) { const float e = expf(z - mx); if (float_order_key(e / sum_pre) >= p_key) m2 += __float2ull_rn(e * SMP_FIX); });
        m2 = smp_block_sum64<THREADS>(m2, red_q);
        sum = (float)m2 * (1.0f / SMP_FIX);                // soft-max over the surviving logits only
    }
    if (a.probs_out || a.kept_out) {
        float* po = a.probs_out ? a.probs_out + (size_t)b * V : nullptr;
        unsigned char* ko = a.kept_out ? a.kept_out + (size_t)b * V : nullptr;
        for (int i4 = tid; i4 < V4; i4 += THREADS) {
            if (po) reinterpret_cast<float4*>(po)[i4] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ko) reinterpret_cast<uchar4*>(ko)[i4] = make_uchar4(0, 0, 0, 0);
        }
        __syncthreads();
        for_kept([&](int i, float z) {
            const float e = expf(z - mx);
            if (float_order_key(e / sum_pre) >= p_key) { if (po) po[i] = e / sum; if (ko) ko[i] = 1; }
        });
    }
    SMP_STAMP(3);
    // ---- draw: arg-max of p (greedy) or of p / q (exponential race); lowest index wins ties
    float best = -1.f; int besti = 0x7fffffff;
    const float* nz = a.noise ? a.noise + ((size_t)(a.noise_per_step ? step : 0) * a.B + b) * V : nullptr;
    for_kept([&](int i, float z) {
        const float e = expf(z - mx);
        if (float_order_key(e / sum_pre) >= p_key && e > 0.f) {
            float sv = e / sum;
            if (sample_logits) sv = sv / (nz ? nz[i] : exp1_noise(seed_lo, seed_hi, i, noise_row, step));
            if (sv > best || (sv == best && i < besti)) { best = sv; besti = i; }
        }
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    __syncthreads();
    if (lane == 0) { red_f[warp] = best; red_i[warp] = besti; }
    __syncthreads();
    if (tid == 0) {
        float bb = red_f[0]; int bi = red_i[0];
        for (int w = 1; w < NW; ++w)
            if (red_f[w] > bb || (red_f[w] == bb && red_i[w] < bi)) { bb = red_f[w]; bi = red_i[w]; }
        s_tok = bi;
        if (a.tokens_ld > 0) a.idx_out[(size_t)b * a.tokens_ld + step] = bi;
        else a.idx_out[b] = bi;
        if (a.tok_buf) { a.tok_buf[b] = bi; if (a.use_cfg) a.tok_buf[b + a.B] = bi; }
    }
    __syncthreads();

    SMP_STAMP(4);
    // ---- fused tail: next step's input rows (cond half b, uncond half b+B)
    if (a.h_out) {
        const int tok = s_tok;
        if (a.dtype == CAR_BF16) {
            write_next_h<bf16>(a, b, tok, pos + 1, red_f);
            if (a.use_cfg) write_next_h<bf16>(a, b + a.B, tok, pos + 1, red_f);
        } else {
            write_next_h<float>(a, b, tok, pos + 1, red_f);
            if (a.use_cfg) write_next_h<float>(a, b + a.B, tok, pos + 1, red_f);
        }
    }
    // ---- the last block to finish advances the device-side position
    if (a.done_ctr) {
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            const int old = atomicAdd(a.done_ctr, 1);
            if (old == a.B - 1) {
                *a.done_ctr = 0;
                if (a.pos_ptr) *a.pos_ptr = pos + 1;
            }
        }
    }
}

__global__ void __launch_bounds__(SMP_THREADS) sample_kernel(SampleArgs a) {
    __shared__ __align__(16) unsigned char smp_scratch[SMP_SCRATCH];
    sample_body<SMP_THREADS>(a, blockIdx.x, smp_scratch);
}
