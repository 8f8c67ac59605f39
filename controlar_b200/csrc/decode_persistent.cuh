// decode_persistent.cuh — the whole conditional-decoding loop (N-1 decode steps + CFG + sampling) as ONE persistent
// cooperative kernel, one 512-thread CTA per SM.  Replaces, per generated token (reference file:line):
//   decode_one_token + decode_n_tokens      autoregressive/models/generate.py:95-131
//   Transformer.forward (decode branch)     autoregressive/models/gpt_t2i.py:444-470
//   TransformerBlock / Attention / FeedForward / RMSNorm / KVCache.update   gpt_t2i.py:187-306
//
// Why it is built this way:
//   * At B_eff = 16 a decode step is a chain of 5 all-to-all dependent phases per layer (qkv | attention | wo |
//     w1w3 | w2); each per-kernel link of the launch chain costs several times the time the data needs.  Here the CTAs stay
//     resident and the chain link is a tagged-packet exchange through L2 instead
//     of a kernel boundary (or a grid barrier + gather, 2.2 us).
//   * Weights do not depend on activations: every CTA streams ITS weight slices, in consumption order, with
//     cp.async.bulk into an 8 x 20 KB shared-memory ring that runs ahead of the compute — across phases, layers and
//     tokens — so HBM stays busy while the dependent chain waits on L2 latency.
//   * Activations cross CTAs as 8-byte packets {bf16 pair, tag}; the consumer polls the data itself
//     (ld.relaxed.gpu — a weak .cg load can be served from a stale far-die copy) until the tag equals the expected
//     epoch.  No fence, no counter, one L2 round trip.  Packets are laid out as the consumer's mma A fragments, so
//     they go from L2 straight into registers.
//   * Attention splits the flattened (sequence, head, key) space evenly over the CTAs; a (b, h) that straddles two
//     CTAs is combined by its owner from the helper's tagged partial.  The one true grid barrier per token sits in
//     front of the sampler (it also orders the KV-cache rows written with plain stores).
// Arithmetic (rounding points, fixed reduction orders) follows the per-kernel chain in gemm_skinny.cuh/attention.cuh.
#pragma once
#include "common.cuh"
#include "sampler.cuh"
#include "pk_plan.h"

constexpr int PK_WARPS = 16, PK_THREADS = PK_WARPS * 32;
constexpr int PK_NSLOT = 8;                          // ring slots (power of two)
constexpr int PK_UNIT_KS = 40;                       // k32-steps per streamed unit (one 8-column block, <= 40 steps)
constexpr int PK_SLOT_BYTES = PK_UNIT_KS * 512;      // 20 KB
constexpr int PK_NBMAX = 4;                          // 8-column blocks per batch (accumulator registers)
constexpr int PK_RED = 144;                          // floats per (warp, block) in the reduction buffer (128 + 16 pad)
constexpr int PK_MAXSEG = 6;                         // attention segments per CTA
constexpr int PK_SMEM_RING = PK_NSLOT * PK_SLOT_BYTES;
constexpr int PK_SMEM_RED = PK_WARPS * PK_NBMAX * PK_RED * 4;
constexpr int PK_MAXA = 7;                           // k32-steps per warp (K <= 16 * 7 * 32 = 3584)
constexpr int PK_MAXA_NORM = 3;                      // ... of the RMS-normalised GEMMs (K = dim <= 1536)
constexpr int PK_MAXL = 64;                          // layers (shared-memory pointer tables)
constexpr int PK_SMEM_MISC = 16 * 16 * 4 + 128 + 128 + 2 * 2 * 32 * 8 + 3 * 6 * 128     // ssq, mbarriers, stream cursor, residual and control pairs, q/k/v rows
                             + 1024 + 4 * PK_MAXL * 8 + PK_WARPS * PK_MAXA_NORM * 32 * 2;   // attention plan, pointer tables, norm weights
constexpr int PK_SMEM_TOTAL = PK_SMEM_RING + PK_SMEM_RED + PK_SMEM_MISC;

struct PkParams {
    int dim, F, V, L, H, T, S, n_img, b_eff, B;
    float eps;
    const float* cs;                   // [b_eff] control strength per row
    const bf16* tok_emb; const bf16* norm_w; const uint4* w_out;
    const uint4* const* wqkv; const uint4* const* wo; const uint4* const* w13; const uint4* const* w2;
    const bf16* const* attn_norm; const bf16* const* ffn_norm;
    bf16* const* kc; bf16* const* vc;
    const bf16* ctrl[3]; int has_ctrl;
    const float* rope; const int* emb_mask;
    float* logits;
    const int* part;                   // [4][grid + 1] block offsets per CTA: qkv blocks, d-column blocks (wo, w2), w1/w3 pairs, head blocks
    uint2* h2[2]; uint2* h1[2]; uint2* att[2]; uint2* act[2]; uint2* qkv[2]; uint2* partial[2];
    int part_slots;                    // helper slots per (b, h) in `partial`
    unsigned int tag_base;             // tags of this launch are tag_base + 1 ...
    unsigned int* bar; unsigned int bar_base;
    SampleArgs smp;
    int n_steps;                       // tokens to produce (decode iterations = n_steps - 1)
    const int* forced; int forced_ld;  // teacher forcing (parity tests): token fed to the next step = forced[b * forced_ld + step] instead of the sampled one
    long long* step_ts;                // optional [n_steps]: globaltimer (ns) when CTA 0 enters step s (bench: ms/step vs context length)
    float* trace;                      // optional [n_steps][b_eff][V] fp32: raw model logits of every step (trace[0] = prefill logits, copied by the host)
    long long* dbg; int dbg_step;      // PK_TRACE builds: [grid][64] globaltimer stamps (ns) of one step / layer 3
};

// ---------------------------------------------------------------------------------------------------------
// primitives
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 pk_ld128(const void* p) {
    uint4 r;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ uint2 pk_ld64(const void* p) {
    uint2 r;
    asm volatile("ld.relaxed.gpu.global.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void pk_st128(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.relaxed.gpu.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void pk_st64(void* p, uint32_t a, uint32_t b) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint32_t pk_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void pk_mbar_init(uint64_t* b, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(pk_smem(b)), "r"(count)); }
__device__ __forceinline__ void pk_mbar_expect(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(pk_smem(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void pk_mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t ok = 0, spins = 0;
    while (!ok) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(pk_smem(b)), "r"(parity) : "memory");
        if (!ok && ++spins > (1u << 24)) __trap();       // never hang the box
    }
}
// L2 eviction priority (per-instruction cache hint).  Weight units pass through L2 once per token and K/V rows are read once
// per layer and token, so neither is ever re-read from L2: both are marked evict-first and give way to the lines that are
// (activation packets, attention partials, the K/V rows this token writes).  Measured: DESIGN §5.
__device__ __forceinline__ uint64_t pk_pol_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void pk_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(pk_smem(dst)), "l"(src), "r"(bytes), "r"(pk_smem(bar)), "l"(pk_pol_evict_first()) : "memory");
}
__device__ __forceinline__ uint4 pk_ld_kv(const void* p, uint64_t pol) {
    uint4 r;
    asm volatile("ld.global.cg.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void pk_grid_sync(unsigned int* bar, unsigned int& gen) {
    __syncthreads();
    if (threadIdx.x == 0) {
        gen += gridDim.x;
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(bar) : "memory");
        unsigned int spins = 0;
        while (true) {
            unsigned int v;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
            if ((int)(v - gen) >= 0) break;
            if (++spins > (1u << 26)) __trap();
        }
    }
    __syncthreads();
}
__device__ __forceinline__ uint32_t pk_pack(float a, float b) {
    __nv_bfloat162 pk = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&pk);
}
__device__ __forceinline__ long long pk_now() { long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void pk_spin_check(unsigned int& spins) { if (++spins > (1u << 24)) __trap(); }

// A-fragment packet layout of a [16][K] activation tile (H1, H2, ATT, ACT): for k32-step s, pair slot p = 0..3 and lane
// (g, t) one 16-byte packet {pair(row g, k = 32s + 8t + 2p), tag, pair(row g + 8, same k), tag} at 16-byte index
// (4s + p) * 32 + lane — a warp's load of one p is 512 contiguous bytes.  uint2 index of (row r, column k):
__device__ __forceinline__ size_t pk_a_index(int r, int k) {
    const int s = k >> 5, t = (k >> 3) & 3, p = (k >> 1) & 3, g = r & 7, hi = r >> 3;
    return ((size_t)((s * 4 + p) * 32 + g * 4 + t)) * 2 + hi;
}

extern __shared__ __align__(128) unsigned char pk_smem_raw[];

struct PkSmem {
    unsigned char* ring;     // [PK_NSLOT][PK_SLOT_BYTES]
    float* red;              // [PK_WARPS][PK_NBMAX][PK_RED]   (attention scratch aliases it)
    float* ssq;              // [PK_WARPS][16]
    uint64_t* full;          // [PK_NSLOT]
    struct PkStream* st;     // weight-stream cursor (touched by the producer thread only)
    uint2* own;              // [2][32] residual-stream pairs of the d-column blocks this CTA owns {rows g, rows g + 8}
    uint2* ctl;              // [2][32] the same pairs' control add of the next layer group, rnd(cs[r] * c)
    uint32_t* qrow;          // [3][PK_MAXSEG][32] q / newest k / newest v of the attention segments (bf16 pairs)
    PkAttnPlan* plan;        // this token's attention work split (pk_plan.h)
    const bf16** kvp;        // [L][2] K / V cache base of every layer (copied from the pointer arrays once per launch)
    const bf16** nwp;        // [L][2] attention_norm / ffn_norm weights of every layer
    bf16* nw;                // [<= 1536] the phase's RMSNorm weights, staged by cp.async while the CTA waits for its A packets
};
static_assert(sizeof(PkAttnPlan) <= 1024 && PKP_WARPS == PK_WARPS && PKP_MAXSEG == PK_MAXSEG, "plan layout");
__device__ __forceinline__ PkSmem pk_smem_layout() {
    PkSmem sm;
    unsigned char* q = pk_smem_raw;
    sm.ring = q; q += PK_SMEM_RING;
    sm.red = reinterpret_cast<float*>(q); q += PK_SMEM_RED;
    sm.ssq = reinterpret_cast<float*>(q); q += 16 * 16 * 4;
    sm.full = reinterpret_cast<uint64_t*>(q); q += 128;
    sm.st = reinterpret_cast<PkStream*>(q); q += 128;
    sm.own = reinterpret_cast<uint2*>(q); q += 2 * 32 * 8;
    sm.ctl = reinterpret_cast<uint2*>(q); q += 2 * 32 * 8;
    sm.qrow = reinterpret_cast<uint32_t*>(q); q += 3 * 6 * 128;
    sm.plan = reinterpret_cast<PkAttnPlan*>(q); q += 1024;
    sm.kvp = reinterpret_cast<const bf16**>(q); q += 2 * PK_MAXL * 8;
    sm.nwp = reinterpret_cast<const bf16**>(q); q += 2 * PK_MAXL * 8;
    sm.nw = reinterpret_cast<bf16*>(q);
    return sm;
}


// ---------------------------------------------------------------------------------------------------------
// weight stream: the producer thread walks the CTA's units in consumption order
// ---------------------------------------------------------------------------------------------------------
struct PkCursor { int step, l, phase, blk, sub; bool done; };
struct PkStream {
    PkCursor c;                     // next unit to copy into the ring
    unsigned int issued;
    int lo[5], hi[5];               // block ranges per phase (0 qkv, 1 wo, 2 w13, 3 w2, 4 head)
};

__device__ __forceinline__ int pk_phase_ks(const PkParams& P, int phase) { return (phase == 3 ? P.F : P.dim) >> 5; }

__device__ __forceinline__ void pk_cursor_next_phase(const PkParams& P, PkCursor& c) {
    if (c.phase == 4) { c.phase = 0; c.l = 0; ++c.step; if (c.step >= P.n_steps - 1) c.done = true; }
    else if (c.phase == 3) { c.phase = 0; ++c.l; }
    else ++c.phase;
}
// position the cursor on the next phase with a non-empty block range; sets done at the end of the stream
__device__ __forceinline__ void pk_cursor_skip_empty(const PkParams& P, const PkStream& st, PkCursor& c) {
    while (!c.done) {
        if (c.phase < 4 && c.l >= P.L) c.phase = 4;
        if (st.lo[c.phase] < st.hi[c.phase]) { c.blk = st.lo[c.phase]; c.sub = 0; return; }
        pk_cursor_next_phase(P, c);
    }
}
// the unit under the cursor (global address, bytes), then advance
__device__ __forceinline__ const uint4* pk_cursor_take(const PkParams& P, const PkStream& st, PkCursor& c, uint32_t& bytes) {
    const int KS = pk_phase_ks(P, c.phase);
    const uint4* W = c.phase == 0 ? P.wqkv[c.l] : c.phase == 1 ? P.wo[c.l] : c.phase == 2 ? P.w13[c.l] : c.phase == 3 ? P.w2[c.l] : P.w_out;
    const int ks0 = c.sub * PK_UNIT_KS, nks = min(PK_UNIT_KS, KS - ks0);
    const uint4* src = W + ((size_t)c.blk * KS + ks0) * 32;
    bytes = (uint32_t)nks * 512u;
    if ((c.sub + 1) * PK_UNIT_KS < KS) { ++c.sub; return src; }
    c.sub = 0;
    if (++c.blk < st.hi[c.phase]) return src;
    pk_cursor_next_phase(P, c);
    pk_cursor_skip_empty(P, st, c);
    return src;
}
__device__ __forceinline__ void pk_stream_issue(const PkParams& P, const PkSmem& sm, PkStream& st) {
    uint32_t bytes;
    const uint4* src = pk_cursor_take(P, st, st.c, bytes);
    const int slot = st.issued % PK_NSLOT;
    pk_mbar_expect(&sm.full[slot], bytes);
    pk_bulk_g2s(sm.ring + (size_t)slot * PK_SLOT_BYTES, src, bytes, &sm.full[slot]);
    ++st.issued;
}

// ---------------------------------------------------------------------------------------------------------
// A operand: poll the tagged packets of this warp's k-steps (s = warp + 16 i) straight into mma fragments
// ---------------------------------------------------------------------------------------------------------
// one round: up to 4 k-steps = 16 x 16 B per lane in flight
template <int I0, int CNT, bool FULL>
__device__ __forceinline__ void pk_poll_round(const unsigned char* __restrict__ base, int nst, int warp, int lane, unsigned int tag,
                                              bool need_lo, bool need_hi, uint32_t (&alo)[PK_MAXA][4], uint32_t (&ahi)[PK_MAXA][4]) {
    // k-steps past the end re-read step 0 and are ignored (unconditional first loads keep the 16-byte results in registers);
    // a k-step whose packets have not all arrived is re-read alone
    uint4 v[CNT][4];
    const unsigned char* rec[CNT];
#pragma unroll
    for (int u = 0; u < CNT; ++u) rec[u] = base + ((size_t)((I0 + u < nst) ? warp + (I0 + u) * PK_WARPS : 0) * 128 + lane) * 16;
#pragma unroll
    for (int u = 0; u < CNT; ++u)
#pragma unroll
        for (int p = 0; p < 4; ++p) v[u][p] = pk_ld128(rec[u] + p * 512);
    unsigned int spins = 0;
    while (true) {
        bool any_bad = false;
#pragma unroll
        for (int u = 0; u < CNT; ++u) {
            unsigned int b = 0;
#pragma unroll
            for (int p = 0; p < 4; ++p) b |= ((FULL || need_lo) ? (v[u][p].y ^ tag) : 0u) | ((FULL || need_hi) ? (v[u][p].w ^ tag) : 0u);
            if (I0 + u < nst && b != 0u) {
                any_bad = true;
#pragma unroll
                for (int p = 0; p < 4; ++p) v[u][p] = pk_ld128(rec[u] + p * 512);
            }
        }
        if (!any_bad) break;
        __nanosleep(40);
        pk_spin_check(spins);
    }
#pragma unroll
    for (int u = 0; u < CNT; ++u) {
        const bool in = I0 + u < nst;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            alo[I0 + u][p] = (in && (FULL || need_lo)) ? v[u][p].x : 0u;
            ahi[I0 + u][p] = (in && (FULL || need_hi)) ? v[u][p].z : 0u;
        }
    }
}

// Cheap arrival hint before the full poll: warp 0 watches the first packet of 32 of the K/8 producer blocks (a different
// subset per CTA) with back-off; the other warps wait at the CTA barrier.  SM count x 32 eight-byte loads per round instead of
// the whole tile from every waiting thread — waiting CTAs must not eat the L2 bandwidth of the ones still producing.
__device__ __forceinline__ void pk_prepoll(const uint2* buf, int K, unsigned int tag) {
    const int nblk = K >> 3;
    if (threadIdx.x < 32) {
        const uint2* pkt = buf + pk_a_index(0, (int)((blockIdx.x * 7u + threadIdx.x * (unsigned)max(1, nblk >> 5)) % (unsigned)nblk) * 8);
        unsigned int spins = 0;
        while (!__all_sync(0xffffffffu, pk_ld64(pkt).y == tag)) { __nanosleep(120); pk_spin_check(spins); }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------
// GEMM phase.  kind: 0 qkv (+RoPE, KV append) | 1 wo (+residual) | 2 w1/w3 (+SwiGLU) | 3 w2 (+residual, control add)
//              | 4 head (logits).  out[16, 8 nblk] = epi( norm?(A[16, K]) x Wp^T ), K split over the 16 warps.
// rnd(s * c) of a bf16x2 control pair, repacked: each product rounded to bf16 as the control add rounds it, so the w2 epilogue's
// rnd(h + that) is the add at strength s.  Formed when the pair is loaded and parked in shared memory (PkSmem::ctl), so the
// per-row strength holds no register across the GEMM phase.
__device__ __forceinline__ uint32_t pk_scaled_pair(float s, uint32_t c) {
    float c0, c1;
    unpack_bf16x2(c, c0, c1);
    return pk_pack(rnd<bf16>(s * c0), rnd<bf16>(s * c1));
}

// ---------------------------------------------------------------------------------------------------------
// Buffers by kind (l = layer, par = l & 1, tag = tag(step, l)):
//   0 qkv : A = H2[par]            out = QKV[par]                 norm = attention_norm[l]
//   1 wo  : A = ATT[par]           out = H1[par]                  residual = own pairs (layer 0: H2[0] from the sampler)
//   2 w13 : A = H1[par]            out = ACT[par]                 norm = ffn_norm[l]
//   3 w2  : A = ACT[par]           out = H2[par ^ 1], tag + 1     residual = own pairs, control add for layer l + 1
//   4 head: A = H2[par] (l = L)    out = logits                   norm = norm
__device__ __forceinline__ const uint2* pk_a_buf(const PkParams& P, int kind, int par) {
    return kind == 1 ? P.att[par] : kind == 2 ? P.h1[par] : kind == 3 ? P.act[par] : P.h2[par];
}
__device__ __forceinline__ const bf16* pk_ctrl_next(const PkParams& P, int l) {
    const int step3 = P.L / 3;
    return (P.has_ctrl && (l + 1) < P.L && (l + 1) % step3 == 0) ? P.ctrl[(l + 1) / step3] : nullptr;
}

__device__ __forceinline__ unsigned int pk_gemm_phase(const PkParams& P, const int kind, const int l, const int pos,
                                                       const unsigned int tag, int blk_lo, int blk_hi, unsigned int cons, long long* dbg, long long* wdbg_base,
                                                       float* trace_rows = nullptr) {
    const PkSmem sm = pk_smem_layout();
    const int par = l & 1;
    const bool NORM = (kind == 0 || kind == 2 || kind == 4);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int K = kind == 3 ? P.F : P.dim;
    const int KS = K >> 5;
    const int nsub = (KS + PK_UNIT_KS - 1) / PK_UNIT_KS;
    const int nst = (KS - warp + PK_WARPS - 1) / PK_WARPS;
    const int M = P.b_eff;
#ifdef PK_TRACE
    const bool stamp = dbg != nullptr && tid == 0;
#else
    constexpr bool stamp = false;
#endif
    if (blk_lo >= blk_hi) return cons;                 // this CTA owns no columns of this phase
    if (stamp) dbg[0] = pk_now();
    long long* const wdbg = (wdbg_base != nullptr && lane == 0) ? wdbg_base + warp * 16 : nullptr;   // per-warp stamps (dev)
#ifdef PK_TRACE
#define PK_W(k) do { if (wdbg) wdbg[k] = pk_now(); } while (0)
#else
#define PK_W(k) do { } while (0)
#endif
    PK_W(0);

    // epilogue identity of this thread (fixed across batches): block ej of the batch, row pair eg, column pair ecp
    const int ej = tid >> 7, eq = tid & 127, ei = eq >> 2, er = eq & 3, eg = ei >> 2, ecp = ei & 3;
    // residual pairs / control pairs (scaled by their rows' strengths) needed by the epilogue are requested before the A poll
    if (kind == 1 && l == 0 && er == 0 && ej < 2 && blk_lo + ej < blk_hi) {
        const int n = (blk_lo + ej) * 8 + 2 * ecp;
        const uint2* pp = P.h2[0] + pk_a_index(eg, n);
        uint4 v;
        unsigned int spins = 0;
        do { v = pk_ld128(pp); if (!(eg < M) || (v.y == tag && (!(eg + 8 < M) || v.w == tag))) break; pk_spin_check(spins); } while (true);
        sm.own[ej * 32 + ei] = make_uint2(v.x, v.z);
    }
    if (kind == 3 && er == 0 && blk_lo + ej < blk_hi) {
        const bf16* ctrl = pk_ctrl_next(P, l);
        const int n = (blk_lo + ej) * 8 + 2 * ecp;
        const int p = pos - P.T + 1;
        if (ctrl != nullptr && p >= 0 && p < P.n_img) {
            uint32_t lo = 0, hi = 0;
            if (eg < M) lo = pk_scaled_pair(__ldg(P.cs + eg), __ldg(reinterpret_cast<const unsigned int*>(ctrl + ((size_t)eg * P.n_img + p) * P.dim + n)));
            if (eg + 8 < M) hi = pk_scaled_pair(__ldg(P.cs + eg + 8), __ldg(reinterpret_cast<const unsigned int*>(ctrl + ((size_t)(eg + 8) * P.n_img + p) * P.dim + n)));
            sm.ctl[(ej & 1) * 32 + ei] = make_uint2(lo, hi);
        }
    }

    if (NORM) {   // this phase's RMSNorm weights -> shared memory, asynchronously, while we wait for the A packets
        const bf16* nwg = kind == 0 ? sm.nwp[2 * l] : kind == 2 ? sm.nwp[2 * l + 1] : P.norm_w;
        if (tid < (K >> 3))
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(pk_smem(sm.nw + tid * 8)), "l"(nwg + tid * 8) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    // ---- A fragments (+ RMSNorm).  Normalised GEMMs have K = dim (<= 3 k-steps per warp, one poll round, norm weights
    // prefetched); the w2 GEMM (K = ffn) polls in two rounds.
    uint32_t alo[PK_MAXA][4], ahi[PK_MAXA][4];
    {
        const unsigned char* base = reinterpret_cast<const unsigned char*>(pk_a_buf(P, kind, par));
        const bool need_lo = g < M, need_hi = g + 8 < M;
        if (kind != 3) {
            pk_prepoll(pk_a_buf(P, kind, par), K, tag);
            PK_W(1);
            if (M == 16) pk_poll_round<0, PK_MAXA_NORM, true>(base, nst, warp, lane, tag, true, true, alo, ahi);
            else pk_poll_round<0, PK_MAXA_NORM, false>(base, nst, warp, lane, tag, need_lo, need_hi, alo, ahi);
#pragma unroll
            for (int i = PK_MAXA_NORM; i < PK_MAXA; ++i)
#pragma unroll
                for (int p = 0; p < 4; ++p) { alo[i][p] = 0u; ahi[i][p] = 0u; }
        } else {
            pk_prepoll(pk_a_buf(P, kind, par), K, tag);
            PK_W(1);
            if (M == 16) {
                pk_poll_round<0, 4, true>(base, nst, warp, lane, tag, true, true, alo, ahi);
                pk_poll_round<4, 3, true>(base, nst, warp, lane, tag, true, true, alo, ahi);
            } else {
                pk_poll_round<0, 4, false>(base, nst, warp, lane, tag, need_lo, need_hi, alo, ahi);
                pk_poll_round<4, 3, false>(base, nst, warp, lane, tag, need_lo, need_hi, alo, ahi);
            }
        }
    }
    if (stamp) dbg[1] = pk_now();
    PK_W(2);
    if (NORM) asm volatile("cp.async.wait_group 0;" ::: "memory");   // own chunk landed; the CTA barrier below publishes all of them
    if (NORM) {
        float s_lo = 0.f, s_hi = 0.f;
#pragma unroll
        for (int i = 0; i < PK_MAXA_NORM; ++i)
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                float a, b;
                unpack_bf16x2(alo[i][p], a, b); s_lo = fmaf(a, a, s_lo); s_lo = fmaf(b, b, s_lo);
                unpack_bf16x2(ahi[i][p], a, b); s_hi = fmaf(a, a, s_hi); s_hi = fmaf(b, b, s_hi);
            }
        s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 1); s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 2);
        s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 1); s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 2);
        if (t == 0) { sm.ssq[warp * 16 + g] = s_lo; sm.ssq[warp * 16 + g + 8] = s_hi; }
    }

    bool first = true;
    for (int b0 = blk_lo; b0 < blk_hi;) {
        int nb = min(blk_hi - b0, min(PK_NBMAX, PK_NSLOT / nsub));
        if (kind == 2 && nb > 1) nb &= ~1;             // w1/w3 blocks travel in pairs
        const int nunits = nb * nsub;
        // ---- wait for the batch's weight units (one thread per unit); ssq partials become visible
        if (first) PK_W(3);
        if (tid < nunits) { const unsigned int u = cons + tid; pk_mbar_wait(&sm.full[u % PK_NSLOT], (u / PK_NSLOT) & 1); }
        __syncthreads();
        if (first) PK_W(4);
        if (NORM && first) {
            uint4 nwv[PK_MAXA_NORM];
            // row sums of squares: lane i adds row (i & 15) over the 16 warps in order, rsqrt, then rows g / g + 8 by shuffle
            float qs = 0.f;
#pragma unroll
            for (int w = 0; w < PK_WARPS; ++w) qs += sm.ssq[w * 16 + (lane & 15)];
            const float rs = rsqrtf(qs / (float)K + P.eps);
            const float r_lo = __shfl_sync(0xffffffffu, rs, g), r_hi = __shfl_sync(0xffffffffu, rs, g + 8);
            // unconditional definition (a conditionally initialised array would live in local memory); k-steps past the end read step 0
#pragma unroll
            for (int i = 0; i < PK_MAXA_NORM; ++i)
                nwv[i] = *reinterpret_cast<const uint4*>(sm.nw + ((i < nst) ? warp + i * PK_WARPS : 0) * 32 + t * 8);
#pragma unroll
            for (int i = 0; i < PK_MAXA_NORM; ++i) {
                if (i < nst) {
                    const uint32_t wi[4] = {nwv[i].x, nwv[i].y, nwv[i].z, nwv[i].w};
#pragma unroll
                    for (int p = 0; p < 4; ++p) {
                        // RMSNorm.forward (gpt_t2i.py:193-198): (x.float() * rstd).type_as(x) * weight — an fp32 product
                        // rounded to bf16, then a bf16 x bf16 product rounded to bf16 (exact in fp32, so HMUL2.BF16 is the same)
                        const __nv_bfloat162 w2 = *reinterpret_cast<const __nv_bfloat162*>(&wi[p]);
                        float a, b;
                        unpack_bf16x2(alo[i][p], a, b);
                        __nv_bfloat162 x = __floats2bfloat162_rn(a * r_lo, b * r_lo);
                        x = __hmul2(x, w2);
                        alo[i][p] = *reinterpret_cast<uint32_t*>(&x);
                        unpack_bf16x2(ahi[i][p], a, b);
                        x = __floats2bfloat162_rn(a * r_hi, b * r_hi);
                        x = __hmul2(x, w2);
                        ahi[i][p] = *reinterpret_cast<uint32_t*>(&x);
                    }
                }
            }
        }
        if (stamp && first) dbg[2] = pk_now();
        if (first) PK_W(5);
        // ---- MMA: this warp's k-steps against the batch's blocks, B fragments from the ring (32-bit shared addresses).
        // No per-k-step predicates: a k-step past the end has an all-zero A fragment and re-reads the last real k-step's
        // weights (finite), so it contributes exactly 0.
        float acc[PK_NBMAX][4];
#pragma unroll
        for (int j = 0; j < PK_NBMAX; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
        const uint32_t ring_s = pk_smem(sm.ring) + lane * 16;
        if (kind != 3) {   // K = dim: one unit per block (host-checked: dim <= 40 k32-steps), slot of block j = (cons + j) mod 8
            uint32_t soff[PK_NBMAX];
#pragma unroll
            for (int j = 0; j < PK_NBMAX; ++j) soff[j] = ring_s + ((cons + j) & (PK_NSLOT - 1)) * PK_SLOT_BYTES;
#pragma unroll
            for (int i = 0; i < PK_MAXA_NORM; ++i) {
                const uint32_t koff = (uint32_t)min(warp + i * PK_WARPS, KS - 1) * 512u;
#pragma unroll
                for (int j = 0; j < PK_NBMAX; ++j) {
                    if (j < nb) {
                        uint4 wf;
                        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wf.x), "=r"(wf.y), "=r"(wf.z), "=r"(wf.w) : "r"(soff[j] + koff));
                        mma_bf16_16816(acc[j], alo[i][0], ahi[i][0], alo[i][1], ahi[i][1], wf.x, wf.y);
                        mma_bf16_16816(acc[j], alo[i][2], ahi[i][2], alo[i][3], ahi[i][3], wf.z, wf.w);
                    }
                }
            }
        } else {           // K = ffn: up to 3 units per block (nb <= PK_NSLOT / nsub blocks per batch: 2 for XL, 4 for small models)
#pragma unroll
            for (int i = 0; i < PK_MAXA; ++i) {
                const int s = min(warp + i * PK_WARPS, KS - 1);
                const int sub = s / PK_UNIT_KS, so = s - sub * PK_UNIT_KS;
                const uint32_t koff = ring_s + so * 512;
#pragma unroll
                for (int j = 0; j < PK_NBMAX; ++j) {
                    if (j < nb) {
                        uint4 wf;
                        const uint32_t addr = koff + ((cons + j * nsub + sub) & (PK_NSLOT - 1)) * PK_SLOT_BYTES;
                        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(wf.x), "=r"(wf.y), "=r"(wf.z), "=r"(wf.w) : "r"(addr));
                        mma_bf16_16816(acc[j], alo[i][0], ahi[i][0], alo[i][1], ahi[i][1], wf.x, wf.y);
                        mma_bf16_16816(acc[j], alo[i][2], ahi[i][2], alo[i][3], ahi[i][3], wf.z, wf.w);
                    }
                }
            }
        }
        if (first) PK_W(6);
#pragma unroll
        for (int j = 0; j < PK_NBMAX; ++j) {
            if (j < nb) {
                float* rp = sm.red + (size_t)(warp * PK_NBMAX + j) * PK_RED;
                *reinterpret_cast<float2*>(rp + g * 8 + 2 * t) = make_float2(acc[j][0], acc[j][1]);
                *reinterpret_cast<float2*>(rp + 80 + g * 8 + 2 * t) = make_float2(acc[j][2], acc[j][3]);
            }
        }
        if (first) PK_W(7);
        __syncthreads();
        if (stamp && first) dbg[3] = pk_now();
        if (first) PK_W(8);
        cons += nunits;
        if (tid == PK_THREADS - 32) {                  // the batch's slots are free again: keep the stream ahead.  (Issuing after this
            PkStream& st = *sm.st;                     // warp's epilogue instead was measured 2 us per layer SLOWER: the weight stream
            while (!st.c.done && st.issued < cons + PK_NSLOT) pk_stream_issue(P, sm, st);   // falls behind, r2 GPU calls 2 / 3)
        }
        {
            const int bb = b0, cnt = nb;
   // blocks bb .. bb + cnt - 1 are in the reduction buffer
            // ---- fixed-order cross-warp reduction; lane er == 0 of every quad ends up with the 2 x 2 values
            //      (rows eg, eg + 8) x (columns 2 ecp, 2 ecp + 1) of block ej
            const int jj = kind == 2 ? 2 * ej : ej;        // kind 2: the thread sums the w1 block and the w3 block of pair ej
            const bool active = jj < cnt;
            const int e = (er < 2) ? (eg * 8 + 2 * ecp + (er & 1)) : (80 + eg * 8 + 2 * ecp + (er & 1));
            float val = 0.f;
            if (active) {
    #pragma unroll
                for (int w = 0; w < PK_WARPS; ++w) val += sm.red[(size_t)(w * PK_NBMAX + jj) * PK_RED + e];
                if (kind == 2) {
                    float val3 = 0.f;
    #pragma unroll
                    for (int w = 0; w < PK_WARPS; ++w) val3 += sm.red[(size_t)(w * PK_NBMAX + jj + 1) * PK_RED + e];
                    // FeedForward.forward gpt_t2i.py:217: w2(silu(w1 x) * w3 x), every intermediate in bf16
                    val = rnd<bf16>(silu_f(rnd<bf16>(val))) * rnd<bf16>(val3);
                }
            }
            if (first) PK_W(9);
            const int qb = lane & ~3;
            const float v00 = val;
            const float v01 = __shfl_sync(0xffffffffu, val, qb + 1);
            const float v10 = __shfl_sync(0xffffffffu, val, qb + 2);
            const float v11 = __shfl_sync(0xffffffffu, val, qb + 3);
            if (active && er == 0) {
                const int r_lo = eg, r_hi = eg + 8;
                if (kind == 0) {
                    const int n = (bb + ej) * 8 + 2 * ecp;
                    const int sec = n / P.dim, w = n - sec * P.dim;
                    const int head = w >> 6, el = w & 63;
                    float2 cs2 = make_float2(1.f, 0.f);
                    if (sec < 2) cs2 = __ldg(reinterpret_cast<const float2*>(P.rope + ((size_t)pos * 32 + (el >> 1)) * 2));
                    float a0 = rnd<bf16>(v00), a1 = rnd<bf16>(v01), c0 = rnd<bf16>(v10), c1 = rnd<bf16>(v11);
                    if (sec < 2) {   // apply_rotary_emb gpt_t2i.py:522-532 (interleaved pairs, fp32, then cast)
                        const float x0 = a0 * cs2.x - a1 * cs2.y, x1 = a1 * cs2.x + a0 * cs2.y;
                        const float y0 = c0 * cs2.x - c1 * cs2.y, y1 = c1 * cs2.x + c0 * cs2.y;
                        a0 = x0; a1 = x1; c0 = y0; c1 = y1;
                    }
                    const uint32_t p_lo = pk_pack(a0, a1), p_hi = pk_pack(c0, c1);
                    // packets for the attention phase: [sec][b][head][el/8][(el%8)/2]
                    uint2* ob = P.qkv[par];
                    if (r_lo < M) pk_st64(ob + ((((size_t)sec * 16 + r_lo) * P.H + head) * 8 + (el >> 3)) * 4 + ((el & 7) >> 1), p_lo, tag);
                    if (r_hi < M) pk_st64(ob + ((((size_t)sec * 16 + r_hi) * P.H + head) * 8 + (el >> 3)) * 4 + ((el & 7) >> 1), p_hi, tag);
                    if (sec > 0) {   // KVCache.update gpt_t2i.py:227-235 (read by later tokens; ordered by the per-token barrier)
                        bf16* cache = const_cast<bf16*>(sm.kvp[2 * l + (sec - 1)]);
                        if (r_lo < M) *reinterpret_cast<uint32_t*>(cache + (((size_t)r_lo * P.H + head) * P.S + pos) * 64 + el) = p_lo;
                        if (r_hi < M) *reinterpret_cast<uint32_t*>(cache + (((size_t)r_hi * P.H + head) * P.S + pos) * 64 + el) = p_hi;
                    }
                } else if (kind == 1 || kind == 3) {
                    const int n = (bb + ej) * 8 + 2 * ecp;
                    float o0, o1, o2, o3, h0, h1, h2, h3;
                    const uint2 prev = sm.own[(ej & 1) * 32 + ei];
                    unpack_bf16x2(prev.x, h0, h1);
                    unpack_bf16x2(prev.y, h2, h3);
                    o0 = rnd<bf16>(h0 + rnd<bf16>(v00)); o1 = rnd<bf16>(h1 + rnd<bf16>(v01));   // h + drop_path(...) gpt_t2i.py:305-306
                    o2 = rnd<bf16>(h2 + rnd<bf16>(v10)); o3 = rnd<bf16>(h3 + rnd<bf16>(v11));
                    if (kind == 3) {   // gpt_t2i.py:466 — h += cs * ctrl[:, pos - T + 1] ahead of the next layer group
                        const int p = pos - P.T + 1;
                        if (pk_ctrl_next(P, l) != nullptr && p >= 0 && p < P.n_img) {
                            float c0, c1, c2, c3;
                            const uint2 cp = sm.ctl[(ej & 1) * 32 + ei];
                            unpack_bf16x2(cp.x, c0, c1); unpack_bf16x2(cp.y, c2, c3);
                            if (r_lo < M) { o0 = rnd<bf16>(o0 + c0); o1 = rnd<bf16>(o1 + c1); }
                            if (r_hi < M) { o2 = rnd<bf16>(o2 + c2); o3 = rnd<bf16>(o3 + c3); }
                        }
                    }
                    const uint32_t p_lo = pk_pack(o0, o1), p_hi = pk_pack(o2, o3);
                    sm.own[(ej & 1) * 32 + ei] = make_uint2(p_lo, p_hi);
                    const unsigned int otag = kind == 3 ? tag + 1u : tag;
                    pk_st128((kind == 3 ? P.h2[par ^ 1] : P.h1[par]) + pk_a_index(r_lo, n), p_lo, otag, p_hi, otag);
                } else if (kind == 2) {
                    const int n = ((bb >> 1) + ej) * 8 + 2 * ecp;   // activation column
                    pk_st128(P.act[par] + pk_a_index(r_lo, n), pk_pack(v00, v01), tag, pk_pack(v10, v11), tag);
                } else {
                    const int n = (bb + ej) * 8 + 2 * ecp;
                    // logits = output(norm(h)).float()  gpt_t2i.py:469-470 (bf16 head output, then fp32)
                    if (r_lo < M) *reinterpret_cast<float2*>(P.logits + (size_t)r_lo * P.V + n) = make_float2(rnd<bf16>(v00), rnd<bf16>(v01));
                    if (r_hi < M) *reinterpret_cast<float2*>(P.logits + (size_t)r_hi * P.V + n) = make_float2(rnd<bf16>(v10), rnd<bf16>(v11));
                    if (trace_rows != nullptr) {
                        if (r_lo < M) *reinterpret_cast<float2*>(trace_rows + (size_t)r_lo * P.V + n) = make_float2(rnd<bf16>(v00), rnd<bf16>(v01));
                        if (r_hi < M) *reinterpret_cast<float2*>(trace_rows + (size_t)r_hi * P.V + n) = make_float2(rnd<bf16>(v10), rnd<bf16>(v11));
                    }
                }
            }
        }
        if (stamp && first) dbg[4] = pk_now();
        if (first) PK_W(10);
        b0 += nb;
        first = false;
    }
    return cons;
}

// ---------------------------------------------------------------------------------------------------------
// attention phase: the flattened (b, h, key) space is cut into gridDim.x equal ranges (work split: pk_plan.h, computed once
// per token into shared memory — it depends on the context length only, not on the layer)
// ---------------------------------------------------------------------------------------------------------
// publish one segment's merged (m, l, acc[e]) (thread e = head dimension, 64 threads = two warps): the helper's tagged
// partial, or the attention output row (combined with the helpers' partials) as A-fragment packets for the wo GEMM
__device__ __forceinline__ void pk_attn_finalize(const PkParams& P, float Mx, float Ls, float a, const PkSegPlan& sgm, int e, unsigned int tag,
                                                 int par) {
    const int first_cta = sgm.first_cta;
    uint2* pb = P.partial[par] + ((size_t)sgm.bh * P.part_slots) * 66;
    if (!sgm.owner) {
        uint2* mine = pb + (size_t)((int)blockIdx.x - first_cta) * 66;
        pk_st64(mine + 2 + e, __float_as_uint(a), tag);
        if (e == 0) pk_st64(mine, __float_as_uint(Mx), tag);
        if (e == 1) pk_st64(mine + 1, __float_as_uint(Ls), tag);
        return;
    }
    if (sgm.ks > 0) {   // combine the helpers' partials (CTAs first_cta .. blockIdx.x - 1) in index order, then ours
        const int nh = (int)blockIdx.x - first_cta;
        float Mc = -INFINITY, Lc = 0.f, ac = 0.f;
        for (int hI = 0; hI <= nh; ++hI) {
            float mh, lh, ah;
            if (hI < nh) {
                const uint2* src = pb + (size_t)hI * 66;
                uint2 pm, pl, pa;
                unsigned int spins = 0;
                do {
                    pm = pk_ld64(src); pl = pk_ld64(src + 1); pa = pk_ld64(src + 2 + e);
                    if (pm.y == tag && pl.y == tag && pa.y == tag) break;
                    __nanosleep(32);
                    pk_spin_check(spins);
                } while (true);
                mh = __uint_as_float(pm.x); lh = __uint_as_float(pl.x); ah = __uint_as_float(pa.x);
            } else { mh = Mx; lh = Ls; ah = a; }
            const float m_new = fmaxf(Mc, mh);
            const float wa = Mc == -INFINITY ? 0.f : __expf(Mc - m_new);
            const float wb = mh == -INFINITY ? 0.f : __expf(mh - m_new);
            Lc = Lc * wa + lh * wb; ac = ac * wa + ah * wb; Mc = m_new;
        }
        Ls = Lc; a = ac;
    }
    const float o = rnd<bf16>(a / Ls);           // SDPA output in the model dtype
    const float o1 = __shfl_down_sync(0xffffffffu, o, 1);
    if ((e & 1) == 0) pk_st64(P.att[par] + pk_a_index(sgm.b, sgm.hd * 64 + e), pk_pack(o, o1), tag);
}

// Work split: the CTA's flat range is cut into 16 contiguous warp ranges; a warp range touches at most two (b, h) pairs
// ("parts").  Within a part the four 8-lane row slots of the warp take rows k0 + sub + 4 i, the loads of two blocks of 4 rows
// per slot in flight at once; the slots are merged with shuffles and the warp leaves one partial per part in shared memory:
// entry (warp, part) = {-, m, l, -, acc[64]}.
__device__ __forceinline__ void pk_attn_phase(const PkParams& P, int layer, int pos, unsigned int tag, int par, const int* klo, long long* dbg) {
    const PkSmem sm = pk_smem_layout();
    constexpr int EPL = 8, UNR = 4, ENT = 68;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, sub = lane >> 3, cl = lane & 7;
    const PkAttnPlan& pl = *sm.plan;
    if (!pl.active) return;                                // more CTAs than keys (only for tiny contexts)
    const int n = pos + 1;                                 // keys 0 .. pos; key `pos` is the token being decoded (== pl.n)
    const int nseg = pl.nseg, pair_lo = pl.pair_lo;
#ifdef PK_TRACE
    const bool stamp = dbg != nullptr && tid == 0;
#else
    constexpr bool stamp = false;
#endif
    if (stamp) dbg[0] = pk_now();
    const uint2* qkvb = P.qkv[par];
    const bf16* kc = sm.kvp[2 * layer];
    const bf16* vc = sm.kvp[2 * layer + 1];
    float* sc = sm.red;                                    // [PK_WARPS][2][ENT]
    const uint64_t kv_pol = pk_pol_evict_first();

    // q (and, for owner segments, this token's k and v) of every segment -> shared memory, polled in parallel:
    // warp sg, lanes 0-7 q, 8-15 k, 16-23 v (lane & 7 = 16-byte chunk = 4 packets)
    if (warp < nseg && lane < 24) {
        const PkSegPlan& q = pl.seg[warp];
        const int sec = lane >> 3;
        if (sec == 0 || q.owner) {
            const uint2* qp = qkvb + (((size_t)(sec * 16 + q.b) * P.H + q.hd) * 8 + (lane & 7)) * 4;
            uint4 v0, v1;
            unsigned int spins = 0;
            do {
                v0 = pk_ld128(qp); v1 = pk_ld128(qp + 2);
                if (v0.y == tag && v0.w == tag && v1.y == tag && v1.w == tag) break;
                __nanosleep(32);
                pk_spin_check(spins);
            } while (true);
            *reinterpret_cast<uint4*>(sm.qrow + (sec * PK_MAXSEG + warp) * 32 + (lane & 7) * 4) = make_uint4(v0.x, v0.z, v1.x, v1.z);
        }
    }
    if (stamp) dbg[1] = pk_now();
    __syncthreads();                                       // q/k/v rows visible; the scratch aliases the previous phase's reduction buffer

#pragma unroll 1
    for (int part = 0; part < 2; ++part) {
        float* ent = sc + (size_t)(warp * 2 + part) * ENT;
        const int4 pt = *reinterpret_cast<const int4*>(&pl.part[warp][part]);   // {bh, b, k0, k1}
        const int bh = pt.x, b = pt.y, k0 = pt.z, k1 = pt.w;
        if (k0 >= k1) continue;                            // (warp-uniform)
        const int sg = bh - pair_lo;
        float qf[EPL];
        {
            const uint4 qq = *reinterpret_cast<const uint4*>(sm.qrow + sg * 32 + cl * 4);
            unpack_bf16x2(qq.x, qf[0], qf[1]); unpack_bf16x2(qq.y, qf[2], qf[3]);
            unpack_bf16x2(qq.z, qf[4], qf[5]); unpack_bf16x2(qq.w, qf[6], qf[7]);
        }
        const bf16* kbase = kc + ((size_t)bh * P.S) * 64 + cl * EPL;
        const bf16* vbase = vc + ((size_t)bh * P.S) * 64 + cl * EPL;
        const int* mrow = P.emb_mask ? P.emb_mask + (size_t)b * P.T : nullptr;
        float m_run = -INFINITY, l_run = 0.f, acc[EPL];
#pragma unroll
        for (int e = 0; e < EPL; ++e) acc[e] = 0.f;
        // Two blocks of 4 x UNR keys in flight: the loads of block i + 1 are issued before block i is consumed, so the
        // HBM / L2 latency of the K / V rows overlaps the arithmetic (same 64 raw registers as one 8-row block).
        // Rows past the end re-read the part's last row (unconditional loads, weight 0).
        uint4 kA[UNR], vA[UNR], kB[UNR], vB[UNR];
        int mA[UNR], mB[UNR];
        auto load_block = [&](uint4 (&kr)[UNR], uint4 (&vr)[UNR], int (&mk)[UNR], const int rb) {
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int rr = min(rb + sub + 4 * u, k1 - 1);
                kr[u] = pk_ld_kv(kbase + (size_t)rr * 64, kv_pol); vr[u] = pk_ld_kv(vbase + (size_t)rr * 64, kv_pol);
                mk[u] = (mrow != nullptr && rr < P.T) ? __ldg(mrow + rr) : 1;
            }
        };
        // scores of the block's (up to UNR) keys first, ONE running-max update and rescale per block, then the
        // probability-weighted sum: exp(s - m) and 8 FFMA per key (soft-max is invariant to the reference maximum)
        auto use_block = [&](uint4 (&kr)[UNR], uint4 (&vr)[UNR], const int (&mk)[UNR], const int rb) {
            float scu[UNR];
            float mb = -INFINITY;
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int r = rb + sub + 4 * u;
                if (r == n - 1 && r < k1) {   // the newest key / value is this token's: from the QKV packets (owner segments only), not from the cache
                    kr[u] = *reinterpret_cast<const uint4*>(sm.qrow + (1 * PK_MAXSEG + sg) * 32 + cl * 4);
                    vr[u] = *reinterpret_cast<const uint4*>(sm.qrow + (2 * PK_MAXSEG + sg) * 32 + cl * 4);
                }
                float kf[EPL];
                unpack_bf16x2(kr[u].x, kf[0], kf[1]); unpack_bf16x2(kr[u].y, kf[2], kf[3]);
                unpack_bf16x2(kr[u].z, kf[4], kf[5]); unpack_bf16x2(kr[u].w, kf[6], kf[7]);
                float s = 0.f;
#pragma unroll
                for (int e = 0; e < EPL; ++e) s = fmaf(qf[e], kf[e], s);
                s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2); s += __shfl_xor_sync(0xffffffffu, s, 4);
                scu[u] = (r < k1 && mk[u] != 0) ? s * 0.125f : -INFINITY;      // 1/sqrt(head_dim = 64); masked / past-the-end -> weight 0
                mb = fmaxf(mb, scu[u]);
            }
            const float m_new = fmaxf(m_run, mb);
            if (m_new != -INFINITY) {                     // (uniform over the 8 lanes of a row slot)
                const float corr = __expf(m_run - m_new);   // exp(-inf) = 0 on the first block
                l_run *= corr;
#pragma unroll
                for (int e = 0; e < EPL; ++e) acc[e] *= corr;
#pragma unroll
                for (int u = 0; u < UNR; ++u) {
                    float vf[EPL];
                    unpack_bf16x2(vr[u].x, vf[0], vf[1]); unpack_bf16x2(vr[u].y, vf[2], vf[3]);
                    unpack_bf16x2(vr[u].z, vf[4], vf[5]); unpack_bf16x2(vr[u].w, vf[6], vf[7]);
                    const float p = __expf(scu[u] - m_new);
                    l_run += p;
#pragma unroll
                    for (int e = 0; e < EPL; ++e) acc[e] = fmaf(p, vf[e], acc[e]);
                }
                m_run = m_new;
            }
        };
        // Captions are left-padded: the blocks of 4 x UNR keys that lie wholly inside the sequence's leading masked keys come
        // before any key with weight, so they leave (m, l, acc) at its initial state and are not read.  The remaining blocks
        // keep their offsets from k0, so the arithmetic is exactly that of the whole range.
        const int kfirst = k0 + ((max(min(klo[b], k1), k0) - k0) / (4 * UNR)) * (4 * UNR);
        load_block(kA, vA, mA, kfirst);
        for (int rb = kfirst; rb < k1; rb += 8 * UNR) {    // warp-uniform trip count
            load_block(kB, vB, mB, rb + 4 * UNR);
            use_block(kA, vA, mA, rb);
            load_block(kA, vA, mA, rb + 8 * UNR);
            if (rb + 4 * UNR < k1) use_block(kB, vB, mB, rb + 4 * UNR);
        }
        // merge the warp's four row slots (lanes 8 apart), fixed order
#pragma unroll
        for (int o = 8; o <= 16; o <<= 1) {
            const float m_o = __shfl_xor_sync(0xffffffffu, m_run, o);
            const float l_o = __shfl_xor_sync(0xffffffffu, l_run, o);
            const float m_new = fmaxf(m_run, m_o);
            const float wA = m_run == -INFINITY ? 0.f : __expf(m_run - m_new);
            const float wB = m_o == -INFINITY ? 0.f : __expf(m_o - m_new);
            l_run = l_run * wA + l_o * wB;
#pragma unroll
            for (int e = 0; e < EPL; ++e) {
                const float a_o = __shfl_xor_sync(0xffffffffu, acc[e], o);
                acc[e] = acc[e] * wA + a_o * wB;
            }
            m_run = m_new;
        }
        if (sub == 0) {
            if (cl == 0) { ent[1] = m_run; ent[2] = l_run; }
#pragma unroll
            for (int e = 0; e < EPL; ++e) ent[4 + cl * EPL + e] = acc[e];
        }
    }
    __syncthreads();
    if (stamp) dbg[2] = pk_now();
    // ---- finalise: two warps per segment (thread e = dimension) merge the entries of their pair in warp order.  Only the
    // warps whose range touches the pair are visited (a handful, not all 32 entries): this section runs on two warps alone.
    {
        const int sg = warp >> 1, e = tid & 63;
        if (sg < nseg) {
            const PkSegPlan& q = pl.seg[sg];
            const int w0 = q.w0, w1 = q.w1;
            const unsigned int pm = q.part_mask;
            float Mx = -INFINITY;
            for (int w = w0; w <= w1; ++w) Mx = fmaxf(Mx, sc[(w * 2 + (int)((pm >> w) & 1u)) * ENT + 1]);
            float Ls = 0.f, a = 0.f;
            for (int w = w0; w <= w1; ++w) {
                const float* en = sc + (w * 2 + (int)((pm >> w) & 1u)) * ENT;
                const float mi = en[1];
                const float wt = (mi == -INFINITY) ? 0.f : __expf(mi - Mx);
                Ls += en[2] * wt;
                a += en[4 + e] * wt;
            }
            pk_attn_finalize(P, Mx, Ls, a, q, e, tag, par);
        }
    }
    if (stamp) dbg[3] = pk_now();
}

// ---------------------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------------------
// next-token input rows as H2 packets: h = tok_embeddings[tok] (+ cs[b] * ctrl0[b][pos_next - T + 1])  gpt_t2i.py:445,466
__device__ __forceinline__ void pk_write_embedding(const PkParams& P, uint2* h2, unsigned int tag, int row, int tok, int pos_next) {
    const bf16* e = P.tok_emb + (size_t)tok * P.dim;
    const int p = pos_next - P.T + 1;
    const bf16* c = (P.has_ctrl && p >= 0 && p < P.n_img) ? P.ctrl[0] + ((size_t)row * P.n_img + p) * P.dim : nullptr;
    const float s = c ? __ldg(P.cs + row) : 0.f;
    for (int k2 = threadIdx.x; k2 < (P.dim >> 1); k2 += PK_THREADS) {
        float v0, v1;
        unpack_bf16x2(*reinterpret_cast<const uint32_t*>(e + 2 * k2), v0, v1);
        if (c) {
            float c0, c1;
            unpack_bf16x2(*reinterpret_cast<const uint32_t*>(c + 2 * k2), c0, c1);
            v0 = rnd<bf16>(v0 + rnd<bf16>(s * c0)); v1 = rnd<bf16>(v1 + rnd<bf16>(s * c1));
        }
        pk_st64(h2 + pk_a_index(row, 2 * k2), pk_pack(v0, v1), tag);
    }
}

// Out of line: the kernel is one large function under a 128-register cap, and ptxas' allocation for the layer loop shifts with
// unrelated code (a smaller sampler can make the layers slower).  The outlined sampler gets its own register allocation and keeps
// the loop's code independent of it; the GEMM and attention phases stay inlined (measured faster than outlined).
__device__ __noinline__ void pk_sample(const SampleArgs& a, int b) {
    static_assert(SMP_SCRATCH <= PK_SMEM_RED, "the sampler's scratch aliases the reduction buffer");
    sample_body<PK_THREADS>(a, b, pk_smem_raw + PK_SMEM_RING);
}

__global__ void __launch_bounds__(PK_THREADS, 1) pk_decode_kernel(const __grid_constant__ PkParams P) {
    __shared__ int s_tok;
    __shared__ int s_lo[5], s_hi[5];                       // this CTA's block ranges per GEMM kind
    __shared__ int s_klo[16];                              // leading masked caption keys per sequence (pk_attn_phase)
    const PkSmem sm = pk_smem_layout();
    const int tid = threadIdx.x;
    const int G = gridDim.x;
    if (tid == 0) {
        for (int s = 0; s < PK_NSLOT; ++s) pk_mbar_init(&sm.full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid < P.b_eff) {                                   // (host-checked: b_eff <= 16)
        int k = 0;
        if (P.emb_mask != nullptr)
            while (k < P.T && __ldg(P.emb_mask + (size_t)tid * P.T + k) == 0) ++k;
        s_klo[tid] = k;
    }
    __syncthreads();
    if (tid < P.L) {   // (host-checked: L <= PK_MAXL)
        sm.kvp[2 * tid] = P.kc[tid]; sm.kvp[2 * tid + 1] = P.vc[tid];
        sm.nwp[2 * tid] = P.attn_norm[tid]; sm.nwp[2 * tid + 1] = P.ffn_norm[tid];
    }
    if (tid == PK_THREADS - 32) {
        const int* pt = P.part;
        PkStream& st = *sm.st;
        st.lo[0] = pt[0 * (G + 1) + blockIdx.x]; st.hi[0] = pt[0 * (G + 1) + blockIdx.x + 1];
        st.lo[1] = pt[1 * (G + 1) + blockIdx.x]; st.hi[1] = pt[1 * (G + 1) + blockIdx.x + 1];
        st.lo[2] = 2 * pt[2 * (G + 1) + blockIdx.x]; st.hi[2] = 2 * pt[2 * (G + 1) + blockIdx.x + 1];
        st.lo[3] = st.lo[1]; st.hi[3] = st.hi[1];
        st.lo[4] = pt[3 * (G + 1) + blockIdx.x]; st.hi[4] = pt[3 * (G + 1) + blockIdx.x + 1];
        for (int i = 0; i < 5; ++i) { s_lo[i] = st.lo[i]; s_hi[i] = st.hi[i]; }
        st.c.step = 0; st.c.l = 0; st.c.phase = 0; st.c.blk = 0; st.c.sub = 0; st.c.done = P.n_steps <= 1;
        st.issued = 0;
        pk_cursor_skip_empty(P, st, st.c);
        while (!st.c.done && st.issued < PK_NSLOT) pk_stream_issue(P, sm, st);   // ring priming
    }
    __syncthreads();
    unsigned int cons = 0;
    unsigned int gen = P.bar_base;
    const unsigned int tstride = (unsigned int)P.L + 1u;

    for (int step = 0; step < P.n_steps; ++step) {
        const int pos = P.T - 1 + step;                    // logits of this position are sampled now
        const unsigned int tag0 = P.tag_base + (unsigned int)step * tstride + 1u;   // tag(step, 0)
#ifdef PK_TRACE
        const bool dbg_step = P.dbg != nullptr && step == P.dbg_step;
#else
        constexpr bool dbg_step = false;
#endif
        long long* const dbg_cta = P.dbg + (size_t)blockIdx.x * 64;
        if (dbg_step && tid == 0) dbg_cta[0] = pk_now();
        if (P.step_ts != nullptr && blockIdx.x == 0 && tid == 0) P.step_ts[step] = pk_now();
        // ---------------- sampler (+ embedding of the sampled token for position pos + 1) ----------------
        if ((int)blockIdx.x < P.B) {
            SampleArgs a = P.smp;
            a.pos_ptr = nullptr; a.done_ctr = nullptr; a.pos_val = pos; a.step = step; a.ssq_rows = nullptr;
            a.h_out = nullptr; a.tok_buf = nullptr;
            a.dbg_ts = (dbg_step && blockIdx.x == 0) ? dbg_cta + 48 : nullptr;   // (slots 8 .. 47: the five phases of layer 3)
            pk_sample(a, blockIdx.x);
            __syncthreads();
            if (tid == 0) s_tok = P.forced != nullptr ? __ldg(P.forced + (size_t)blockIdx.x * P.forced_ld + step)
                                                      : ld_cg(a.idx_out + (size_t)blockIdx.x * a.tokens_ld + step);
            __syncthreads();
            if (step + 1 < P.n_steps) {
                const int tok = s_tok;
                pk_write_embedding(P, P.h2[0], tag0, blockIdx.x, tok, pos + 1);
                if (P.smp.use_cfg) pk_write_embedding(P, P.h2[0], tag0, blockIdx.x + P.B, tok, pos + 1);
            }
        }
        if (dbg_step && tid == 0) dbg_cta[1] = pk_now();
        if (step + 1 == P.n_steps) break;
        const int p = pos + 1;                             // position being decoded
        // attention work split of this token (context length p + 1): 38 threads fill one record each; the previous
        // token's readers are behind the grid barrier
        if (tid < 2 * PK_WARPS + PK_MAXSEG) pkp_fill(*sm.plan, tid, (int)blockIdx.x, (int)gridDim.x, P.b_eff * P.H, P.H, p + 1);
        __syncthreads();
        // layers 0 .. L-1: phases qkv | attention | wo | w1w3 | w2 ; pseudo-layer L: the head.  One call site per
        // phase kind keeps the loop body small enough for the instruction cache.
        for (int l = 0; l <= P.L; ++l) {
            const int par = l & 1;
            const unsigned int tag = tag0 + (unsigned int)l;
            const int nph = l < P.L ? 5 : 1;
            for (int ph = 0; ph < nph; ++ph) {
                long long* dbg = (dbg_step && l == 3) ? dbg_cta + 8 + 8 * ph : (dbg_step && l == P.L) ? dbg_cta + 56 : nullptr;   // (head: slots 56 .. 60)
                if (l < P.L && ph == 1) { pk_attn_phase(P, l, p, tag, par, s_klo, dbg); continue; }
                const int kind = l == P.L ? 4 : (ph == 0 ? 0 : ph - 1);
                cons = pk_gemm_phase(P, kind, l, p, tag, s_lo[kind], s_hi[kind], cons, dbg,
                              (dbg != nullptr && (int)blockIdx.x == 77 % (int)gridDim.x) ? P.dbg + (size_t)gridDim.x * 64 + (size_t)ph * 256 : nullptr,
                              (kind == 4 && P.trace != nullptr) ? P.trace + (size_t)(step + 1) * P.b_eff * P.V : nullptr);
            }
        }
        if (dbg_step && tid == 0) dbg_cta[3] = pk_now();
        pk_grid_sync(P.bar, gen);                          // logits complete; KV rows of this token ordered
        if (dbg_step && tid == 0) dbg_cta[4] = pk_now();
    }
}
