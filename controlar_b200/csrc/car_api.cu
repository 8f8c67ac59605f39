// car_api.cu — C-ABI entry points (include/controlar_b200.h) and the host-side chaining of the AR kernels.
#include <vector>
#include <cstring>
#include <cstdio>
#include <cstdlib>
#include <cmath>

#include "common.cuh"
#include "gemm_skinny.cuh"
#include "attention.cuh"
#include "sampler.cuh"
#include "misc.cuh"
#include "decode_persistent.cuh"
#include "gemm.h"
#include "t5.cuh"
#include <algorithm>

thread_local std::string g_car_err;
std::atomic<long long> g_car_launches{0};

// ---------------------------------------------------------------------------------------------------------
// structures
// ---------------------------------------------------------------------------------------------------------
struct CarModel : CarOwned {
    CarModelDesc d;
    // borrowed originals
    const void *tok_emb, *norm, *output, *cap_fc1, *cap_fc2, *label_table, *cond_fc1, *cond_fc2, *ctl_fc1[3], *ctl_fc2[3];
    std::vector<const void*> attention_norm, wqkv, wo, ffn_norm, w1, w3, w2;
    // owned GEMM-ready copies: bf16 -> fragment-packed; fp32 -> plain (only w13 is an owned interleaved copy)
    std::vector<void*> g_wqkv, g_wo, g_w13, g_w2;
    void *g_output, *g_cap_fc1, *g_cap_fc2, *g_cond_fc1, *g_cond_fc2, *g_ctl_fc1[3], *g_ctl_fc2[3];
    unsigned int pack_gen = 0;       // bumped by every (re)pack: states refresh their device pointer tables when it moves
    size_t esize() const { return d.dtype == CAR_BF16 ? 2 : 4; }
};

struct CarState : CarOwned {
    CarModel* m;
    int b_eff, S, N, T;
    std::vector<void*> kc, vc;
    const float* rope;
    int* emb_mask = nullptr;       // [b_eff][T] or null (= all ones)
    int* emb_mask_store;
    // decode scratch (b_eff rows)
    void *h, *q, *attn, *act;
    float* logits;       // [b_eff][V]
    int *tok, *pos, *done_ctr, *tickets, *tokens;
    float* attn_part;
    int nsplit;
    // control tokens [3][b_eff][N][d]
    void* ctrl[3];
    bool has_ctrl = false;
    // per-image sampling (car_state_set_row_sampling); empty: the launch's CarSampling and car_prefill's control_strength
    std::vector<CarRowSampling> row_sp;
    std::vector<float> cs_rows;        // [b_eff] host staging of the per-row strengths
    float* cs_dev = nullptr;           // [b_eff] control strength of each row, read by every control add (set by car_prefill)
    SmpRow* smp_rows = nullptr;        // [b_eff] sampling parameters per image read by the sampler (the first B are used)
    // prefill scratch
    void *hP, *qP, *attnP, *actP, *t1, *t2;
    void *qkvP = nullptr, *gP = nullptr, *uP = nullptr;     // dense prefill path (bf16): qkv [rows][3d], w1 / w3 outputs [rows][F]
    bool prefilled = false;
    // decode graph
    cudaGraphExec_t gexec = nullptr;
    cudaStream_t cap_stream = nullptr;   // capture happens on a private stream (the legacy default stream cannot capture)
    // what the captured graph bakes in besides the state's buffers: the per-launch CFG parameters, the noise and the weight packing
    bool graph_ok = false; unsigned int graph_pack_gen = 0;
    float graph_cfg_scale = 0.f; int graph_cfg_interval = 0;
    const float* gnoise = nullptr;
    // persistent decode kernel (decode_persistent.cuh)
    void** pk_ptrs = nullptr;          // device arrays of per-layer pointers [8][L]
    int* pk_part = nullptr;            // [4][grid + 1] block offsets per CTA
    uint2 *pk_h2[2], *pk_h1[2], *pk_att[2], *pk_act[2], *pk_qkv[2], *pk_partial[2];
    int pk_part_slots = 0, pk_grid = 0; bool pk_ok = false; unsigned int pk_ptrs_gen = 0;
    unsigned int* pk_bar = nullptr; unsigned int pk_bar_count = 0, pk_tag_gen = 0;
    size_t pk_pkt_bytes = 0; void* pk_pkt_base = nullptr;
    long long* pk_step_ts = nullptr;   // caller-provided device buffer [N] for per-step timestamps (car_state_set_step_timer) or null
    // wide decode route (bf16, 32 < b_eff <= 64): gemm_wide on the borrowed weights, RMSNorm into xn, one split-K workspace
    bool wide = false;
    void* xn = nullptr;                // [b_eff][dim] normalised rows
    float* wide_part = nullptr; size_t wide_part_bytes = 0;
    int* wide_tickets = nullptr; int wide_n_tickets = 0;
    long long graph_launches = 0;      // launches in one replay of the decode graph

    // Releases the graph and the capture stream; the device memory goes with CarOwned.  It must not read `m`: a layout change
    // destroys the old CarModel (gpt_t2i.setup_caches) before the state built on it is closed.
    ~CarState() {
        if (gexec) cudaGraphExecDestroy(gexec);
        if (cap_stream) cudaStreamDestroy(cap_stream);
    }
};

// Device buffers that other SMs POLL (packet tags, barrier counters) are initialised with SM stores, not cudaMemset: a
// recycled allocation that was zeroed by cudaMemset has been observed to still return the previous owner's packets to strong
// polling loads (tests/test_ar_gpu.py run as a whole failed deterministically until tags were made unique per state).  Two defences: this fill kernel, and tags that are unique process-wide (pk_alloc_tags).
__global__ void fill_u32_kernel(unsigned int* __restrict__ p, unsigned int v, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
static int fill_u32(void* p, unsigned int v, size_t bytes, cudaStream_t st) {
    const size_t n = bytes / 4;
    CAR_LAUNCH(fill_u32_kernel, (unsigned)std::min<size_t>((n + 255) / 256, 1184), 256, 0, st, (unsigned int*)p, v, n);
    return CAR_OK;
}
// Process-wide tag allocator of the persistent decode kernel: every launch gets a fresh, never-reused range of packet tags, so
// a packet left in memory by ANY earlier launch or state can never be mistaken for a current one.  (2^32 tags last for ~10^5
// full-size generate() calls; on wrap-around every state re-zeroes its packet buffers before its next launch.)
static std::atomic<unsigned int> g_pk_tag_next{1u};
static std::atomic<unsigned int> g_pk_tag_gen{0u};
static unsigned int pk_alloc_tags(unsigned int span, unsigned int* gen_out) {
    for (;;) {
        unsigned int base = g_pk_tag_next.load();
        if (base > 0xF0000000u || base + span < base) {            // wrap: new generation, tags restart at 1
            unsigned int expected = base;
            if (g_pk_tag_next.compare_exchange_strong(expected, 1u)) g_pk_tag_gen.fetch_add(1u);
            continue;
        }
        if (g_pk_tag_next.compare_exchange_weak(base, base + span)) { *gen_out = g_pk_tag_gen.load(); return base; }
    }
}

extern "C" const char* car_last_error(void) { return g_car_err.c_str(); }
extern "C" int car_version(void) { return 100; }
extern "C" int64_t car_launch_count(int32_t reset) {
    long long v = g_car_launches.load();
    if (reset) g_car_launches.store(0);
    return v;
}

// ---------------------------------------------------------------------------------------------------------
// skinny GEMM dispatch
// ---------------------------------------------------------------------------------------------------------
template <int NB, int U, bool NORM>
static int launch_skinny_bf16_inst(cudaStream_t st, const bf16* A, int lda, const void* Wp, const bf16* nw, float eps,
                                   int M, int nblk, int K, const EpiParams& ep) {
    const size_t smem = skinny_smem_bytes(K, NB);
    static DevOnce once;
    if (once.first()) {
        CAR_CUDA(cudaFuncSetAttribute(skinny_gemm_bf16<NB, U, NORM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        CAR_CUDA(cudaFuncSetAttribute(skinny_gemm_bf16<NB, U, NORM>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
    if (smem > 200 * 1024) CAR_FAIL(CAR_ERR_UNSUPPORTED, "K too large for the shared-memory activation tile");
    dim3 grid((nblk + NB - 1) / NB, (M + 15) / 16);
    if (grid.y == 1) {   // decode shape: never more than one wave of CTAs; a CTA strides over its column groups
        int occ = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, skinny_gemm_bf16<NB, U, NORM>, SK_THREADS, smem);
        const unsigned cap = (unsigned)sm_count() * (unsigned)std::max(1, std::min(occ, 2));
        if (grid.x > cap) grid.x = cap;
    }
    CAR_LAUNCH_PDL((skinny_gemm_bf16<NB, U, NORM>), grid, dim3(SK_THREADS), smem, st, A, lda, (const uint4*)Wp, nw, eps, K, nblk, ep);
    return CAR_OK;
}

template <int NB, bool NORM>
static int launch_skinny_bf16_u(cudaStream_t st, int U, const bf16* A, int lda, const void* Wp, const bf16* nw, float eps,
                                int M, int nblk, int K, const EpiParams& ep) {
    switch (U) {
        case 5: if (NB <= 2) return launch_skinny_bf16_inst<NB, (NB <= 2 ? 5 : 4), NORM>(st, A, lda, Wp, nw, eps, M, nblk, K, ep);
        case 7: if (NB <= 2) return launch_skinny_bf16_inst<NB, (NB <= 2 ? 7 : 4), NORM>(st, A, lda, Wp, nw, eps, M, nblk, K, ep);
        case 2: if (NB == 8) return launch_skinny_bf16_inst<NB, (NB == 8 ? 2 : 4), NORM>(st, A, lda, Wp, nw, eps, M, nblk, K, ep);
        default: return launch_skinny_bf16_inst<NB, (NB == 8 ? 2 : 4), NORM>(st, A, lda, Wp, nw, eps, M, nblk, K, ep);
    }
}

// W: bf16 -> packed (pack_weight_bf16_kernel) ; fp32 -> plain [N][K].  N = 8*nblk rows of W.
static int launch_skinny(cudaStream_t st, int dtype, const void* A, int lda, const void* W, const void* nw, float eps,
                         int M, int N, int K, EpiParams ep, bool norm) {
    if (K % 64 != 0 || N % 8 != 0) CAR_FAIL(CAR_ERR_UNSUPPORTED, "skinny GEMM needs K % 64 == 0 and N % 8 == 0");
    if (M <= 0) return CAR_OK;
    ep.M = M;
    const int nblk = N / 8;
    if (dtype == CAR_F32) {
        dim3 grid((nblk + 1) / 2, (M + 15) / 16);
        if (norm) CAR_LAUNCH((skinny_gemm_f32<true>), grid, SK_THREADS, 0, st, (const float*)A, lda, (const float*)W, (const float*)nw, eps, K, nblk, ep);
        else CAR_LAUNCH((skinny_gemm_f32<false>), grid, SK_THREADS, 0, st, (const float*)A, lda, (const float*)W, (const float*)nw, eps, K, nblk, ep);
        return CAR_OK;
    }
    const int mtiles = (M + 15) / 16;
    const int nsteps = ((K >> 5) + SK_WARPS - 1) / SK_WARPS;
    int U = 4;
    if (nsteps % 7 == 0) U = 7; else if (nsteps % 5 == 0) U = 5;
    int NB;
    if (mtiles > 1) NB = 4;                       // M-tiled (prefill): maximise reuse of the activation tile
    else {
        // one wave: ceil(nblk / NB) <= SM count where possible (register use makes these 1 CTA / SM kernels)
        const int want = (nblk + sm_count() - 1) / sm_count();
        NB = want > 4 ? 8 : (want > 2 ? 4 : (want > 1 ? 2 : 1));
    }
    if (ep.kind == EPI_SWIGLU && NB == 1) NB = 2;
    if (NB == 8) U = 2; else if (NB * U > 16) U = 4;   // register budget
    const bf16* Ab = (const bf16*)A; const bf16* nwb = (const bf16*)nw;
#define CAR_SK(NB_) (norm ? launch_skinny_bf16_u<NB_, true>(st, U, Ab, lda, W, nwb, eps, M, nblk, K, ep) \
                          : launch_skinny_bf16_u<NB_, false>(st, U, Ab, lda, W, nwb, eps, M, nblk, K, ep))
    switch (NB) {
        case 8: return CAR_SK(8);
        case 4: return CAR_SK(4);
        case 2: return CAR_SK(2);
        default: return CAR_SK(1);
    }
#undef CAR_SK
}

// ---------------------------------------------------------------------------------------------------------
// model
// ---------------------------------------------------------------------------------------------------------
static int pack_one(CarModel* m, cudaStream_t st, const void* w, const void* w3, int N, int K, bool interleave, void** dst,
                    bool allocate) {
    // N = rows of the logical (possibly interleaved) matrix
    if (m->d.dtype == CAR_BF16) {
        if (allocate) CAR_TRY(m->alloc(dst, (size_t)N * K * 2));
        const int nblk = N / 8;
        const long long total = (long long)nblk * (K / 32) * 32;
        const int blocks = (int)std::min<long long>((total + 255) / 256, 4096);
        CAR_LAUNCH(pack_weight_bf16_kernel, blocks, 256, 0, st, (const bf16*)w, (const bf16*)w3, (uint4*)*dst, nblk, K, interleave ? 1 : 0);
    } else {
        if (!interleave) { *dst = const_cast<void*>(w); return CAR_OK; }
        if (allocate) CAR_TRY(m->alloc(dst, (size_t)N * K * 4));
        CAR_LAUNCH(interleave_rows_f32_kernel, 2048, 256, 0, st, (const float*)w, (const float*)w3, (float*)*dst, N / 2, K);
    }
    return CAR_OK;
}

static int model_pack_all(CarModel* m, const CarWeights* w, cudaStream_t st, bool allocate) {
    const CarModelDesc& d = m->d;
    const int L = d.n_layer;
    m->tok_emb = w->tok_embeddings; m->norm = w->norm; m->output = w->output;
    m->cap_fc1 = w->cap_fc1; m->cap_fc2 = w->cap_fc2; m->label_table = w->label_table;
    m->cond_fc1 = w->cond_fc1; m->cond_fc2 = w->cond_fc2;
    for (int j = 0; j < 3; ++j) { m->ctl_fc1[j] = w->ctl_fc1[j]; m->ctl_fc2[j] = w->ctl_fc2[j]; }
    m->attention_norm.assign(w->attention_norm, w->attention_norm + L);
    m->wqkv.assign(w->wqkv, w->wqkv + L); m->wo.assign(w->wo, w->wo + L);
    m->ffn_norm.assign(w->ffn_norm, w->ffn_norm + L);
    m->w1.assign(w->w1, w->w1 + L); m->w3.assign(w->w3, w->w3 + L); m->w2.assign(w->w2, w->w2 + L);
    if (allocate) { m->g_wqkv.assign(L, nullptr); m->g_wo.assign(L, nullptr); m->g_w13.assign(L, nullptr); m->g_w2.assign(L, nullptr); }
    for (int l = 0; l < L; ++l) {
        CAR_TRY(pack_one(m, st, m->wqkv[l], nullptr, 3 * d.dim, d.dim, false, &m->g_wqkv[l], allocate));
        CAR_TRY(pack_one(m, st, m->wo[l], nullptr, d.dim, d.dim, false, &m->g_wo[l], allocate));
        CAR_TRY(pack_one(m, st, m->w1[l], m->w3[l], 2 * d.ffn_dim, d.dim, true, &m->g_w13[l], allocate));
        CAR_TRY(pack_one(m, st, m->w2[l], nullptr, d.dim, d.ffn_dim, false, &m->g_w2[l], allocate));
    }
    ++m->pack_gen;
    CAR_TRY(pack_one(m, st, m->output, nullptr, d.vocab_size, d.dim, false, &m->g_output, allocate));
    if (d.model_type == 1) {
        if (!m->cap_fc1 || !m->cap_fc2) CAR_FAIL(CAR_ERR_ARG, "t2i model needs cap_fc1/cap_fc2");
        CAR_TRY(pack_one(m, st, m->cap_fc1, nullptr, d.dim, d.caption_dim, false, &m->g_cap_fc1, allocate));
        CAR_TRY(pack_one(m, st, m->cap_fc2, nullptr, d.dim, d.dim, false, &m->g_cap_fc2, allocate));
    } else if (!m->label_table) CAR_FAIL(CAR_ERR_ARG, "c2i model needs label_table");
    CAR_TRY(pack_one(m, st, m->cond_fc1, nullptr, d.dim, d.dim, false, &m->g_cond_fc1, allocate));
    CAR_TRY(pack_one(m, st, m->cond_fc2, nullptr, d.dim, d.dim, false, &m->g_cond_fc2, allocate));
    for (int j = 0; j < 3; ++j) {
        CAR_TRY(pack_one(m, st, m->ctl_fc1[j], nullptr, d.dim, d.dim, false, &m->g_ctl_fc1[j], allocate));
        CAR_TRY(pack_one(m, st, m->ctl_fc2[j], nullptr, d.dim, d.dim, false, &m->g_ctl_fc2[j], allocate));
    }
    return CAR_OK;
}

extern "C" int car_model_create(const CarModelDesc* desc, const CarWeights* w, void* stream, CarModel** out) {
    if (!desc || !w || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    const CarModelDesc& d = *desc;
    if (d.dtype != CAR_BF16 && d.dtype != CAR_F32) CAR_FAIL(CAR_ERR_ARG, "dtype must be CAR_BF16 or CAR_F32");
    if (d.n_head <= 0 || d.dim != d.n_head * 64) CAR_FAIL(CAR_ERR_UNSUPPORTED, "head_dim must be 64");
    if (d.n_layer <= 0 || d.n_layer % 3 != 0) CAR_FAIL(CAR_ERR_UNSUPPORTED, "n_layer must be a multiple of 3 (gpt_t2i.py:320,457)");
    if (d.dim % 64 || d.ffn_dim % 64 || d.vocab_size % 8) CAR_FAIL(CAR_ERR_UNSUPPORTED, "dim, ffn_dim must be multiples of 64; vocab of 8");
    if (d.model_type == 1 && d.caption_dim % 64) CAR_FAIL(CAR_ERR_UNSUPPORTED, "caption_dim must be a multiple of 64");
    if (d.cls_token_num < 1 || d.cls_token_num > 256) CAR_FAIL(CAR_ERR_UNSUPPORTED, "cls_token_num must be in [1,256]");
    CarModel* m = new CarModel();
    m->d = d;
    int r = model_pack_all(m, w, (cudaStream_t)stream, true);
    if (r != CAR_OK) { delete m; return r; }
    *out = m;
    return CAR_OK;
}

extern "C" int car_model_repack(CarModel* m, const CarWeights* w, void* stream) {
    if (!m || !w) CAR_FAIL(CAR_ERR_ARG, "null argument");
    return model_pack_all(m, w, (cudaStream_t)stream, false);
}

extern "C" int car_model_destroy(CarModel* m) {
    delete m;
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// state
// ---------------------------------------------------------------------------------------------------------
// block ownership of the persistent decode kernel: counts per CTA balanced on streamed bytes per token
static void pk_partition(const CarModelDesc& d, int G, std::vector<int>& table) {
    const int nQ = 3 * d.dim / 8, nD = d.dim / 8, nP = d.ffn_dim / 8, nH = d.vocab_size / 8;
    const double L = d.n_layer;
    const double wQ = L * 16.0 * d.dim, wD = L * 16.0 * (d.dim + d.ffn_dim), wP = L * 32.0 * d.dim, wH = 16.0 * d.dim;
    std::vector<double> load(G, 0.0);
    std::vector<int> cQ(G, 0), cD(G, 0), cP(G, 0), cH(G, 0);
    for (int i = 0; i < nD; ++i) { cD[i % G] += 1; load[i % G] += wD; }
    auto spread = [&](int n, double w, std::vector<int>& cnt) {
        for (int i = 0; i < n; ++i) {
            int best = 0;
            for (int c = 1; c < G; ++c) if (load[c] < load[best] - 1e-9) best = c;
            cnt[best] += 1; load[best] += w;
        }
    };
    spread(nP, wP, cP); spread(nQ, wQ, cQ);
    (void)wH;
    for (int i = 0; i < nH; ++i) cH[i % G] += 1;      // the head ends in a grid barrier: its latency, not its bytes, is what counts
    table.assign(4 * (G + 1), 0);
    const std::vector<int>* cs[4] = {&cQ, &cD, &cP, &cH};
    for (int k = 0; k < 4; ++k)
        for (int c = 0; c < G; ++c) table[k * (G + 1) + c + 1] = table[k * (G + 1) + c] + (*cs[k])[c];
}

// per-layer device pointers of the persistent kernel: packed weights (library-owned), norm weights (borrowed from the module: they
// move when a parameter tensor is replaced, hence the refresh in launch_pk after car_model_repack), KV caches
static std::vector<const void*> pk_pointer_table(const CarState* s) {
    const int L = s->m->d.n_layer;
    std::vector<const void*> hp(8 * L);
    for (int l = 0; l < L; ++l) {
        hp[0 * L + l] = s->m->g_wqkv[l]; hp[1 * L + l] = s->m->g_wo[l]; hp[2 * L + l] = s->m->g_w13[l]; hp[3 * L + l] = s->m->g_w2[l];
        hp[4 * L + l] = s->m->attention_norm[l]; hp[5 * L + l] = s->m->ffn_norm[l]; hp[6 * L + l] = s->kc[l]; hp[7 * L + l] = s->vc[l];
    }
    return hp;
}

static int pk_state_setup(CarState* s) {
    const CarModelDesc& d = s->m->d;
    const int G = sm_count(), L = d.n_layer;
    s->pk_grid = G;
    const int nbh = s->b_eff * d.n_head;
    // shapes the kernel is instantiated for (else car_generate falls back to the per-kernel graph chain)
    s->pk_ok = s->b_eff <= 16 && d.dim % 32 == 0 && d.dim <= 16 * 3 * 32 && d.dim <= PK_UNIT_KS * 32 /* one ring unit per block of the K = dim GEMMs */ && d.ffn_dim % 32 == 0 && d.ffn_dim <= 16 * 7 * 32 &&
               d.dim / 8 <= 2 * G && d.vocab_size <= 16384 && d.ffn_dim % 8 == 0 && nbh <= 5 * G &&
               2 * ((d.ffn_dim / 32 + PK_UNIT_KS - 1) / PK_UNIT_KS) <= PK_NSLOT && L <= PK_MAXL;
    if (!s->pk_ok) return CAR_OK;
    std::vector<const void*> hp = pk_pointer_table(s);
    std::vector<int> table;
    pk_partition(d, G, table);
    s->pk_part_slots = G / std::max(1, nbh) + 3;
    // packet buffers: two parities of H2, H1, ATT (K = dim), ACT (K = ffn), QKV, PARTIAL; one allocation, zeroed (tag 0 = never)
    const size_t a_d = (size_t)(d.dim / 32) * 2048, a_f = (size_t)(d.ffn_dim / 32) * 2048;
    const size_t qkv_b = (size_t)3 * 16 * d.n_head * 8 * 4 * 8, part_b = (size_t)nbh * s->pk_part_slots * 66 * 8;
    const size_t total = 2 * (3 * a_d + a_f + qkv_b + part_b);
    CAR_TRY(s->alloc(&s->pk_ptrs, hp.size() * sizeof(void*)));
    CAR_TRY(s->alloc(&s->pk_part, table.size() * sizeof(int)));
    CAR_TRY(s->alloc(&s->pk_bar, 64));
    CAR_TRY(s->alloc(&s->pk_pkt_base, total));
    s->pk_pkt_bytes = total;
    unsigned char* q = (unsigned char*)s->pk_pkt_base;
    for (int par = 0; par < 2; ++par) {
        s->pk_h2[par] = (uint2*)q; q += a_d; s->pk_h1[par] = (uint2*)q; q += a_d; s->pk_att[par] = (uint2*)q; q += a_d;
        s->pk_act[par] = (uint2*)q; q += a_f; s->pk_qkv[par] = (uint2*)q; q += qkv_b; s->pk_partial[par] = (uint2*)q; q += part_b;
    }
    CAR_CUDA(cudaMemcpy(s->pk_ptrs, hp.data(), hp.size() * sizeof(void*), cudaMemcpyHostToDevice));
    s->pk_ptrs_gen = s->m->pack_gen;
    CAR_CUDA(cudaMemcpy(s->pk_part, table.data(), table.size() * sizeof(int), cudaMemcpyHostToDevice));
    CAR_TRY(fill_u32(s->pk_bar, 0u, 64, nullptr));
    CAR_TRY(fill_u32(s->pk_pkt_base, 0u, total, nullptr));
    CAR_CUDA(cudaStreamSynchronize(nullptr));          // state creation is rare; the caller's stream may not be ordered after the NULL stream
    return CAR_OK;
}

// the wide decode route: every decode-step GEMM through gemm_wide (gemm.h) with one workspace sized for the largest of them.  Taken
// above 32 rows: on an H100 at GPT-XL it is faster than the skinny chain at 50 and 64 rows and slower at 32, where its separate
// RMSNorm launches and split-K partials cost more than the second weight pass of the chain's two 16-row tiles (DESIGN §4.2).
static bool wide_route(const CarModelDesc& d, int b_eff) { return d.dtype == CAR_BF16 && b_eff > 32 && b_eff <= 64; }
static int wide_state_setup(CarState* s) {
    const CarModelDesc& d = s->m->d;
    const int M = s->b_eff;
    const WidePlan plans[5] = {gemm_wide_plan(M, 3 * d.dim, d.dim, false), gemm_wide_plan(M, d.dim, d.dim, false),
                               gemm_wide_plan(M, d.ffn_dim, d.dim, true), gemm_wide_plan(M, d.dim, d.ffn_dim, false),
                               gemm_wide_plan(M, d.vocab_size, d.dim, false)};
    for (const WidePlan& w : plans) {
        s->wide_part_bytes = std::max(s->wide_part_bytes, w.part_bytes);
        s->wide_n_tickets = std::max(s->wide_n_tickets, w.tiles);
    }
    CAR_TRY(s->alloc(&s->xn, (size_t)M * d.dim * 2));
    CAR_TRY(s->alloc(&s->wide_part, s->wide_part_bytes));
    CAR_TRY(s->alloc(&s->wide_tickets, (size_t)s->wide_n_tickets * 4));
    CAR_TRY(fill_u32(s->wide_tickets, 0u, (size_t)s->wide_n_tickets * 4, nullptr));
    CAR_CUDA(cudaStreamSynchronize(nullptr));
    s->wide = true;
    return CAR_OK;
}

// key splits of the decode attention: about four CTAs per SM over all (b, h) rows, at most 16 per row
static int attn_decode_nsplit(int bh) { return std::max(1, std::min(16, (4 * sm_count() + bh - 1) / bh)); }

// everything car_state_create allocates and initialises; on failure the caller deletes the half-built state
static int state_init(CarState* s, void* const* k_cache, void* const* v_cache) {
    const CarModelDesc& d = s->m->d;
    const int b_eff = s->b_eff;
    s->kc.assign(k_cache, k_cache + d.n_layer); s->vc.assign(v_cache, v_cache + d.n_layer);
    CAR_CUDA(cudaStreamCreateWithFlags(&s->cap_stream, cudaStreamNonBlocking));
    const size_t es = s->m->esize();
    const size_t dd = d.dim, F = d.ffn_dim, V = d.vocab_size;
    const size_t MP = (size_t)b_eff * s->T, MC = (size_t)b_eff * s->N;
    s->nsplit = attn_decode_nsplit(b_eff * d.n_head);
    CAR_TRY(s->alloc(&s->h, b_eff * dd * es)); CAR_TRY(s->alloc(&s->q, b_eff * dd * es));
    CAR_TRY(s->alloc(&s->attn, b_eff * dd * es)); CAR_TRY(s->alloc(&s->act, b_eff * F * es));
    CAR_TRY(s->alloc(&s->logits, b_eff * V * 4)); CAR_TRY(s->alloc(&s->tok, b_eff * 4)); CAR_TRY(s->alloc(&s->pos, 4 * 4));
    CAR_TRY(s->alloc(&s->tickets, (size_t)b_eff * d.n_head * 4));
    CAR_TRY(s->alloc(&s->tokens, (size_t)b_eff * s->N * 4));
    CAR_TRY(s->alloc(&s->attn_part, (size_t)b_eff * d.n_head * s->nsplit * AD_PART * 4));
    for (int j = 0; j < 3; ++j) CAR_TRY(s->alloc(&s->ctrl[j], MC * dd * es));
    CAR_TRY(s->alloc(&s->hP, MP * dd * es)); CAR_TRY(s->alloc(&s->qP, MP * dd * es));
    CAR_TRY(s->alloc(&s->attnP, MP * dd * es)); CAR_TRY(s->alloc(&s->actP, MP * F * es));
    CAR_TRY(s->alloc(&s->t1, std::max(MC, MP) * dd * es)); CAR_TRY(s->alloc(&s->t2, std::max(MC, MP) * dd * es));
    if (d.dtype == CAR_BF16) {
        CAR_TRY(s->alloc(&s->qkvP, MP * 3 * dd * es)); CAR_TRY(s->alloc(&s->gP, MP * F * es)); CAR_TRY(s->alloc(&s->uP, MP * F * es));
    }
    CAR_TRY(s->alloc(&s->emb_mask_store, MP * 4));
    CAR_TRY(s->alloc(&s->cs_dev, (size_t)b_eff * 4)); CAR_TRY(s->alloc(&s->smp_rows, (size_t)b_eff * sizeof(SmpRow)));
    s->cs_rows.assign(b_eff, 1.f);
    CAR_CUDA(cudaMemcpy(s->cs_dev, s->cs_rows.data(), (size_t)b_eff * 4, cudaMemcpyHostToDevice));
    CAR_CUDA(cudaMemset(s->tickets, 0, (size_t)b_eff * d.n_head * 4));
    CAR_CUDA(cudaMemset(s->pos, 0, 16));
    s->done_ctr = s->pos + 1;
    s->pk_tag_gen = g_pk_tag_gen.load();
    if (wide_route(d, b_eff)) CAR_TRY(wide_state_setup(s));
    return d.dtype == CAR_BF16 ? pk_state_setup(s) : CAR_OK;     // persistent decode kernel resources (bf16 only)
}

extern "C" int car_state_create(CarModel* m, int32_t b_eff, int32_t S, int32_t N, void* const* k_cache, void* const* v_cache,
                                const float* rope_table, CarState** out) {
    if (!m || !k_cache || !v_cache || !rope_table || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (b_eff <= 0 || N <= 0) CAR_FAIL(CAR_ERR_ARG, "need b_eff > 0, N > 0");
    const CarModelDesc& d = m->d;
    if (S < d.cls_token_num + N) CAR_FAIL(CAR_ERR_ARG, "need S >= T + N");
    if (N > d.block_size) CAR_FAIL(CAR_ERR_ARG, "N exceeds block_size (RoPE table rows)");
    CarState* s = new CarState();
    s->m = m; s->b_eff = b_eff; s->S = S; s->N = N; s->T = d.cls_token_num; s->rope = rope_table;
    const int rc = state_init(s, k_cache, v_cache);
    if (rc != CAR_OK) { delete s; return rc; }
    *out = s;
    return CAR_OK;
}

extern "C" int car_state_set_emb_mask(CarState* s, const int32_t* emb_mask_dev, void* stream) {
    if (!s) CAR_FAIL(CAR_ERR_ARG, "null state");
    if (!emb_mask_dev) { s->emb_mask = nullptr; return CAR_OK; }
    CAR_CUDA(cudaMemcpyAsync(s->emb_mask_store, emb_mask_dev, (size_t)s->b_eff * s->T * 4, cudaMemcpyDeviceToDevice,
                             (cudaStream_t)stream));
    s->emb_mask = s->emb_mask_store;
    return CAR_OK;
}

// host checks of per-image parameters that arrive from outside the library
static int check_rows(const CarRowSampling* rows, int B) {
    for (int b = 0; b < B; ++b) {
        const CarRowSampling& r = rows[b];
        if (!(r.temperature > 0.f) || !std::isfinite(r.temperature)) CAR_FAIL(CAR_ERR_ARG, "row " + std::to_string(b) + ": need temperature > 0");
        if (!(r.top_p > 0.f && r.top_p <= 1.f)) CAR_FAIL(CAR_ERR_ARG, "row " + std::to_string(b) + ": need 0 < top_p <= 1");
        if (r.top_k < 0) CAR_FAIL(CAR_ERR_ARG, "row " + std::to_string(b) + ": need top_k >= 0");
        if (!std::isfinite(r.control_strength)) CAR_FAIL(CAR_ERR_ARG, "row " + std::to_string(b) + ": control_strength must be finite");
    }
    return CAR_OK;
}

extern "C" int car_state_set_row_sampling(CarState* s, const CarRowSampling* rows, int32_t B) {
    if (!s) CAR_FAIL(CAR_ERR_ARG, "null state");
    if (!rows) { s->row_sp.clear(); return CAR_OK; }
    if (B <= 0 || (B != s->b_eff && 2 * B != s->b_eff)) CAR_FAIL(CAR_ERR_ARG, "B must be the state's b_eff, or b_eff / 2 with CFG");
    CAR_TRY(check_rows(rows, B));
    s->row_sp.assign(rows, rows + B);
    return CAR_OK;
}

extern "C" int car_state_set_step_timer(CarState* s, int64_t* step_ns_dev) {
    if (!s) CAR_FAIL(CAR_ERR_ARG, "null state");
    s->pk_step_ts = (long long*)step_ns_dev;
    return CAR_OK;
}

extern "C" int car_state_destroy(CarState* s) {
    delete s;
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// kernel chains
// ---------------------------------------------------------------------------------------------------------
// The three attention launches (attention.cuh), shared by the model chains and by car_op_attn_decode / car_op_attn_prefill so that
// the unit tests exercise exactly the launch the product makes.  Caches [B, H, S, 64]; emb_mask [B][mask_ld] gates key columns < Tpre.
static int launch_attn_decode(int dtype, cudaStream_t st, const void* q, const void* kc, const void* vc, const int* emb_mask, int mask_ld,
                              const int* pos, int B, int H, int S, int Tpre, int nsplit, float* part, int* tickets, void* out) {
    const dim3 grid(B * H, nsplit);
    if (dtype == CAR_BF16)
        CAR_LAUNCH_PDL((attn_decode_kernel<bf16>), grid, dim3(AD_THREADS), 0, st, (const bf16*)q, (const bf16*)kc, (const bf16*)vc,
                       emb_mask, mask_ld, pos, H, S, Tpre, nsplit, part, tickets, (bf16*)out);
    else
        CAR_LAUNCH_PDL((attn_decode_kernel<float>), grid, dim3(AD_THREADS), 0, st, (const float*)q, (const float*)kc, (const float*)vc,
                       emb_mask, mask_ld, pos, H, S, Tpre, nsplit, part, tickets, (float*)out);
    return CAR_OK;
}

static int launch_attn_prefill(int dtype, cudaStream_t st, const void* q, const void* kc, const void* vc, const int* emb_mask,
                               int mask_ld, int B, int H, int S, int Tq, int Tpre, void* out) {
    const unsigned blocks = (unsigned)(((long long)B * H * Tq + 3) / 4);
    if (dtype == CAR_BF16)
        CAR_LAUNCH((attn_prefill_kernel<bf16>), blocks, 128, 0, st, (const bf16*)q, (const bf16*)kc, (const bf16*)vc, emb_mask, mask_ld,
                   B, H, S, Tq, Tpre, (bf16*)out);
    else
        CAR_LAUNCH((attn_prefill_kernel<float>), blocks, 128, 0, st, (const float*)q, (const float*)kc, (const float*)vc, emb_mask, mask_ld,
                   B, H, S, Tq, Tpre, (float*)out);
    return CAR_OK;
}

static int launch_attn_prefill_mma(cudaStream_t st, const void* q, const void* kc, const void* vc, const int* emb_mask, int mask_ld,
                                   int B, int H, int S, int Tq, int Tpre, void* out) {
    CAR_LAUNCH(attn_prefill_mma_kernel, dim3((Tq + 63) / 64, H, B), 128, 0, st, (const bf16*)q, (const bf16*)kc, (const bf16*)vc,
               emb_mask, mask_ld, H, S, Tq, Tpre, (bf16*)out);
    return CAR_OK;
}

static EpiParams epi_base(int kind) {
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.kind = kind;
    ep.rpb = 1;
    return ep;
}

// ---------------------------------------------------------------------------------------------------------
// dense (M >= 128 rows) bf16 path of the prefill: tiled tensor-core GEMM on the ORIGINAL [N][K] weights
// ---------------------------------------------------------------------------------------------------------
static int dense_linear(cudaStream_t st, const void* A, int lda, const void* W, int M, int N, int K, int act, const void* resid, int ldr,
                        void* out, int ldo) {
    DenseP p = dp_plain((const bf16*)A, lda, (const bf16*)W, K, M, N, K, out, ldo);
    p.act = act; p.resid = (const bf16*)resid; p.ldr = ldr;
    return gemm(st, p);
}
static bool use_dense(const CarState* s, int rows) { return s->m->d.dtype == CAR_BF16 && rows >= 64 && s->qkvP != nullptr; }

// one prefill block on the dense path (same rounding points as the skinny chain)
static int enqueue_block_dense(CarState* s, int l, cudaStream_t st) {
    CarModel* m = s->m;
    const CarModelDesc& d = m->d;
    const int dim = d.dim, F = d.ffn_dim, rows = s->b_eff * s->T;
    CAR_LAUNCH((rmsnorm_rows_kernel<bf16>), rows, 256, 0, st, (const bf16*)s->hP, (const bf16*)m->attention_norm[l], (bf16*)s->t1, dim, d.norm_eps);
    CAR_TRY(dense_linear(st, s->t1, dim, m->wqkv[l], rows, 3 * dim, dim, ACT_NONE, nullptr, 0, s->qkvP, 3 * dim));
    CAR_LAUNCH(rope_kv_write_kernel, sm_count() * 8, 256, 0, st, (const bf16*)s->qkvP, s->rope, (bf16*)s->qP, (bf16*)s->kc[l], (bf16*)s->vc[l], rows, s->T, dim,
               d.n_head, s->S);
    // prefix attention on the tensor cores (attention.cuh): 64 query rows per CTA
    CAR_TRY(launch_attn_prefill_mma(st, s->qP, s->kc[l], s->vc[l], s->emb_mask, s->T, s->b_eff, d.n_head, s->S, s->T, s->T, s->attnP));
    CAR_TRY(dense_linear(st, s->attnP, dim, m->wo[l], rows, dim, dim, ACT_NONE, s->hP, dim, s->hP, dim));
    CAR_LAUNCH((rmsnorm_rows_kernel<bf16>), rows, 256, 0, st, (const bf16*)s->hP, (const bf16*)m->ffn_norm[l], (bf16*)s->t1, dim, d.norm_eps);
    CAR_TRY(dense_linear(st, s->t1, dim, m->w1[l], rows, F, dim, ACT_NONE, nullptr, 0, s->gP, F));
    CAR_TRY(dense_linear(st, s->t1, dim, m->w3[l], rows, F, dim, ACT_NONE, nullptr, 0, s->uP, F));
    CAR_LAUNCH(swiglu_kernel, sm_count() * 8, 256, 0, st, (const bf16*)s->gP, (const bf16*)s->uP, (bf16*)s->actP, (long long)rows * F);
    CAR_TRY(dense_linear(st, s->actP, F, m->w2[l], rows, dim, F, ACT_NONE, s->hP, dim, s->hP, dim));
    return CAR_OK;
}

// one GEMM of a block or of the head, RMSNorm `nw` in front when given.  Decode steps of the wide route: rmsnorm_rows_kernel then
// gemm_wide on the borrowed [N][K] weights W (and W3 = w3 for SwiGLU); otherwise the skinny kernel on the packed copy Wp (N rows,
// 2N when W3 is given: w1 / w3 interleaved) with the norm fused.
static int block_linear(CarState* s, bool decode, cudaStream_t st, const void* A, int lda, const void* Wp, const void* W, const void* W3,
                        const void* nw, int rows, int N, int K, const EpiParams& ep) {
    const CarModelDesc& d = s->m->d;
    if (decode && s->wide) {
        if (nw) {
            CAR_LAUNCH((rmsnorm_rows_kernel<bf16>), rows, 256, 0, st, (const bf16*)A, (const bf16*)nw, (bf16*)s->xn, K, d.norm_eps);
            A = s->xn; lda = K;
        }
        return gemm_wide(st, (const bf16*)A, lda, (const bf16*)W, (const bf16*)W3, rows, N, K, ep, s->wide_part, s->wide_part_bytes,
                         s->wide_tickets, s->wide_n_tickets);
    }
    return launch_skinny(st, d.dtype, A, lda, Wp, nw, nw ? d.norm_eps : 0.f, rows, W3 ? 2 * N : N, K, ep, nw != nullptr);
}

// one transformer block on `rows` rows; decode (rpb = 1, pos from device scalar) or prefill (rpb = T, pos = t)
static int enqueue_block(CarState* s, int l, bool decode, cudaStream_t st) {
    CarModel* m = s->m;
    const CarModelDesc& d = m->d;
    const int dt = d.dtype, dim = d.dim, F = d.ffn_dim;
    const int rows = decode ? s->b_eff : s->b_eff * s->T;
    void* h = decode ? s->h : s->hP;
    void* q = decode ? s->q : s->qP;
    void* attn = decode ? s->attn : s->attnP;
    void* act = decode ? s->act : s->actP;
    const int rpb = decode ? 1 : s->T;
    const int* posp = decode ? s->pos : nullptr;

    EpiParams e1 = epi_base(EPI_QKV);
    e1.rpb = rpb; e1.pos_ptr = posp; e1.rope = s->rope; e1.kc = s->kc[l]; e1.vc = s->vc[l]; e1.q = q; e1.S = s->S;
    e1.H = d.n_head; e1.d = dim;
    CAR_TRY(block_linear(s, decode, st, h, dim, m->g_wqkv[l], m->wqkv[l], nullptr, m->attention_norm[l], rows, 3 * dim, dim, e1));

    if (decode)
        CAR_TRY(launch_attn_decode(dt, st, s->q, s->kc[l], s->vc[l], s->emb_mask, s->T, s->pos, s->b_eff, d.n_head, s->S, s->T, s->nsplit,
                                   s->attn_part, s->tickets, s->attn));
    else
        CAR_TRY(launch_attn_prefill(dt, st, s->qP, s->kc[l], s->vc[l], s->emb_mask, s->T, s->b_eff, d.n_head, s->S, s->T, s->T, s->attnP));

    EpiParams e2 = epi_base(EPI_RESID);
    e2.rpb = rpb; e2.pos_ptr = posp; e2.h = h; e2.ldh = dim;
    CAR_TRY(block_linear(s, decode, st, attn, dim, m->g_wo[l], m->wo[l], nullptr, nullptr, rows, dim, dim, e2));

    EpiParams e3 = epi_base(EPI_SWIGLU);
    e3.rpb = rpb; e3.out = act; e3.ldo = F;
    CAR_TRY(block_linear(s, decode, st, h, dim, m->g_w13[l], m->w1[l], m->w3[l], m->ffn_norm[l], rows, F, dim, e3));

    EpiParams e4 = epi_base(EPI_RESID);
    e4.rpb = rpb; e4.pos_ptr = posp; e4.h = h; e4.ldh = dim;
    const int step3 = d.n_layer / 3;
    if (decode && s->has_ctrl && (l + 1) < d.n_layer && (l + 1) % step3 == 0) {
        // control add of the NEXT layer group fused here (gpt_t2i.py:466)
        e4.ctrl = s->ctrl[(l + 1) / step3]; e4.n_img = s->N; e4.T = s->T; e4.cs = s->cs_dev;
    }
    return block_linear(s, decode, st, act, F, m->g_w2[l], m->w2[l], nullptr, nullptr, rows, dim, F, e4);
}

static int enqueue_head(CarState* s, const void* hrows, int rows, float* logits, bool decode, cudaStream_t st) {
    CarModel* m = s->m;
    const CarModelDesc& d = m->d;
    EpiParams e = epi_base(EPI_LOGITS);
    e.logits = logits; e.ldl = d.vocab_size;
    return block_linear(s, decode, st, hrows, d.dim, m->g_output, m->output, nullptr, m->norm, rows, d.vocab_size, d.dim, e);
}

static int enqueue_decode_layers(CarState* s, float* logits, cudaStream_t st) {
    for (int l = 0; l < s->m->d.n_layer; ++l) CAR_TRY(enqueue_block(s, l, true, st));
    return enqueue_head(s, s->h, s->b_eff, logits, true, st);
}

static int enqueue_mlp(CarState* s, const void* x, int rows, int K, const void* fc1, const void* fc2, const void* fc1_plain,
                       const void* fc2_plain, void* tmp, void* out, cudaStream_t st) {
    const CarModelDesc& d = s->m->d;
    if (use_dense(s, rows) && K % 8 == 0) {      // MLP.forward gpt_t2i.py:165-181: fc2(gelu_tanh(fc1 x)), bias-free
        CAR_TRY(dense_linear(st, x, K, fc1_plain, rows, d.dim, K, ACT_GELU_TANH, nullptr, 0, tmp, d.dim));
        return dense_linear(st, tmp, d.dim, fc2_plain, rows, d.dim, d.dim, ACT_NONE, nullptr, 0, out, d.dim);
    }
    EpiParams a = epi_base(EPI_STORE);
    a.out = tmp; a.ldo = d.dim; a.act = 1;
    CAR_TRY(launch_skinny(st, d.dtype, x, K, fc1, nullptr, 0.f, rows, d.dim, K, a, false));
    EpiParams b = epi_base(EPI_STORE);
    b.out = out; b.ldo = d.dim; b.act = 0;
    return launch_skinny(st, d.dtype, tmp, d.dim, fc2, nullptr, 0.f, rows, d.dim, d.dim, b, false);
}

template <typename T>
static int prefill_small_kernels(CarState* s, int l, cudaStream_t st) {
    const CarModelDesc& d = s->m->d;
    const int step3 = d.n_layer / 3;
    if (s->has_ctrl && l % step3 == 0)
        CAR_LAUNCH((prefill_ctrl_add_kernel<T>), s->b_eff, 256, 0, st, (T*)s->hP, (const T*)s->ctrl[l / step3], s->T, s->N, d.dim, s->cs_dev);
    return CAR_OK;
}

extern "C" int car_prefill(CarState* s, const void* cond, const void* condition, float control_strength, float* logits_out,
                           int32_t all_rows, void* stream) {
    if (!s || !cond) CAR_FAIL(CAR_ERR_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    CarModel* m = s->m;
    const CarModelDesc& d = m->d;
    const int rows = s->b_eff * s->T;
    // the control strength of every row, read by each control add of this prefill and of the decode that follows: image r mod B's
    // when per-image sampling is set (an unconditional row takes its partner's), else control_strength
    for (int r = 0; r < s->b_eff; ++r)
        s->cs_rows[r] = s->row_sp.empty() ? control_strength : s->row_sp[r % s->row_sp.size()].control_strength;
    CAR_CUDA(cudaMemcpyAsync(s->cs_dev, s->cs_rows.data(), (size_t)s->b_eff * 4, cudaMemcpyHostToDevice, st));
    s->has_ctrl = condition != nullptr;
    s->graph_ok = false;
    // 1. prefix embeddings: CaptionEmbedder MLP (gpt_t2i.py:156-162) or LabelEmbedder gather (:89-97)
    if (d.model_type == 1) CAR_TRY(enqueue_mlp(s, cond, rows, d.caption_dim, m->g_cap_fc1, m->g_cap_fc2, m->cap_fc1, m->cap_fc2, s->t1, s->hP, st));
    else {
        if (d.dtype == CAR_BF16) CAR_LAUNCH((gather_rows_kernel<bf16>), rows, 256, 0, st, (const bf16*)m->label_table, (const int*)cond, (bf16*)s->hP, d.dim, (const bf16*)nullptr, 0, 0, nullptr);
        else CAR_LAUNCH((gather_rows_kernel<float>), rows, 256, 0, st, (const float*)m->label_table, (const int*)cond, (float*)s->hP, d.dim, (const float*)nullptr, 0, 0, nullptr);
    }
    // 2. control tokens: condition_mlp then the three condition_layers MLPs (gpt_t2i.py:438-442)
    if (condition) {
        const int crow = s->b_eff * s->N;
        CAR_TRY(enqueue_mlp(s, condition, crow, d.dim, m->g_cond_fc1, m->g_cond_fc2, m->cond_fc1, m->cond_fc2, s->t1, s->t2, st));
        for (int j = 0; j < 3; ++j)
            CAR_TRY(enqueue_mlp(s, s->t2, crow, d.dim, m->g_ctl_fc1[j], m->g_ctl_fc2[j], m->ctl_fc1[j], m->ctl_fc2[j], s->t1, s->ctrl[j], st));
    }
    // 3. blocks
    for (int l = 0; l < d.n_layer; ++l) {
        if (d.dtype == CAR_BF16) CAR_TRY(prefill_small_kernels<bf16>(s, l, st)); else CAR_TRY(prefill_small_kernels<float>(s, l, st));
        if (use_dense(s, rows)) CAR_TRY(enqueue_block_dense(s, l, st));
        else CAR_TRY(enqueue_block(s, l, false, st));
    }
    // 4. head: last prefix row always (feeds car_generate); all rows on request (forward() parity)
    if (d.dtype == CAR_BF16) CAR_LAUNCH((take_last_row_kernel<bf16>), s->b_eff, 256, 0, st, (const bf16*)s->hP, (bf16*)s->h, s->T, d.dim);
    else CAR_LAUNCH((take_last_row_kernel<float>), s->b_eff, 256, 0, st, (const float*)s->hP, (float*)s->h, s->T, d.dim);
    CAR_TRY(enqueue_head(s, s->h, s->b_eff, s->logits, false, st));
    if (logits_out) {
        if (all_rows) CAR_TRY(enqueue_head(s, s->hP, rows, logits_out, false, st));
        else CAR_CUDA(cudaMemcpyAsync(logits_out, s->logits, (size_t)s->b_eff * d.vocab_size * 4, cudaMemcpyDeviceToDevice, st));
    }
    CAR_LAUNCH(set_int_kernel, 1, 1, 0, st, s->pos, s->T - 1);
    s->prefilled = true;
    return CAR_OK;
}

extern "C" int car_decode_step(CarState* s, const int32_t* tok, int32_t pos, float* logits_out, void* stream) {
    if (!s || !tok || !logits_out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (pos < s->T || pos >= s->S) CAR_FAIL(CAR_ERR_ARG, "pos out of range");
    cudaStream_t st = (cudaStream_t)stream;
    const CarModelDesc& d = s->m->d;
    CAR_LAUNCH(set_int_kernel, 1, 1, 0, st, s->pos, pos);
    const int p = pos - s->T + 1;
    if (d.dtype == CAR_BF16)
        CAR_LAUNCH((gather_rows_kernel<bf16>), s->b_eff, 256, 0, st, (const bf16*)s->m->tok_emb, (const int*)tok, (bf16*)s->h, d.dim,
                   (const bf16*)(s->has_ctrl ? s->ctrl[0] : nullptr), s->N, p, s->cs_dev);
    else
        CAR_LAUNCH((gather_rows_kernel<float>), s->b_eff, 256, 0, st, (const float*)s->m->tok_emb, (const int*)tok, (float*)s->h, d.dim,
                   (const float*)(s->has_ctrl ? s->ctrl[0] : nullptr), s->N, p, s->cs_dev);
    return enqueue_decode_layers(s, logits_out, st);
}

// ---------------------------------------------------------------------------------------------------------
// sampling
// ---------------------------------------------------------------------------------------------------------
static int fill_sample_args(SampleArgs& a, const CarSampling* sp, int b_eff, int V) {
    memset(&a, 0, sizeof(a));
    a.V = V;
    a.use_cfg = sp->cfg_scale > 1.0f ? 1 : 0;
    if (a.use_cfg && (b_eff % 2)) CAR_FAIL(CAR_ERR_ARG, "cfg_scale > 1 needs an even number of rows");
    a.B = a.use_cfg ? b_eff / 2 : b_eff;
    a.cfg_on = 1; a.cfg_scale = sp->cfg_scale; a.cfg_interval = sp->cfg_interval;
    return CAR_OK;
}

static SmpRow smp_row(float temperature, int top_k, float top_p, int sample_logits, uint64_t seed, uint32_t noise_row) {
    SmpRow r;
    r.inv_temp = 1.0f / fmaxf(temperature, 1e-5f);
    r.top_k = top_k; r.top_p = top_p; r.sample_logits = sample_logits;
    r.seed_lo = (uint32_t)(seed & 0xffffffffu); r.seed_hi = (uint32_t)(seed >> 32); r.noise_row = noise_row; r.pad = 0u;
    return r;
}

// the sampler's parameters of B images: rows[b] when given, else every image from sp, its Philox counter word the image index
static std::vector<SmpRow> smp_rows(const CarSampling* sp, const CarRowSampling* rows, int B) {
    std::vector<SmpRow> out(B);
    for (int b = 0; b < B; ++b)
        out[b] = rows ? smp_row(rows[b].temperature, rows[b].top_k, rows[b].top_p, rows[b].sample_logits, rows[b].seed, rows[b].noise_row)
                      : smp_row(sp->temperature, sp->top_k, sp->top_p, sp->sample_logits, sp->seed, (uint32_t)b);
    return out;
}

static int launch_sampler(const SampleArgs& a, cudaStream_t st) {
    if (a.V % 4 != 0 || a.V < 4) CAR_FAIL(CAR_ERR_UNSUPPORTED, "the fused sampler needs a vocabulary size that is a multiple of 4");
    CAR_LAUNCH(sample_kernel, a.B, SMP_THREADS, 0, st, a);
    return CAR_OK;
}

// the standalone sampler: the per-image parameters go to a stream-ordered temporary
static int launch_sampler_host_rows(SampleArgs& a, const std::vector<SmpRow>& rows, cudaStream_t st) {
    void* d = nullptr;
    CAR_CUDA(cudaMallocAsync(&d, rows.size() * sizeof(SmpRow), st));
    const cudaError_t e = cudaMemcpyAsync(d, rows.data(), rows.size() * sizeof(SmpRow), cudaMemcpyHostToDevice, st);
    int r = CAR_OK;
    if (e != cudaSuccess) { g_car_err = std::string(__func__) + ": " + cudaGetErrorString(e); r = CAR_ERR_CUDA; }
    else { a.rows = (const SmpRow*)d; r = launch_sampler(a, st); }
    cudaFreeAsync(d, st);
    return r;
}

static int standalone_sample_args(SampleArgs& a, const CarSampling* sp, const float* logits, int b_eff, int V, int cfg_on, int step,
                                  const float* noise, int32_t* idx_out, float* probs_out, uint8_t* kept_out) {
    CAR_TRY(fill_sample_args(a, sp, b_eff, V));
    a.logits = logits; a.cfg_on = cfg_on; a.cfg_interval = -1; a.step = step; a.noise = noise;
    a.idx_out = idx_out; a.tokens_ld = 0; a.probs_out = probs_out; a.kept_out = kept_out;
    return CAR_OK;
}

extern "C" int car_sample(const float* logits, int32_t b_eff, int32_t V, const CarSampling* sp, int32_t cfg_on, int32_t step,
                          const float* noise, int32_t* idx_out, float* probs_out, uint8_t* kept_out, void* stream) {
    if (!logits || !sp || !idx_out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    SampleArgs a;
    CAR_TRY(standalone_sample_args(a, sp, logits, b_eff, V, cfg_on, step, noise, idx_out, probs_out, kept_out));
    return launch_sampler_host_rows(a, smp_rows(sp, nullptr, a.B), (cudaStream_t)stream);
}

extern "C" int car_sample_rows(const float* logits, int32_t b_eff, int32_t V, const CarRowSampling* rows, int32_t B, float cfg_scale,
                               int32_t cfg_on, int32_t step, const float* noise, int32_t* idx_out, float* probs_out, uint8_t* kept_out,
                               void* stream) {
    if (!logits || !rows || !idx_out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (b_eff <= 0 || B != (cfg_scale > 1.0f ? b_eff / 2 : b_eff)) CAR_FAIL(CAR_ERR_ARG, "B must be b_eff, or b_eff / 2 when cfg_scale > 1");
    CAR_TRY(check_rows(rows, B));
    CarSampling sp{1.0f, 0, 1.0f, 1, cfg_scale, -1, 0ull};
    SampleArgs a;
    CAR_TRY(standalone_sample_args(a, &sp, logits, b_eff, V, cfg_on, step, noise, idx_out, probs_out, kept_out));
    return launch_sampler_host_rows(a, smp_rows(&sp, rows, B), (cudaStream_t)stream);
}

// the decode loop's sampler arguments; uploads the per-image parameters of this launch (car_state_set_row_sampling or sp)
static int loop_sample_args(CarState* s, const CarSampling* sp, const float* noise, cudaStream_t st, SampleArgs& a) {
    const CarModelDesc& d = s->m->d;
    CAR_TRY(fill_sample_args(a, sp, s->b_eff, d.vocab_size));
    if (!s->row_sp.empty() && (int)s->row_sp.size() != a.B)
        CAR_FAIL(CAR_ERR_ARG, "the row sampling set on the state has " + std::to_string(s->row_sp.size()) + " images, the launch " +
                              std::to_string(a.B) + " (cfg_scale decides whether b_eff counts the unconditional rows)");
    const std::vector<SmpRow> rows = smp_rows(sp, s->row_sp.empty() ? nullptr : s->row_sp.data(), a.B);
    CAR_CUDA(cudaMemcpyAsync(s->smp_rows, rows.data(), rows.size() * sizeof(SmpRow), cudaMemcpyHostToDevice, st));
    a.rows = s->smp_rows;
    a.logits = s->logits; a.noise = noise; a.noise_per_step = noise ? 1 : 0;
    a.idx_out = s->tokens; a.tokens_ld = s->N; a.probs_out = nullptr;
    a.h_out = s->h; a.tok_emb = s->m->tok_emb; a.ctrl0 = s->has_ctrl ? s->ctrl[0] : nullptr; a.d = d.dim; a.n_img = s->N;
    a.T = s->T; a.cs = s->cs_dev; a.dtype = d.dtype; a.tok_buf = s->tok; a.pos_ptr = s->pos; a.done_ctr = s->done_ctr;
    return CAR_OK;
}

// the whole decode loop as one persistent cooperative kernel (decode_persistent.cuh)
static int launch_pk(CarState* s, const SampleArgs& a, int n_tokens, cudaStream_t st, const int32_t* forced = nullptr, float* trace = nullptr) {
    const CarModelDesc& d = s->m->d;
    const int L = d.n_layer;
    if (s->pk_ptrs_gen != s->m->pack_gen) {   // car_model_repack since the table was uploaded: the borrowed norm-weight pointers may have moved
        const std::vector<const void*> hp = pk_pointer_table(s);
        CAR_CUDA(cudaMemcpyAsync(s->pk_ptrs, hp.data(), hp.size() * sizeof(void*), cudaMemcpyHostToDevice, st));
        CAR_CUDA(cudaStreamSynchronize(st));                      // hp is a host temporary
        s->pk_ptrs_gen = s->m->pack_gen;
    }
    unsigned int tag_gen = 0;
    const unsigned int tag_base = pk_alloc_tags((unsigned int)n_tokens * (unsigned int)(L + 1) + 8u, &tag_gen);
    if (tag_gen != s->pk_tag_gen) {       // the process-wide tag counter wrapped since this state's packets were last zeroed
        CAR_TRY(fill_u32(s->pk_pkt_base, 0u, s->pk_pkt_bytes, st));
        s->pk_tag_gen = tag_gen;
    }
    PkParams P;
    memset(&P, 0, sizeof(P));
    P.dim = d.dim; P.F = d.ffn_dim; P.V = d.vocab_size; P.L = L; P.H = d.n_head; P.T = s->T; P.S = s->S; P.n_img = s->N;
    P.b_eff = s->b_eff; P.B = a.B; P.eps = d.norm_eps; P.cs = s->cs_dev;
    P.tok_emb = (const bf16*)s->m->tok_emb; P.norm_w = (const bf16*)s->m->norm; P.w_out = (const uint4*)s->m->g_output;
    void** pp = s->pk_ptrs;
    P.wqkv = (const uint4* const*)(pp + 0 * L); P.wo = (const uint4* const*)(pp + 1 * L); P.w13 = (const uint4* const*)(pp + 2 * L);
    P.w2 = (const uint4* const*)(pp + 3 * L); P.attn_norm = (const bf16* const*)(pp + 4 * L); P.ffn_norm = (const bf16* const*)(pp + 5 * L);
    P.kc = (bf16* const*)(pp + 6 * L); P.vc = (bf16* const*)(pp + 7 * L);
    for (int j = 0; j < 3; ++j) P.ctrl[j] = (const bf16*)s->ctrl[j];
    P.has_ctrl = s->has_ctrl ? 1 : 0;
    P.rope = s->rope; P.emb_mask = s->emb_mask; P.logits = s->logits; P.part = s->pk_part;
    for (int par = 0; par < 2; ++par) {
        P.h2[par] = s->pk_h2[par]; P.h1[par] = s->pk_h1[par]; P.att[par] = s->pk_att[par]; P.act[par] = s->pk_act[par];
        P.qkv[par] = s->pk_qkv[par]; P.partial[par] = s->pk_partial[par];
    }
    P.part_slots = s->pk_part_slots; P.tag_base = tag_base; P.bar = s->pk_bar; P.bar_base = s->pk_bar_count;
    P.smp = a; P.n_steps = n_tokens;
    P.forced = forced; P.forced_ld = n_tokens; P.trace = trace; P.step_ts = s->pk_step_ts;
    if (trace) CAR_CUDA(cudaMemcpyAsync(trace, s->logits, (size_t)s->b_eff * d.vocab_size * 4, cudaMemcpyDeviceToDevice, st));
    static DevOnce once;
    if (once.first()) {
        CAR_CUDA(cudaFuncSetAttribute(pk_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PK_SMEM_TOTAL));
    }
    int occ = 0;
    CAR_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, pk_decode_kernel, PK_THREADS, PK_SMEM_TOTAL));
    if (occ < 1) CAR_FAIL(CAR_ERR_UNSUPPORTED, "persistent decode kernel does not fit on an SM");
#ifdef PK_TRACE
    // phase timings of one decode step (CAR_DBG=<step>), printed to stderr after the launch
    static const int trace_step = [] { const char* e = getenv("CAR_DBG"); return e ? atoi(e) : 0; }();
    static long long* mdbg = nullptr;
    const size_t dbg_n = (size_t)s->pk_grid * 64 + 5 * 256;
    if (trace_step) {
        if (!mdbg) { cudaMalloc(&mdbg, dbg_n * 8); }
        cudaMemsetAsync(mdbg, 0, dbg_n * 8, st);
        P.dbg = mdbg; P.dbg_step = std::max(0, std::min(n_tokens - 2, trace_step));
    }
#endif
    void* args[] = {&P};
    CAR_CUDA(cudaLaunchCooperativeKernel((const void*)pk_decode_kernel, dim3(s->pk_grid), dim3(PK_THREADS), args, PK_SMEM_TOTAL, st));
    s->pk_bar_count += (unsigned int)(n_tokens - 1) * (unsigned int)s->pk_grid;        // one grid barrier per decoded token
    g_car_launches.fetch_add(1, std::memory_order_relaxed);
#ifdef PK_TRACE
    if (trace_step) {
        cudaStreamSynchronize(st);
        std::vector<long long> t(dbg_n);
        cudaMemcpy(t.data(), mdbg, dbg_n * 8, cudaMemcpyDeviceToHost);
        const int G = s->pk_grid;
        long long t0 = t[0];
        for (int c = 0; c < G; ++c) if (t[(size_t)c * 64]) t0 = std::min(t0, t[(size_t)c * 64]);
        auto stat = [&](int slot, const char* name) {
            std::vector<long long> v;
            for (int c = 0; c < G; ++c) if (t[(size_t)c * 64 + slot]) v.push_back(t[(size_t)c * 64 + slot] - t0);
            if (v.empty()) return;
            std::sort(v.begin(), v.end());
            int amax = 0;
            for (int c = 0; c < G; ++c) if (t[(size_t)c * 64 + slot] - t0 == v.back()) amax = c;
            fprintf(stderr, "[pk] %-22s n=%3zu  min %8.2f  med %8.2f  max %8.2f us (CTA %d)\n", name, v.size(), v.front() * 1e-3, v[v.size() / 2] * 1e-3,
                    v.back() * 1e-3, amax);
        };
        fprintf(stderr, "[pk] step %d, times relative to the first CTA entering the sampler; layer 3 phases\n", P.dbg_step);
        stat(0, "step start"); stat(1, "sampler done");
        if (t[48]) fprintf(stderr, "[pk] sampler top-k of CTA 0: histogram built %.2f | boundary bin found %.2f | candidates gathered %.2f\n",
                           (t[53] - t[48]) * 1e-3, (t[54] - t[48]) * 1e-3, (t[55] - t[48]) * 1e-3);
        if (t[48]) fprintf(stderr, "[pk] sampler of CTA 0 (us after its start): loads issued %.2f | row in registers + CFG %.2f | top-k done %.2f | soft-max done %.2f | race done %.2f | CTA done %.2f\n",
                           0.0, (t[49] - t[48]) * 1e-3, (t[50] - t[48]) * 1e-3, (t[51] - t[48]) * 1e-3, (t[52] - t[48]) * 1e-3, (t[1] - t[48]) * 1e-3);
        const char* nm[5] = {"qkv", "attn", "wo", "w13", "w2"};
        for (int k = 0; k < 5; ++k) {
            char buf[64];
            const char* sub[5] = {"start", k == 1 ? "q polled" : "A polled", k == 1 ? "keys done" : "weights+norm", k == 1 ? "end" : "mma done", "end"};
            for (int j = 0; j < (k == 1 ? 4 : 5); ++j) { snprintf(buf, sizeof buf, "L3 %s %s", nm[k], sub[j]); stat(8 + 8 * k + j, buf); }
        }
        {
            const char* sub[5] = {"head start", "head A polled", "head weights+norm", "head mma done (batch 0)", "head end (batch 0)"};
            for (int j = 0; j < 5; ++j) stat(56 + j, sub[j]);
        }
        stat(3, "head done"); stat(4, "barrier passed");
        {   // per-warp stamps of one CTA (77): min / max over the 16 warps, relative to the phase's first stamp
            const char* wn[11] = {"start", "prepoll", "A loaded", "ssq out", "sync1", "normed", "mma", "red out", "sync2", "reduced", "end"};
            const char* pn[5] = {"qkv", "attn", "wo", "w13", "w2"};
            for (int ph = 0; ph < 5; ++ph) {
                if (ph == 1) continue;
                const long long* w = t.data() + (size_t)G * 64 + (size_t)ph * 256;
                long long base = 0;
                for (int k = 0; k < 16; ++k) if (w[k * 16] && (!base || w[k * 16] < base)) base = w[k * 16];
                if (!base) continue;
                fprintf(stderr, "[pk warp] %-3s", pn[ph]);
                for (int sI = 0; sI < 11; ++sI) {
                    long long mn = 0, mx = 0;
                    for (int k = 0; k < 16; ++k) { const long long v = w[k * 16 + sI]; if (!v) continue; if (!mn || v < mn) mn = v; if (v > mx) mx = v; }
                    if (mn) fprintf(stderr, " | %s %.2f-%.2f", wn[sI], (mn - base) * 1e-3, (mx - base) * 1e-3);
                }
                fprintf(stderr, "\n");
            }
        }
    }
#endif
    return CAR_OK;
}

extern "C" int car_generate(CarState* s, const CarSampling* sp, int32_t n_tokens, const float* noise, int32_t* tokens_out,
                            void* stream) {
    if (!s || !sp || !tokens_out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (!s->prefilled) CAR_FAIL(CAR_ERR_STATE, "car_generate must follow car_prefill on the same state");
    if (n_tokens < 1 || n_tokens > s->N) CAR_FAIL(CAR_ERR_ARG, "n_tokens must be in [1, N]");
    cudaStream_t st = (cudaStream_t)stream;
    SampleArgs a;
    CAR_TRY(loop_sample_args(s, sp, noise, st, a));
    if (s->m->d.dtype == CAR_BF16 && s->pk_ok) {
        CAR_TRY(launch_pk(s, a, n_tokens, st));
        CAR_CUDA(cudaMemcpy2DAsync(tokens_out, (size_t)n_tokens * 4, s->tokens, (size_t)s->N * 4, (size_t)n_tokens * 4, a.B,
                                   cudaMemcpyDeviceToDevice, st));
        CAR_LAUNCH(set_int_kernel, 1, 1, 0, st, s->pos, s->T - 1 + n_tokens);
        s->prefilled = false;
        return CAR_OK;
    }
    // token 0 from the prefill logits (generate.py:198); its fused tail writes h for position T and bumps pos
    CAR_TRY(launch_sampler(a, st));
    if (n_tokens > 1) {
        if (!s->graph_ok || s->graph_cfg_scale != sp->cfg_scale || s->graph_cfg_interval != sp->cfg_interval || s->gnoise != noise ||
            s->graph_pack_gen != s->m->pack_gen) {
            if (s->gexec) { cudaGraphExecDestroy(s->gexec); s->gexec = nullptr; }
            cudaGraph_t g = nullptr;
            const long long launched_before = g_car_launches.load();   // captured nodes are not launches yet
            CAR_CUDA(cudaStreamBeginCapture(s->cap_stream, cudaStreamCaptureModeRelaxed));
            int r = enqueue_decode_layers(s, s->logits, s->cap_stream);
            if (r == CAR_OK) r = launch_sampler(a, s->cap_stream);
            cudaError_t ce = cudaStreamEndCapture(s->cap_stream, &g);
            s->graph_launches = g_car_launches.load() - launched_before;
            g_car_launches.store(launched_before);
            if (r != CAR_OK) { if (g) cudaGraphDestroy(g); return r; }
            if (ce != cudaSuccess) CAR_FAIL(CAR_ERR_CUDA, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce));
            ce = cudaGraphInstantiate(&s->gexec, g, 0);
            cudaGraphDestroy(g);
            if (ce != cudaSuccess) CAR_FAIL(CAR_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(ce));
            s->graph_ok = true; s->graph_cfg_scale = sp->cfg_scale; s->graph_cfg_interval = sp->cfg_interval; s->gnoise = noise;
            s->graph_pack_gen = s->m->pack_gen;
        }
        for (int i = 1; i < n_tokens; ++i) CAR_CUDA(cudaGraphLaunch(s->gexec, st));
        g_car_launches.fetch_add(s->graph_launches * (n_tokens - 1), std::memory_order_relaxed);
    }
    const int B = a.B;
    CAR_CUDA(cudaMemcpy2DAsync(tokens_out, (size_t)n_tokens * 4, s->tokens, (size_t)s->N * 4, (size_t)n_tokens * 4, B,
                               cudaMemcpyDeviceToDevice, st));
    s->prefilled = false;
    return CAR_OK;
}

// teacher forcing on the per-kernel chain: row r (image r mod B; a CFG pair shares its token) is fed forced[image][step]
__global__ void forced_tokens_kernel(const int* __restrict__ forced, int ld, int step, int B, int b_eff, int* __restrict__ tok) {
    for (int r = threadIdx.x; r < b_eff; r += blockDim.x) tok[r] = forced[(size_t)(r % B) * ld + step];
}

// the per-kernel chain's decode loop (wide route included), teacher-forced: per step the sampler (its fused tail advances the position), the forced token's
// embedding (+ control add) in place of the sampled one, the layers and the head
static int chain_forced_loop(CarState* s, const SampleArgs& a, int n_tokens, const int32_t* forced, float* trace, cudaStream_t st) {
    const CarModelDesc& d = s->m->d;
    const size_t row_bytes = (size_t)s->b_eff * d.vocab_size * 4;
    if (trace) CAR_CUDA(cudaMemcpyAsync(trace, s->logits, row_bytes, cudaMemcpyDeviceToDevice, st));
    for (int i = 0; i < n_tokens; ++i) {
        CAR_TRY(launch_sampler(a, st));
        if (i + 1 == n_tokens) break;
        CAR_LAUNCH(forced_tokens_kernel, 1, 64, 0, st, (const int*)forced, n_tokens, i, a.B, s->b_eff, s->tok);
        CAR_LAUNCH((gather_rows_kernel<bf16>), s->b_eff, 256, 0, st, (const bf16*)s->m->tok_emb, (const int*)s->tok, (bf16*)s->h, d.dim,
                   (const bf16*)(s->has_ctrl ? s->ctrl[0] : nullptr), s->N, i + 1, s->cs_dev);
        CAR_TRY(enqueue_decode_layers(s, s->logits, st));
        if (trace) CAR_CUDA(cudaMemcpyAsync(trace + (size_t)(i + 1) * s->b_eff * d.vocab_size, s->logits, row_bytes, cudaMemcpyDeviceToDevice, st));
    }
    return CAR_OK;
}

// teacher-forced run of the product decode loop (parity tests): the token fed to step i + 1 is forced[b][i]; the sampler still
// runs and tokens_out holds what it would have chosen at every step given the forced prefix; logits_trace (optional) receives the
// raw model logits of every step.  bf16: the persistent kernel where it runs, else the per-kernel chain (wide route above 32 rows).
extern "C" int car_generate_forced(CarState* s, const CarSampling* sp, int32_t n_tokens, const float* noise, const int32_t* forced_tokens,
                                   float* logits_trace, int32_t* tokens_out, void* stream) {
    if (!s || !sp || !tokens_out || !forced_tokens) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (!s->prefilled) CAR_FAIL(CAR_ERR_STATE, "car_generate_forced must follow car_prefill on the same state");
    if (n_tokens < 1 || n_tokens > s->N) CAR_FAIL(CAR_ERR_ARG, "n_tokens must be in [1, N]");
    if (s->m->d.dtype != CAR_BF16) CAR_FAIL(CAR_ERR_UNSUPPORTED, "teacher forcing through the device-side loop is bf16 only; use car_decode_step");
    cudaStream_t st = (cudaStream_t)stream;
    SampleArgs a;
    CAR_TRY(loop_sample_args(s, sp, noise, st, a));
    if (s->pk_ok) CAR_TRY(launch_pk(s, a, n_tokens, st, forced_tokens, logits_trace));
    else CAR_TRY(chain_forced_loop(s, a, n_tokens, forced_tokens, logits_trace, st));
    CAR_CUDA(cudaMemcpy2DAsync(tokens_out, (size_t)n_tokens * 4, s->tokens, (size_t)s->N * 4, (size_t)n_tokens * 4, a.B,
                               cudaMemcpyDeviceToDevice, st));
    CAR_LAUNCH(set_int_kernel, 1, 1, 0, st, s->pos, s->T - 1 + n_tokens);
    s->prefilled = false;
    return CAR_OK;
}

extern "C" int64_t car_decode_step_bytes(const CarState* s, int32_t n_context) {
    if (!s) return -1;
    const CarModelDesc& d = s->m->d;
    const int64_t es = d.dtype == CAR_BF16 ? 2 : 4;
    const int64_t P = (int64_t)d.n_layer * (4LL * d.dim * d.dim + 3LL * d.dim * d.ffn_dim) + (int64_t)d.vocab_size * d.dim;
    const int64_t kappa = 2LL * d.n_layer * d.dim * es;
    return es * P + (int64_t)s->b_eff * kappa * n_context + (int64_t)s->b_eff * kappa + 4LL * s->b_eff * d.vocab_size;
}

// ---------------------------------------------------------------------------------------------------------
// building-block ops for unit tests
// ---------------------------------------------------------------------------------------------------------
extern "C" int car_op_linear(int32_t dtype, const void* x, const void* w, const void* bias, void* y, int32_t M, int32_t N,
                             int32_t K, int32_t act, void* stream) {
    if (!x || !w || !y) CAR_FAIL(CAR_ERR_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    EpiParams e = epi_base(EPI_STORE);
    e.out = y; e.ldo = N; e.act = act; e.bias = bias;
    if (dtype == CAR_F32) return launch_skinny(st, dtype, x, K, w, nullptr, 0.f, M, N, K, e, false);
    void* packed = nullptr;
    CAR_CUDA(cudaMallocAsync(&packed, (size_t)N * K * 2, st));
    const int nblk = N / 8;
    const long long total = (long long)nblk * (K / 32) * 32;
    CAR_LAUNCH(pack_weight_bf16_kernel, (int)std::min<long long>((total + 255) / 256, 4096), 256, 0, st, (const bf16*)w,
               (const bf16*)nullptr, (uint4*)packed, nblk, K, 0);
    int r = launch_skinny(st, dtype, x, K, packed, nullptr, 0.f, M, N, K, e, false);
    cudaFreeAsync(packed, st);
    return r;
}

// the dense (M >= 64 rows) tensor-core linear of the prefill / MLP path, exposed for unit tests and micro-benchmarks:
// y[M,N] = act(x[M,K] · w[N,K]^T) (+ resid), bf16, fp32 accumulate, routed by gemm() (gemm.cu): the wgmma kernel when N is a
// multiple of 8 and y, resid 16-byte aligned, otherwise the mma.sync kernel; K % 8 != 0 or misaligned x, w are refused (gemm.h)
extern "C" int car_op_dense_linear(const void* x, const void* w, const void* resid, void* y, int32_t M, int32_t N, int32_t K, int32_t act,
                                   void* stream) {
    if (!x || !w || !y) CAR_FAIL(CAR_ERR_ARG, "null argument");
    return dense_linear((cudaStream_t)stream, x, K, w, M, N, K, act ? ACT_GELU_TANH : ACT_NONE, resid, N, y, N);
}

// the library's GEMM front end (gemm.h), for conformance tests: the descriptor is copied field by field into a DenseP
static DenseP dense_p(const CarGemmDesc& d) {
    DenseP p;
    memset(&p, 0, sizeof(p));
    p.A = (const bf16*)d.A; p.B = (const bf16*)d.B; p.M = d.M; p.N = d.N; p.K = d.K; p.lda = d.lda; p.ldb = d.ldb;
    p.sA = d.sA; p.sB = d.sB; p.sC = d.sC; p.sR = d.sR;
    p.amode = d.amode; p.Hs = d.Hs; p.Ws = d.Ws; p.Cin = d.Cin; p.Ho = d.Ho; p.Wo = d.Wo; p.ups = d.ups;
    p.alpha = d.alpha; p.bias = (const bf16*)d.bias; p.bias_along_m = d.bias_along_m; p.bias_f = d.bias_f; p.resid_f = d.resid_f;
    p.act = d.act; p.scale = (const bf16*)d.scale; p.resid = (const bf16*)d.resid; p.ldr = d.ldr; p.C = d.C; p.ldc = d.ldc;
    p.out_mode = d.out_mode; p.kh = d.kh; p.kw = d.kw; p.ws = d.ws;
    p.osy = d.osy; p.osx = d.osx; p.oay = d.oay; p.oax = d.oax; p.oH = d.oH; p.oW = d.oW;
    return p;
}
extern "C" int car_op_gemm_route(const CarGemmDesc* d, int32_t batch) {
    if (!d) CAR_FAIL(CAR_ERR_ARG, "null descriptor");
    return gemm_route(dense_p(*d), batch);
}
extern "C" int car_op_gemm(const CarGemmDesc* d, int32_t batch, void* stream) {
    if (!d) CAR_FAIL(CAR_ERR_ARG, "null descriptor");
    return gemm((cudaStream_t)stream, dense_p(*d), batch);
}
extern "C" int car_op_gemm_f32(const void* A, const void* B, int32_t M, int32_t N, int32_t K, const float* bias, const float* resid, float* out,
                               int32_t ldc, void* stream) {
    return gemm_f32((cudaStream_t)stream, (const bf16*)A, (const bf16*)B, M, N, K, bias, resid, out, ldc);
}
extern "C" int car_op_gemm_f32_conv3(const void* src, int32_t fh, int32_t fw, const void* B, int32_t nimg, int32_t H, int32_t W, int32_t cin,
                                     int32_t N, const float* bias, const float* resid, float* out, void* stream) {
    return gemm_f32_conv3((cudaStream_t)stream, (const bf16*)src, fh, fw, (const bf16*)B, nimg, H, W, cin, N, bias, resid, out);
}

extern "C" int car_op_rmsnorm(int32_t dtype, const void* x, const void* w, void* y, int32_t M, int32_t K, float eps, void* stream) {
    if (!x || !w || !y) CAR_FAIL(CAR_ERR_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == CAR_BF16) CAR_LAUNCH((rmsnorm_rows_kernel<bf16>), M, 256, 0, st, (const bf16*)x, (const bf16*)w, (bf16*)y, K, eps);
    else CAR_LAUNCH((rmsnorm_rows_kernel<float>), M, 256, 0, st, (const float*)x, (const float*)w, (float*)y, K, eps);
    return CAR_OK;
}

// shape and mask checks common to the two attention ops
static int attn_op_check(int dtype, const void* q, const void* kc, const void* vc, const int32_t* emb_mask, int mask_ld, int B, int H,
                         int S, int Tpre, const void* out) {
    if (!q || !kc || !vc || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (dtype != CAR_BF16 && dtype != CAR_F32) CAR_FAIL(CAR_ERR_ARG, "dtype must be CAR_BF16 or CAR_F32");
    if (B <= 0 || H <= 0 || S <= 0 || B > 65535 || H > 65535 || (long long)B * H > (1 << 30)) CAR_FAIL(CAR_ERR_ARG, "need 0 < B, H <= 65535 and S > 0");
    if (Tpre < 0) CAR_FAIL(CAR_ERR_ARG, "Tpre must be >= 0");
    if (emb_mask && mask_ld < Tpre) CAR_FAIL(CAR_ERR_ARG, "mask_ld must be >= Tpre");
    if (((uintptr_t)kc | (uintptr_t)vc) % 16) CAR_FAIL(CAR_ERR_ARG, "k_cache and v_cache must be 16-byte aligned");
    return CAR_OK;
}

extern "C" int car_op_attn_decode(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, const int32_t* emb_mask,
                                  int32_t mask_ld, const int32_t* pos_dev, int32_t B, int32_t H, int32_t S, int32_t Tpre, int32_t nsplit,
                                  float* part, int32_t* tickets, void* out, void* stream) {
    CAR_TRY(attn_op_check(dtype, q, k_cache, v_cache, emb_mask, mask_ld, B, H, S, Tpre, out));
    if (!pos_dev || !part || !tickets) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (nsplit < 0 || nsplit > 16) CAR_FAIL(CAR_ERR_ARG, "nsplit must be in [0, 16]");
    cudaStream_t st = (cudaStream_t)stream;
    // the kernel reads pos on the device; read it back to check the invariant car_decode_step guarantees by pos >= T: the key at
    // pos is an image key, so every row has at least one unmasked key (the decode kernel does not force the diagonal)
    int32_t pos = -1;
    CAR_CUDA(cudaMemcpyAsync(&pos, pos_dev, sizeof(pos), cudaMemcpyDeviceToHost, st));
    CAR_CUDA(cudaStreamSynchronize(st));
    if (pos < Tpre || pos >= S) CAR_FAIL(CAR_ERR_ARG, "need Tpre <= *pos_dev < S");
    return launch_attn_decode(dtype, st, q, k_cache, v_cache, emb_mask, mask_ld, pos_dev, B, H, S, Tpre,
                              nsplit ? nsplit : attn_decode_nsplit(B * H), part, tickets, out);
}

extern "C" int car_op_attn_prefill(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, const int32_t* emb_mask,
                                   int32_t mask_ld, int32_t B, int32_t H, int32_t S, int32_t Tq, int32_t Tpre, int32_t impl, void* out,
                                   void* stream) {
    CAR_TRY(attn_op_check(dtype, q, k_cache, v_cache, emb_mask, mask_ld, B, H, S, Tpre, out));
    if (Tq < 1 || Tq > 256) CAR_FAIL(CAR_ERR_ARG, "Tq must be in [1, 256]");
    if (Tq > S || Tpre > Tq) CAR_FAIL(CAR_ERR_ARG, "need Tpre <= Tq <= S");
    if (impl != 0 && impl != 1) CAR_FAIL(CAR_ERR_ARG, "impl must be 0 (scalar) or 1 (tensor cores)");
    cudaStream_t st = (cudaStream_t)stream;
    if (impl == 0) return launch_attn_prefill(dtype, st, q, k_cache, v_cache, emb_mask, mask_ld, B, H, S, Tq, Tpre, out);
    if (dtype != CAR_BF16) CAR_FAIL(CAR_ERR_UNSUPPORTED, "the tensor-core prefill attention is bf16 only");
    if (((uintptr_t)q | (uintptr_t)out) % 4) CAR_FAIL(CAR_ERR_ARG, "q and out must be 4-byte aligned");
    return launch_attn_prefill_mma(st, q, k_cache, v_cache, emb_mask, mask_ld, B, H, S, Tq, Tpre, out);
}

// ---------------------------------------------------------------------------------------------------------
// T5 text encoder forward (SURVEY.md §8 row f3): language/t5.py:58-79 -> HF T5EncoderModel(...).last_hidden_state, bf16.
// v1.1 / flan architecture: gated gelu_new feed-forward, no biases, RMS layer norm (eps 1e-6), relative position bias of block 0
// shared by every block, no 1/sqrt(d) scaling.  GEMMs: dense_linear (wgmma); glue: t5.cuh.
// ---------------------------------------------------------------------------------------------------------
struct CarT5 : CarOwned {
    CarT5Desc d;
    const void *embed, *rel_bias, *final_norm;
    std::vector<const void*> ln1, wq, wk, wv, wo, ln2, wi0, wi1, wo2;
    int max_rows;
    bf16 *h, *x, *q, *k, *v, *att, *g, *u, *act;
};

static int t5_init(CarT5* t) {
    const CarT5Desc& d = t->d;
    const size_t R = (size_t)t->max_rows, inner = (size_t)d.n_heads * 64;
    CAR_TRY(t->alloc(&t->h, R * d.d_model * 2)); CAR_TRY(t->alloc(&t->x, R * d.d_model * 2));
    CAR_TRY(t->alloc(&t->q, R * inner * 2)); CAR_TRY(t->alloc(&t->k, R * inner * 2)); CAR_TRY(t->alloc(&t->v, R * inner * 2));
    CAR_TRY(t->alloc(&t->att, R * inner * 2));
    CAR_TRY(t->alloc(&t->g, R * d.d_ff * 2)); CAR_TRY(t->alloc(&t->u, R * d.d_ff * 2)); CAR_TRY(t->alloc(&t->act, R * d.d_ff * 2));
    return CAR_OK;
}

extern "C" int car_t5_create(const CarT5Desc* desc, const CarT5Weights* w, int32_t max_rows, void* stream, CarT5** out) {
    if (!desc || !w || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    (void)stream;
    const CarT5Desc& d = *desc;
    if (d.dtype != CAR_BF16) CAR_FAIL(CAR_ERR_UNSUPPORTED, "the T5 encoder is built for bf16 checkpoints (the reference's default torch_dtype, language/t5.py:22)");
    if (d.d_kv != 64 || d.d_model % 8 || d.d_ff % 8 || d.n_heads <= 0 || d.n_layers <= 0 || max_rows <= 0 || d.num_buckets % 2)
        CAR_FAIL(CAR_ERR_UNSUPPORTED, "shape not supported (d_kv 64, dims multiple of 8)");
    CarT5* t = new CarT5();
    t->d = d; t->embed = w->embed; t->rel_bias = w->rel_bias; t->final_norm = w->final_norm; t->max_rows = max_rows;
    const int L = d.n_layers;
    auto cp = [&](std::vector<const void*>& v, const void* const* src) { v.assign(src, src + L); };
    cp(t->ln1, w->ln1); cp(t->wq, w->q); cp(t->wk, w->k); cp(t->wv, w->v); cp(t->wo, w->o); cp(t->ln2, w->ln2);
    cp(t->wi0, w->wi_0); cp(t->wi1, w->wi_1); cp(t->wo2, w->wo);
    const int rc = t5_init(t);
    if (rc != CAR_OK) { delete t; return rc; }
    *out = t;
    return CAR_OK;
}
extern "C" int car_t5_destroy(CarT5* t) {
    delete t;
    return CAR_OK;
}
// ids int32 [B][L], mask int32 [B][L] (1 = token, 0 = padding) -> last_hidden_state bf16 [B][L][d_model]
extern "C" int car_t5_forward(CarT5* t, const int32_t* ids, const int32_t* mask, int32_t B, int32_t L, void* out, void* stream) {
    if (!t || !ids || !mask || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || L <= 0 || (long long)B * L > t->max_rows) CAR_FAIL(CAR_ERR_ARG, "batch x length beyond the capacity given to car_t5_create");
    cudaStream_t st = (cudaStream_t)stream;
    const CarT5Desc& d = t->d;
    const int R = B * L, dm = d.d_model, inner = d.n_heads * 64, F = d.d_ff;
    const size_t att_smem = (size_t)T5A_WARPS * L * 4;
    if (att_smem > 48 * 1024) CAR_FAIL(CAR_ERR_UNSUPPORTED, "sequence too long for the T5 attention kernel (L <= 3072)");
    CAR_LAUNCH(t5_embed_kernel, R, 128, 0, st, (const int*)ids, (const bf16*)t->embed, t->h, R, dm);
    for (int l = 0; l < d.n_layers; ++l) {
        // T5LayerSelfAttention (modeling_t5.py: layer_norm -> SelfAttention -> residual)
        CAR_LAUNCH((rmsnorm_rows_kernel<bf16>), R, 256, 0, st, (const bf16*)t->h, (const bf16*)t->ln1[l], t->x, dm, d.eps);
        CAR_TRY(dense_linear(st, t->x, dm, t->wq[l], R, inner, dm, ACT_NONE, nullptr, 0, t->q, inner));
        CAR_TRY(dense_linear(st, t->x, dm, t->wk[l], R, inner, dm, ACT_NONE, nullptr, 0, t->k, inner));
        CAR_TRY(dense_linear(st, t->x, dm, t->wv[l], R, inner, dm, ACT_NONE, nullptr, 0, t->v, inner));
        CAR_LAUNCH(t5_attention_kernel, (unsigned)(((long long)B * d.n_heads * L + T5A_WARPS - 1) / T5A_WARPS), T5A_WARPS * 32, att_smem, st,
                   (const bf16*)t->q, (const bf16*)t->k, (const bf16*)t->v, (const bf16*)t->rel_bias, (const int*)mask, B, d.n_heads, L, d.num_buckets,
                   d.max_distance, t->att);
        CAR_TRY(dense_linear(st, t->att, inner, t->wo[l], R, dm, inner, ACT_NONE, t->h, dm, t->h, dm));          // hidden + attention_output
        // T5LayerFF: layer_norm -> wi_0 / wi_1 -> gelu_new(.) * . -> wo -> residual
        CAR_LAUNCH((rmsnorm_rows_kernel<bf16>), R, 256, 0, st, (const bf16*)t->h, (const bf16*)t->ln2[l], t->x, dm, d.eps);
        CAR_TRY(dense_linear(st, t->x, dm, t->wi0[l], R, F, dm, ACT_NONE, nullptr, 0, t->g, F));
        CAR_TRY(dense_linear(st, t->x, dm, t->wi1[l], R, F, dm, ACT_NONE, nullptr, 0, t->u, F));
        CAR_LAUNCH(t5_geglu_kernel, gsz((long long)R * F), 256, 0, st, (const bf16*)t->g, (const bf16*)t->u, t->act,
                   (long long)R * F);
        CAR_TRY(dense_linear(st, t->act, F, t->wo2[l], R, dm, F, ACT_NONE, t->h, dm, t->h, dm));
    }
    CAR_LAUNCH((rmsnorm_rows_kernel<bf16>), R, 256, 0, st, (const bf16*)t->h, (const bf16*)t->final_norm, (bf16*)out, dm, d.eps);
    return CAR_OK;
}
