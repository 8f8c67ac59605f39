// car_train.cu — C-ABI entry points of training: the transformer's (car_train_*, car_dropout_keep_mask, car_adamw_step) and the
// trainable control encoder's (car_dino_train_*).  Both backwards run their linear layers through one set of helpers.
#include <cmath>

#include "common.cuh"
#include "gemm.h"
#include "misc.h"
#include "train.cuh"
#include "train_bwd.cuh"
#include "dropout.cuh"

// car_vision.cu instantiates resize_patchify_kernel<float> too: internal linkage keeps the two instantiations from sharing one host stub.
namespace {
#include "patch_embed.cuh"
}
#include "dino_train.cuh"

// ---- linear-layer backward helpers of both handles: the two GEMMs of a layer's backward on the [N][K] x [M][K]^T tensor-core
// kernels and the deterministic column sums, over the scratch each handle carves: W^T (dgrad); dY^T, X^T and the bf16 weight
// gradient (wgrad); partial column sums and the bias gradients' column sums
struct TrScratch { Buf<bf16> wT, yT, xT, dWb; Buf<float> part, colv; };

// dynamic shared memory of the plain attention kernels (TRA_WARPS warps x floats_per_warp); above 48 KB the opt-in attribute is set on
// every call (cheap, and correct on every device of the process — no process-wide "already set" flag)
static int tr_attn_smem(size_t floats_per_warp, const void* fn, size_t* bytes) {
    *bytes = (size_t)TRA_WARPS * floats_per_warp * 4;
    if (*bytes > 200 * 1024) CAR_FAIL(CAR_ERR_UNSUPPORTED, "sequence too long for the plain attention kernels");
    if (*bytes > 48 * 1024) CAR_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return CAR_OK;
}
// autocast's bf16 copy of an fp32 tensor
static int tr_cast(cudaStream_t st, const void* src, bf16* dst, long long n) {
    CAR_LAUNCH(tr_cast_bf16_kernel, gsz(n), 256, 0, st, (const float*)src, dst, n);
    return CAR_OK;
}
// dX [rows][K] = bf16(dY [rows][N] . W [N][K] (+ resid)): needs W^T as the K-major operand
static int tr_dgrad(cudaStream_t st, const TrScratch& sc, const bf16* dY, const bf16* W, int rows, int N, int K, const bf16* resid, bf16* dX) {
    CAR_TRY(car_fits("tr_dgrad", sc.wT, (size_t)N * K));
    CAR_LAUNCH(tr_transpose_pad_kernel, dim3((N + 31) / 32, (K + 31) / 32), dim3(32, 8), 0, st, W, (bf16*)sc.wT, N, K, N);
    DenseP p = dp_plain(dY, N, sc.wT, N, rows, K, N, dX, K);
    p.resid = resid; p.ldr = K;
    return gemm(st, p);
}
// sc.dWb [N][K] = bf16(dY^T . X), dY [rows][N], X [rows][K]: both operands transposed, the row extent zero-padded to 64
static int tr_wgrad(cudaStream_t st, const TrScratch& sc, const bf16* dY, const bf16* X, int rows, int N, int K) {
    const int Rp = (rows + 63) / 64 * 64;
    CAR_TRY(car_fits("tr_wgrad", sc.yT, (size_t)N * Rp)); CAR_TRY(car_fits("tr_wgrad", sc.xT, (size_t)K * Rp));
    CAR_TRY(car_fits("tr_wgrad", sc.dWb, (size_t)N * K));
    CAR_LAUNCH(tr_transpose_pad_kernel, dim3(Rp / 32, (N + 31) / 32), dim3(32, 8), 0, st, dY, (bf16*)sc.yT, rows, N, Rp);
    CAR_LAUNCH(tr_transpose_pad_kernel, dim3(Rp / 32, (K + 31) / 32), dim3(32, 8), 0, st, X, (bf16*)sc.xT, rows, K, Rp);
    return gemm(st, dp_plain(sc.yT, Rp, sc.xT, Rp, N, K, Rp, (bf16*)sc.dWb, K));
}
// the fp32 gradient dst [N][K] of an autocast weight copy from sc.dWb + off, rows of ld elements (columns >= K are padding); null dst: none
static int tr_weight_grad(cudaStream_t st, const TrScratch& sc, size_t off, int N, int K, int ld, float* dst) {
    if (dst) CAR_LAUNCH(tr_bf16_to_f32_2d_kernel, gsz((long long)N * K), 256, 0, st, (const bf16*)sc.dWb + off, ld, dst, N, K);
    return CAR_OK;
}
// grad [N][K] fp32 = float(bf16(dY^T . X)) of one whole weight; null grad: nothing is computed
static int tr_wgrad_f32(cudaStream_t st, const TrScratch& sc, const bf16* dY, const bf16* X, int rows, int N, int K, float* grad) {
    if (!grad) return CAR_OK;
    CAR_TRY(tr_wgrad(st, sc, dY, X, rows, N, K));
    return tr_weight_grad(st, sc, 0, N, K, K, grad);
}
// dst[k] = sum_r src[r][k] (fp32 or bf16 rows, deterministic two-pass column sum)
template <typename T> static int tr_colsum(cudaStream_t st, const TrScratch& sc, const T* src, int rows, int K, float* dst) {
    CAR_TRY(car_fits("tr_colsum", sc.part, (size_t)TR_COLSUM_CHUNKS * K));
    CAR_LAUNCH(tr_colsum_part_kernel, dim3((K + 31) / 32, TR_COLSUM_CHUNKS), dim3(32, 8), 0, st, src, (float*)sc.part, rows, K);
    CAR_LAUNCH(tr_colsum_final_kernel, (K + 255) / 256, 256, 0, st, (const float*)sc.part, dst, K);
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// training forward (SURVEY.md §8 row f1): Transformer.forward(idx, cond_idx, targets, mask, valid, condition) in train mode,
// fp32 parameters under bf16 autocast — gpt_t2i.py:420-431,451-484.  First correct path: prefill GEMM kernels + train.cuh glue.
// ---------------------------------------------------------------------------------------------------------
struct CarTrain : CarOwned {
    CarModelDesc d;
    CarTrainWeights w;
    std::vector<const void*> attention_norm, wqkv, wo, ffn_norm, w1, w3, w2;   // borrowed fp32
    // carved once by car_train_create (train_carve) for (maxB, maxN)
    std::vector<Buf<bf16>> b_wqkv, b_wo, b_w1, b_w3, b_w2;                     // bf16 casts, refreshed every forward
    Buf<bf16> b_out, b_cap1, b_cap2, b_cond1, b_cond2, b_ctl1[3], b_ctl2[3], b_ad1, b_ad2;
    int maxB, maxN, maxS;
    const float* rope;
    Buf<float> h, nll;
    Buf<bf16> x, qkv, q, kc, vc, att, g, u, act, o, cin, ctmp, ctok, cadd, lg;
    // ---- backward (car_train_backward): the stream saved at every block input, gradient / transpose workspaces ----
    Buf<float> hs, dh, h0, scr, lse, dsum;
    Buf<bf16> capx, x2, db, dact, dg, du, dx, datt, dq, dk, dv, dqkv, dlg;
    Buf<bf16> m_t, m_a, m_da, m_dt, dctok, dcin, dadd;
    TrScratch sc;
    // arguments of the last car_train_forward (borrowed until car_train_backward returns)
    int fB = 0, fN = 0;
    const int32_t *f_idx = nullptr, *f_targets = nullptr;
    const void *f_cond = nullptr, *f_feat = nullptr;
    const uint8_t *f_drop = nullptr, *f_mask = nullptr;
    const float* f_valid = nullptr;
    bool fwd_ok = false;
    // dropout (car_train_set_dropout): the settings the next forward takes, and the ones the last forward ran with (its backward's)
    struct DropCfg { float tok_p = 0.f, resid_p = 0.f, ffn_p = 0.f; std::vector<float> path; const uint64_t* seed = nullptr; };
    DropCfg drop_next, drop_fwd;
};

// keep = fp32(1 - p), scale = fp32(1 / keep): the values ATen's CUDA dropout derives from p (native_dropout -> keep probability in
// double, cast to the fp32 accumulate type, scale = 1.0 / keep)
static void tr_keep_scale(float p, float* keep, float* scale) {
    *keep = (float)(1.0 - (double)p);
    *scale = (float)(1.0 / (double)*keep);
}
// the dropout of one site of layer l under the settings c; every part off when its p (or rate) is 0
static TrDrop tr_drop(const CarTrain::DropCfg& c, int site, int l) {
    TrDrop r{c.seed, site, l};
    const float p = site == CAR_DROP_TOKEN ? c.tok_p : (site == CAR_DROP_RESID ? c.resid_p : c.ffn_p);
    if (p > 0.f) tr_keep_scale(p, &r.keep, &r.scale);
    const float rate = (site != CAR_DROP_TOKEN && !c.path.empty()) ? c.path[l] : 0.f;
    if (rate > 0.f) {                                          // utils/drop_path.py: bernoulli_(keep).div_(keep) on a bf16 tensor
        float unused;
        tr_keep_scale(rate, &r.path_keep, &unused);
        r.path_site = site == CAR_DROP_RESID ? CAR_DROP_PATH_ATTN : CAR_DROP_PATH_FFN;
        r.path_mult = __bfloat162float(__float2bfloat16_rn(1.f / r.path_keep));
    }
    return r;
}

// MLP.forward gpt_t2i.py:177-181 on bf16 operands: out = fc2(gelu_tanh(fc1 x))
static int tr_mlp(cudaStream_t st, const bf16* x, int rows, int K, const bf16* fc1, const bf16* fc2, int d, Buf<bf16> tmp, Buf<bf16> out) {
    CAR_TRY(car_fits("tr_mlp", tmp, (size_t)rows * d)); CAR_TRY(car_fits("tr_mlp", out, (size_t)rows * d));
    DenseP p = dp_plain(x, K, fc1, K, rows, d, K, tmp, d);
    p.act = ACT_GELU_TANH;
    CAR_TRY(gemm(st, p));
    return gemm(st, dp_plain(tmp, d, fc2, d, rows, d, d, out, d));
}

// Every buffer of the handle, sized for max_batch samples of max_img_tokens image tokens: the bf16 autocast copies of the weights, the
// forward's activations, the stream saved at every block input and the backward's gradients and scratch.  A buffer that serves several
// stages is taken at the largest of its uses, and its writers check it with car_fits.
static int train_carve(CarTrain* t) {
    const CarModelDesc& d = t->d;
    const int L = d.n_layer;
    const size_t dim = d.dim, F = d.ffn_dim, V = d.vocab_size, T = d.cls_token_num, H = d.n_head, ad = t->w.adapter_dim;
    const size_t cap = d.model_type == 1 ? d.caption_dim : 8;
    const size_t R = (size_t)t->maxB * t->maxS, RC = (size_t)t->maxB * t->maxN, BT = (size_t)t->maxB * T, Rp = (R + 63) / 64 * 64;
    t->b_wqkv.resize(L); t->b_wo.resize(L); t->b_w1.resize(L); t->b_w3.resize(L); t->b_w2.resize(L);
    return t->ws.carve([&](Carve& c) {
        for (int l = 0; l < L; ++l) {
            t->b_wqkv[l] = c.take<bf16>(3 * dim * dim); t->b_wo[l] = c.take<bf16>(dim * dim);
            t->b_w1[l] = c.take<bf16>(F * dim); t->b_w3[l] = c.take<bf16>(F * dim); t->b_w2[l] = c.take<bf16>(dim * F);
        }
        t->b_out = c.take<bf16>(V * dim);
        t->b_cap1 = c.take<bf16>(d.model_type == 1 ? dim * d.caption_dim : 0); t->b_cap2 = c.take<bf16>(d.model_type == 1 ? dim * dim : 0);
        t->b_cond1 = c.take<bf16>(dim * dim); t->b_cond2 = c.take<bf16>(dim * dim);
        for (int j = 0; j < 3; ++j) { t->b_ctl1[j] = c.take<bf16>(dim * dim); t->b_ctl2[j] = c.take<bf16>(dim * dim); }
        t->b_ad1 = c.take<bf16>(dim * ad); t->b_ad2 = c.take<bf16>(dim * dim);
        // forward
        t->h = c.take<float>(R * dim); t->nll = c.take<float>(RC);
        t->x = c.take<bf16>(std::max(R * dim, BT * std::max((size_t)d.caption_dim, dim)));
        t->qkv = c.take<bf16>(R * 3 * dim); t->q = c.take<bf16>(R * dim); t->kc = c.take<bf16>(R * dim); t->vc = c.take<bf16>(R * dim);
        t->att = c.take<bf16>(R * dim); t->g = c.take<bf16>(R * F); t->u = c.take<bf16>(R * F); t->act = c.take<bf16>(R * F);
        t->o = c.take<bf16>(R * dim);
        t->cin = c.take<bf16>(RC * dim); t->ctmp = c.take<bf16>(std::max(RC, BT) * dim); t->ctok = c.take<bf16>(RC * dim);
        t->cadd = c.take<bf16>(RC * dim); t->lg = c.take<bf16>(RC * V);
        // backward
        t->hs = c.take<float>((size_t)L * R * dim); t->dh = c.take<float>(R * dim); t->h0 = c.take<float>(R * dim);
        t->scr = c.take<float>(R * dim); t->sc.part = c.take<float>((size_t)TR_COLSUM_CHUNKS * dim);
        t->lse = c.take<float>((size_t)t->maxB * H * t->maxS); t->dsum = c.take<float>((size_t)t->maxB * H * t->maxS);
        t->capx = c.take<bf16>(BT * cap);
        t->x2 = c.take<bf16>(R * dim); t->db = c.take<bf16>(R * dim); t->dact = c.take<bf16>(R * F);
        t->dg = c.take<bf16>(R * F); t->du = c.take<bf16>(R * F); t->dx = c.take<bf16>(R * dim);
        t->datt = c.take<bf16>(R * dim); t->dq = c.take<bf16>(R * dim); t->dk = c.take<bf16>(R * dim);
        t->dv = c.take<bf16>(R * dim); t->dqkv = c.take<bf16>(R * 3 * dim); t->dlg = c.take<bf16>(RC * V);
        // the linear layers' N x K: the head V x dim, the blocks' 3 dim x dim, F x dim, dim x F, the MLPs' dim x {dim, caption, adapter}
        for (Buf<bf16>* b : {&t->sc.wT, &t->sc.dWb}) *b = c.take<bf16>(dim * std::max({3 * dim, F, V, cap, ad}));
        t->sc.yT = c.take<bf16>(std::max({3 * dim, F, V}) * Rp); t->sc.xT = c.take<bf16>(std::max({F, dim, cap, ad}) * Rp);
        for (Buf<bf16>* b : {&t->m_t, &t->m_a, &t->m_da, &t->m_dt, &t->dadd}) *b = c.take<bf16>(std::max(RC, BT) * dim);
        t->dctok = c.take<bf16>(RC * dim); t->dcin = c.take<bf16>(RC * dim);
    });
}

extern "C" int car_train_create(const CarModelDesc* desc, const CarTrainWeights* w, int32_t max_batch, int32_t max_img_tokens,
                                const float* rope_table, void* stream, CarTrain** out) {
    if (!desc || !w || !out || !rope_table) CAR_FAIL(CAR_ERR_ARG, "null argument");
    const CarModelDesc& d = *desc;
    if (d.dtype != CAR_F32) CAR_FAIL(CAR_ERR_UNSUPPORTED, "training forward takes the fp32 master weights (bf16 autocast is applied inside)");
    if (d.n_head <= 0 || d.dim != d.n_head * 64 || d.n_layer % 3 != 0 || d.ffn_dim % 8 != 0 || d.vocab_size % 8 != 0 || w->adapter_dim % 8 != 0 ||
        (d.model_type == 1 && d.caption_dim % 8 != 0))
        CAR_FAIL(CAR_ERR_UNSUPPORTED, "shape not supported (head_dim 64, dims multiple of 8, n_layer multiple of 3)");
    if (max_batch <= 0 || max_img_tokens <= 0) CAR_FAIL(CAR_ERR_ARG, "bad capacity");
    (void)stream;
    CarTrain* t = new CarTrain();
    t->d = d; t->w = *w; t->rope = rope_table;
    t->maxB = max_batch; t->maxN = max_img_tokens; t->maxS = d.cls_token_num + max_img_tokens - 1;
    const CarWeights& cw = w->w;
    auto copyp = [&](std::vector<const void*>& v, const void* const* src) { v.assign(src, src + d.n_layer); };
    copyp(t->attention_norm, cw.attention_norm); copyp(t->wqkv, cw.wqkv); copyp(t->wo, cw.wo); copyp(t->ffn_norm, cw.ffn_norm);
    copyp(t->w1, cw.w1); copyp(t->w3, cw.w3); copyp(t->w2, cw.w2);
    const int rc = train_carve(t);
    if (rc != CAR_OK) { delete t; return rc; }
    *out = t;
    return CAR_OK;
}

extern "C" int car_train_destroy(CarTrain* t) {
    delete t;
    return CAR_OK;
}

// One TransformerBlock (gpt_t2i.py:303-307) on the fp32 stream t->h, preceded by the control add of gpt_t2i.py:458-460 when the
// block opens a third of the stack.  for_bwd: the recompute of car_train_backward — keeps the block input (after the control
// add) in t->h0, the attention-side norm output in t->x, the feed-forward-side one in t->x2, and stops before w2 (t->h then
// holds the stream between the two halves).
static int tr_block_fwd(CarTrain* t, cudaStream_t st, int l, int B, int n_img, const uint8_t* mask, bool has_feat, bool for_bwd) {
    const CarModelDesc& d = t->d;
    const int L = d.n_layer, dim = d.dim, F = d.ffn_dim, T = d.cls_token_num, H = d.n_head;
    const int n = n_img - 1, S = T + n, R = B * S, RC = B * n_img, step3 = L / 3;
    if (has_feat && l % step3 == 0) {
        CAR_TRY(tr_mlp(st, t->ctok, RC, dim, t->b_ctl1[l / step3], t->b_ctl2[l / step3], dim, t->ctmp, t->cadd));
        CAR_LAUNCH(tr_add_rows_kernel, gsz((long long)RC * dim / 4), 256, 0, st, (float*)t->h, (const bf16*)t->cadd, B, n_img, S, T - 1, dim, TrDrop{});
    }
    if (for_bwd) CAR_CUDA(cudaMemcpyAsync(t->h0, t->h, (size_t)R * dim * 4, cudaMemcpyDeviceToDevice, st));
    size_t att_smem = 0;
    CAR_TRY(tr_attn_smem((size_t)S, (const void*)tr_attention_kernel, &att_smem));
    CAR_LAUNCH(tr_rmsnorm_kernel, R, 256, 0, st, (const float*)t->h, (const float*)t->attention_norm[l], (bf16*)t->x, dim, d.norm_eps, S, S, 0);
    CAR_TRY(gemm(st, dp_plain(t->x, dim, t->b_wqkv[l], dim, R, 3 * dim, dim, t->qkv, 3 * dim)));
    CAR_LAUNCH(rope_kv_write_kernel, sm_count() * 8, 256, 0, st, (const bf16*)t->qkv, t->rope, (bf16*)t->q, (bf16*)t->kc, (bf16*)t->vc, R, S, dim, H, S);
    CAR_LAUNCH(tr_attention_kernel, (unsigned)(((long long)B * H * S + TRA_WARPS - 1) / TRA_WARPS), TRA_WARPS * 32, att_smem, st, (const bf16*)t->q,
               (const bf16*)t->kc, (const bf16*)t->vc, mask, B, H, S, (bf16*)t->att, 1);
    CAR_TRY(gemm(st, dp_plain(t->att, dim, t->b_wo[l], dim, R, dim, dim, t->o, dim)));
    // h += branch output (gpt_t2i.py:305-306) through the branch's dropout and drop path of the last forward's settings
    CAR_LAUNCH(tr_add_rows_kernel, gsz((long long)R * dim / 4), 256, 0, st, (float*)t->h, (const bf16*)t->o, B, S, S, 0, dim,
               tr_drop(t->drop_fwd, CAR_DROP_RESID, l));
    bf16* xn = for_bwd ? t->x2 : t->x;
    CAR_LAUNCH(tr_rmsnorm_kernel, R, 256, 0, st, (const float*)t->h, (const float*)t->ffn_norm[l], xn, dim, d.norm_eps, S, S, 0);
    CAR_TRY(gemm(st, dp_plain(xn, dim, t->b_w1[l], dim, R, F, dim, t->g, F)));
    CAR_TRY(gemm(st, dp_plain(xn, dim, t->b_w3[l], dim, R, F, dim, t->u, F)));
    CAR_LAUNCH(swiglu_kernel, sm_count() * 8, 256, 0, st, (const bf16*)t->g, (const bf16*)t->u, (bf16*)t->act, (long long)R * F);
    if (for_bwd) return CAR_OK;
    CAR_TRY(gemm(st, dp_plain(t->act, F, t->b_w2[l], F, R, dim, F, t->o, dim)));
    CAR_LAUNCH(tr_add_rows_kernel, gsz((long long)R * dim / 4), 256, 0, st, (float*)t->h, (const bf16*)t->o, B, S, S, 0, dim,
               tr_drop(t->drop_fwd, CAR_DROP_FFN, l));
    return CAR_OK;
}

extern "C" int car_train_forward(CarTrain* t, int32_t B, int32_t n_img, const int32_t* idx, const void* cond, const void* feat,
                                 const uint8_t* drop_ids, const uint8_t* mask, const int32_t* targets, const float* valid,
                                 float* logits_out, float* loss_out, void* stream) {
    if (!t || !idx || !cond || !drop_ids) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || B > t->maxB || n_img < 2 || n_img > t->maxN) CAR_FAIL(CAR_ERR_ARG, "batch / token count beyond the capacity given to car_train_create");
    if ((loss_out != nullptr) != (targets != nullptr)) CAR_FAIL(CAR_ERR_ARG, "loss_out and targets go together");
    cudaStream_t st = (cudaStream_t)stream;
    const CarModelDesc& d = t->d;
    const int L = d.n_layer, dim = d.dim, F = d.ffn_dim, V = d.vocab_size, T = d.cls_token_num;
    const int n = n_img - 1, S = T + n, R = B * S, RC = B * n_img;
    if (S > T + d.block_size) CAR_FAIL(CAR_ERR_ARG, "sequence longer than the RoPE table");
    t->fwd_ok = false;
    t->drop_fwd = t->drop_next;
    const TrDrop dtok = tr_drop(t->drop_fwd, CAR_DROP_TOKEN, 0);
    // 0. autocast: bf16 copies of every nn.Linear weight, re-cast each forward (the fp32 masters may have been stepped)
    for (int l = 0; l < L; ++l) {
        CAR_TRY(tr_cast(st, t->wqkv[l], t->b_wqkv[l], (long long)3 * dim * dim)); CAR_TRY(tr_cast(st, t->wo[l], t->b_wo[l], (long long)dim * dim));
        CAR_TRY(tr_cast(st, t->w1[l], t->b_w1[l], (long long)F * dim)); CAR_TRY(tr_cast(st, t->w3[l], t->b_w3[l], (long long)F * dim));
        CAR_TRY(tr_cast(st, t->w2[l], t->b_w2[l], (long long)dim * F));
    }
    CAR_TRY(tr_cast(st, t->w.w.output, t->b_out, (long long)V * dim));
    if (d.model_type == 1) { CAR_TRY(tr_cast(st, t->w.w.cap_fc1, t->b_cap1, (long long)dim * d.caption_dim)); CAR_TRY(tr_cast(st, t->w.w.cap_fc2, t->b_cap2, (long long)dim * dim)); }
    if (feat) {
        CAR_TRY(tr_cast(st, t->w.w.cond_fc1, t->b_cond1, (long long)dim * dim)); CAR_TRY(tr_cast(st, t->w.w.cond_fc2, t->b_cond2, (long long)dim * dim));
        for (int j = 0; j < 3; ++j) { CAR_TRY(tr_cast(st, t->w.w.ctl_fc1[j], t->b_ctl1[j], (long long)dim * dim)); CAR_TRY(tr_cast(st, t->w.w.ctl_fc2[j], t->b_ctl2[j], (long long)dim * dim)); }
        CAR_TRY(tr_cast(st, t->w.adapter_fc1, t->b_ad1, (long long)dim * t->w.adapter_dim)); CAR_TRY(tr_cast(st, t->w.adapter_fc2, t->b_ad2, (long long)dim * dim));
    }
    // 1. prefix rows: CaptionEmbedder (token_drop, cap_proj) gpt_t2i.py:145-162 or LabelEmbedder :78-97; image-token rows :423;
    //    tok_dropout (:430) applied by the writes of both
    if (d.model_type == 1) {
        CAR_LAUNCH(tr_caption_select_kernel, gsz((long long)B * T * d.caption_dim), 256, 0, st, (const float*)cond, (const float*)t->w.cap_uncond,
                   drop_ids, (bf16*)t->capx, B, T, d.caption_dim);
        CAR_TRY(tr_mlp(st, t->capx, B * T, d.caption_dim, t->b_cap1, t->b_cap2, dim, t->ctmp, t->o));
        CAR_LAUNCH(tr_put_rows_bf16_kernel, gsz((long long)B * T * dim / 4), 256, 0, st, (const bf16*)t->o, (float*)t->h, B, T, S, 0, dim, dtok);
    } else {
        CAR_LAUNCH(tr_embed_rows_kernel, B, 256, 0, st, (const float*)t->w.w.label_table, (const int*)cond, 1, drop_ids, t->w.num_classes, (float*)t->h, B, 1, S, 0, dim, dtok);
    }
    CAR_LAUNCH(tr_embed_rows_kernel, B * n, 256, 0, st, (const float*)t->w.w.tok_embeddings, (const int*)idx, n, (const unsigned char*)nullptr, 0, (float*)t->h, B, n, S, T, dim, dtok);
    // 2. control tokens: adapter_mlp -> token_drop -> condition_mlp  gpt_t2i.py:424-427 (feat = the control encoder's output tokens)
    if (feat) {
        CAR_TRY(tr_mlp(st, (const bf16*)feat, RC, t->w.adapter_dim, t->b_ad1, t->b_ad2, dim, t->ctmp, t->cin));
        CAR_LAUNCH(tr_select_uncond_kernel, gsz((long long)RC * dim), 256, 0, st, (bf16*)t->cin, (const float*)t->w.cond_uncond, drop_ids, B, (long long)n_img * dim);
        CAR_TRY(tr_mlp(st, t->cin, RC, dim, t->b_cond1, t->b_cond2, dim, t->ctmp, t->ctok));
    }
    // 3. blocks  gpt_t2i.py:456-468; the stream at every block input is kept for the backward's recompute
    for (int l = 0; l < L; ++l) {
        CAR_CUDA(cudaMemcpyAsync(t->hs + (size_t)l * R * dim, t->h, (size_t)R * dim * 4, cudaMemcpyDeviceToDevice, st));
        CAR_TRY(tr_block_fwd(t, st, l, B, n_img, mask, feat != nullptr, false));
    }
    // 4. head on rows T-1 .. S-1 of every sample (gpt_t2i.py:469-473), loss :474-481
    CAR_LAUNCH(tr_rmsnorm_kernel, RC, 256, 0, st, (const float*)t->h, (const float*)t->w.w.norm, (bf16*)t->x, dim, d.norm_eps, n_img, S, T - 1);
    CAR_TRY(gemm(st, dp_plain(t->x, dim, t->b_out, dim, RC, V, dim, t->lg, V)));
    if (targets) {
        CAR_LAUNCH(tr_ce_rows_kernel, RC, 256, 0, st, (const bf16*)t->lg, (const int*)targets, logits_out, (float*)t->nll, V);
        CAR_LAUNCH(tr_ce_reduce_kernel, 1, 1024, 0, st, (const float*)t->nll, valid, B, n_img, loss_out);
    } else if (logits_out) {
        CAR_LAUNCH(tr_put_rows_bf16_kernel, gsz((long long)RC * V / 4), 256, 0, st, (const bf16*)t->lg, logits_out, 1, RC, RC, 0, V, TrDrop{});
    }
    t->fB = B; t->fN = n_img; t->f_idx = idx; t->f_cond = cond; t->f_feat = feat; t->f_drop = drop_ids; t->f_mask = mask; t->f_targets = targets;
    t->f_valid = valid;
    t->fwd_ok = targets != nullptr;
    return CAR_OK;
}

// RMSNorm backward on `rows` output rows (row map like tr_rmsnorm_kernel) + the weight gradient
static int tr_norm_bwd(CarTrain* t, cudaStream_t st, const float* h, const void* w, const bf16* dy, int rows, int nrows, int S, int row0, float* gw) {
    const int dim = t->d.dim;
    CAR_LAUNCH(tr_rmsnorm_bwd_kernel, rows, 256, 0, st, h, (const float*)w, dy, (float*)t->dh, (float*)t->scr, dim, t->d.norm_eps, nrows, S, row0);
    if (gw) CAR_TRY(tr_colsum(st, t->sc, (const float*)t->scr, rows, dim, gw));
    return CAR_OK;
}
// MLP backward (gpt_t2i.py:177-181: fc2(gelu_tanh(fc1 x)), no bias), recomputing the two intermediates.  dX (optional) = bf16(dT . fc1 (+ resid))
static int tr_mlp_bwd(CarTrain* t, cudaStream_t st, const bf16* x, int rows, int K, const bf16* fc1, const bf16* fc2, const bf16* dY,
                      const bf16* resid, bf16* dX, float* g1, float* g2) {
    const int dim = t->d.dim;
    for (const Buf<bf16>* b : {&t->m_t, &t->m_a, &t->m_da, &t->m_dt}) CAR_TRY(car_fits("tr_mlp_bwd", *b, (size_t)rows * dim));
    CAR_TRY(gemm(st, dp_plain(x, K, fc1, K, rows, dim, K, t->m_t, dim)));
    CAR_LAUNCH(tr_gelu_kernel, gsz((long long)rows * dim), 256, 0, st, (const bf16*)t->m_t, (bf16*)t->m_a, (long long)rows * dim);
    CAR_TRY(tr_wgrad_f32(st, t->sc, dY, t->m_a, rows, dim, dim, g2));
    CAR_TRY(tr_dgrad(st, t->sc, dY, fc2, rows, dim, dim, nullptr, t->m_da));
    CAR_LAUNCH(tr_gelu_bwd_kernel, gsz((long long)rows * dim), 256, 0, st, (const bf16*)t->m_t, (const bf16*)t->m_da, (bf16*)t->m_dt, (long long)rows * dim);
    CAR_TRY(tr_wgrad_f32(st, t->sc, t->m_dt, x, rows, dim, K, g1));
    if (dX) CAR_TRY(tr_dgrad(st, t->sc, t->m_dt, fc1, rows, dim, K, resid, dX));
    return CAR_OK;
}

// Backward of the last car_train_forward(targets != NULL) on this handle: writes d loss / d parameter (fp32, OVERWRITTEN, scaled
// by *loss_grad when given) through the non-NULL pointers of `g` (a CarTrainWeights whose fields point at gradient buffers of the
// parameters' shapes) and d loss / d feat (bf16 [B, n_img, adapter_dim]) when d_feat is given.
extern "C" int car_train_backward(CarTrain* t, const CarTrainWeights* g, void* d_feat, const float* loss_grad, void* stream) {
    if (!t || !g) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (!t->fwd_ok) CAR_FAIL(CAR_ERR_ARG, "car_train_backward needs a preceding car_train_forward with targets on the same handle");
    cudaStream_t st = (cudaStream_t)stream;
    const CarModelDesc& d = t->d;
    const int L = d.n_layer, dim = d.dim, F = d.ffn_dim, V = d.vocab_size, T = d.cls_token_num, H = d.n_head;
    if (dim % 64 != 0 || F % 64 != 0 || V % 64 != 0) CAR_FAIL(CAR_ERR_UNSUPPORTED, "backward: dim, ffn_dim and vocab_size must be multiples of 64");
    const int B = t->fB, n_img = t->fN, n = n_img - 1, S = T + n, R = B * S, RC = B * n_img, step3 = L / 3;
    const bool has_feat = t->f_feat != nullptr;
    const uint8_t* mask = t->f_mask;
    const TrScratch& sc = t->sc;
    size_t smem_q = 0, smem_kv = 0;
    CAR_TRY(tr_attn_smem((size_t)2 * S + 128, (const void*)tr_attn_bwd_q_kernel, &smem_q));
    CAR_TRY(tr_attn_smem((size_t)2 * S + 128, (const void*)tr_attn_bwd_kv_kernel, &smem_kv));
    const unsigned att_grid = (unsigned)(((long long)B * H * S + TRA_WARPS - 1) / TRA_WARPS);
    t->fwd_ok = false;                                         // the recompute below overwrites the forward's buffers
    // ---- head: loss -> logits -> output projection -> final norm (gpt_t2i.py:469-481) ----
    CAR_LAUNCH(tr_rmsnorm_kernel, RC, 256, 0, st, (const float*)t->h, (const float*)t->w.w.norm, (bf16*)t->x, dim, d.norm_eps, n_img, S, T - 1);
    CAR_LAUNCH(tr_ce_grad_kernel, RC, 256, 0, st, (const bf16*)t->lg, (const int*)t->f_targets, t->f_valid, loss_grad, B, n_img, (bf16*)t->dlg, V);
    CAR_TRY(tr_wgrad_f32(st, sc, t->dlg, t->x, RC, V, dim, (float*)g->w.output));
    CAR_TRY(tr_dgrad(st, sc, t->dlg, t->b_out, RC, V, dim, nullptr, t->dx));
    CAR_CUDA(cudaMemsetAsync(t->dh, 0, (size_t)R * dim * 4, st));
    CAR_TRY(tr_norm_bwd(t, st, t->h, t->w.w.norm, t->dx, RC, n_img, S, T - 1, (float*)g->w.norm));
    // ---- blocks, last to first: recompute from the saved input stream, then feed-forward half, attention half, control add ----
    bool first_ctl = true;
    for (int l = L - 1; l >= 0; --l) {
        CAR_CUDA(cudaMemcpyAsync(t->h, t->hs + (size_t)l * R * dim, (size_t)R * dim * 4, cudaMemcpyDeviceToDevice, st));
        CAR_TRY(tr_block_fwd(t, st, l, B, n_img, mask, has_feat, true));
        // feed-forward: h_out = h_mid + drop_path(ffn_dropout(w2(silu(w1 x2) * w3 x2)))
        CAR_LAUNCH(tr_take_rows_bf16_kernel, gsz((long long)R * dim / 4), 256, 0, st, (const float*)t->dh, (bf16*)t->db, B, S, S, 0, dim,
                   tr_drop(t->drop_fwd, CAR_DROP_FFN, l));
        CAR_TRY(tr_wgrad_f32(st, sc, t->db, t->act, R, dim, F, g->w.w2 ? (float*)g->w.w2[l] : nullptr));
        CAR_TRY(tr_dgrad(st, sc, t->db, t->b_w2[l], R, dim, F, nullptr, t->dact));
        CAR_LAUNCH(tr_swiglu_bwd_kernel, sm_count() * 8, 256, 0, st, (const bf16*)t->g, (const bf16*)t->u, (const bf16*)t->dact, (bf16*)t->dg, (bf16*)t->du, (long long)R * F);
        CAR_TRY(tr_wgrad_f32(st, sc, t->dg, t->x2, R, F, dim, g->w.w1 ? (float*)g->w.w1[l] : nullptr));
        CAR_TRY(tr_wgrad_f32(st, sc, t->du, t->x2, R, F, dim, g->w.w3 ? (float*)g->w.w3[l] : nullptr));
        CAR_TRY(tr_dgrad(st, sc, t->dg, t->b_w1[l], R, F, dim, nullptr, t->dx));
        CAR_TRY(tr_dgrad(st, sc, t->du, t->b_w3[l], R, F, dim, t->dx, t->dx));
        CAR_TRY(tr_norm_bwd(t, st, t->h, t->ffn_norm[l], t->dx, R, S, S, 0, g->w.ffn_norm ? (float*)g->w.ffn_norm[l] : nullptr));
        // attention: h_mid = h0 + drop_path(resid_dropout(wo(sdpa(rope(wqkv x1)))))
        CAR_LAUNCH(tr_take_rows_bf16_kernel, gsz((long long)R * dim / 4), 256, 0, st, (const float*)t->dh, (bf16*)t->db, B, S, S, 0, dim,
                   tr_drop(t->drop_fwd, CAR_DROP_RESID, l));
        CAR_TRY(tr_wgrad_f32(st, sc, t->db, t->att, R, dim, dim, g->w.wo ? (float*)g->w.wo[l] : nullptr));
        CAR_TRY(tr_dgrad(st, sc, t->db, t->b_wo[l], R, dim, dim, nullptr, t->datt));
        CAR_LAUNCH(tr_attn_bwd_q_kernel, att_grid, TRA_WARPS * 32, smem_q, st, (const bf16*)t->q, (const bf16*)t->kc, (const bf16*)t->vc, mask,
                   (const bf16*)t->datt, B, H, S, (float*)t->lse, (float*)t->dsum, (bf16*)t->dq, 1);
        CAR_LAUNCH(tr_attn_bwd_kv_kernel, att_grid, TRA_WARPS * 32, smem_kv, st, (const bf16*)t->q, (const bf16*)t->kc, (const bf16*)t->vc, mask,
                   (const bf16*)t->datt, (const float*)t->lse, (const float*)t->dsum, B, H, S, (bf16*)t->dk, (bf16*)t->dv, 1);
        CAR_LAUNCH(tr_rope_bwd_kernel, sm_count() * 8, 256, 0, st, (const bf16*)t->dq, (const bf16*)t->dk, (const bf16*)t->dv, t->rope, (bf16*)t->dqkv, R, S, dim, H, S);
        CAR_TRY(tr_wgrad_f32(st, sc, t->dqkv, t->x, R, 3 * dim, dim, g->w.wqkv ? (float*)g->w.wqkv[l] : nullptr));
        CAR_TRY(tr_dgrad(st, sc, t->dqkv, t->b_wqkv[l], R, 3 * dim, dim, nullptr, t->dx));
        CAR_TRY(tr_norm_bwd(t, st, t->h0, t->attention_norm[l], t->dx, R, S, S, 0, g->w.attention_norm ? (float*)g->w.attention_norm[l] : nullptr));
        // control add h[:, T-1:] += condition_layers[j](condition_token)
        if (has_feat && l % step3 == 0) {
            const int j = l / step3;
            CAR_TRY(car_fits("car_train_backward", t->dadd, (size_t)RC * dim));
            CAR_LAUNCH(tr_take_rows_bf16_kernel, gsz((long long)RC * dim / 4), 256, 0, st, (const float*)t->dh, (bf16*)t->dadd, B, n_img, S, T - 1, dim,
                       TrDrop{});
            CAR_TRY(tr_mlp_bwd(t, st, t->ctok, RC, dim, t->b_ctl1[j], t->b_ctl2[j], t->dadd, first_ctl ? nullptr : (const bf16*)t->dctok, t->dctok,
                               (float*)g->w.ctl_fc1[j], (float*)g->w.ctl_fc2[j]));
            first_ctl = false;
        }
    }
    // ---- embeddings and the prefix / control front ends; dh is the gradient of tok_dropout's output, its mask applies first ----
    const TrDrop dtok = tr_drop(t->drop_fwd, CAR_DROP_TOKEN, 0);
    if (g->w.tok_embeddings) {
        CAR_CUDA(cudaMemsetAsync((void*)g->w.tok_embeddings, 0, (size_t)V * dim * 4, st));
        CAR_LAUNCH(tr_embed_grad_kernel, B * n, 256, 0, st, (const float*)t->dh, (const int*)t->f_idx, n, (const unsigned char*)nullptr, 0,
                   (float*)g->w.tok_embeddings, B, n, S, T, dim, dtok);
    }
    if (d.model_type == 1) {
        CAR_TRY(car_fits("car_train_backward", t->dadd, (size_t)B * T * dim));
        CAR_LAUNCH(tr_take_rows_bf16_kernel, gsz((long long)B * T * dim / 4), 256, 0, st, (const float*)t->dh, (bf16*)t->dadd, B, T, S, 0, dim, dtok);
        CAR_TRY(tr_mlp_bwd(t, st, t->capx, B * T, d.caption_dim, t->b_cap1, t->b_cap2, t->dadd, nullptr, nullptr, (float*)g->w.cap_fc1, (float*)g->w.cap_fc2));
    } else if (g->w.label_table) {
        CAR_CUDA(cudaMemsetAsync((void*)g->w.label_table, 0, (size_t)(t->w.num_classes + 1) * dim * 4, st));
        CAR_LAUNCH(tr_embed_grad_kernel, B, 256, 0, st, (const float*)t->dh, (const int*)t->f_cond, 1, t->f_drop, t->w.num_classes,
                   (float*)g->w.label_table, B, 1, S, 0, dim, dtok);
    }
    if (has_feat) {
        CAR_TRY(tr_mlp_bwd(t, st, t->cin, RC, dim, t->b_cond1, t->b_cond2, t->dctok, nullptr, t->dcin, (float*)g->w.cond_fc1, (float*)g->w.cond_fc2));
        CAR_LAUNCH(tr_zero_dropped_kernel, gsz((long long)RC * dim), 256, 0, st, (bf16*)t->dcin, t->f_drop, B, (long long)n_img * dim);
        CAR_TRY(tr_mlp_bwd(t, st, (const bf16*)t->f_feat, RC, t->w.adapter_dim, t->b_ad1, t->b_ad2, t->dcin, nullptr, (bf16*)d_feat,
                           (float*)g->adapter_fc1, (float*)g->adapter_fc2));
    }
    return CAR_OK;
}

static bool tr_prob_ok(float p) { return p >= 0.f && p < 1.f; }           // (false for NaN)

// dropout settings of the next car_train_forward; every check happens before the handle is touched
extern "C" int car_train_set_dropout(CarTrain* t, const CarTrainDropout* cfg) {
    if (!t) CAR_FAIL(CAR_ERR_ARG, "null argument");
    CarTrain::DropCfg c;
    if (cfg) {
        if (!tr_prob_ok(cfg->token_p) || !tr_prob_ok(cfg->resid_p) || !tr_prob_ok(cfg->ffn_p))
            CAR_FAIL(CAR_ERR_ARG, "dropout probabilities must lie in [0, 1)");
        if (cfg->n_layer < 0 || (cfg->drop_path == nullptr) != (cfg->n_layer == 0))
            CAR_FAIL(CAR_ERR_ARG, "drop_path and n_layer go together");
        bool any = cfg->token_p > 0.f || cfg->resid_p > 0.f || cfg->ffn_p > 0.f;
        for (int l = 0; l < cfg->n_layer; ++l) {
            if (!tr_prob_ok(cfg->drop_path[l])) CAR_FAIL(CAR_ERR_ARG, "drop-path rates must lie in [0, 1)");
            any = any || cfg->drop_path[l] > 0.f;
        }
        if (any && cfg->seed == nullptr) CAR_FAIL(CAR_ERR_ARG, "dropout needs a device seed");
        c.tok_p = cfg->token_p; c.resid_p = cfg->resid_p; c.ffn_p = cfg->ffn_p;
        if (cfg->drop_path) c.path.assign(cfg->drop_path, cfg->drop_path + cfg->n_layer);
        c.seed = any ? cfg->seed : nullptr;
    }
    if (!c.path.empty() && (int)c.path.size() != t->d.n_layer) CAR_FAIL(CAR_ERR_ARG, "drop_path needs one rate per layer");
    t->drop_next = c;
    return CAR_OK;
}

extern "C" int car_dropout_keep_mask(const uint64_t* seed_dev, int32_t site, int32_t layer, int32_t B, int32_t rows, int32_t cols, float p,
                                     uint8_t* out, void* stream) {
    if (!seed_dev || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (site < CAR_DROP_TOKEN || site > CAR_DROP_PATH_FFN) CAR_FAIL(CAR_ERR_ARG, "site must be 0 (token) .. 4 (drop path, feed-forward)");
    if (layer < 0 || layer > 0xFFFF || B <= 0 || rows <= 0 || cols <= 0) CAR_FAIL(CAR_ERR_ARG, "bad layer or shape");
    if (!tr_prob_ok(p)) CAR_FAIL(CAR_ERR_ARG, "p must lie in [0, 1)");
    float keep = 1.f, scale;
    tr_keep_scale(p, &keep, &scale);
    CAR_LAUNCH(car_dropout_mask_kernel, gsz((long long)B * rows * cols), 256, 0, (cudaStream_t)stream, seed_dev, site, layer, B, rows, cols, keep, out);
    return CAR_OK;
}

// fused AdamW step over a device-resident tensor table (train.cuh); bias corrections from the step count (1-based)
extern "C" int car_adamw_step(const void* tensors_dev, const void* chunks_dev, int32_t n_chunks, float lr, float beta1, float beta2, float eps,
                              int32_t step, void* stream) {
    if (!tensors_dev || !chunks_dev) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (n_chunks <= 0 || step < 1) CAR_FAIL(CAR_ERR_ARG, "n_chunks must be positive and step 1-based");
    const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
    CAR_LAUNCH(adamw_multi_kernel, n_chunks, 256, 0, (cudaStream_t)stream, (const CarAdamWTensorDev*)tensors_dev, (const int2*)chunks_dev, lr, beta1, beta2,
               eps, bc1, sqrtf(bc2));
    return CAR_OK;
}

// =========================================================================================================
// Trainable control encoder (dino_train.cuh): Dinov2_Adapter / ViT_Adapter forward with fp32 parameters under bf16 autocast, and
// its backward to every encoder parameter.  The fp32 masters are borrowed and re-cast to bf16 by every forward (an optimizer step
// changes them in place); the forward keeps the fp32 stream at every block input, the backward recomputes each block from it.
// =========================================================================================================
struct CarDinoTrain : CarOwned {
    CarDinoDesc d;
    int kpatch, kpad;
    const float *cls, *pos, *patch_w, *patch_b, *ln_w, *ln_b;
    struct Layer { const float *n1w, *n1b, *qw, *qb, *kw, *kb, *vw, *vb, *ow, *ob, *ls1, *n2w, *n2b, *f1w, *f1b, *f2w, *f2b, *ls2;
                   bf16 *w_qkv, *b_qkv, *w_o, *b_o, *w_fc1, *b_fc1, *w_fc2, *b_fc2; };
    std::vector<Layer> L;
    bf16 *w_patch, *b_patch;                 // owned bf16 casts, refreshed by every forward
    int fB = 0, fH = 0, fW = 0;              // shape of the last forward; its backward carves the same workspace
    bool fwd_ok = false;
};

struct DtBufs {
    Buf<bf16> patches, ptok, xn, qkv, q, kc, vc, ctx, o, xn2, pre, act, y2, db, dact, dctx, dq, dk, dv, dqkv, dxn;
    Buf<float> posi, hs, xm, dx, scr, lse, dsum, dposi, ptmp;
    TrScratch sc;
};

// the one list of takes of a forward and of its backward (same shape => same offsets: the saved streams survive in between)
static int dt_carve(CarDinoTrain* m, int B, int h, int w, DtBufs& s) {
    const CarDinoDesc& d = m->d;
    const size_t C = d.hidden, F = 4 * C, hw = (size_t)h * w, rows = (size_t)B * (hw + 1), Rp = (rows + 63) / 64 * 64;
    const size_t KP = m->kpad, BHT = (size_t)B * d.heads * (hw + 1), maxK = std::max(F, KP);
    return m->ws.carve([&](Carve& c) {
        s.patches = c.take<bf16>((size_t)B * hw * KP); s.ptok = c.take<bf16>((size_t)B * hw * C);
        s.posi = c.take<float>(hw * C); s.hs = c.take<float>((size_t)(d.layers + 1) * rows * C); s.xm = c.take<float>(rows * C);
        s.xn = c.take<bf16>(rows * C); s.qkv = c.take<bf16>(rows * 3 * C); s.q = c.take<bf16>(rows * C);
        s.kc = c.take<bf16>(rows * C); s.vc = c.take<bf16>(rows * C); s.ctx = c.take<bf16>(rows * C); s.o = c.take<bf16>(rows * C);
        s.xn2 = c.take<bf16>(rows * C); s.pre = c.take<bf16>(rows * F); s.act = c.take<bf16>(rows * F); s.y2 = c.take<bf16>(rows * C);
        // backward
        s.dx = c.take<float>(rows * C); s.scr = c.take<float>(rows * C); s.sc.part = c.take<float>((size_t)TR_COLSUM_CHUNKS * F);
        s.sc.colv = c.take<float>(F); s.lse = c.take<float>(BHT); s.dsum = c.take<float>(BHT);
        s.dposi = c.take<float>(hw * C); s.ptmp = c.take<float>((size_t)d.pos_grid * w * C);
        s.db = c.take<bf16>(rows * C); s.dact = c.take<bf16>(rows * F); s.dctx = c.take<bf16>(rows * C);
        s.dq = c.take<bf16>(rows * C); s.dk = c.take<bf16>(rows * C); s.dv = c.take<bf16>(rows * C);
        s.dqkv = c.take<bf16>(rows * 3 * C); s.dxn = c.take<bf16>(rows * C);
        s.sc.yT = c.take<bf16>(F * Rp); s.sc.xT = c.take<bf16>(maxK * Rp); s.sc.wT = c.take<bf16>(F * C);
        s.sc.dWb = c.take<bf16>(std::max(F * C, C * KP));
    });
}

// Y [rows][N] bf16 = X [rows][K] . W [N][K]^T + bias (nn.Linear on autocast's bf16 operands)
static int dt_linear(cudaStream_t st, const bf16* X, const bf16* W, const bf16* bias, int rows, int N, int K, bf16* Y) {
    DenseP p = dp_plain(X, K, W, K, rows, N, K, Y, N);
    p.bias = bias;
    return gemm(st, p);
}
// the bias gradients of nn.Linear layers whose bf16 output gradients are the `parts` column blocks of dY [rows][parts * N]
static int dt_bias_grad(cudaStream_t st, const TrScratch& sc, const bf16* dY, int rows, int N, int parts, float* const* dst) {
    bool any = false;
    for (int j = 0; j < parts; ++j) any = any || dst[j];
    if (!any) return CAR_OK;
    CAR_TRY(car_fits("dt_bias_grad", sc.colv, (size_t)parts * N));
    CAR_TRY(tr_colsum(st, sc, dY, rows, parts * N, (float*)sc.colv));
    for (int j = 0; j < parts; ++j)
        if (dst[j]) CAR_LAUNCH(dt_round_bf16_kernel, (N + 255) / 256, 256, 0, st, (const float*)sc.colv + (size_t)j * N, dst[j], N);
    return CAR_OK;
}

extern "C" int car_dino_train_create(const CarDinoDesc* desc, const CarDinoWeights* w, void* stream, CarDinoTrain** out) {
    if (!desc || !w || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    const CarDinoDesc& d = *desc;
    if (d.dtype != CAR_F32) CAR_FAIL(CAR_ERR_UNSUPPORTED, "the trainable encoder takes the fp32 master weights (bf16 autocast is applied inside)");
    if (d.hidden <= 0 || d.hidden % 64 || d.heads * 64 != d.hidden) CAR_FAIL(CAR_ERR_UNSUPPORTED, "head_dim must be 64");
    if (d.patch != 14 && d.patch != 16) CAR_FAIL(CAR_ERR_UNSUPPORTED, "patch size must be 14 (DINOv2) or 16 (ViT-S/16)");
    if (d.layers <= 0 || d.pos_grid <= 0 || (d.resize_mode != 0 && d.resize_mode != 1)) CAR_FAIL(CAR_ERR_ARG, "bad layers, pos_grid or resize_mode");
    if (!w->cls_token || !w->pos_emb || !w->patch_w || !w->patch_b || !w->ln_w || !w->ln_b) CAR_FAIL(CAR_ERR_ARG, "null weight");
    const void* const* arrays[] = {w->n1_w, w->n1_b, w->q_w, w->q_b, w->k_w, w->k_b, w->v_w, w->v_b, w->o_w, w->o_b, w->n2_w, w->n2_b,
                                   w->fc1_w, w->fc1_b, w->fc2_w, w->fc2_b};
    for (const void* const* a : arrays) {
        if (!a) CAR_FAIL(CAR_ERR_ARG, "null weight array");
        for (int l = 0; l < d.layers; ++l) if (!a[l]) CAR_FAIL(CAR_ERR_ARG, "null weight");
    }
    if ((w->ls1 == nullptr) != (w->ls2 == nullptr)) CAR_FAIL(CAR_ERR_ARG, "ls1 and ls2 go together (both NULL: no LayerScale, ViT)");
    for (int l = 0; w->ls1 && l < d.layers; ++l) if (!w->ls1[l] || !w->ls2[l]) CAR_FAIL(CAR_ERR_ARG, "null weight");
    (void)stream;
    CarDinoTrain* m = new CarDinoTrain();
    m->d = d;
    const size_t C = d.hidden;
    m->kpatch = 3 * d.patch * d.patch;
    m->kpad = (m->kpatch + 31) & ~31;
    m->cls = (const float*)w->cls_token; m->pos = (const float*)w->pos_emb; m->patch_w = (const float*)w->patch_w;
    m->patch_b = (const float*)w->patch_b; m->ln_w = (const float*)w->ln_w; m->ln_b = (const float*)w->ln_b;
    int r = m->alloc(&m->w_patch, C * m->kpad * 2);
    if (r == CAR_OK) r = m->alloc(&m->b_patch, C * 2);
    m->L.resize(d.layers);
    for (int l = 0; l < d.layers && r == CAR_OK; ++l) {
        CarDinoTrain::Layer& Ly = m->L[l];
        auto f = [&](const void* const* a) { return a ? (const float*)a[l] : nullptr; };
        Ly.n1w = f(w->n1_w); Ly.n1b = f(w->n1_b); Ly.qw = f(w->q_w); Ly.qb = f(w->q_b); Ly.kw = f(w->k_w); Ly.kb = f(w->k_b);
        Ly.vw = f(w->v_w); Ly.vb = f(w->v_b); Ly.ow = f(w->o_w); Ly.ob = f(w->o_b); Ly.ls1 = f(w->ls1); Ly.n2w = f(w->n2_w);
        Ly.n2b = f(w->n2_b); Ly.f1w = f(w->fc1_w); Ly.f1b = f(w->fc1_b); Ly.f2w = f(w->fc2_w); Ly.f2b = f(w->fc2_b); Ly.ls2 = f(w->ls2);
        r = m->alloc(&Ly.w_qkv, 3 * C * C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.b_qkv, 3 * C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.w_o, C * C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.b_o, C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.w_fc1, 4 * C * C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.b_fc1, 4 * C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.w_fc2, 4 * C * C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.b_fc2, C * 2);
    }
    if (r != CAR_OK) { delete m; return r; }
    *out = m;
    return CAR_OK;
}

extern "C" int car_dino_train_destroy(CarDinoTrain* m) {
    delete m;
    return CAR_OK;
}

// One encoder block (Dinov2Layer.forward / ViTLayer.forward) on the fp32 stream x [B*Tn][C].  for_bwd: the backward's recompute —
// stops after fc2, before the second residual add (x then holds the stream between the two halves).
static int dt_block(CarDinoTrain* m, cudaStream_t st, DtBufs& s, int l, int B, int Tn, float* x, bool for_bwd) {
    const CarDinoDesc& d = m->d;
    const CarDinoTrain::Layer& Ly = m->L[l];
    const int C = d.hidden, F = 4 * C, H = d.heads, rows = B * Tn;
    size_t smem = 0;
    CAR_TRY(tr_attn_smem((size_t)Tn, (const void*)tr_attention_kernel, &smem));
    CAR_LAUNCH(dt_layernorm_kernel, rows, 128, 0, st, (const float*)x, Ly.n1w, Ly.n1b, (bf16*)s.xn, (float*)nullptr, C, d.eps, Tn, Tn, 0);
    CAR_TRY(dt_linear(st, s.xn, Ly.w_qkv, Ly.b_qkv, rows, 3 * C, C, s.qkv));
    CAR_LAUNCH(rope_kv_write_kernel, sm_count() * 8, 256, 0, st, (const bf16*)s.qkv, (const float*)nullptr, (bf16*)s.q, (bf16*)s.kc, (bf16*)s.vc,
               rows, Tn, C, H, Tn);
    CAR_LAUNCH(tr_attention_kernel, (unsigned)(((long long)B * H * Tn + TRA_WARPS - 1) / TRA_WARPS), TRA_WARPS * 32, smem, st, (const bf16*)s.q,
               (const bf16*)s.kc, (const bf16*)s.vc, (const unsigned char*)nullptr, B, H, Tn, (bf16*)s.ctx, 0);
    CAR_TRY(dt_linear(st, s.ctx, Ly.w_o, Ly.b_o, rows, C, C, s.o));
    CAR_LAUNCH(dt_layerscale_add_kernel, gsz((long long)rows * C), 256, 0, st, x, (const bf16*)s.o, Ly.ls1, (long long)rows * C, C);
    CAR_LAUNCH(dt_layernorm_kernel, rows, 128, 0, st, (const float*)x, Ly.n2w, Ly.n2b, (bf16*)s.xn2, (float*)nullptr, C, d.eps, Tn, Tn, 0);
    CAR_TRY(dt_linear(st, s.xn2, Ly.w_fc1, Ly.b_fc1, rows, F, C, s.pre));
    CAR_LAUNCH(dt_gelu_erf_kernel, gsz((long long)rows * F), 256, 0, st, (const bf16*)s.pre, (bf16*)s.act, (long long)rows * F);
    CAR_TRY(dt_linear(st, s.act, Ly.w_fc2, Ly.b_fc2, rows, C, F, s.y2));
    if (!for_bwd) CAR_LAUNCH(dt_layerscale_add_kernel, gsz((long long)rows * C), 256, 0, st, x, (const bf16*)s.y2, Ly.ls2, (long long)rows * C, C);
    return CAR_OK;
}

// image fp32 [B,3,H,W] -> feat fp32 [B, (H/16)(W/16), hidden] (last_hidden_state without the CLS row)
extern "C" int car_dino_train_forward(CarDinoTrain* m, const float* image, int32_t B, int32_t H, int32_t W, float* feat, void* stream) {
    if (!m || !image || !feat) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || H <= 0 || W <= 0 || H % 16 || W % 16) CAR_FAIL(CAR_ERR_ARG, "B must be positive, H and W positive multiples of 16");
    cudaStream_t st = (cudaStream_t)stream;
    const CarDinoDesc& d = m->d;
    const int C = d.hidden, F = 4 * C, h = H / 16, w = W / 16, hw = h * w, Tn = hw + 1, rows = B * Tn, KP = m->kpad;
    m->fwd_ok = false;
    DtBufs s;
    CAR_TRY(dt_carve(m, B, h, w, s));
    // 0. autocast: bf16 copies of the patch projection and of every nn.Linear (weights and biases), re-cast every forward
    CAR_LAUNCH(dt_cast_pad_kernel, gsz((long long)C * KP), 256, 0, st, m->patch_w, m->w_patch, C, m->kpatch, KP);
    CAR_TRY(tr_cast(st, m->patch_b, m->b_patch, C));
    const long long CC = (long long)C * C;
    for (const CarDinoTrain::Layer& Ly : m->L) {
        CAR_TRY(tr_cast(st, Ly.qw, Ly.w_qkv, CC)); CAR_TRY(tr_cast(st, Ly.kw, Ly.w_qkv + CC, CC)); CAR_TRY(tr_cast(st, Ly.vw, Ly.w_qkv + 2 * CC, CC));
        CAR_TRY(tr_cast(st, Ly.qb, Ly.b_qkv, C)); CAR_TRY(tr_cast(st, Ly.kb, Ly.b_qkv + C, C)); CAR_TRY(tr_cast(st, Ly.vb, Ly.b_qkv + 2 * C, C));
        CAR_TRY(tr_cast(st, Ly.ow, Ly.w_o, CC)); CAR_TRY(tr_cast(st, Ly.ob, Ly.b_o, C));
        CAR_TRY(tr_cast(st, Ly.f1w, Ly.w_fc1, 4 * CC)); CAR_TRY(tr_cast(st, Ly.f1b, Ly.b_fc1, F));
        CAR_TRY(tr_cast(st, Ly.f2w, Ly.w_fc2, 4 * CC)); CAR_TRY(tr_cast(st, Ly.f2b, Ly.b_fc2, C));
    }
    // 1. resize (fp32) + patchify, patch projection on bf16 operands (dinov2_adapter.py:16-24, Dinov2PatchEmbeddings)
    CAR_LAUNCH((resize_patchify_kernel<float>), gsz((long long)B * hw * KP), 256, 0, st, image, (bf16*)s.patches, B, H, W, h, w, KP, d.resize_mode, d.patch);
    {
        DenseP p = dp_plain(s.patches, KP, m->w_patch, KP, B * hw, C, KP, (bf16*)s.ptok, C);
        p.bias = m->b_patch;
        CAR_TRY(gemm(st, p));
    }
    // 2. CLS row + fp32 bicubic position embeddings -> the fp32 stream hs[0]
    CAR_LAUNCH((pos_embed_interp_kernel<float, float>), gsz((long long)hw * C), 256, 0, st, m->pos, (float*)s.posi, d.pos_grid, h, w, C);
    CAR_LAUNCH(dt_assemble_kernel, gsz((long long)rows * C), 256, 0, st, (const bf16*)s.ptok, m->cls, m->pos, (const float*)s.posi, (float*)s.hs, B, hw, C);
    // 3. blocks: hs[l + 1] = block_l(hs[l])
    const size_t RC = (size_t)rows * C;
    for (int l = 0; l < d.layers; ++l) {
        float* x = s.hs + (size_t)(l + 1) * RC;
        CAR_CUDA(cudaMemcpyAsync(x, s.hs + (size_t)l * RC, RC * 4, cudaMemcpyDeviceToDevice, st));
        CAR_TRY(dt_block(m, st, s, l, B, Tn, x, false));
    }
    // 4. final LayerNorm on the patch rows (dinov2_adapter.py:29 drops the CLS row)
    CAR_LAUNCH(dt_layernorm_kernel, B * hw, 128, 0, st, (const float*)(s.hs + (size_t)d.layers * RC), m->ln_w, m->ln_b, (bf16*)nullptr, feat, C, d.eps,
               hw, Tn, 1);
    m->fB = B; m->fH = h; m->fW = w;
    m->fwd_ok = true;
    return CAR_OK;
}

// Backward of the last car_dino_train_forward on this handle from d_feat (fp32, the forward's feat shape): writes d loss / d parameter
// (fp32, OVERWRITTEN) through the non-NULL pointers of `g` (a CarDinoWeights whose fields point at gradient buffers of the
// parameters' shapes; NULL skips a tensor).
extern "C" int car_dino_train_backward(CarDinoTrain* m, const float* d_feat, const CarDinoWeights* g, void* stream) {
    if (!m || !d_feat || !g) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (!m->fwd_ok) CAR_FAIL(CAR_ERR_STATE, "car_dino_train_backward needs a preceding car_dino_train_forward on the same handle");
    cudaStream_t st = (cudaStream_t)stream;
    const CarDinoDesc& d = m->d;
    const int B = m->fB, h = m->fH, w = m->fW, C = d.hidden, F = 4 * C, H = d.heads, hw = h * w, Tn = hw + 1, rows = B * Tn, G = d.pos_grid;
    const size_t RC = (size_t)rows * C, CC = (size_t)C * C;
    DtBufs s;
    CAR_TRY(dt_carve(m, B, h, w, s));
    const TrScratch& sc = s.sc;
    m->fwd_ok = false;                                          // the recompute below overwrites the forward's buffers
    size_t smem_q = 0, smem_kv = 0;
    CAR_TRY(tr_attn_smem((size_t)2 * Tn + 128, (const void*)tr_attn_bwd_q_kernel, &smem_q));
    CAR_TRY(tr_attn_smem((size_t)2 * Tn + 128, (const void*)tr_attn_bwd_kv_kernel, &smem_kv));
    const unsigned att_grid = (unsigned)(((long long)B * H * Tn + TRA_WARPS - 1) / TRA_WARPS);
    auto at = [](const void* const* a, int l) { return a ? (float*)a[l] : (float*)nullptr; };
    // final LayerNorm
    CAR_CUDA(cudaMemsetAsync(s.dx, 0, RC * 4, st));
    CAR_LAUNCH(dt_layernorm_bwd_kernel<float>, B * hw, 128, 0, st, (const float*)(s.hs + (size_t)d.layers * RC), m->ln_w, d_feat, (float*)s.dx,
               (float*)s.scr, C, d.eps, hw, Tn, 1);
    if (g->ln_w) CAR_TRY(tr_colsum(st, sc, (const float*)s.scr, B * hw, C, (float*)g->ln_w));
    if (g->ln_b) CAR_TRY(tr_colsum(st, sc, d_feat, B * hw, C, (float*)g->ln_b));
    for (int l = d.layers - 1; l >= 0; --l) {
        const CarDinoTrain::Layer& Ly = m->L[l];
        const float* x0 = s.hs + (size_t)l * RC;
        CAR_CUDA(cudaMemcpyAsync(s.xm, x0, RC * 4, cudaMemcpyDeviceToDevice, st));
        CAR_TRY(dt_block(m, st, s, l, B, Tn, s.xm, true));
        // feed-forward half: x_out = x_mid + ls2 * fc2(gelu(fc1(norm2(x_mid))))
        CAR_LAUNCH(dt_layerscale_bwd_kernel, gsz((long long)RC), 256, 0, st, (const float*)s.dx, (const bf16*)s.y2, Ly.ls2, (bf16*)s.db,
                   at(g->ls2, l) ? (float*)s.scr : (float*)nullptr, (long long)RC, C);
        if (at(g->ls2, l)) CAR_TRY(tr_colsum(st, sc, (const float*)s.scr, rows, C, at(g->ls2, l)));
        CAR_TRY(tr_wgrad_f32(st, sc, s.db, s.act, rows, C, F, at(g->fc2_w, l)));
        { float* b[1] = {at(g->fc2_b, l)}; CAR_TRY(dt_bias_grad(st, sc, s.db, rows, C, 1, b)); }
        CAR_TRY(tr_dgrad(st, sc, s.db, Ly.w_fc2, rows, C, F, nullptr, s.dact));
        CAR_LAUNCH(dt_gelu_erf_bwd_kernel, gsz((long long)rows * F), 256, 0, st, (const bf16*)s.pre, (const bf16*)s.dact, (bf16*)s.dact, (long long)rows * F);
        CAR_TRY(tr_wgrad_f32(st, sc, s.dact, s.xn2, rows, F, C, at(g->fc1_w, l)));
        { float* b[1] = {at(g->fc1_b, l)}; CAR_TRY(dt_bias_grad(st, sc, s.dact, rows, F, 1, b)); }
        CAR_TRY(tr_dgrad(st, sc, s.dact, Ly.w_fc1, rows, F, C, nullptr, s.dxn));
        CAR_LAUNCH(dt_layernorm_bwd_kernel<bf16>, rows, 128, 0, st, (const float*)s.xm, Ly.n2w, (const bf16*)s.dxn, (float*)s.dx, (float*)s.scr, C, d.eps,
                   Tn, Tn, 0);
        if (at(g->n2_w, l)) CAR_TRY(tr_colsum(st, sc, (const float*)s.scr, rows, C, at(g->n2_w, l)));
        if (at(g->n2_b, l)) CAR_TRY(tr_colsum(st, sc, (const bf16*)s.dxn, rows, C, at(g->n2_b, l)));
        // attention half: x_mid = x0 + ls1 * o(sdpa(q, k, v)(norm1(x0)))
        CAR_LAUNCH(dt_layerscale_bwd_kernel, gsz((long long)RC), 256, 0, st, (const float*)s.dx, (const bf16*)s.o, Ly.ls1, (bf16*)s.db,
                   at(g->ls1, l) ? (float*)s.scr : (float*)nullptr, (long long)RC, C);
        if (at(g->ls1, l)) CAR_TRY(tr_colsum(st, sc, (const float*)s.scr, rows, C, at(g->ls1, l)));
        CAR_TRY(tr_wgrad_f32(st, sc, s.db, s.ctx, rows, C, C, at(g->o_w, l)));
        { float* b[1] = {at(g->o_b, l)}; CAR_TRY(dt_bias_grad(st, sc, s.db, rows, C, 1, b)); }
        CAR_TRY(tr_dgrad(st, sc, s.db, Ly.w_o, rows, C, C, nullptr, s.dctx));
        CAR_LAUNCH(tr_attn_bwd_q_kernel, att_grid, TRA_WARPS * 32, smem_q, st, (const bf16*)s.q, (const bf16*)s.kc, (const bf16*)s.vc,
                   (const unsigned char*)nullptr, (const bf16*)s.dctx, B, H, Tn, (float*)s.lse, (float*)s.dsum, (bf16*)s.dq, 0);
        CAR_LAUNCH(tr_attn_bwd_kv_kernel, att_grid, TRA_WARPS * 32, smem_kv, st, (const bf16*)s.q, (const bf16*)s.kc, (const bf16*)s.vc,
                   (const unsigned char*)nullptr, (const bf16*)s.dctx, (const float*)s.lse, (const float*)s.dsum, B, H, Tn, (bf16*)s.dk, (bf16*)s.dv, 0);
        CAR_LAUNCH(tr_rope_bwd_kernel, sm_count() * 8, 256, 0, st, (const bf16*)s.dq, (const bf16*)s.dk, (const bf16*)s.dv, (const float*)nullptr,
                   (bf16*)s.dqkv, rows, Tn, C, H, Tn);
        if (at(g->q_w, l) || at(g->k_w, l) || at(g->v_w, l)) {
            CAR_TRY(tr_wgrad(st, sc, s.dqkv, s.xn, rows, 3 * C, C));
            CAR_TRY(tr_weight_grad(st, sc, 0, C, C, C, at(g->q_w, l)));
            CAR_TRY(tr_weight_grad(st, sc, CC, C, C, C, at(g->k_w, l)));
            CAR_TRY(tr_weight_grad(st, sc, 2 * CC, C, C, C, at(g->v_w, l)));
        }
        { float* b[3] = {at(g->q_b, l), at(g->k_b, l), at(g->v_b, l)}; CAR_TRY(dt_bias_grad(st, sc, s.dqkv, rows, C, 3, b)); }
        CAR_TRY(tr_dgrad(st, sc, s.dqkv, Ly.w_qkv, rows, 3 * C, C, nullptr, s.dxn));
        CAR_LAUNCH(dt_layernorm_bwd_kernel<bf16>, rows, 128, 0, st, x0, Ly.n1w, (const bf16*)s.dxn, (float*)s.dx, (float*)s.scr, C, d.eps, Tn, Tn, 0);
        if (at(g->n1_w, l)) CAR_TRY(tr_colsum(st, sc, (const float*)s.scr, rows, C, at(g->n1_w, l)));
        if (at(g->n1_b, l)) CAR_TRY(tr_colsum(st, sc, (const bf16*)s.dxn, rows, C, at(g->n1_b, l)));
    }
    // embeddings: CLS row and position table (fp32), patch tokens (bf16 gradient of the cast) -> patch projection
    float* dpos = (float*)g->pos_emb;
    CAR_LAUNCH(dt_embed_bwd_kernel, gsz((long long)Tn * C), 256, 0, st, (const float*)s.dx, (float*)g->cls_token, dpos,
               dpos ? (float*)s.dposi : (float*)nullptr, B, Tn, C);
    if (dpos) {
        CAR_LAUNCH(dt_cubic_t_kernel, gsz((long long)G * w * C), 256, 0, st, (const float*)s.dposi, (float*)s.ptmp, G, h, 1, w * C);
        CAR_LAUNCH(dt_cubic_t_kernel, gsz((long long)G * G * C), 256, 0, st, (const float*)s.ptmp, dpos + C, G, w, G, C);
    }
    if (g->patch_w || g->patch_b) {
        CAR_LAUNCH(tr_take_rows_bf16_kernel, gsz((long long)B * hw * C / 4), 256, 0, st, (const float*)s.dx, (bf16*)s.db, B, hw, Tn, 1, C, TrDrop{});
        if (g->patch_w) {
            CAR_TRY(tr_wgrad(st, sc, s.db, s.patches, B * hw, C, m->kpad));
            CAR_TRY(tr_weight_grad(st, sc, 0, C, m->kpatch, m->kpad, (float*)g->patch_w));
        }
        float* b[1] = {(float*)g->patch_b};
        CAR_TRY(dt_bias_grad(st, sc, s.db, B * hw, C, 1, b));
    }
    return CAR_OK;
}
