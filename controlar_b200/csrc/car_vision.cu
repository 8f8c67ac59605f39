// car_vision.cu — C-ABI entry points for the control encoder (DINOv2) and the VQGAN tokenizer.
#include <vector>
#include <cstdio>
#include <algorithm>

#include "common.cuh"
#include "gemm.h"
#include "vision.cuh"
#include "frontend.cuh"
#include "lineart.cuh"
#include "dpt.cuh"
#include "midas.cuh"
#include "groupnorm.cuh"

template <typename... KArgs, typename... Args>
static int launch_on(cudaStream_t st, void (*kernel)(KArgs...), unsigned grid, unsigned block, Args... args) {
    CAR_LAUNCH(kernel, grid, block, 0, st, args...);
    return CAR_OK;
}

// A split-bf16 weight of the fp32-grade networks (split3.cuh): W3 bf16 [n][kh][kw][cin3] = [ w_hi | w_hi | w_lo ] per tap, cin3 =
// 3 x the padded input channels (the channels per pixel of its S3 source), and the fp32 bias [n] (null: none)
struct X3W { bf16* w; const float* b; int n, cin3, kh, kw; };

// Reader of the flat tensor list a create call takes (device pointers in state-dict order, fp32), copying and packing each tensor
// into memory the handle owns.  The list comes from the caller: the constructor refuses a null entry before any CUDA call, and every
// read is bounds-checked.  The first error sticks — later calls allocate, copy and launch nothing, and return null — and finish()
// returns it; messages name the entry point `fn`.
struct TensorReader {
    const char* fn;
    const void* const* t;
    int n, i = 0, rc = CAR_OK;
    cudaStream_t st;
    CarOwned* m;

    TensorReader(const char* fn, const void* const* t, int n, void* stream, CarOwned* m)
        : fn(fn), t(t), n(n), st((cudaStream_t)stream), m(m) {
        for (int k = 0; k < n && rc == CAR_OK; ++k)
            if (!t[k]) fail(CAR_ERR_ARG, "null tensor");
    }
    bool ok() const { return rc == CAR_OK; }
    void fail(int code, const std::string& msg) {
        if (rc != CAR_OK) return;
        rc = code;
        g_car_err = std::string(fn) + ": " + msg;
    }
    void cuda(cudaError_t e, const char* what) {
        if (e != cudaSuccess) fail(CAR_ERR_CUDA, std::string(what) + " -> " + cudaGetErrorString(e));
    }
    const float* next() {
        if (ok() && i >= n) fail(CAR_ERR_ARG, "tensor list too short");
        return ok() ? (const float*)t[i++] : nullptr;
    }
    void skip(int k) {
        for (int j = 0; j < k; ++j) next();
    }
    void* alloc(size_t bytes) {
        void* p = nullptr;
        if (ok() && m->alloc(&p, bytes) != CAR_OK) fail(CAR_ERR_CUDA, g_car_err);
        return ok() ? p : nullptr;
    }
    void copy(float* dst, const float* src, long long count) {
        if (ok()) cuda(cudaMemcpyAsync(dst, src, (size_t)count * 4, cudaMemcpyDeviceToDevice, st), "copy");
    }
    template <typename... KArgs, typename... Args> void launch(void (*kernel)(KArgs...), unsigned grid, unsigned block, Args... args) {
        if (ok() && launch_on(st, kernel, grid, block, args...) != CAR_OK) fail(CAR_ERR_CUDA, g_car_err);
    }
    // one launch of a grid-stride packing kernel over `total` elements
    template <typename... KArgs, typename... Args> void pack(void (*kernel)(KArgs...), long long total, Args... args) {
        if (ok()) launch(kernel, gsz(total), 256, args...);
    }
    float* f32(const float* src, long long count) {
        float* p = (float*)alloc((size_t)count * 4);
        copy(p, src, count);
        return p;
    }
    float* f32(long long count) { return f32(next(), count); }
    float* zeros(long long count) {
        float* p = (float*)alloc((size_t)count * 4);
        if (ok()) cuda(cudaMemsetAsync(p, 0, (size_t)count * 4, st), "memset");
        return p;
    }
    // split-bf16 weight: fp32 [n][cin][k][k] at src -> W3 [n][k][k][3 cin_pad], with the fp32 bias b
    X3W x3(const float* src, int n, int cin, int k, int cin_pad, const float* b) {
        const long long n3 = (long long)n * k * k * cin_pad;
        X3W w{(bf16*)alloc((size_t)n3 * 3 * 2), b, n, 3 * cin_pad, k, k};
        pack(conv_weight_pack_x3_kernel, n3, src, w.w, n, cin, k, k, cin_pad);
        return w;
    }
    // the next tensor as a split-bf16 weight, then (bias) the one after it as its bias
    X3W x3(int n, int cin, int k, int cin_pad, bool bias = true) {
        X3W w = x3(next(), n, cin, k, cin_pad, nullptr);
        if (bias) w.b = f32(n);
        return w;
    }
    // the create's last step: the whole list was read and nothing failed
    int finish() {
        if (ok() && i != n) fail(CAR_ERR_ARG, "tensor list length does not match the architecture");
        return rc;
    }
};

// =========================================================================================================
// DINOv2 control encoder
// =========================================================================================================
struct CarDino : CarOwned {
    CarDinoDesc d;
    // bf16 GEMM-ready weights
    bf16* w_patch;                      // [C][kpad]  (k = 3 * patch^2 = 588 -> 608 for DINOv2, 768 for ViT-S/16)
    int kpatch, kpad;
    const void *b_patch, *cls, *pos, *ln_w, *ln_b;
    struct Layer { bf16 *w_qk, *b_qk, *w_v; const void *b_v, *w_o, *b_o, *ls1, *ls2, *n1w, *n1b, *n2w, *n2b, *w_fc1, *b_fc1, *w_fc2, *b_fc2; };
    std::vector<Layer> L;
    bf16 *ad_fc1, *ad_fc2;              // adapter_mlp (bias-free)
    int ad_dim;
};

template <typename TI>
static int to_bf16(cudaStream_t st, CarOwned* m, const void* src, long long n, bf16** dst) {
    CAR_TRY(m->alloc(dst, (size_t)n * 2));
    CAR_LAUNCH((cast_to_bf16_kernel<TI>), gsz(n), 256, 0, st, (const TI*)src, *dst, n);
    return CAR_OK;
}
static int to_bf16_any(cudaStream_t st, int dtype, CarOwned* m, const void* src, long long n, bf16** dst) {
    return dtype == CAR_BF16 ? to_bf16<bf16>(st, m, src, n, dst) : to_bf16<float>(st, m, src, n, dst);
}

extern "C" int car_dino_create(const CarDinoDesc* desc, const CarDinoWeights* w, void* stream, CarDino** out) {
    if (!desc || !w || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    const CarDinoDesc& d = *desc;
    if (d.hidden % 64 || d.heads * 64 != d.hidden) CAR_FAIL(CAR_ERR_UNSUPPORTED, "DINOv2 head_dim must be 64");
    if (d.patch != 14 && d.patch != 16) CAR_FAIL(CAR_ERR_UNSUPPORTED, "patch size must be 14 (DINOv2) or 16 (ViT-S/16)");
    cudaStream_t st = (cudaStream_t)stream;
    CarDino* m = new CarDino();
    m->d = d;
    const int C = d.hidden, dt = d.dtype;
    int r = CAR_OK;
    auto T = [&](int rc) { if (r == CAR_OK) r = rc; };
    // patch projection [C][3*P*P] -> [C][kpad] zero padded (k-tiles of 32)
    m->kpatch = 3 * d.patch * d.patch;
    m->kpad = (m->kpatch + 31) & ~31;
    {
        bf16* tmp = nullptr;
        T(to_bf16_any(st, dt, m, w->patch_w, (long long)C * m->kpatch, &tmp));
        if (r == CAR_OK) r = m->alloc(&m->w_patch, (size_t)C * m->kpad * 2);
        if (r == CAR_OK) {
            cudaMemsetAsync(m->w_patch, 0, (size_t)C * m->kpad * 2, st);
            cudaMemcpy2DAsync(m->w_patch, (size_t)m->kpad * 2, tmp, (size_t)m->kpatch * 2, (size_t)m->kpatch * 2, C, cudaMemcpyDeviceToDevice, st);
        }
    }
    auto cv = [&](const void* src, long long n) -> const void* {   // bf16 view of a (possibly fp32) vector / matrix
        bf16* p = nullptr;
        T(to_bf16_any(st, dt, m, src, n, &p));
        return p;
    };
    m->b_patch = cv(w->patch_b, C); m->cls = w->cls_token; m->pos = w->pos_emb;
    m->ln_w = cv(w->ln_w, C); m->ln_b = cv(w->ln_b, C);
    m->L.resize(d.layers);
    for (int l = 0; l < d.layers && r == CAR_OK; ++l) {
        CarDino::Layer& Ly = m->L[l];
        // q and k fused into one [2C][C] weight (+bias); v kept separate (computed transposed)
        r = m->alloc(&Ly.w_qk, (size_t)2 * C * C * 2);
        if (r == CAR_OK) r = m->alloc(&Ly.b_qk, (size_t)2 * C * 2);
        if (r != CAR_OK) break;
        const bf16 *wq = (const bf16*)cv(w->q_w[l], (long long)C * C), *wk = (const bf16*)cv(w->k_w[l], (long long)C * C);
        const bf16 *bq = (const bf16*)cv(w->q_b[l], C), *bk = (const bf16*)cv(w->k_b[l], C);
        if (r != CAR_OK) break;
        cudaMemcpyAsync(Ly.w_qk, wq, (size_t)C * C * 2, cudaMemcpyDeviceToDevice, st);
        cudaMemcpyAsync(Ly.w_qk + (size_t)C * C, wk, (size_t)C * C * 2, cudaMemcpyDeviceToDevice, st);
        cudaMemcpyAsync(Ly.b_qk, bq, (size_t)C * 2, cudaMemcpyDeviceToDevice, st);
        cudaMemcpyAsync(Ly.b_qk + C, bk, (size_t)C * 2, cudaMemcpyDeviceToDevice, st);
        Ly.w_v = (bf16*)cv(w->v_w[l], (long long)C * C); Ly.b_v = cv(w->v_b[l], C);
        Ly.w_o = cv(w->o_w[l], (long long)C * C); Ly.b_o = cv(w->o_b[l], C);
        Ly.ls1 = cv(w->ls1[l], C); Ly.ls2 = cv(w->ls2[l], C);
        Ly.n1w = cv(w->n1_w[l], C); Ly.n1b = cv(w->n1_b[l], C); Ly.n2w = cv(w->n2_w[l], C); Ly.n2b = cv(w->n2_b[l], C);
        Ly.w_fc1 = cv(w->fc1_w[l], (long long)4 * C * C); Ly.b_fc1 = cv(w->fc1_b[l], 4 * C);
        Ly.w_fc2 = cv(w->fc2_w[l], (long long)4 * C * C); Ly.b_fc2 = cv(w->fc2_b[l], C);
    }
    m->ad_fc1 = m->ad_fc2 = nullptr; m->ad_dim = d.adapter_out_dim;
    if (w->adapter_fc1 && d.adapter_out_dim > 0) {
        m->ad_fc1 = (bf16*)cv(w->adapter_fc1, (long long)d.adapter_out_dim * C);
        m->ad_fc2 = (bf16*)cv(w->adapter_fc2, (long long)d.adapter_out_dim * d.adapter_out_dim);
    }
    if (r != CAR_OK) { delete m; return r; }
    *out = m;
    return CAR_OK;
}

extern "C" int car_dino_destroy(CarDino* m) {
    delete m;
    return CAR_OK;
}

template <typename TI>
static int dino_forward_t(CarDino* m, const TI* image, int B, int H, int W, void* out, int apply_mlp, cudaStream_t st) {
    const CarDinoDesc& d = m->d;
    const int C = d.hidden, h = H / 16, w = W / 16, hw = h * w, Tn = hw + 1, heads = d.heads;
    const int Tp = (Tn + 31) & ~31;                      // key axis of V^T, zero padded (vit_attention_kernel reads it in 8-key chunks)
    const long long rows = (long long)B * Tn;
    // workspace (every buffer is sized for its one use)
    const int KP = m->kpad;
    bf16 *patches, *ptok, *posi, *x, *xn, *qk, *vT, *ctx, *hid, *feat, *mlp_h;
    CAR_TRY(m->ws.carve([&](Carve& c) {
        patches = c.take<bf16>((size_t)B * hw * KP);
        ptok = c.take<bf16>((size_t)B * hw * C);
        posi = c.take<bf16>((size_t)hw * C);
        x = c.take<bf16>(rows * C);
        xn = c.take<bf16>(rows * C);
        qk = c.take<bf16>(rows * 2 * C);
        vT = c.take<bf16>((size_t)B * C * Tp);
        ctx = c.take<bf16>(rows * C);
        hid = c.take<bf16>(rows * 4 * C);
        feat = c.take<bf16>((size_t)B * hw * C);
        mlp_h = c.take<bf16>((size_t)B * hw * std::max(m->ad_dim, 1));
    }));

    CAR_CUDA(cudaMemsetAsync(vT, 0, (size_t)B * C * Tp * 2, st));   // padded key columns must be finite (x 0 prob)
    // 1. resize to (h*P, w*P) + patchify (dinov2_adapter.py:16-24; ViT: P = 16, no resize), patch projection + bias
    CAR_LAUNCH((resize_patchify_kernel<TI>), gsz((long long)B * hw * KP), 256, 0, st, image, patches, B, H, W, h, w, KP, d.resize_mode, d.patch);
    {
        DenseP p = dp_plain(patches, KP, m->w_patch, KP, B * hw, C, KP, ptok, C);
        p.bias = (const bf16*)m->b_patch;
        CAR_TRY(gemm(st, p));
    }
    // 2. CLS + interpolated position embeddings
    CAR_LAUNCH((pos_embed_interp_kernel<TI>), gsz((long long)hw * C), 256, 0, st, (const TI*)m->pos, posi, d.pos_grid, h, w, C);
    CAR_LAUNCH((dino_assemble_kernel<TI>), gsz(rows * C), 256, 0, st, ptok, (const TI*)m->cls, (const TI*)m->pos, posi, x, B, hw, C);
    // 3. encoder layers (modeling_dinov2.py Dinov2Layer.forward)
    const float scale = 0.125f;
    for (int l = 0; l < d.layers; ++l) {
        const CarDino::Layer& Ly = m->L[l];
        CAR_LAUNCH(layernorm_kernel, (unsigned)rows, 128, 0, st, x, (const bf16*)Ly.n1w, (const bf16*)Ly.n1b, xn, C, d.eps, (long long)C, (long long)C);
        {   // q | k  : [rows][2C]
            DenseP p = dp_plain(xn, C, Ly.w_qk, C, (int)rows, 2 * C, C, qk, 2 * C);
            p.bias = Ly.b_qk;
            CAR_TRY(gemm(st, p));
        }
        {   // V^T per image: [C][Tp] = Wv[C][C] · xn_b[Tn][C]^T  (+ bias along M); padded key columns stay 0-weighted
            DenseP p = dp_plain(Ly.w_v, C, xn, C, C, Tn, C, vT, Tp);
            p.sB = (long long)Tn * C; p.sC = (long long)C * Tp; p.bias = (const bf16*)Ly.b_v; p.bias_along_m = 1;
            CAR_TRY(gemm(st, p, B));
        }
        // fused attention (vision.cuh): scores / probabilities never leave the SM.  hidden % 64 == 0 (car_dino_create) and the
        // 256-byte aligned workspace give the kernel its 16-byte aligned rows.
        CAR_LAUNCH(vit_attention_kernel, dim3((Tn + 63) / 64, heads, B), 128, 0, st, (const bf16*)qk, (const bf16*)vT, ctx, Tn, Tp, C, scale);
        {   // x = x + ls1 * (dense(ctx) + b)
            DenseP p = dp_plain(ctx, C, (const bf16*)Ly.w_o, C, (int)rows, C, C, x, C);
            p.bias = (const bf16*)Ly.b_o; p.scale = (const bf16*)Ly.ls1; p.resid = x; p.ldr = C;
            CAR_TRY(gemm(st, p));
        }
        CAR_LAUNCH(layernorm_kernel, (unsigned)rows, 128, 0, st, x, (const bf16*)Ly.n2w, (const bf16*)Ly.n2b, xn, C, d.eps, (long long)C, (long long)C);
        {
            DenseP p = dp_plain(xn, C, (const bf16*)Ly.w_fc1, C, (int)rows, 4 * C, C, hid, 4 * C);
            p.bias = (const bf16*)Ly.b_fc1; p.act = ACT_GELU_ERF;
            CAR_TRY(gemm(st, p));
        }
        {
            DenseP p = dp_plain(hid, 4 * C, (const bf16*)Ly.w_fc2, 4 * C, (int)rows, C, 4 * C, x, C);
            p.bias = (const bf16*)Ly.b_fc2; p.scale = (const bf16*)Ly.ls2; p.resid = x; p.ldr = C;
            CAR_TRY(gemm(st, p));
        }
    }
    // 4. final LayerNorm, drop CLS (dinov2_adapter.py:29): rows of image b start at token 1
    bf16* fdst = apply_mlp ? feat : (bf16*)out;
    for (int b = 0; b < B; ++b)
        CAR_LAUNCH(layernorm_kernel, (unsigned)hw, 128, 0, st, x + ((size_t)b * Tn + 1) * C, (const bf16*)m->ln_w, (const bf16*)m->ln_b,
                   fdst + (size_t)b * hw * C, C, d.eps, (long long)C, (long long)C);
    // 5. optional adapter_mlp (generate.py:138): fc2(gelu_tanh(fc1 x)), bias-free
    if (apply_mlp) {
        if (!m->ad_fc1) CAR_FAIL(CAR_ERR_STATE, "adapter_mlp weights were not registered");
        DenseP p1 = dp_plain(feat, C, m->ad_fc1, C, B * hw, m->ad_dim, C, mlp_h, m->ad_dim);
        p1.act = ACT_GELU_TANH;
        CAR_TRY(gemm(st, p1));
        DenseP p2 = dp_plain(mlp_h, m->ad_dim, m->ad_fc2, m->ad_dim, B * hw, m->ad_dim, m->ad_dim, out, m->ad_dim);
        CAR_TRY(gemm(st, p2));
    }
    return CAR_OK;
}

extern "C" int car_dino_forward(CarDino* m, const void* image, int32_t B, int32_t H, int32_t W, void* out_bf16, int32_t apply_mlp,
                                void* stream) {
    if (!m || !image || !out_bf16) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (H % 16 || W % 16 || B <= 0) CAR_FAIL(CAR_ERR_ARG, "H and W must be multiples of 16");
    if (m->d.dtype == CAR_BF16) return dino_forward_t<bf16>(m, (const bf16*)image, B, H, W, out_bf16, apply_mlp, (cudaStream_t)stream);
    return dino_forward_t<float>(m, (const float*)image, B, H, W, out_bf16, apply_mlp, (cudaStream_t)stream);
}

// =========================================================================================================
// VQGAN tokenizer
// =========================================================================================================
struct ConvW { bf16* w; bf16* b; int cin, cin_pad, cout, k; };
struct NormW { bf16 *w, *b; int c; };
struct NormF { float *w, *b; };                                          // fp32 affine of a norm in the fp32-grade networks
template <typename Conv, typename Norm> struct ResT { Norm n1, n2; Conv c1, c2, nin; bool has_nin; };
template <typename Conv, typename Norm> struct AttnT { Norm n; Conv q, k, v, o; };
using ResW = ResT<ConvW, NormW>;                                         // decoder: bf16
using AttnW = AttnT<ConvW, NormW>;
using ResX3 = ResT<X3W, NormF>;                                          // encoder: fp32 grade
using AttnX3 = AttnT<X3W, NormF>;

struct CarVQ : CarOwned {
    CarVQDesc d;
    float* codebook_n;                 // l2-normalised fp32 [n_codes][e_dim]
    // decoder
    ConvW post_quant, d_conv_in, d_conv_out; NormW d_norm_out;
    ResW d_mid0, d_mid2; AttnW d_mid1;
    std::vector<std::vector<ResW>> d_res; std::vector<std::vector<AttnW>> d_attn; std::vector<ConvW> d_up; std::vector<bool> d_has_up;
    // encoder
    X3W quant_conv, e_conv_in, e_conv_out; NormF e_norm_out;
    ResX3 e_mid0, e_mid2; AttnX3 e_mid1;
    std::vector<std::vector<ResX3>> e_res; std::vector<std::vector<AttnX3>> e_attn; std::vector<X3W> e_down; std::vector<bool> e_has_down;
};

static bf16* take_bf16(TensorReader& tc, const float* src, long long n) {
    bf16* p = (bf16*)tc.alloc((size_t)n * 2);
    tc.pack(cast_to_bf16_kernel<float>, n, src, p, n);
    return p;
}
static void take_conv(TensorReader& tc, int cout, int cin, int k, ConvW* c) {
    c->cin = cin; c->cout = cout; c->k = k; c->cin_pad = (cin + 31) & ~31;
    const float* w = tc.next();
    const long long n = (long long)cout * k * k * c->cin_pad;
    c->w = (bf16*)tc.alloc((size_t)n * 2);
    tc.pack(conv_weight_pack_kernel<float>, n, w, c->w, cout, cin, k, k, c->cin_pad);
    c->b = take_bf16(tc, tc.next(), cout);
}
static void take_conv(TensorReader& tc, int cout, int cin, int k, X3W* c) { *c = tc.x3(cout, cin, k, (cin + 31) & ~31); }
static void take_norm(TensorReader& tc, int c, NormW* nw) {
    nw->c = c;
    nw->w = take_bf16(tc, tc.next(), c);
    nw->b = take_bf16(tc, tc.next(), c);
}
static void take_norm(TensorReader& tc, int c, NormF* nf) { nf->w = tc.f32(c); nf->b = tc.f32(c); }
// canonical order inside a ResnetBlock: norm1.{w,b} conv1.{w,b} norm2.{w,b} conv2.{w,b} [nin_shortcut.{w,b}]
template <typename Conv, typename Norm> static void take_res(TensorReader& tc, int cin, int cout, ResT<Conv, Norm>* r) {
    take_norm(tc, cin, &r->n1); take_conv(tc, cout, cin, 3, &r->c1);
    take_norm(tc, cout, &r->n2); take_conv(tc, cout, cout, 3, &r->c2);
    r->has_nin = cin != cout;
    if (r->has_nin) take_conv(tc, cout, cin, 1, &r->nin);
}
// AttnBlock: norm.{w,b} q.{w,b} k.{w,b} v.{w,b} proj_out.{w,b}
template <typename Conv, typename Norm> static void take_attn(TensorReader& tc, int c, AttnT<Conv, Norm>* a) {
    take_norm(tc, c, &a->n); take_conv(tc, c, c, 1, &a->q); take_conv(tc, c, c, 1, &a->k);
    take_conv(tc, c, c, 1, &a->v); take_conv(tc, c, c, 1, &a->o);
}

extern "C" int car_vq_create(const CarVQDesc* desc, const void* const* tensors, int32_t n_tensors, void* stream, CarVQ** out) {
    if (!desc || !tensors || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (desc->embed_dim > 8 || desc->n_levels > 8 || desc->ch % 32) CAR_FAIL(CAR_ERR_UNSUPPORTED, "unsupported VQ shape");
    CarVQ* m = new CarVQ();
    m->d = *desc;
    const CarVQDesc& d = m->d;
    TensorReader tc(__func__, tensors, n_tensors, stream, m);
    const int ch = d.ch, nres = d.n_levels, nrb = d.num_res_blocks;
    // ---- encoder (vq_model.py:65-125)
    take_conv(tc, ch, 3, 3, &m->e_conv_in);
    m->e_res.resize(nres); m->e_attn.resize(nres); m->e_down.resize(nres); m->e_has_down.assign(nres, false);
    int block_in = ch;
    for (int lvl = 0; lvl < nres; ++lvl) {
        block_in = ch * (lvl == 0 ? 1 : d.ch_mult[lvl - 1]);
        const int block_out = ch * d.ch_mult[lvl];
        for (int b = 0; b < nrb; ++b) {
            ResX3 r; take_res(tc, block_in, block_out, &r); m->e_res[lvl].push_back(r);
            block_in = block_out;
            if (lvl == nres - 1) { AttnX3 a; take_attn(tc, block_in, &a); m->e_attn[lvl].push_back(a); }
        }
        if (lvl != nres - 1) { take_conv(tc, block_in, block_in, 3, &m->e_down[lvl]); m->e_has_down[lvl] = true; }
    }
    take_res(tc, block_in, block_in, &m->e_mid0); take_attn(tc, block_in, &m->e_mid1);
    take_res(tc, block_in, block_in, &m->e_mid2);
    take_norm(tc, block_in, &m->e_norm_out); take_conv(tc, d.z_channels, block_in, 3, &m->e_conv_out);
    // ---- decoder (vq_model.py:129-195)
    block_in = ch * d.ch_mult[nres - 1];
    take_conv(tc, block_in, d.z_channels, 3, &m->d_conv_in);
    take_res(tc, block_in, block_in, &m->d_mid0); take_attn(tc, block_in, &m->d_mid1);
    take_res(tc, block_in, block_in, &m->d_mid2);
    m->d_res.resize(nres); m->d_attn.resize(nres); m->d_up.resize(nres); m->d_has_up.assign(nres, false);
    for (int idx = 0; idx < nres; ++idx) {
        const int lvl = nres - 1 - idx;
        const int block_out = ch * d.ch_mult[lvl];
        for (int b = 0; b < nrb + 1; ++b) {
            ResW r; take_res(tc, block_in, block_out, &r); m->d_res[idx].push_back(r);
            block_in = block_out;
            if (lvl == nres - 1) { AttnW a; take_attn(tc, block_in, &a); m->d_attn[idx].push_back(a); }
        }
        if (lvl != 0) { take_conv(tc, block_in, block_in, 3, &m->d_up[idx]); m->d_has_up[idx] = true; }
    }
    take_norm(tc, block_in, &m->d_norm_out); take_conv(tc, 3, block_in, 3, &m->d_conv_out);
    // ---- quantiser + 1x1 convs
    const float* codebook = tc.next();
    m->codebook_n = (float*)tc.alloc((size_t)d.codebook_size * d.embed_dim * 4);
    tc.launch(codebook_normalize_kernel, (d.codebook_size + 255) / 256, 256, codebook, m->codebook_n, d.codebook_size, d.embed_dim);
    take_conv(tc, d.embed_dim, d.z_channels, 1, &m->quant_conv);
    take_conv(tc, d.z_channels, d.embed_dim, 1, &m->post_quant);
    const int rc = tc.finish();
    if (rc != CAR_OK) { delete m; return rc; }
    *out = m;
    return CAR_OK;
}
extern "C" int car_vq_destroy(CarVQ* m) {
    delete m;
    return CAR_OK;
}

// ---- layer helpers on NHWC bf16 activations ----
struct Act { bf16* p; int B, H, W, C; long long n() const { return (long long)B * H * W * C; } };

static int conv_fwd(cudaStream_t st, const ConvW& c, const Act& x, int ups, int stride2, Buf<bf16> out, const bf16* resid, int Ho, int Wo,
                    float* out_nchw_f32 = nullptr) {
    if (x.C != c.cin_pad && !(c.k == 1 && x.C == c.cin_pad)) CAR_FAIL(CAR_ERR_STATE, "conv input channel mismatch");
    if (!out_nchw_f32) CAR_TRY(car_fits(__func__, out, (size_t)x.B * Ho * Wo * c.cout));
    DenseP p;
    memset(&p, 0, sizeof(p));
    p.A = x.p; p.B = c.w; p.M = x.B * Ho * Wo; p.N = c.cout; p.K = c.k * c.k * c.cin_pad; p.ldb = p.K; p.alpha = 1.f;
    if (c.k == 1) { p.amode = A_PLAIN; p.lda = x.C; }
    else { p.amode = stride2 ? A_CONV3x3S2 : A_CONV3x3; p.Hs = x.H; p.Ws = x.W; p.Cin = c.cin_pad; p.ups = ups; }
    p.Ho = Ho; p.Wo = Wo;
    p.bias = c.b;
    if (out_nchw_f32) { p.C = out_nchw_f32; p.out_mode = 2; }
    else { p.C = out; p.ldc = c.cout; p.resid = resid; p.ldr = c.cout; }
    return gemm(st, p);
}
static int gn_fwd(cudaStream_t st, const NormW& nw, const Act& x, Buf<bf16> y, int swish, float* stats) {
    const int G = 32;
    const int C8 = x.C / 8;
    CAR_TRY(car_fits(__func__, y, (size_t)x.n()));
    if (x.C % 64 == 0 && 256 % C8 == 0 && x.H * x.W >= 4 * GN_CHUNKS && ((uintptr_t)x.p % 16) == 0 && ((uintptr_t)y.p % 16) == 0 &&
        ((uintptr_t)nw.w % 16) == 0 && ((uintptr_t)nw.b % 16) == 0) {
        // coalesced two-stage statistics + 16-byte apply (vision.cuh); `stats` has room for the partial sums behind the [B*32][2] block
        float* part = stats + (size_t)x.B * G * 2;
        CAR_LAUNCH(groupnorm_partial_kernel, dim3(GN_CHUNKS, x.B), 256, 0, st, (const bf16*)x.p, part, x.H * x.W, x.C);
        CAR_LAUNCH(groupnorm_finish_kernel, x.B, 32, 0, st, (const float*)part, stats, x.H * x.W, x.C);
        CAR_LAUNCH(groupnorm_apply8_kernel, gsz(x.n() / 8), 256, 0, st, (const bf16*)x.p, (const float*)stats, (const bf16*)nw.w, (const bf16*)nw.b, y, x.n() / 8,
                   x.H * x.W, x.C, swish);
        return CAR_OK;
    }
    CAR_LAUNCH(groupnorm_stats_kernel, x.B * G, 512, 0, st, x.p, stats, x.H * x.W, x.C, G);
    CAR_LAUNCH(groupnorm_apply_kernel, gsz(x.n()), 256, 0, st, x.p, stats, nw.w, nw.b, y, x.n(), x.H * x.W, x.C, G, swish);
    return CAR_OK;
}

struct VqScratch { Buf<bf16> a, b, t0, t1, t2; float* stats; float* S; bf16* P; Buf<bf16> vT; };   // a / b: the ping-pong activations

// ResnetBlock.forward (vq_model.py:300-315): x + conv2(swish(GN(conv1(swish(GN(x))))))  [+ 1x1 shortcut]
static int res_fwd(cudaStream_t st, const ResW& r, Act& x, Buf<bf16> out, VqScratch& s) {
    Act a = x;
    CAR_TRY(gn_fwd(st, r.n1, x, s.t0, 1, s.stats));
    a.p = s.t0;
    CAR_TRY(conv_fwd(st, r.c1, a, 0, 0, s.t1, nullptr, x.H, x.W));
    Act b{s.t1, x.B, x.H, x.W, r.c1.cout};
    CAR_TRY(gn_fwd(st, r.n2, b, s.t0, 1, s.stats));
    b.p = s.t0;
    const bf16* sc = x.p;
    if (r.has_nin) { CAR_TRY(conv_fwd(st, r.nin, x, 0, 0, s.t2, nullptr, x.H, x.W)); sc = s.t2; }
    CAR_TRY(conv_fwd(st, r.c2, b, 0, 0, out, sc, x.H, x.W));
    x.p = out; x.C = r.c2.cout;
    return CAR_OK;
}
// AttnBlock.forward (vq_model.py:328-352): single head over H*W tokens, scale C^-0.5
static int attn_fwd(cudaStream_t st, const AttnW& a, Act& x, Buf<bf16> out, VqScratch& s) {
    const int C = x.C, hw = x.H * x.W, B = x.B;
    const int hwp = (hw + 31) & ~31;
    CAR_TRY(gn_fwd(st, a.n, x, s.t0, 0, s.stats));
    Act xn{s.t0, B, x.H, x.W, C};
    Buf<bf16> q = s.t1, k = s.t2;
    CAR_TRY(conv_fwd(st, a.q, xn, 0, 0, q, nullptr, x.H, x.W));
    CAR_TRY(conv_fwd(st, a.k, xn, 0, 0, k, nullptr, x.H, x.W));
    CAR_TRY(car_fits(__func__, s.vT, (size_t)B * C * hwp));
    {   // V^T [B][C][hwp]
        DenseP p = dp_plain(a.v.w, C, xn.p, C, C, hw, C, s.vT, hwp);
        p.sB = (long long)hw * C; p.sC = (long long)C * hwp; p.bias = a.v.b; p.bias_along_m = 1;
        CAR_TRY(gemm(st, p, B));
    }
    {
        DenseP p = dp_plain(q, C, k, C, hw, hw, C, s.S, hwp);
        p.sA = (long long)hw * C; p.sB = (long long)hw * C; p.sC = (long long)hw * hwp; p.alpha = 1.0f / sqrtf((float)C); p.out_mode = 1;
        CAR_TRY(gemm(st, p, B));
    }
    CAR_LAUNCH(softmax_rows_kernel, (unsigned)((long long)B * hw), 256, 0, st, s.S, s.P, hw, hwp, hwp);
    {
        DenseP p = dp_plain(s.P, hwp, s.vT, hwp, hw, C, hwp, q, C);     // ctx overwrites q
        p.sA = (long long)hw * hwp; p.sB = (long long)C * hwp; p.sC = (long long)hw * C;
        CAR_TRY(gemm(st, p, B));
    }
    Act ctx{q, B, x.H, x.W, C};
    CAR_TRY(conv_fwd(st, a.o, ctx, 0, 0, out, x.p, x.H, x.W));
    x.p = out;
    return CAR_OK;
}

// the decoder's scratch buffers, in carve order
static void vq_scratch(Carve& c, const CarVQDesc& d, int B, int Hmax, int Wmax, int h16, int w16, int Cfull, VqScratch& s) {
    const size_t act = (size_t)B * Hmax * Wmax * Cfull;                // largest activation (ch channels at full res)
    const int hw = h16 * w16, hwp = (hw + 31) & ~31, Cmax = d.ch * d.ch_mult[d.n_levels - 1];
    s.a = c.take<bf16>(act); s.b = c.take<bf16>(act);
    s.t0 = c.take<bf16>(act); s.t1 = c.take<bf16>(act); s.t2 = c.take<bf16>(act);
    s.stats = c.take<float>((size_t)B * 32 * 2 * (1 + GN_CHUNKS));
    s.S = c.take<float>((size_t)B * hw * hwp); s.P = c.take<bf16>((size_t)B * hw * hwp);
    s.vT = c.take<bf16>((size_t)B * Cmax * hwp);
}

// VQModel.decode_code (vq_model.py:53-56): codes int32 [B][h*w] -> image fp32 NCHW [B][3][16h][16w] (VQ-16)
// VQModel.decode (vq_model.py:48-51): quant fp32 NCHW [B][e][h][w] -> image
static int vq_decode_impl(CarVQ* m, const int32_t* codes, const float* quant, int32_t B, int32_t h, int32_t w, float* out, void* stream) {
    if (!m || !(codes || quant) || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const CarVQDesc& d = m->d;
    const int up = 1 << (d.n_levels - 1);
    VqScratch s; bf16* zbuf;
    CAR_TRY(m->ws.carve([&](Carve& c) {
        vq_scratch(c, d, B, h * up, w * up, h, w, d.ch, s);
        zbuf = c.take<bf16>((size_t)B * h * w * 32);
    }));
    CAR_CUDA(cudaMemsetAsync(s.vT, 0, s.vT.cap * 2, st));
    // get_codebook_entry (vq_model.py:262-277) + post_quant_conv
    if (codes) CAR_LAUNCH(codebook_lookup_kernel, gsz((long long)B * h * w * 32), 256, 0, st, m->codebook_n, codes, zbuf, (long long)B * h * w, d.embed_dim, 32, d.codebook_size);
    else CAR_LAUNCH((nchw_to_nhwc_bf16_kernel<float>), gsz((long long)B * h * w * 32), 256, 0, st, quant, zbuf, B, d.embed_dim, h * w, 32);
    Act x{zbuf, B, h, w, 32};
    CAR_TRY(conv_fwd(st, m->post_quant, x, 0, 0, s.a, nullptr, h, w));
    x = Act{s.a, B, h, w, d.z_channels};
    Buf<bf16> cur = s.b;
    auto flip = [&](bf16* used) { return used == s.a ? s.b : s.a; };
    CAR_TRY(conv_fwd(st, m->d_conv_in, x, 0, 0, cur, nullptr, h, w));
    x = Act{cur, B, h, w, m->d_conv_in.cout};
    CAR_TRY(res_fwd(st, m->d_mid0, x, flip(x.p), s));
    CAR_TRY(attn_fwd(st, m->d_mid1, x, flip(x.p), s));
    CAR_TRY(res_fwd(st, m->d_mid2, x, flip(x.p), s));
    for (int idx = 0; idx < d.n_levels; ++idx) {
        for (size_t b = 0; b < m->d_res[idx].size(); ++b) {
            CAR_TRY(res_fwd(st, m->d_res[idx][b], x, flip(x.p), s));
            if (!m->d_attn[idx].empty()) CAR_TRY(attn_fwd(st, m->d_attn[idx][b], x, flip(x.p), s));
        }
        if (m->d_has_up[idx]) {   // Upsample (vq_model.py:368-379): nearest x2, then the 3x3 convolution
            Buf<bf16> o = flip(x.p);
            if (x.C % WG_CBLK == 0) {   // materialise the up-sampled tensor (bandwidth-trivial) so the convolution is a plain TMA box walk
                CAR_TRY(car_fits("upsample2x", s.t2, (size_t)x.n() * 4));
                CAR_LAUNCH(upsample2x_nhwc_kernel, gsz((long long)B * x.H * 2 * x.W * 2 * (x.C / 8)), 256, 0, st, (const bf16*)x.p, s.t2, B, x.H, x.W, x.C);
                Act u{s.t2, B, x.H * 2, x.W * 2, x.C};
                CAR_TRY(conv_fwd(st, m->d_up[idx], u, 0, 0, o, nullptr, u.H, u.W));
            } else {                              // nearest x2 folded into the conv's addressing (mma.sync kernel)
                CAR_TRY(conv_fwd(st, m->d_up[idx], x, 1, 0, o, nullptr, x.H * 2, x.W * 2));
            }
            x = Act{o, B, x.H * 2, x.W * 2, m->d_up[idx].cout};
        }
    }
    CAR_TRY(gn_fwd(st, m->d_norm_out, x, s.t0, 1, s.stats));
    Act y{s.t0, B, x.H, x.W, x.C};
    if (m->d_conv_out.cout == 3 && m->d_conv_out.cin_pad == y.C && y.C % 8 == 0 && 27 * y.C * 2 <= 48 * 1024) {
        CAR_LAUNCH(conv3x3_to3_kernel, gsz((long long)B * y.H * y.W), 256, (size_t)27 * y.C * 2, st, (const bf16*)y.p, (const bf16*)m->d_conv_out.w,
                   (const bf16*)m->d_conv_out.b, out, B, y.H, y.W, y.C);
        return CAR_OK;
    }
    return conv_fwd(st, m->d_conv_out, y, 0, 0, Buf<bf16>{}, nullptr, x.H, x.W, out);
}

extern "C" int car_vq_decode_code(CarVQ* m, const int32_t* codes, int32_t B, int32_t h, int32_t w, float* out, void* stream) {
    if (!codes) CAR_FAIL(CAR_ERR_ARG, "null codes");
    return vq_decode_impl(m, codes, nullptr, B, h, w, out, stream);
}
extern "C" int car_vq_decode(CarVQ* m, const float* quant, int32_t B, int32_t h, int32_t w, float* out, void* stream) {
    if (!quant) CAR_FAIL(CAR_ERR_ARG, "null quant");
    return vq_decode_impl(m, nullptr, quant, B, h, w, out, stream);
}

// ---- VQModel.encode (vq_model.py:41-46) at fp32 grade: the split-bf16 ("x3") path of split3.cuh ----
// fp32 NHWC activations; every convolution = one launch of the bf16 implicit-GEMM kernel over tripled K, fp32 output / bias / residual.
struct ActF { float* p; int B, H, W, C; long long npix() const { return (long long)B * H * W; } long long n() const { return npix() * C; } };
struct EncScratch { Buf<bf16> t3, x3; Buf<float> h1, sc, gnp, stats; Buf<float> qf, kf, vf, ctx; float *S, *P; Buf<bf16> q3, k3, P3, vT3; };

// fp32 rows x [M][N] -> S3 rows (mode X3_ROWS_A, X3_ROWS_A_GELU) or W3 rows (X3_ROWS_B) [M][3N]
static int split3_rows(cudaStream_t st, const float* x, Buf<bf16> y, long long M, int N, int mode = X3_ROWS_A) {
    CAR_TRY(car_fits(__func__, y, (size_t)M * N * 3));
    CAR_LAUNCH(split3_rows_kernel, gsz(M * N), 256, 0, st, x, y, M, N, mode);
    return CAR_OK;
}
// image fp32 NCHW (- sub[c]) -> padded S3 NHWC frame (split3.cuh image_split3_kernel)
static int image_split3(cudaStream_t st, const float* x, const float* sub, Buf<bf16> y, X3Image q) {
    const long long n = (long long)q.B * (q.pt + q.H + q.pb) * (q.pl + q.W + q.pr) * q.Cpad;
    CAR_TRY(car_fits(__func__, y, (size_t)n * 3));
    CAR_LAUNCH(image_split3_kernel, gsz(n), 256, 0, st, x, sub, y, q);
    return CAR_OK;
}
// mma.sync implicit GEMM (gemm.h A_PLAIN for a 1x1 weight, else A_CONV3x3 or, with stride2, A_CONV3x3S2): S3 activations
// [B][Hs][Ws][w.cin3] -> out fp32 [B][Ho][Wo][w.n] = conv + bias (+ fp32 residual of the same shape), then act
static int x3_mma(cudaStream_t st, const X3W& w, const bf16* a3, int B, int Hs, int Ws, int stride2, Buf<float> out, const float* resid, int Ho, int Wo,
                  int act = ACT_NONE) {
    CAR_TRY(car_fits(__func__, out, (size_t)B * Ho * Wo * w.n));
    DenseP p;
    memset(&p, 0, sizeof(p));
    p.A = a3; p.B = w.w; p.M = B * Ho * Wo; p.N = w.n; p.K = w.kh * w.kw * w.cin3; p.ldb = p.K; p.alpha = 1.f;
    if (w.kh == 1) { p.amode = A_PLAIN; p.lda = w.cin3; }
    else { p.amode = stride2 ? A_CONV3x3S2 : A_CONV3x3; p.Hs = Hs; p.Ws = Ws; p.Cin = w.cin3; p.ups = 0; }
    p.Ho = Ho; p.Wo = Wo;
    p.bias_f = w.b; p.C = out; p.ldc = w.n; p.out_mode = 1; p.resid_f = resid; p.ldr = w.n; p.act = act;
    return gemm(st, p);
}
// fp32 GroupNorm statistics (groupnorm.cuh) of x [B][HW][C], cpg channels per group (InstanceNorm: 1) -> stats [B][C/cpg][2];
// part holds the two [B][gn_nch(HW)][C] partial sums
static int gn_stats(cudaStream_t st, const float* x, int B, int HW, int C, int cpg, float eps, Buf<float> part, Buf<float> stats) {
    if (C % 32 || cpg < 1 || 32 % cpg) CAR_FAIL(CAR_ERR_STATE, "group statistics need C % 32 == 0 and cpg dividing 32");
    const int nch = gn_nch(HW);
    const size_t np = (size_t)B * nch * C;
    CAR_TRY(car_fits(__func__, part, 2 * np));
    CAR_TRY(car_fits(__func__, stats, (size_t)B * (C / cpg) * 2));
    const dim3 grid(C / 32, B, nch);
    CAR_LAUNCH(gn_partial_kernel<false>, grid, GN_THREADS, 0, st, x, nullptr, part, HW, C, cpg);
    CAR_LAUNCH(gn_partial_kernel<true>, grid, GN_THREADS, 0, st, x, (const float*)part, part + np, HW, C, cpg);
    CAR_LAUNCH(gn_finish_kernel, dim3(C / 32, B), 32, 0, st, (const float*)part, (const float*)(part + np), stats, HW, C, cpg, nch, eps);
    return CAR_OK;
}
// GroupNorm(32) of x [B][H][W][C] (+ resid, itself normalised when rn.stats) (act) (max-pool) -> S3 frame y, fp32 carrier when given
static int gn_apply_s3(cudaStream_t st, const float* x, GnAffine gn, const float* resid, GnAffine rn, float* carrier, Buf<bf16> y, int B, int H, int W,
                       int C, GnApply a) {
    if (C % GN_GROUPS) CAR_FAIL(CAR_ERR_STATE, "GroupNorm(32) needs C % 32 == 0");
    if (a.pool && a.act != GN_ACT_RELU) CAR_FAIL(CAR_ERR_STATE, "the GroupNorm max-pool follows ReLU only");
    const long long n = (long long)B * a.Hp * a.Wp * C;
    CAR_TRY(car_fits(__func__, y, (size_t)n * 3));
    CAR_LAUNCH(gn_apply_s3_kernel, gsz(n), 256, 0, st, x, gn, resid, rn, carrier, y, B, H, W, C, a);
    return CAR_OK;
}
// GroupNorm(32, eps 1e-6) (act) of an encoder activation -> S3 rows y3
static int gn_x3(cudaStream_t st, const NormF& nw, const ActF& x, Buf<bf16> y3, int act, EncScratch& s) {
    CAR_TRY(gn_stats(st, x.p, x.B, x.H * x.W, x.C, x.C / GN_GROUPS, 1e-6f, s.gnp, s.stats));
    return gn_apply_s3(st, x.p, GnAffine{s.stats, nw.w, nw.b}, nullptr, GnAffine{}, nullptr, y3, x.B, x.H, x.W, x.C, GnApply{0, 0, x.H, x.W, act, 0});
}
// ResnetBlock.forward (vq_model.py:300-315)
static int res_x3(cudaStream_t st, const ResX3& r, ActF& x, Buf<float> out, EncScratch& s) {
    CAR_TRY(gn_x3(st, r.n1, x, s.t3, GN_ACT_SWISH, s));
    CAR_TRY(x3_mma(st, r.c1, s.t3, x.B, x.H, x.W, 0, s.h1, nullptr, x.H, x.W));
    ActF h{s.h1, x.B, x.H, x.W, r.c1.n};
    CAR_TRY(gn_x3(st, r.n2, h, s.t3, GN_ACT_SWISH, s));
    const float* sc = x.p;
    if (r.has_nin) {
        CAR_TRY(split3_rows(st, x.p, s.x3, x.npix(), x.C));
        CAR_TRY(x3_mma(st, r.nin, s.x3, x.B, x.H, x.W, 0, s.sc, nullptr, x.H, x.W));
        sc = s.sc;
    }
    CAR_TRY(x3_mma(st, r.c2, s.t3, x.B, x.H, x.W, 0, out, sc, x.H, x.W));
    x.p = out; x.C = r.c2.n;
    return CAR_OK;
}
// AttnBlock.forward (vq_model.py:328-352): single head over H*W tokens, scale C^-0.5, everything fp32-grade
static int attn_x3(cudaStream_t st, const AttnX3& a, ActF& x, Buf<float> out, EncScratch& s) {
    const int C = x.C, hw = x.H * x.W, B = x.B;
    const int hwp = (hw + 31) & ~31;
    const long long rows = (long long)B * hw;
    CAR_TRY(gn_x3(st, a.n, x, s.t3, GN_ACT_NONE, s));
    CAR_TRY(x3_mma(st, a.q, s.t3, B, x.H, x.W, 0, s.qf, nullptr, x.H, x.W));
    CAR_TRY(x3_mma(st, a.k, s.t3, B, x.H, x.W, 0, s.kf, nullptr, x.H, x.W));
    CAR_TRY(x3_mma(st, a.v, s.t3, B, x.H, x.W, 0, s.vf, nullptr, x.H, x.W));
    CAR_TRY(split3_rows(st, s.qf, s.q3, rows, C));
    CAR_TRY(split3_rows(st, s.kf, s.k3, rows, C, X3_ROWS_B));
    {   // scores [B][hw][hwp] fp32
        DenseP p = dp_plain(s.q3, 3 * C, s.k3, 3 * C, hw, hw, 3 * C, s.S, hwp);
        p.sA = (long long)hw * 3 * C; p.sB = (long long)hw * 3 * C; p.sC = (long long)hw * hwp; p.alpha = 1.0f / sqrtf((float)C); p.out_mode = 1;
        CAR_TRY(gemm(st, p, B));
    }
    CAR_LAUNCH(softmax_rows_f32_kernel, (unsigned)rows, 256, 0, st, (const float*)s.S, s.P, hw, hwp);
    CAR_TRY(split3_rows(st, s.P, s.P3, rows, hwp));
    CAR_TRY(car_fits(__func__, s.vT3, (size_t)B * C * hwp * 3));
    CAR_TRY(car_fits(__func__, s.ctx, (size_t)rows * C));
    CAR_LAUNCH(transpose_split3b_kernel, gsz((long long)B * C * hwp), 256, 0, st, (const float*)s.vf, s.vT3, B, hw, hwp, C);
    {   // context [B][hw][C] fp32
        DenseP p = dp_plain(s.P3, 3 * hwp, s.vT3, 3 * hwp, hw, C, 3 * hwp, s.ctx, C);
        p.sA = (long long)hw * 3 * hwp; p.sB = (long long)C * 3 * hwp; p.sC = (long long)hw * C; p.out_mode = 1;
        CAR_TRY(gemm(st, p, B));
    }
    CAR_TRY(split3_rows(st, s.ctx, s.q3, rows, C));             // (q3 is free again)
    CAR_TRY(x3_mma(st, a.o, s.q3, B, x.H, x.W, 0, out, x.p, x.H, x.W));
    x.p = out;
    return CAR_OK;
}

// VQModel.encode (vq_model.py:41-46): image fp32 NCHW [B][3][H][W] -> indices int32 [B*h*w] (+ quant fp32 [B][e][h][w])
extern "C" int car_vq_encode(CarVQ* m, const float* img, int32_t B, int32_t H, int32_t W, int32_t* idx_out, float* quant_out,
                             void* stream) {
    if (!m || !img || !idx_out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const CarVQDesc& d = m->d;
    const int down = 1 << (d.n_levels - 1);
    if (H % down || W % down) CAR_FAIL(CAR_ERR_ARG, "image size must be a multiple of the down-sampling factor");
    const int h = H / down, w = W / down;
    const size_t npix = (size_t)B * h * w;
    const int hw = h * w, hwp = (hw + 31) & ~31, Cmax = d.ch * d.ch_mult[d.n_levels - 1];
    // workspace: fp32 activations (largest: ch channels at full resolution) and their S3 forms
    const size_t actf = (size_t)B * H * W * d.ch, act3 = actf * 3;
    const size_t af = npix * Cmax, a3 = af * 3;
    Buf<float> fA, fB, zf; EncScratch s; Buf<bf16> img3; float* zq;
    CAR_TRY(m->ws.carve([&](Carve& c) {
        fA = c.take<float>(actf); fB = c.take<float>(actf);
        s.h1 = c.take<float>(actf); s.sc = c.take<float>(actf);
        s.t3 = c.take<bf16>(act3); s.x3 = c.take<bf16>(act3);
        img3 = c.take<bf16>((size_t)B * H * W * 32 * 3);
        s.gnp = c.take<float>(2 * (size_t)B * GN_MAX_CHUNKS * Cmax);
        s.stats = c.take<float>((size_t)B * GN_GROUPS * 2);
        s.qf = c.take<float>(af); s.kf = c.take<float>(af); s.vf = c.take<float>(af); s.ctx = c.take<float>(af);
        s.q3 = c.take<bf16>(a3); s.k3 = c.take<bf16>(a3);
        s.S = c.take<float>((size_t)B * hw * hwp); s.P = c.take<float>((size_t)B * hw * hwp);
        s.P3 = c.take<bf16>((size_t)B * hw * hwp * 3); s.vT3 = c.take<bf16>((size_t)B * Cmax * hwp * 3);
        zf = c.take<float>(npix * 8); zq = c.take<float>(npix * 8);
    }));

    CAR_TRY(image_split3(st, img, nullptr, img3, X3Image{B, 3, H, W, 32, 0, 0, 0, 0, 0}));
    auto flip = [&](float* used) { return used == fA ? fB : fA; };
    CAR_TRY(x3_mma(st, m->e_conv_in, img3, B, H, W, 0, fA, nullptr, H, W));
    ActF x{fA, B, H, W, m->e_conv_in.n};
    for (int lvl = 0; lvl < d.n_levels; ++lvl) {
        for (size_t b = 0; b < m->e_res[lvl].size(); ++b) {
            CAR_TRY(res_x3(st, m->e_res[lvl][b], x, flip(x.p), s));
            if (!m->e_attn[lvl].empty()) CAR_TRY(attn_x3(st, m->e_attn[lvl][b], x, flip(x.p), s));
        }
        if (m->e_has_down[lvl]) {   // Downsample (vq_model.py:382-397): pad (0,1,0,1), 3x3 stride 2
            Buf<float> o = flip(x.p);
            CAR_TRY(split3_rows(st, x.p, s.x3, x.npix(), x.C));
            CAR_TRY(x3_mma(st, m->e_down[lvl], s.x3, B, x.H, x.W, 1, o, nullptr, x.H / 2, x.W / 2));
            x = ActF{o, B, x.H / 2, x.W / 2, m->e_down[lvl].n};
        }
    }
    CAR_TRY(res_x3(st, m->e_mid0, x, flip(x.p), s));
    CAR_TRY(attn_x3(st, m->e_mid1, x, flip(x.p), s));
    CAR_TRY(res_x3(st, m->e_mid2, x, flip(x.p), s));
    CAR_TRY(gn_x3(st, m->e_norm_out, x, s.t3, GN_ACT_SWISH, s));
    Buf<float> zc = flip(x.p);
    CAR_TRY(x3_mma(st, m->e_conv_out, s.t3, B, x.H, x.W, 0, zc, nullptr, x.H, x.W));               // [npix][z_channels]
    CAR_TRY(split3_rows(st, zc, s.x3, (long long)npix, d.z_channels));
    CAR_TRY(x3_mma(st, m->quant_conv, s.x3, B, x.H, x.W, 0, zf, nullptr, x.H, x.W));               // [npix][embed_dim] fp32
    CAR_LAUNCH(vq_argmin_kernel, (unsigned)((npix + 127) / 128), 128, 0, st, (const float*)zf, m->codebook_n, idx_out, quant_out ? zq : nullptr, (long long)npix, d.embed_dim, d.codebook_size);
    if (quant_out) CAR_LAUNCH(nhwc_to_nchw_f32_kernel, gsz((long long)npix * d.embed_dim), 256, 0, st, zq, quant_out, B, h * w, d.embed_dim);
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// antialiased bilinear resize (row f2): width pass into tmp, height pass into out
// ---------------------------------------------------------------------------------------------------------
extern "C" int car_resize_bilinear_aa(const float* in, int32_t B, int32_t Cc, int32_t H, int32_t W, float* out, int32_t OH, int32_t OW,
                                      float* tmp, void* stream) {
    if (!in || !out || !tmp) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || Cc <= 0 || H <= 0 || W <= 0 || OH <= 0 || OW <= 0) CAR_FAIL(CAR_ERR_ARG, "bad shape");
    cudaStream_t st = (cudaStream_t)stream;
    const long long n1 = (long long)B * Cc * H * OW, n2 = (long long)B * Cc * OH * OW;
    CAR_LAUNCH(resize_aa_axis_kernel, gsz(n1), 256, 0, st, in, tmp, (long long)B * Cc * H, W, OW, 1);
    CAR_LAUNCH(resize_aa_axis_kernel, gsz(n2), 256, 0, st, (const float*)tmp, out, (long long)B * Cc, H, OH, OW);
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// control-map / prompt front-end (row f3): Canny edges (condition/canny.py:14) and caption left-padding (sample_t2i.py:146-156)
// ---------------------------------------------------------------------------------------------------------
extern "C" int64_t car_canny_workspace_bytes(int32_t H, int32_t W) {
    const int64_t n = (int64_t)H * W;
    return ((n * 2 + 255) / 256 * 256) * 3 + (n + 255) / 256 * 256 + 256;     // mag u16, xs i16, ys i16, map u8, changed flag
}
// img uint8 [H][W][C] (device) -> edges uint8 [H][W] in {0, 255}.  restart != 0: gradients + non-maximum suppression + thresholds,
// then `sweeps` hysteresis sweeps; restart == 0: `sweeps` more sweeps on the map left in `work`.  *changed_dev (int32 in device
// memory) is 1 afterwards iff the LAST sweep still grew an edge — the caller repeats with restart = 0 until it reads 0
// (the reference's cv2 call is synchronous host code; here only that convergence check needs the host).
extern "C" int car_canny_u8(const uint8_t* img, int32_t H, int32_t W, int32_t C, int32_t low, int32_t high, uint8_t* edges_out, void* work,
                            int32_t sweeps, int32_t restart, int32_t* changed_dev, void* stream) {
    if (!img || !edges_out || !work || !changed_dev) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (H <= 0 || W <= 0 || C <= 0 || C > 4 || sweeps < 1) CAR_FAIL(CAR_ERR_ARG, "bad shape");
    cudaStream_t st = (cudaStream_t)stream;
    const long long n = (long long)H * W;
    const size_t a2 = ((size_t)n * 2 + 255) / 256 * 256;
    unsigned short* mag = (unsigned short*)work;
    short* xs = (short*)((char*)work + a2);
    short* ys = (short*)((char*)work + 2 * a2);
    unsigned char* map = (unsigned char*)work + 3 * a2;
    if (low > high) std::swap(low, high);
    if (restart) {
        CAR_LAUNCH(canny_grad_kernel, gsz(n), 256, 0, st, img, H, W, C, mag, xs, ys);
        CAR_LAUNCH(canny_nms_kernel, gsz(n), 256, 0, st, (const unsigned short*)mag, (const short*)xs, (const short*)ys, H, W, low, high, map);
    }
    dim3 grid((W + CH_T - 1) / CH_T, (H + CH_T - 1) / CH_T);
    for (int s = 0; s < sweeps; ++s) {
        CAR_CUDA(cudaMemsetAsync(changed_dev, 0, 4, st));
        CAR_LAUNCH(canny_hyst_kernel, grid, CH_T * CH_T / 4, 0, st, map, H, W, changed_dev);
    }
    CAR_LAUNCH(canny_finish_kernel, gsz(n), 256, 0, st, (const unsigned char*)map, edges_out, n);
    return CAR_OK;
}

// caption_embs [B][L][row_bytes] (any dtype, row_bytes % 16 == 0), emb_masks int64 [B][L] -> rotated embeddings + flipped masks
extern "C" int car_left_pad_captions(const void* embs, const int64_t* masks, int32_t B, int32_t L, int32_t row_bytes, void* embs_out,
                                     int64_t* masks_out, void* stream) {
    if (!embs || !masks || !embs_out || !masks_out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || L <= 0 || row_bytes <= 0 || row_bytes % 16) CAR_FAIL(CAR_ERR_ARG, "row size must be a positive multiple of 16 bytes");
    if (((uintptr_t)embs % 16) || ((uintptr_t)embs_out % 16)) CAR_FAIL(CAR_ERR_ARG, "embeddings must be 16-byte aligned");
    CAR_LAUNCH(left_pad_pack_kernel, B * L, 128, 0, (cudaStream_t)stream, (const uint4*)embs, (const long long*)masks, (uint4*)embs_out,
               (long long*)masks_out, L, row_bytes / 16);
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// HED soft-edge detector (row f3): condition/hed.py:17-84 — 13 ReLU 3x3 convolutions in five blocks with 2x2 max-pooling between
// them, a 1x1 projection per block, bilinear resize of the five maps, mean, sigmoid.  fp32 in the reference => fp32-grade here.
// ---------------------------------------------------------------------------------------------------------
struct CarHED : CarOwned {
    std::vector<X3W> conv;             // 13, in forward order
    float* norm;                       // [3]
    float* pw[5]; float* pb[5];        // projection weights [C] / bias [1]
};
static const int HED_BLK[5][3] = {{3, 64, 2}, {64, 128, 2}, {128, 256, 3}, {256, 512, 3}, {512, 512, 3}};

// tensors (fp32, device), in order: norm [3]; per block: conv0.weight, conv0.bias, conv1.weight, ... , projection.weight [C], projection.bias [1]
extern "C" int car_hed_create(const void* const* tensors, int32_t n_tensors, void* stream, CarHED** out) {
    if (!tensors || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (n_tensors != 1 + 2 * 13 + 2 * 5) CAR_FAIL(CAR_ERR_ARG, "HED expects 37 tensors (norm, 13 x (weight, bias), 5 x (projection weight, bias))");
    CarHED* m = new CarHED();
    TensorReader tc(__func__, tensors, n_tensors, stream, m);
    m->norm = tc.f32(3);
    for (int b = 0; b < 5; ++b) {
        int cin = HED_BLK[b][0];
        const int cout = HED_BLK[b][1];
        for (int i = 0; i < HED_BLK[b][2]; ++i) {
            m->conv.push_back(tc.x3(cout, cin, 3, (cin + 31) & ~31));
            cin = cout;
        }
        m->pw[b] = tc.f32(cout); m->pb[b] = tc.f32(1);
    }
    const int rc = tc.finish();
    if (rc != CAR_OK) { delete m; return rc; }
    *out = m;
    return CAR_OK;
}
extern "C" int car_hed_destroy(CarHED* m) {
    delete m;
    return CAR_OK;
}
// image fp32 NCHW [B][3][H][W] (values 0..255) -> edge fp32 [B][H][W] in [0, 255]; proj_out (optional): the five projection maps
// back to back, map k = [B][hk][wk] with hk = H >> k (floor), wk = W >> k
extern "C" int car_hed_forward(CarHED* m, const float* img, int32_t B, int32_t H, int32_t W, float* edge_out, float* proj_out, void* stream) {
    if (!m || !img || !edge_out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || H < 16 || W < 16) CAR_FAIL(CAR_ERR_ARG, "image must be at least 16 x 16");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t full = (size_t)B * H * W;
    size_t proj_elems = 0;
    { int h = H, w = W; for (int k = 0; k < 5; ++k) { proj_elems += (size_t)B * h * w; h /= 2; w /= 2; } }
    const size_t actf = full * 64, act3 = actf * 3;                             // largest activation: 64 channels at full resolution
    Buf<float> fA, fB; Buf<bf16> s3, img3; float* maps;
    CAR_TRY(m->ws.carve([&](Carve& c) {
        fA = c.take<float>(actf); fB = c.take<float>(actf);
        s3 = c.take<bf16>(act3);
        img3 = c.take<bf16>(full * 32 * 3);
        maps = c.take<float>(proj_elems);
    }));
    CAR_TRY(image_split3(st, img, m->norm, img3, X3Image{B, 3, H, W, 32, 0, 0, 0, 0, 0}));
    HedMaps hm;
    int h = H, w = W, ci = 0, curC = 3;
    float* cur = nullptr;                                                       // the one live fp32 activation (NHWC); ping-pong fA / fB
    auto other = [&](float* p) { return p == fA ? fB : fA; };
    size_t moff = 0;
    for (int b = 0; b < 5; ++b) {
        if (b > 0) {                                                            // down_sampling=True (:28-30)
            Buf<float> o = other(cur);
            CAR_TRY(car_fits("maxpool2", o, (size_t)B * (h / 2) * (w / 2) * curC));
            CAR_LAUNCH(maxpool2_nhwc_f32_kernel, gsz((long long)B * (h / 2) * (w / 2) * curC), 256, 0, st, (const float*)cur, o, B, h, w, curC);
            h /= 2; w /= 2; cur = o;
        }
        for (int i = 0; i < HED_BLK[b][2]; ++i, ++ci) {
            const X3W& c = m->conv[ci];
            const bf16* a3 = img3;
            if (ci > 0) { CAR_TRY(split3_rows(st, cur, s3, (long long)B * h * w, curC)); a3 = s3; }
            Buf<float> o = other(cur);
            CAR_TRY(x3_mma(st, c, a3, B, h, w, 0, o, nullptr, h, w, ACT_RELU));   // conv + bias, ReLU (:31-33)
            cur = o; curC = c.n;
        }
        float* mp = maps + moff;
        CAR_LAUNCH(hed_proj_kernel, (unsigned)(((long long)B * h * w * 32 + 255) / 256), 256, 0, st, (const float*)cur, (const float*)m->pw[b], (const float*)m->pb[b], mp,
                   (long long)B * h * w, curC);
        hm.p[b] = mp; hm.h[b] = h; hm.w[b] = w;
        moff += (size_t)B * h * w;
    }
    CAR_LAUNCH(hed_merge_kernel, gsz((long long)full), 256, 0, st, hm, B, H, W, edge_out);
    if (proj_out) CAR_CUDA(cudaMemcpyAsync(proj_out, maps, proj_elems * 4, cudaMemcpyDeviceToDevice, st));
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// LineArt detector (row f3): condition/lineart.py:8-86 — 7x7 stem, two stride-2 downsampling convolutions, three residual blocks,
// two transposed convolutions, 7x7 head + sigmoid, InstanceNorm2d (no parameters) after every convolution but the head.  fp32 in
// the reference => fp32-grade here: fp32 activations, every convolution but the head on the split-bf16 window GEMM (lineart.cuh).
// ---------------------------------------------------------------------------------------------------------
struct CarLineArt : CarOwned {
    X3W stem, down[2], res[6], up[2][4];              // up[i][(a, b)]: parity class (a, b), the four back to back in one allocation (lineart.cuh)
    float *head_w, *head_b;                           // [64][7][7], [1]
};

// ConvTranspose2d(3, stride 2, pad 1, output_padding 1) weight [cin][cout][3][3] -> the W3 of its four parity classes (a, b), each
// a (1 + a) x (1 + b) window, packed back to back in one allocation (lineart.cuh); then the bias
static void la_convT(TensorReader& tc, X3W (&up)[4], int cin, int cout) {
    const long long n3 = 9LL * cout * cin;
    const float* w = tc.next();
    bf16* w3 = (bf16*)tc.alloc((size_t)n3 * 3 * 2);
    tc.pack(convT_weight_pack_x3_kernel, n3, w, w3, cin, cout, cin);
    const float* b = tc.f32(cout);
    size_t off = 0;
    for (int cls = 0; cls < 4; ++cls) {
        up[cls] = X3W{w3 ? w3 + off : nullptr, b, cout, 3 * cin, 1 + (cls >> 1), 1 + (cls & 1)};
        off += (size_t)cout * up[cls].kh * up[cls].kw * 3 * cin;
    }
}

// tensors (fp32, device), state-dict order: model0.1, model1.0, model1.3, model2.{0,1,2}.conv_block.{1,5}, model3.0, model3.3,
// model4.1 — each weight then bias
extern "C" int car_lineart_create(const void* const* tensors, int32_t n_tensors, void* stream, CarLineArt** out) {
    if (!tensors || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (n_tensors != 24) CAR_FAIL(CAR_ERR_ARG, "LineArt expects 24 tensors (12 x (weight, bias) in state-dict order)");
    CarLineArt* m = new CarLineArt();
    TensorReader tc(__func__, tensors, n_tensors, stream, m);
    m->stem = tc.x3(64, 3, 7, 8);                     // 3 input channels padded to 8 (16-byte chunks), not 32
    m->down[0] = tc.x3(128, 64, 3, 64);
    m->down[1] = tc.x3(256, 128, 3, 128);
    for (int i = 0; i < 6; ++i) m->res[i] = tc.x3(256, 256, 3, 256);
    la_convT(tc, m->up[0], 256, 128);
    la_convT(tc, m->up[1], 128, 64);
    m->head_w = tc.f32(64 * 49); m->head_b = tc.f32(1);
    const int rc = tc.finish();
    if (rc != CAR_OK) { delete m; return rc; }
    *out = m;
    return CAR_OK;
}
extern "C" int car_lineart_destroy(CarLineArt* m) {
    delete m;
    return CAR_OK;
}

// one window convolution (gemm.h A_WIN) with the weight's w.kh x w.kw window: S3 source [B][Hs][Ws][w.cin3] -> fp32
// [B][oH][oW][w.n], row (b, oy, ox) of the Ho x Wo grid stored at pixel (osy*oy + oay, osx*ox + oax).  The window kernel reads the
// bias unconditionally: a bias-free weight carries a zero bias.
static int x3_win(cudaStream_t st, const X3W& w, const bf16* a3, int B, int Hs, int Ws, int stride, int Ho, int Wo, Buf<float> out, int oH, int oW,
                  int osy = 1, int osx = 1, int oay = 0, int oax = 0) {
    if (!w.b) CAR_FAIL(CAR_ERR_STATE, "window convolution without a bias");
    CAR_TRY(car_fits(__func__, out, (size_t)B * oH * oW * w.n));
    DenseP p;
    memset(&p, 0, sizeof(p));
    p.A = a3; p.B = w.w; p.M = B * Ho * Wo; p.N = w.n; p.K = w.kh * w.kw * w.cin3; p.ldb = p.K; p.alpha = 1.f;
    p.amode = A_WIN; p.Hs = Hs; p.Ws = Ws; p.Cin = w.cin3; p.Ho = Ho; p.Wo = Wo; p.kh = w.kh; p.kw = w.kw; p.ws = stride;
    p.bias_f = w.b; p.C = out; p.ldc = w.n; p.out_mode = 1;
    p.osy = osy; p.osx = osx; p.oay = oay; p.oax = oax; p.oH = oH; p.oW = oW;
    return gemm(st, p);
}

// image fp32 NCHW [B][3][H][W] (values 0..255) -> map fp32 [B][1][Ho][Wo] in [0, 1], Ho = 4 ceil(ceil(H/2)/2) (likewise Wo)
extern "C" int car_lineart_forward(CarLineArt* m, const float* img, int32_t B, int32_t H, int32_t W, float* out, void* stream) {
    if (!m || !img || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || H <= 4 || W <= 4) CAR_FAIL(CAR_ERR_ARG, "image must be larger than 4 x 4 (the residual blocks' reflection padding needs a 2 x 2 map)");
    cudaStream_t st = (cudaStream_t)stream;
    const int H1 = (H + 1) / 2, W1 = (W + 1) / 2, H2 = (H1 + 1) / 2, W2 = (W1 + 1) / 2, H3 = 2 * H2, W3 = 2 * W2, Ho = 2 * H3, Wo = 2 * W3;
    const size_t Bz = (size_t)B;
    const size_t f_bytes = Bz * 4 * std::max({(size_t)H * W * 64, (size_t)H1 * W1 * 128, (size_t)H2 * W2 * 256, (size_t)H3 * W3 * 128, (size_t)Ho * Wo * 64});
    const size_t s_bytes = Bz * std::max({(size_t)(H + 6) * (W + 6) * 24 * 2, (size_t)(H + 2) * (W + 2) * 192 * 2, (size_t)(H1 + 2) * (W1 + 2) * 384 * 2,
                                          (size_t)(H2 + 2) * (W2 + 2) * 768 * 2, (size_t)(H3 + 1) * (W3 + 1) * 384 * 2, (size_t)(Ho + 6) * (Wo + 6) * 64 * 4});
    const size_t x_bytes = Bz * H2 * W2 * 256 * 4;
    Buf<float> F, part, stats; Buf<char> S; float* X[2];   // S holds S3 (bf16) maps and, for the head, an fp32 map: carved in bytes
    CAR_TRY(m->ws.carve([&](Carve& c) {
        F = c.take<float>(f_bytes / 4);
        S = c.take<char>(s_bytes);
        X[0] = c.take<float>(x_bytes / 4); X[1] = c.take<float>(x_bytes / 4);
        part = c.take<float>(2 * Bz * GN_MAX_CHUNKS * 256);
        stats = c.take<float>(Bz * 256 * 2);
    }));
    bf16* S3 = (bf16*)S.p;
    // InstanceNorm of F [B][h][w][C] (+ resid) (ReLU) -> padded S, optional carrier
    auto inorm = [&](int h, int w, int C, const float* resid, float* carrier, InApply a) -> int {
        CAR_TRY(gn_stats(st, F, B, h * w, C, 1, 1e-5f, part, stats));
        const long long n = (long long)B * (h + a.pt + a.pb) * (w + a.pl + a.pr) * C;
        CAR_TRY(car_fits("inorm", S, (size_t)n * (a.s3 ? 6 : 4)));
        CAR_LAUNCH(instnorm_apply_pad_kernel, gsz(n), 256, 0, st, (const float*)F, (const float*)stats, resid, carrier, S, B, h, w, C, a);
        return CAR_OK;
    };
    const InApply zero1{1, 1, 1, 1, 0, 1, 1}, refl1{1, 1, 1, 1, 1, 1, 1}, zero_br{0, 0, 1, 1, 0, 1, 1};
    // model0: ReflectionPad2d(3), Conv 7x7 3 -> 64, IN, ReLU
    CAR_TRY(image_split3(st, img, nullptr, Buf<bf16>{S3, S.cap / 2}, X3Image{B, 3, H, W, 8, 3, 3, 3, 3, 1}));
    CAR_TRY(x3_win(st, m->stem, S3, B, H + 6, W + 6, 1, H, W, F, H, W));
    CAR_TRY(inorm(H, W, 64, nullptr, nullptr, zero1));
    // model1: 2 x [Conv 3x3 stride 2 pad 1 (zeros), IN, ReLU]
    CAR_TRY(x3_win(st, m->down[0], S3, B, H + 2, W + 2, 2, H1, W1, F, H1, W1));
    CAR_TRY(inorm(H1, W1, 128, nullptr, nullptr, zero1));
    CAR_TRY(x3_win(st, m->down[1], S3, B, H1 + 2, W1 + 2, 2, H2, W2, F, H2, W2));
    CAR_TRY(inorm(H2, W2, 256, nullptr, X[0], refl1));
    // model2: 3 x ResidualBlock: x + [ReflPad 1, Conv, IN, ReLU, ReflPad 1, Conv, IN](x); the fp32 carrier x ping-pongs X[0] / X[1]
    for (int r = 0; r < 3; ++r) {
        CAR_TRY(x3_win(st, m->res[2 * r], S3, B, H2 + 2, W2 + 2, 1, H2, W2, F, H2, W2));
        CAR_TRY(inorm(H2, W2, 256, nullptr, nullptr, refl1));
        CAR_TRY(x3_win(st, m->res[2 * r + 1], S3, B, H2 + 2, W2 + 2, 1, H2, W2, F, H2, W2));
        InApply a = r < 2 ? refl1 : zero_br;          // the last block feeds the transposed convolution
        a.relu = 0;
        CAR_TRY(inorm(H2, W2, 256, X[r & 1], r < 2 ? X[(r + 1) & 1] : nullptr, a));
    }
    // model3: 2 x [ConvTranspose2d 3x3 stride 2 pad 1 output_padding 1, IN, ReLU], four parity classes each
    auto up = [&](const X3W (&c)[4], int h, int w) -> int {
        for (int cls = 0; cls < 4; ++cls) CAR_TRY(x3_win(st, c[cls], S3, B, h + 1, w + 1, 1, h, w, F, 2 * h, 2 * w, 2, 2, cls >> 1, cls & 1));
        return CAR_OK;
    };
    CAR_TRY(up(m->up[0], H2, W2));
    CAR_TRY(inorm(H3, W3, 128, nullptr, nullptr, zero_br));
    CAR_TRY(up(m->up[1], H3, W3));
    // model4: ReflectionPad2d(3), Conv 7x7 64 -> 1, Sigmoid (direct fp32 on the padded fp32 map)
    CAR_TRY(inorm(Ho, Wo, 64, nullptr, nullptr, InApply{3, 3, 3, 3, 1, 0, 1}));
    CAR_LAUNCH(lineart_head_kernel, gsz((long long)B * Ho * Wo * 32), 256, 0, st, (const float*)S.p, (const float*)m->head_w, (const float*)m->head_b, out, B, Ho, Wo);
    return CAR_OK;
}

// ---------------------------------------------------------------------------------------------------------
// DPT depth detector (row f3): transformers DPTForDepthEstimation — ViT encoder, reassemble (readout "project", factors 4, 2, 1,
// 0.5), neck 3x3 convolutions, four fusion stages, depth head.  fp32 in the reference => fp32-grade here: fp32 activations, every
// GEMM and 3x3 stride-1 convolution on the fp32-output wgmma instantiation over split-bf16 operands, the stride-2 convolution on
// the window GEMM (gemm_dense.cuh A_WIN), attention fused (dpt.cuh).  No eager or mma.sync fall-back for the wgmma stages.
// ---------------------------------------------------------------------------------------------------------
struct DptLayer { X3W qkv, o, fc1, fc2; float *ln1w, *ln1b, *ln2w, *ln2b; };
struct DptDecoder {                                     // fusion stages and depth head (shared with MiDaS DPT-Hybrid)
    X3W fproj[4], rcu[4][2][2];                         // fusion layer j: projection, residual_layer{1,2}.convolution{1,2}
    X3W head0, head2;
    float *head4w, *head4b;
};
struct CarDpt : CarOwned {
    CarDptDesc d;
    X3W patch;
    float *cls, *pos;                                   // [C], [1 + g^2][C]
    using Layer = DptLayer;
    std::vector<Layer> L;
    X3W proj[4], resize[4], readout[4], neck[4];        // resize: ConvTranspose2d GEMM (stages 0, 1), 3x3 stride-2 convolution (3)
    DptDecoder dec;
};
static const int DPT_FACTOR[4] = {4, 2, 1, 0};         // 0: the 0.5 stage (3x3 stride-2 convolution)

// ConvTranspose2d(k = s = f): weight [cin][cin][f][f] -> W3 [f^2 cin][3 cin] (dpt.cuh dpt_convT_pack_kernel); the bias repeated per
// (ky, kx)
static X3W dpt_convT(TensorReader& tc, int cin, int f) {
    const int n = f * f * cin;
    const float* w = tc.next();
    X3W L{(bf16*)tc.alloc((size_t)n * cin * 3 * 2), nullptr, n, 3 * cin, 1, 1};
    tc.pack(dpt_convT_pack_kernel, (long long)n * cin, w, L.w, cin, cin, f);
    const float* b = tc.next();
    float* bias = (float*)tc.alloc((size_t)n * 4);
    for (int t = 0; t < f * f; ++t) tc.copy(bias + (size_t)t * cin, b, cin);
    L.b = bias;
    return L;
}

extern "C" int car_dpt_create(const CarDptDesc* desc, const void* const* tensors, int32_t n_tensors, void* stream, CarDpt** out) {
    if (!desc || !tensors || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    const CarDptDesc& d = *desc;
    if (d.hidden <= 0 || d.hidden % 64 || d.n_heads * 64 != d.hidden) CAR_FAIL(CAR_ERR_UNSUPPORTED, "heads must be 64-dimensional (hidden == 64 * heads)");
    if (d.n_layers <= 0 || d.mlp <= 0 || d.mlp % 8 || d.pos_grid <= 0 || !(d.ln_eps > 0.f)) CAR_FAIL(CAR_ERR_ARG, "bad layers / mlp / pos_grid / eps");
    for (int i = 0; i < 4; ++i) {
        if (d.neck[i] <= 0 || d.neck[i] % 64) CAR_FAIL(CAR_ERR_UNSUPPORTED, "neck sizes must be positive multiples of 64");
        if (d.out_indices[i] < 0 || d.out_indices[i] >= d.n_layers || (i && d.out_indices[i] <= d.out_indices[i - 1]))
            CAR_FAIL(CAR_ERR_ARG, "out indices must be ascending encoder layers");
    }
    if (d.fusion <= 0 || d.fusion % 128) CAR_FAIL(CAR_ERR_UNSUPPORTED, "fusion size must be a positive multiple of 128");
    if (n_tensors != 4 + 16 * d.n_layers + 74) CAR_FAIL(CAR_ERR_ARG, "DPT expects 4 + 16 * n_layers + 74 tensors in state-dict order");
    CarDpt* m = new CarDpt();
    m->d = d;
    const int C = d.hidden, F = d.fusion;
    TensorReader tc(__func__, tensors, n_tensors, stream, m);
    // weights [n][cin][kh][kw] (kh = kw = 1: nn.Linear) -> W3 [n][kh][kw][3 cin]
    // dpt.embeddings
    m->cls = tc.f32(C);
    m->pos = tc.f32((long long)(1 + d.pos_grid * d.pos_grid) * C);
    m->patch = tc.x3(C, 3 * 256, 1, 3 * 256);           // [C][3][16][16] read as [C][768]
    // dpt.encoder.layer.{i}: query, key, value (one [3C][3C] GEMM), output.dense, intermediate.dense, output.dense, LN before / after
    m->L.resize(d.n_layers);
    for (int l = 0; l < d.n_layers; ++l) {
        CarDpt::Layer& Ly = m->L[l];
        bf16* qkv = (bf16*)tc.alloc((size_t)3 * C * C * 3 * 2);
        float* qkv_b = (float*)tc.alloc((size_t)3 * C * 4);
        for (int j = 0; j < 3 && tc.ok(); ++j) {
            const float* w = tc.next();
            tc.pack(conv_weight_pack_x3_kernel, (long long)C * C, w, qkv + (size_t)j * C * 3 * C, C, C, 1, 1, C);
            tc.copy(qkv_b + (size_t)j * C, tc.next(), C);
        }
        Ly.qkv = X3W{qkv, qkv_b, 3 * C, 3 * C, 1, 1};
        Ly.o = tc.x3(C, C, 1, C);
        Ly.fc1 = tc.x3(d.mlp, C, 1, C);
        Ly.fc2 = tc.x3(C, d.mlp, 1, d.mlp);
        Ly.ln1w = tc.f32(C); Ly.ln1b = tc.f32(C); Ly.ln2w = tc.f32(C); Ly.ln2b = tc.f32(C);
    }
    tc.skip(2);                                         // dpt.layernorm: applied to last_hidden_state only, which depth does not use
    // neck.reassemble_stage.layers.{i}: projection (1x1), resize
    for (int i = 0; i < 4; ++i) {
        m->proj[i] = tc.x3(d.neck[i], C, 1, C);
        if (DPT_FACTOR[i] > 1) m->resize[i] = dpt_convT(tc, d.neck[i], DPT_FACTOR[i]);
        else if (DPT_FACTOR[i] == 0) m->resize[i] = tc.x3(d.neck[i], d.neck[i], 3, d.neck[i]);
    }
    for (int i = 0; i < 4; ++i) m->readout[i] = tc.x3(C, 2 * C, 1, 2 * C);
    for (int i = 0; i < 4; ++i) m->neck[i] = tc.x3(F, d.neck[i], 3, d.neck[i], false);
    for (int j = 0; j < 4; ++j) {
        m->dec.fproj[j] = tc.x3(F, F, 1, F);
        for (int r = 0; r < 2; ++r)
            for (int c = 0; c < 2; ++c) m->dec.rcu[j][r][c] = tc.x3(F, F, 3, F);
    }
    m->dec.head0 = tc.x3(F / 2, F, 3, F);
    m->dec.head2 = tc.x3(32, F / 2, 3, F / 2);
    m->dec.head4w = tc.f32(32); m->dec.head4b = tc.f32(1);
    const int rc = tc.finish();
    if (rc != CAR_OK) { delete m; return rc; }
    *out = m;
    return CAR_OK;
}
extern "C" int car_dpt_destroy(CarDpt* m) {
    delete m;
    return CAR_OK;
}

// wgmma GEMM (gemm.h gemm_f32): out fp32 [M][ldc] = a3 (S3 rows [M][w.cin3]) · W3^T + bias (+ resid [M][ldc])
static int x3_gemm(cudaStream_t st, const X3W& w, const bf16* a3, int M, Buf<float> out, int ldc, const float* resid = nullptr) {
    CAR_TRY(car_fits(__func__, out, (size_t)(M - 1) * ldc + w.n));
    return gemm_f32(st, a3, w.w, M, w.n, w.kh * w.kw * w.cin3, w.b, resid, out, ldc);
}
// TMA convolution frame: a map smaller than one 16 x 8 pixel box is held in a zero-filled frame of at least that size
static inline int x3_fh(int H) { return std::max(H, WG_TH); }
static inline int x3_fw(int W) { return std::max(W, WG_TW); }
// wgmma 3x3 / pad 1 / stride 1 convolution (gemm.h gemm_f32_conv3): S3 NHWC frame [B][x3_fh(H)][x3_fw(W)][w.cin3] -> fp32 NHWC
// [B][H][W][w.n] (+ resid)
static int x3_conv3(cudaStream_t st, const X3W& w, const bf16* s3, int B, int H, int W, Buf<float> out, const float* resid = nullptr) {
    CAR_TRY(car_fits(__func__, out, (size_t)B * H * W * w.n));
    return gemm_f32_conv3(st, s3, x3_fh(H), x3_fw(W), w.w, B, H, W, w.cin3, w.n, w.b, resid, out);
}
// S3 image producer (dpt.cuh dpt_image_split_kernel)
static int dpt_img(cudaStream_t st, const float* a, const float* b, float* sum_out, Buf<bf16> y, DptImg q) {
    CAR_TRY(car_fits(__func__, y, (size_t)q.B * q.Hp * q.Wp * 3 * q.C));
    CAR_LAUNCH(dpt_image_split_kernel, gsz((long long)q.B * q.Hp * q.Wp * q.C), 256, 0, st, a, b, sum_out, y, q);
    return CAR_OK;
}
static DptImg dpt_frame(int B, int H, int W, int C) { return DptImg{B, H, W, C, x3_fh(H), x3_fw(W), 0, 0, 0, 0, 0}; }

// one pre-LN encoder layer over fp32 rows x [B][T][C] -> dst (x may equal dst); S, T0 and X1 are scratch
static int dpt_layer(cudaStream_t st, const DptLayer& Ly, const float* x, Buf<float> dst, int B, int T, int C, int heads, int mlp, float eps, Buf<bf16> S,
                     Buf<float> T0, Buf<float> X1) {
    const int M = B * T;
    CAR_TRY(car_fits(__func__, S, (size_t)M * 3 * std::max(C, mlp)));   // the LayerNorm, attention and GELU rows written below
    CAR_LAUNCH(dpt_layernorm_split_kernel, M, DPT_LN_THREADS, 0, st, x, (const float*)Ly.ln1w, (const float*)Ly.ln1b, S, C, eps);
    CAR_TRY(x3_gemm(st, Ly.qkv, S, M, T0, 3 * C));
    CAR_LAUNCH(dpt_attention_kernel, dim3((T + DPT_AT_B - 1) / DPT_AT_B, heads, B), 128, 0, st, (const float*)T0, S, T, C);
    CAR_TRY(x3_gemm(st, Ly.o, S, M, X1, C, x));
    CAR_LAUNCH(dpt_layernorm_split_kernel, M, DPT_LN_THREADS, 0, st, (const float*)X1, (const float*)Ly.ln2w, (const float*)Ly.ln2b, S, C, eps);
    CAR_TRY(x3_gemm(st, Ly.fc1, S, M, T0, mlp));
    CAR_TRY(split3_rows(st, T0, S, M, mlp, X3_ROWS_A_GELU));
    CAR_TRY(x3_gemm(st, Ly.fc2, S, M, dst, C, X1));
    return CAR_OK;
}

// fusion, from the coarsest feature: [prev + RCU1(feature)] -> RCU2 -> x2 bilinear (align_corners=True) -> 1x1 projection, then the
// head: conv 3x3 F -> F/2, x2 bilinear (align_corners=True), conv 3x3 F/2 -> 32, ReLU, conv 1x1 32 -> 1, ReLU.
// RCU(r) = conv2(ReLU(conv1(ReLU(r)))) + r; the ReLUs, the add and the upsample are fused into the S3 producers.
// fe[i]: fp32 NHWC [B][sh[i]][sw[i]][F] (i = 0 finest, 2 sh[i] = sh[i-1]); the depth map is [B][H][W] with H = 4 sh[0]
static int dpt_decode(cudaStream_t st, const DptDecoder& w, const Buf<float> fe[4], const int sh[4], const int sw[4], int B, int H, int W, int F,
                      Buf<float> T0, Buf<float> T1, Buf<float> T2, Buf<bf16> S, float* depth) {
    float* prev = nullptr;                              // fp32 [B][s][s][F], in T1
    for (int j = 0; j < 4; ++j) {
        const int i = 3 - j, s = sh[i], t = sw[i];
        DptImg rq = dpt_frame(B, s, t, F);
        rq.relu = 1;
        const float* xin = fe[i];                       // input of residual_layer2
        if (prev) {
            CAR_TRY(dpt_img(st, fe[i], nullptr, nullptr, S, rq));
            CAR_TRY(x3_conv3(st, w.rcu[j][0][0], S, B, s, t, T0));
            CAR_TRY(dpt_img(st, T0, nullptr, nullptr, S, rq));
            CAR_TRY(x3_conv3(st, w.rcu[j][0][1], S, B, s, t, T0, fe[i]));
            CAR_TRY(dpt_img(st, prev, T0, prev, S, rq));                             // prev += RCU1(feature), ReLU'd S3 of it
            xin = prev;
        } else {
            CAR_TRY(dpt_img(st, fe[i], nullptr, nullptr, S, rq));
        }
        CAR_TRY(x3_conv3(st, w.rcu[j][1][0], S, B, s, t, T0));
        CAR_TRY(dpt_img(st, T0, nullptr, nullptr, S, rq));
        CAR_TRY(x3_conv3(st, w.rcu[j][1][1], S, B, s, t, T2, xin));
        DptImg uq{B, 2 * s, 2 * t, F, 2 * s, 2 * t, 0, 0, 0, 1, 0};
        CAR_TRY(dpt_img(st, T2, nullptr, nullptr, S, uq));
        CAR_TRY(x3_gemm(st, w.fproj[j], S, B * 4 * s * t, T1, F));
        prev = T1;
    }
    const int h2 = H / 2, w2 = W / 2;
    CAR_TRY(dpt_img(st, prev, nullptr, nullptr, S, dpt_frame(B, h2, w2, F)));
    CAR_TRY(x3_conv3(st, w.head0, S, B, h2, w2, T0));
    DptImg uq = dpt_frame(B, H, W, F / 2);
    uq.up = 1;
    CAR_TRY(dpt_img(st, T0, nullptr, nullptr, S, uq));
    CAR_TRY(x3_conv3(st, w.head2, S, B, H, W, T2));
    CAR_LAUNCH(dpt_head_kernel, gsz((long long)B * H * W * 32), 256, 0, st, (const float*)T2, (const float*)w.head4w, (const float*)w.head4b, depth,
               (long long)B * H * W);
    return CAR_OK;
}

// pixel_values fp32 NCHW [B][3][H][W] -> predicted_depth fp32 [B][H][W]
extern "C" int car_dpt_forward(CarDpt* m, const float* pixel_values, int32_t B, int32_t H, int32_t W, float* depth, void* stream) {
    if (!m || !pixel_values || !depth) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || H != W || H % 32 || H < 64) CAR_FAIL(CAR_ERR_ARG, "pixel_values must be square with a side that is a multiple of 32 and at least 64");
    cudaStream_t st = (cudaStream_t)stream;
    const CarDptDesc& d = m->d;
    const int C = d.hidden, F = d.fusion, h = H / 16, T = 1 + h * h, M = B * T, Mp = B * h * h;
    const int side[4] = {4 * h, 2 * h, h, h / 2};
    const size_t Bz = (size_t)B;
    // workspace: encoder fp32 rows, fp32 temporaries, the four neck features, one S3 buffer (each operand is consumed before the next
    // is written)
    size_t ft = (size_t)M * std::max(3 * C, d.mlp);
    size_t s3 = std::max({(size_t)M * 3 * std::max(C, d.mlp), (size_t)Mp * 3 * 768, (size_t)Mp * 6 * C});
    for (int i = 0; i < 4; ++i) {
        const int f = DPT_FACTOR[i];
        ft = std::max({ft, (size_t)Mp * C, (size_t)Mp * (f > 1 ? f * f : 1) * d.neck[i]});
        s3 = std::max({s3, (size_t)Mp * 3 * d.neck[i], Bz * (h + 2) * (h + 2) * 3 * d.neck[i],
                       Bz * x3_fh(side[i]) * x3_fw(side[i]) * 3 * std::max(d.neck[i], F)});
    }
    ft = std::max({ft, Bz * 64 * h * h * F, Bz * 256 * h * h * 32});
    s3 = std::max({s3, Bz * 64 * h * h * 3 * F, Bz * 256 * h * h * 3 * (F / 2)});
    Buf<float> X, X1, keep[4], T0, T1, T2, fe[4]; Buf<bf16> S;
    CAR_TRY(m->ws.carve([&](Carve& c) {
        X = c.take<float>((size_t)M * C);
        X1 = c.take<float>((size_t)M * C);
        for (int i = 0; i < 4; ++i) keep[i] = c.take<float>((size_t)M * C);
        T0 = c.take<float>(ft);
        T1 = c.take<float>(ft);
        T2 = c.take<float>(ft);
        for (int i = 0; i < 4; ++i) fe[i] = c.take<float>(Bz * side[i] * side[i] * F);
        S = c.take<bf16>(s3);
    }));

    // ---- embeddings: patch convolution as a GEMM, [CLS], resized position embeddings
    CAR_TRY(car_fits("dpt patchify", S, (size_t)Mp * 3 * 768));
    CAR_LAUNCH(dpt_patchify_kernel, gsz((long long)Mp * 768), 256, 0, st, pixel_values, S, B, h);
    CAR_TRY(x3_gemm(st, m->patch, S, Mp, T0, C));
    CAR_LAUNCH(dpt_assemble_kernel, gsz((long long)M * C), 256, 0, st, (const float*)T0, (const float*)m->cls, (const float*)m->pos, X, B, h, h, d.pos_grid,
               C);
    // ---- encoder: pre-LN layers; the residual stream stays fp32, the out-index layers write their output into keep[]
    float* x = X;
    int kept = 0;
    for (int l = 0; l < d.n_layers; ++l) {
        Buf<float> dst = (kept < 4 && d.out_indices[kept] == l) ? keep[kept++] : X;
        CAR_TRY(dpt_layer(st, m->L[l], x, dst, B, T, C, d.n_heads, d.mlp, d.ln_eps, S, T0, X1));
        x = dst;
        if (kept == 4) break;                           // later layers feed nothing the depth map uses
    }
    // ---- reassemble: readout projection + GELU, 1x1 projection, resize; then the neck's 3x3 convolution -> fe[i] fp32 NHWC
    for (int i = 0; i < 4; ++i) {
        const int Cn = d.neck[i], f = DPT_FACTOR[i], s = side[i];
        CAR_TRY(car_fits("dpt readout split", S, (size_t)Mp * 3 * std::max(2 * C, Cn)));   // this and the two row splits below
        CAR_LAUNCH(dpt_readout_split_kernel, gsz((long long)Mp * 2 * C), 256, 0, st, (const float*)keep[i], S, B, h * h, C);
        CAR_TRY(x3_gemm(st, m->readout[i], S, Mp, T0, C));
        CAR_TRY(split3_rows(st, T0, S, Mp, C, X3_ROWS_A_GELU));
        CAR_TRY(x3_gemm(st, m->proj[i], S, Mp, T1, Cn));                            // [B][h][h][Cn]
        DptImg q = dpt_frame(B, s, s, Cn);
        if (f > 1) {
            CAR_TRY(split3_rows(st, T1, S, Mp, Cn));
            CAR_TRY(x3_gemm(st, m->resize[i], S, Mp, T0, f * f * Cn));           // [B][h][h][f][f][Cn]
            q.shuf = f;
            CAR_TRY(dpt_img(st, T0, nullptr, nullptr, S, q));
        } else if (f == 0) {
            CAR_TRY(dpt_img(st, T1, nullptr, nullptr, S, DptImg{B, h, h, Cn, h + 2, h + 2, 1, 1, 0, 0, 0}));
            CAR_TRY(x3_win(st, m->resize[i], S, B, h + 2, h + 2, 2, s, s, T0, s, s));
            CAR_TRY(dpt_img(st, T0, nullptr, nullptr, S, q));
        } else {
            CAR_TRY(dpt_img(st, T1, nullptr, nullptr, S, q));
        }
        CAR_TRY(x3_conv3(st, m->neck[i], S, B, s, s, fe[i]));
    }
    // ---- fusion and head
    return dpt_decode(st, m->dec, fe, side, side, B, H, W, F, T0, T1, T2, S, depth);
}

// ---------------------------------------------------------------------------------------------------------
// MiDaS DPT-Hybrid depth detector (row f3): condition/midas (DPTDepthModel, backbone vitb_rn50_384) — a ResNet-50 trunk (timm
// ResNetV2: weight-standardised bias-free convolutions, GroupNorm(32), TF "SAME" padding, stages of 3, 4, 9 bottlenecks) whose
// stage-2 map is the token grid of a ViT-B/16 (1x1 projection, [CLS], position embeddings resized to h x w), then reassemble
// (stage outputs 0 and 1 as they are; readout "project" of blocks 8 and 11, 1x1 convolution, and a 3x3/2 convolution for the
// last), the neck's 3x3 convolutions and the DPT fusion and head (dpt_decode).  fp32 in the reference => fp32-grade here: 1x1
// convolutions and GEMMs on x3_gemm, 3x3 stride-1 convolutions on x3_conv3 (wgmma), the stem and the stride-2 convolutions on
// the window GEMM (x3_win), GroupNorm in midas.cuh.  Token grids need not be square.
// ---------------------------------------------------------------------------------------------------------
struct MdBlock { X3W dn, c1, c2, c3; NormF dnn, n1, n2, n3; int cin, mid, out, stride; };
static const int MD_DEPTH[3] = {3, 4, 9}, MD_OUT[3] = {256, 512, 1024};
constexpr int MD_BLOCKS = 16, MD_C = 768, MD_HEADS = 12, MD_MLP = 3072, MD_F = 256, MD_GRID = 24, MD_NT = 368;
struct CarMidas : CarOwned {
    float* zero;                                        // [1024] zeros: the bias of the bias-free window convolutions
    X3W stem;
    NormF stem_n;
    MdBlock blk[MD_BLOCKS];
    X3W patch;                                          // patch_embed.proj: 1x1 convolution 1024 -> 768 with bias
    float *cls, *pos;                                   // [768], [1 + 24^2][768]
    DptLayer L[12];
    X3W readout[2], proj[2], resize4, rn[4];            // act_postprocess{3,4}: readout, 1x1, (3x3/2); scratch.layer{1..4}_rn
    DptDecoder dec;
};

// tensors (fp32, device), state-dict order of controlar_b200.condition.midas.DPTDepthModel: pretrained.model.{cls_token, pos_embed,
// patch_embed.backbone.{stem, stages.*.blocks.*}, patch_embed.proj, blocks.*, norm, head}, pretrained.act_postprocess{3,4},
// scratch.layer{1..4}_rn, scratch.refinenet{1..4}, scratch.output_conv
extern "C" int car_midas_create(const void* const* tensors, int32_t n_tensors, void* stream, CarMidas** out) {
    if (!tensors || !out) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (n_tensors != MD_NT) CAR_FAIL(CAR_ERR_ARG, "MiDaS DPT-Hybrid expects 368 tensors in state-dict order");
    CarMidas* m = new CarMidas();
    TensorReader tc(__func__, tensors, n_tensors, stream, m);
    // weight-standardised bias-free convolution [n][cin][k][k] -> W3 [n][k][k][3 cin_pad]; the standardised fp32 weight goes through
    // `wsd`, re-used in stream order (its largest user is a 3x3 256 -> 256 convolution).  A window convolution (7x7/2 stem, stride-2
    // 1x1 and 3x3) takes the zero bias.
    float* wsd = (float*)tc.alloc((size_t)256 * 256 * 9 * 4);
    m->zero = tc.zeros(1024);
    auto sconv = [&](int n, int cin, int k, int cin_pad, bool window) {
        tc.launch(midas_ws_kernel, n, MD_THREADS, tc.next(), wsd, cin * k * k, 1e-8);
        return tc.x3(wsd, n, cin, k, cin_pad, window ? m->zero : nullptr);
    };
    m->cls = tc.f32(MD_C);
    m->pos = tc.f32((long long)(1 + MD_GRID * MD_GRID) * MD_C);
    m->stem = sconv(64, 3, 7, 8, true);                 // 3 input channels padded to 8 (16-byte chunks)
    take_norm(tc, 64, &m->stem_n);
    int cin = 64, bi = 0;
    for (int s = 0; s < 3; ++s)
        for (int b = 0; b < MD_DEPTH[s]; ++b, ++bi) {
            MdBlock& k = m->blk[bi];
            k.cin = cin; k.out = MD_OUT[s]; k.mid = k.out / 4; k.stride = (s > 0 && b == 0) ? 2 : 1;
            if (b == 0) { k.dn = sconv(k.out, cin, 1, cin, k.stride == 2); take_norm(tc, k.out, &k.dnn); }
            k.c1 = sconv(k.mid, cin, 1, cin, false); take_norm(tc, k.mid, &k.n1);
            k.c2 = sconv(k.mid, k.mid, 3, k.mid, k.stride == 2); take_norm(tc, k.mid, &k.n2);
            k.c3 = sconv(k.out, k.mid, 1, k.mid, false); take_norm(tc, k.out, &k.n3);
            cin = k.out;
        }
    m->patch = tc.x3(MD_C, 1024, 1, 1024);
    for (int l = 0; l < 12; ++l) {                      // blocks.{l}: norm1, attn.qkv (fused), attn.proj, norm2, mlp.fc1, mlp.fc2
        DptLayer& Ly = m->L[l];
        Ly.ln1w = tc.f32(MD_C); Ly.ln1b = tc.f32(MD_C);
        Ly.qkv = tc.x3(3 * MD_C, MD_C, 1, MD_C);
        Ly.o = tc.x3(MD_C, MD_C, 1, MD_C);
        Ly.ln2w = tc.f32(MD_C); Ly.ln2b = tc.f32(MD_C);
        Ly.fc1 = tc.x3(MD_MLP, MD_C, 1, MD_C);
        Ly.fc2 = tc.x3(MD_C, MD_MLP, 1, MD_MLP);
    }
    tc.skip(4);                                         // norm, head: the ViT's final norm and classifier, unused by the depth map
    for (int i = 0; i < 2; ++i) {
        m->readout[i] = tc.x3(MD_C, 2 * MD_C, 1, 2 * MD_C);
        m->proj[i] = tc.x3(MD_C, MD_C, 1, MD_C);
    }
    m->resize4 = tc.x3(MD_C, MD_C, 3, MD_C);
    const int rn_in[4] = {256, 512, MD_C, MD_C};
    for (int i = 0; i < 4; ++i) m->rn[i] = tc.x3(MD_F, rn_in[i], 3, rn_in[i], false);
    for (int r = 1; r <= 4; ++r) {                      // refinenet{r} is fusion layer 4 - r (the coarsest runs first)
        const int j = 4 - r;
        m->dec.fproj[j] = tc.x3(MD_F, MD_F, 1, MD_F);
        for (int u = 0; u < 2; ++u)
            for (int c = 0; c < 2; ++c) m->dec.rcu[j][u][c] = tc.x3(MD_F, MD_F, 3, MD_F);
    }
    m->dec.head0 = tc.x3(MD_F / 2, MD_F, 3, MD_F);
    m->dec.head2 = tc.x3(32, MD_F / 2, 3, MD_F / 2);
    m->dec.head4w = tc.f32(32); m->dec.head4b = tc.f32(1);
    const int rc = tc.finish();
    if (rc != CAR_OK) { delete m; return rc; }
    *out = m;
    return CAR_OK;
}
extern "C" int car_midas_destroy(CarMidas* m) {
    delete m;
    return CAR_OK;
}

// x fp32 NCHW [B][3][H][W] -> depth fp32 [B][H][W]
extern "C" int car_midas_forward(CarMidas* m, const float* x, int32_t B, int32_t H, int32_t W, float* depth, void* stream) {
    if (!m || !x || !depth) CAR_FAIL(CAR_ERR_ARG, "null argument");
    if (B <= 0 || H % 32 || W % 32 || H < 64 || W < 64) CAR_FAIL(CAR_ERR_ARG, "x must be [B][3][H][W] with H and W multiples of 32 and at least 64");
    cudaStream_t st = (cudaStream_t)stream;
    const int C = MD_C, F = MD_F, h = H / 16, w = W / 16, P = h * w, T = 1 + P, M = B * T, Mp = B * P;
    const int sh[4] = {H / 4, H / 8, h, h / 2}, sw[4] = {W / 4, W / 8, w, w / 2};
    const size_t Bz = (size_t)B, HW = (size_t)H * W;
    // workspace: encoder rows, fp32 temporaries, trunk carriers, neck features, GroupNorm partials, one S3 buffer (each operand is
    // consumed before the next is written)
    const size_t ft = std::max({(size_t)M * MD_MLP, Bz * HW / 4 * F, Bz * HW * 32, Bz * HW / 4 * 64});
    const size_t car = Bz * HW / 16 * 256;              // the widest trunk map: stage 0, 256 channels at H/4
    size_t s3 = std::max({Bz * (H + 5) * (W + 5) * 24, (size_t)M * 3 * MD_MLP, (size_t)Mp * 6 * C, Bz * (h + 2) * (w + 2) * 3 * C,
                          Bz * 4 * sh[0] * sw[0] * 3 * F, Bz * x3_fh(H / 2) * x3_fw(W / 2) * 3 * F, Bz * HW * 3 * (F / 2)});
    {
        int hh = H / 4, ww = W / 4, ci = 64;
        for (int s = 0; s < 3; ++s) {
            const int mid = MD_OUT[s] / 4, ho = s ? hh / 2 : hh, wo = s ? ww / 2 : ww;
            s3 = std::max({s3, Bz * hh * ww * 3 * ci, Bz * (hh + 1) * (ww + 1) * 3 * mid, Bz * x3_fh(hh) * x3_fw(ww) * 3 * mid,
                           Bz * ho * wo * 3 * MD_OUT[s]});
            ci = MD_OUT[s]; hh = ho; ww = wo;
        }
        const int rn_in[4] = {256, 512, MD_C, MD_C};
        for (int i = 0; i < 4; ++i) s3 = std::max(s3, Bz * x3_fh(sh[i]) * x3_fw(sw[i]) * 3 * std::max(rn_in[i], F));
    }
    Buf<float> X, X1, K[2], T0, T1, T2, Xa, Xb, Td, fe[4], part, stats, rstats; Buf<bf16> S;
    CAR_TRY(m->ws.carve([&](Carve& c) {
        X = c.take<float>((size_t)M * C);
        X1 = c.take<float>((size_t)M * C);
        K[0] = c.take<float>((size_t)M * C); K[1] = c.take<float>((size_t)M * C);
        T0 = c.take<float>(ft);
        T1 = c.take<float>(ft);
        T2 = c.take<float>(ft);
        Xa = c.take<float>(car);
        Xb = c.take<float>(car);
        Td = c.take<float>(car);
        for (int i = 0; i < 4; ++i) fe[i] = c.take<float>(Bz * sh[i] * sw[i] * F);
        part = c.take<float>(2 * Bz * GN_MAX_CHUNKS * MD_OUT[2]);
        stats = c.take<float>(Bz * GN_GROUPS * 2);
        rstats = c.take<float>(Bz * GN_GROUPS * 2);
        S = c.take<bf16>(s3);
    }));

    // GroupNorm(32, eps 1e-5) statistics of fp32 NHWC [B][hh][ww][Cc] -> stt [B][32][2]
    auto gstats = [&](const float* src, int hh, int ww, int Cc, Buf<float> stt) { return gn_stats(st, src, B, hh * ww, Cc, Cc / GN_GROUPS, 1e-5f, part, stt); };
    // GN(src) (+ resid, normalised by rn when rn.stats) (ReLU) (max-pool) -> S3 frame in S, fp32 carrier when given
    auto gn_apply = [&](const float* src, const NormF& N, const float* resid, GnAffine rn, float* carrier, int hh, int ww, int Cc, GnApply a) {
        return gn_apply_s3(st, src, GnAffine{stats, N.w, N.b}, resid, rn, carrier, S, B, hh, ww, Cc, a);
    };
    const GnAffine none{nullptr, nullptr, nullptr};

    // ---- stem: conv 7x7/2 (SAME: 2 before, 3 after) -> GN + ReLU -> max-pool 3x3/2 (SAME: 0 before, 1 after) -> S3 rows
    CAR_TRY(image_split3(st, x, nullptr, S, X3Image{B, 3, H, W, 8, 2, 2, 3, 3, 0}));
    CAR_TRY(x3_win(st, m->stem, S, B, H + 5, W + 5, 2, H / 2, W / 2, T0, H / 2, W / 2));
    CAR_TRY(gstats(T0, H / 2, W / 2, 64, stats));
    int hh = H / 4, ww = W / 4;
    CAR_TRY(gn_apply(T0, m->stem_n, nullptr, none, nullptr, H / 2, W / 2, 64, GnApply{0, 0, hh, ww, GN_ACT_RELU, 1}));
    // ---- stages: bottlenecks conv1 1x1 -> GN+ReLU -> conv2 3x3 (stride) -> GN+ReLU -> conv3 1x1 -> GN -> + shortcut -> ReLU.  S holds
    // the S3 rows of the block input; xin its fp32 carrier (the identity shortcut); the first block's shortcut is conv 1x1 (stride) + GN.
    float* xin = nullptr;
    int bi = 0;
    for (int s = 0; s < 3; ++s) {
        for (int b = 0; b < MD_DEPTH[s]; ++b, ++bi) {
            const MdBlock& k = m->blk[bi];
            const int ho = hh / k.stride, wo = ww / k.stride, Min = B * hh * ww, Mo = B * ho * wo;
            GnAffine rn = none;
            if (b == 0) {
                if (k.stride == 1) CAR_TRY(x3_gemm(st, k.dn, S, Min, Td, k.out));
                else CAR_TRY(x3_win(st, k.dn, S, B, hh, ww, 2, ho, wo, Td, ho, wo));
                CAR_TRY(gstats(Td, ho, wo, k.out, rstats));
                rn = GnAffine{rstats, k.dnn.w, k.dnn.b};
            }
            CAR_TRY(x3_gemm(st, k.c1, S, Min, T0, k.mid));
            CAR_TRY(gstats(T0, hh, ww, k.mid, stats));
            if (k.stride == 1) {
                CAR_TRY(gn_apply(T0, k.n1, nullptr, none, nullptr, hh, ww, k.mid, GnApply{0, 0, x3_fh(hh), x3_fw(ww), GN_ACT_RELU, 0}));
                CAR_TRY(x3_conv3(st, k.c2, S, B, hh, ww, T1));
            } else {                                    // SAME for 3x3/2 on an even map: no padding before, one after
                CAR_TRY(gn_apply(T0, k.n1, nullptr, none, nullptr, hh, ww, k.mid, GnApply{0, 0, hh + 1, ww + 1, GN_ACT_RELU, 0}));
                CAR_TRY(x3_win(st, k.c2, S, B, hh + 1, ww + 1, 2, ho, wo, T1, ho, wo));
            }
            CAR_TRY(gstats(T1, ho, wo, k.mid, stats));
            CAR_TRY(gn_apply(T1, k.n2, nullptr, none, nullptr, ho, wo, k.mid, GnApply{0, 0, ho, wo, GN_ACT_RELU, 0}));
            CAR_TRY(x3_gemm(st, k.c3, S, Mo, T2, k.out));
            CAR_TRY(gstats(T2, ho, wo, k.out, stats));
            Buf<float> xo = xin == Xa ? Xb : Xa;
            CAR_TRY(car_fits("midas trunk carrier", xo, (size_t)Mo * k.out));
            CAR_TRY(gn_apply(T2, k.n3, b == 0 ? Td : xin, rn, xo, ho, wo, k.out, GnApply{0, 0, ho, wo, GN_ACT_RELU, 0}));
            xin = xo; hh = ho; ww = wo;
        }
        if (s < 2) {                                    // stage outputs 0 and 1 are features 1 and 2: scratch.layer{1,2}_rn
            CAR_TRY(dpt_img(st, xin, nullptr, nullptr, S, dpt_frame(B, hh, ww, MD_OUT[s])));
            CAR_TRY(x3_conv3(st, m->rn[s], S, B, hh, ww, fe[s]));
            CAR_TRY(split3_rows(st, xin, S, (long long)B * hh * ww, MD_OUT[s]));
        }
    }
    // ---- ViT-B/16: tokens = 1x1 projection of the stage-2 map, [CLS], position embeddings resized 24 x 24 -> h x w; blocks 8 and 11
    // write their outputs into K[]
    CAR_TRY(x3_gemm(st, m->patch, S, Mp, T0, C));
    CAR_LAUNCH(dpt_assemble_kernel, gsz((long long)M * C), 256, 0, st, (const float*)T0, (const float*)m->cls, (const float*)m->pos, X, B, h, w, MD_GRID, C);
    float* xv = X;
    for (int l = 0; l < 12; ++l) {
        Buf<float> dst = l == 8 ? K[0] : l == 11 ? K[1] : X;
        CAR_TRY(dpt_layer(st, m->L[l], xv, dst, B, T, C, MD_HEADS, MD_MLP, 1e-6f, S, T0, X1));
        xv = dst;
    }
    // ---- reassemble 3 and 4: readout projection + GELU, 1x1 convolution, (3x3/2 convolution); then scratch.layer{3,4}_rn
    for (int i = 0; i < 2; ++i) {
        CAR_TRY(car_fits("midas readout split", S, (size_t)Mp * 6 * C));   // this and the row split below
        CAR_LAUNCH(dpt_readout_split_kernel, gsz((long long)Mp * 2 * C), 256, 0, st, (const float*)K[i], S, B, P, C);
        CAR_TRY(x3_gemm(st, m->readout[i], S, Mp, T0, C));
        CAR_TRY(split3_rows(st, T0, S, Mp, C, X3_ROWS_A_GELU));
        CAR_TRY(x3_gemm(st, m->proj[i], S, Mp, T1, C));                             // [B][h][w][C]
        if (i == 0) {
            CAR_TRY(dpt_img(st, T1, nullptr, nullptr, S, dpt_frame(B, h, w, C)));
        } else {
            CAR_TRY(dpt_img(st, T1, nullptr, nullptr, S, DptImg{B, h, w, C, h + 2, w + 2, 1, 1, 0, 0, 0}));
            CAR_TRY(x3_win(st, m->resize4, S, B, h + 2, w + 2, 2, sh[3], sw[3], T0, sh[3], sw[3]));
            CAR_TRY(dpt_img(st, T0, nullptr, nullptr, S, dpt_frame(B, sh[3], sw[3], C)));
        }
        CAR_TRY(x3_conv3(st, m->rn[2 + i], S, B, sh[2 + i], sw[2 + i], fe[2 + i]));
    }
    // ---- fusion (refinenet4 .. 1) and head (output_conv)
    return dpt_decode(st, m->dec, fe, sh, sw, B, H, W, F, T0, T1, T2, S, depth);
}
