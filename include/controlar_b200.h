/*
 * controlar_b200.h — C ABI of the H100-native (sm_90a) ControlAR conditional-decoding hot path.
 *
 * The reference (hustvl/ControlAR) has NO native/FFI layer: its boundary for this path is a pure-Python module
 * API (SURVEY.md §8b).  This header is therefore the boundary a maintainer binds *underneath* that Python API
 * (ctypes stub in INTEGRATION.md); each entry point names the reference function(s) it replaces
 * (paths relative to the reference tree).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no exceptions cross the boundary, no torch types.
 *   - every function returns 0 on success, <0 on error; car_last_error() gives the message (thread-local).
 *   - all device pointers are CUDA device memory owned by the CALLER (PyTorch) unless stated; the library only
 *     borrows them for the call, or until car_*_destroy for registered weights / KV caches.
 *   - every op takes a cudaStream_t (as void*) and is asynchronous on it; the library never calls
 *     cudaDeviceSynchronize and never allocates inside a decode step.
 *   - handles are not thread-safe; distinct handles may be used from distinct threads.
 *   - dtype codes: CAR_BF16 = 0, CAR_F32 = 1 (storage type of weights, activations and KV cache).  There is no CAR_F16:
 *     the reference's `--precision fp16` (autoregressive/sample/sample_t2i.py:54,197; default bf16) is refused by the Python shells
 *     with an explicit error.  Reason: the tensor-core operand format (mma.sync / wgmma with bf16 inputs), the
 *     fragment-packed weights and the 8-byte activation packets of the persistent decode kernel are all bf16, and the rounding
 *     points that parity is defined by (SURVEY.md section 8 a-notes) differ between bf16 and fp16; an fp16 twin of every kernel was
 *     not built.  fp16 checkpoints can be run by casting the module to bf16 (or fp32) first.
 */
#ifndef CONTROLAR_B200_H_
#define CONTROLAR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CAR_BF16 0
#define CAR_F32 1

#define CAR_OK 0
#define CAR_ERR_ARG (-1)
#define CAR_ERR_CUDA (-2)
#define CAR_ERR_UNSUPPORTED (-3)
#define CAR_ERR_STATE (-4)

typedef struct CarModel CarModel;   /* packed transformer weights          */
typedef struct CarState CarState;   /* per-generate() state: caches, graph */

/* Shape of gpt_t2i.ModelArgs that matters to the kernels (autoregressive/models/gpt_t2i.py:31-61). */
typedef struct CarModelDesc {
    int32_t dtype;          /* CAR_BF16 | CAR_F32 */
    int32_t dim;            /* d        */
    int32_t n_layer;        /* L, L % 3 == 0 (gpt_t2i.py:320,457) */
    int32_t n_head;         /* H, head_dim = dim / n_head must be 64 */
    int32_t ffn_dim;        /* F (gpt_t2i.py:204-209) */
    int32_t vocab_size;     /* V */
    int32_t cls_token_num;  /* T: 120 (t2i) or 1 (c2i) */
    int32_t block_size;     /* g*g, RoPE table side g (gpt_t2i.py:380-383) */
    int32_t caption_dim;    /* 2048 (t2i) ; 0 for c2i */
    int32_t model_type;     /* 0 = c2i (LabelEmbedder), 1 = t2i (CaptionEmbedder) */
    float   norm_eps;
    float   rope_base;
} CarModelDesc;

/* Device pointers to the reference checkpoint tensors, nn.Linear layout [out, in] row-major, in `dtype`
 * (state-dict keys in comments; SURVEY.md §8b "Checkpoint contract").  Arrays have n_layer entries. */
typedef struct CarWeights {
    const void* tok_embeddings;            /* tok_embeddings.weight            [V, d]   */
    const void* norm;                      /* norm.weight                      [d]      */
    const void* output;                    /* output.weight                    [V, d]   */
    const void* const* attention_norm;     /* layers.i.attention_norm.weight   [d]      */
    const void* const* wqkv;               /* layers.i.attention.wqkv.weight   [3d, d]  */
    const void* const* wo;                 /* layers.i.attention.wo.weight     [d, d]   */
    const void* const* ffn_norm;           /* layers.i.ffn_norm.weight         [d]      */
    const void* const* w1;                 /* layers.i.feed_forward.w1.weight  [F, d]   */
    const void* const* w3;                 /* layers.i.feed_forward.w3.weight  [F, d]   */
    const void* const* w2;                 /* layers.i.feed_forward.w2.weight  [d, F]   */
    const void* cap_fc1;                   /* cls_embedding.cap_proj.fc1.weight [d, caption_dim] (t2i) */
    const void* cap_fc2;                   /* cls_embedding.cap_proj.fc2.weight [d, d]            (t2i) */
    const void* label_table;               /* cls_embedding.embedding_table.weight [classes+1, d] (c2i) */
    const void* cond_fc1;                  /* condition_mlp.cap_proj.fc1.weight [d, d] */
    const void* cond_fc2;                  /* condition_mlp.cap_proj.fc2.weight [d, d] */
    const void* ctl_fc1[3];                /* condition_layers.j.fc1.weight     [d, d] */
    const void* ctl_fc2[3];                /* condition_layers.j.fc2.weight     [d, d] */
} CarWeights;

/* Sampling parameters of generate.sample()/top_k_top_p_filtering (autoregressive/models/generate.py:17-74)
 * plus the CFG knobs of prefill()/decode_one_token() (generate.py:85-110). */
typedef struct CarSampling {
    float    temperature;
    int32_t  top_k;          /* 0 = off */
    float    top_p;          /* 1.0 = off */
    int32_t  sample_logits;  /* 1 = multinomial (exponential race), 0 = arg-max (lowest index wins ties) */
    float    cfg_scale;      /* > 1 => rows [B, 2B) are the unconditional half */
    int32_t  cfg_interval;   /* -1 = always combine (generate.py:121-122) */
    uint64_t seed;           /* Philox key for the in-kernel exponential noise */
} CarSampling;

/* Sampling parameters and control strength of ONE image of a launch (car_state_set_row_sampling, car_sample_rows).
 * cfg_scale and cfg_interval stay per launch (CarSampling).  Checked on the host: temperature > 0, 0 < top_p <= 1, top_k >= 0. */
typedef struct CarRowSampling {
    float    temperature;
    int32_t  top_k;            /* 0 = off */
    float    top_p;            /* 1.0 = off */
    int32_t  sample_logits;    /* 1 = multinomial (exponential race), 0 = arg-max */
    uint64_t seed;             /* Philox key of this image's noise */
    uint32_t noise_row;        /* Philox counter word of this image's noise: 0 makes the draws depend on `seed` alone; the image
                                  index b reproduces the rule of CarSampling, whose one seed keys every image with counter b */
    float    control_strength; /* strength of the control tokens on this image's rows (the unconditional partner's included),
                                  applied by every control add of those rows, as a uniform launch at this strength applies it */
} CarRowSampling;

const char* car_last_error(void);
int car_version(void);

/* ---- model: replaces Transformer.__init__/load_state_dict/.to() weight residency (gpt_t2i.py:310-389) ---- */
int car_model_create(const CarModelDesc* desc, const CarWeights* weights, void* stream, CarModel** out);
/* Re-pack after the caller changed the borrowed weights in place (optimizer step, load_state_dict). */
int car_model_repack(CarModel* m, const CarWeights* weights, void* stream);
int car_model_destroy(CarModel* m);

/* ---- state: replaces Transformer.setup_caches (gpt_t2i.py:391-405) + the mask edit of generate()
 *      (generate.py:184-193).  k_cache[i]/v_cache[i]: caller-allocated [b_eff, H, S, 64] in `dtype`
 *      (the reference's KVCache layout, gpt_t2i.py:220-235) so that model.layers[i].attention.kv_cache stays
 *      inspectable from Python.  emb_mask: int32 [b_eff, T] (1 = attend) or NULL (all ones). ---- */
/*      rope_table: fp32 [T + block_size, 32, 2] (cos, sin) = precompute_freqs_cis_2d (gpt_t2i.py:506-519),
 *      computed by the host shell with the same torch ops so the table is bit-identical; borrowed. */
int car_state_create(CarModel* m, int32_t b_eff, int32_t max_seq /* S */, int32_t n_img_tokens /* N */,
                     void* const* k_cache, void* const* v_cache, const float* rope_table, CarState** out);
int car_state_set_emb_mask(CarState* s, const int32_t* emb_mask_dev, void* stream);
/* Per-image sampling: rows (host, B entries, copied) give image b its own CarRowSampling; B must be b_eff (no CFG) or b_eff / 2
 * (CFG).  The following car_prefill takes each row's control strength (its control_strength argument is then unused), which every
 * control add of that prefill and of the decode after it reads per row; the
 * following car_generate / car_generate_forced take each row's sampling parameters, on every decode route; the CarSampling
 * passed to them then only supplies cfg_scale and cfg_interval.  NULL returns to the scalar behaviour. */
int car_state_set_row_sampling(CarState* s, const CarRowSampling* rows, int32_t B);
int car_state_destroy(CarState* s);

/* ---- prefill: Transformer.forward inference-prefill branch (gpt_t2i.py:433-442,455-470) ----
 * cond:      t2i: [b_eff, T, caption_dim] in dtype;  c2i: int32 [b_eff] class ids.
 * condition: adapter_mlp output [b_eff, N, d] in dtype, or NULL (no control).
 * logits_out: fp32 [b_eff, T, V] when all_rows != 0 else [b_eff, V] (last prefix row only). */
int car_prefill(CarState* s, const void* cond, const void* condition, float control_strength,
                float* logits_out, int32_t all_rows, void* stream);

/* ---- teacher-forced decode step: Transformer.forward KV-cache branch (gpt_t2i.py:444-470) ----
 * tok: int32 [b_eff]; pos: sequence position of `tok` (T <= pos < S); logits_out fp32 [b_eff, V]. */
int car_decode_step(CarState* s, const int32_t* tok, int32_t pos, float* logits_out, void* stream);

/* ---- sampling: generate.sample() + CFG combine (generate.py:59-74,89-90,103-107) on fp32 logits
 * [b_eff, V] -> idx int32 [B] (B = b_eff/2 when cfg_scale > 1).  probs_out (fp32 [B, V]), kept_out (uint8 [B, V]:
 * 1 where the token survives top-k and top-p, also when its probability underflows to 0) and noise
 * (fp32 [B, V] Exp(1) draws; NULL = in-kernel Philox) are optional.  step is the Philox sub-stream index. */
/* car_sample and car_sample_rows stage the per-image parameters in a stream-ordered temporary (cudaMallocAsync, a host-to-device
 * copy, cudaFreeAsync around the launch), so neither can be captured into a CUDA graph; the decode loops do not use them. */
int car_sample(const float* logits, int32_t b_eff, int32_t V, const CarSampling* sp, int32_t cfg_on, int32_t step,
               const float* noise, int32_t* idx_out, float* probs_out, uint8_t* kept_out, void* stream);
/* The same sampler with image b's parameters from rows[b] (host, B entries; B = b_eff / 2 when cfg_scale > 1, else b_eff). */
int car_sample_rows(const float* logits, int32_t b_eff, int32_t V, const CarRowSampling* rows, int32_t B, float cfg_scale,
                    int32_t cfg_on, int32_t step, const float* noise, int32_t* idx_out, float* probs_out, uint8_t* kept_out,
                    void* stream);

/* ---- device-side generation loop: generate()'s prefill-sample + decode_n_tokens (generate.py:113-131,
 * 195-204).  Must follow car_prefill(...) on the same state.  Runs n_tokens sampling steps (the first one on
 * the prefill logits) with no host synchronisation — bf16, B_eff <= 16: ONE persistent cooperative kernel
 * (csrc/decode_persistent.cuh); otherwise a replayed CUDA graph of the per-kernel chain, whose GEMMs are one wgmma weight pass
 * per step (gemm_wide) for bf16 at 32 < B_eff <= 64.  tokens_out int32 [B, n_tokens].
 * noise: optional fp32 [n_tokens, B, V]. ---- */
int car_generate(CarState* s, const CarSampling* sp, int32_t n_tokens, const float* noise,
                 int32_t* tokens_out, void* stream);

/* Measurement hook: when step_ns_dev (device, int64 [N]) is non-NULL, every following car_generate on this state records the
 * GPU globaltimer (ns) at which decode iteration s starts into step_ns_dev[s] (one 8-byte store per token by one thread;
 * bench.py derives ms/step versus context length from it).  NULL switches it off. */
int car_state_set_step_timer(CarState* s, int64_t* step_ns_dev);

/* Teacher-forced run of the same device-side loop (parity instrumentation; the reference equivalent is calling
 * Transformer.forward(idx=forced[:, i], input_pos=[T+i]) step by step, gpt_t2i.py:444-470 / generate.py:97-110).
 * forced_tokens int32 [B, n_tokens] (device): the token fed to step i+1 is forced[b][i]; the sampler still runs and
 * tokens_out[b][i] is its choice given the forced prefix.  logits_trace (optional, device) fp32 [n_tokens, b_eff, V]
 * receives the raw model logits of every step (row 0 = the prefill logits).  bf16 only: the persistent kernel where it
 * runs (B_eff <= 16), else the per-kernel chain step by step (the wide decode route for 32 < B_eff <= 64). */
int car_generate_forced(CarState* s, const CarSampling* sp, int32_t n_tokens, const float* noise,
                        const int32_t* forced_tokens, float* logits_trace, int32_t* tokens_out, void* stream);

/* Algorithmic HBM bytes of one decode step at context length n (SURVEY.md §8d formula). */
int64_t car_decode_step_bytes(const CarState* s, int32_t n_context);
/* Number of kernels the library launched since the counter was last reset (bench.py "gpu_launches"). */
int64_t car_launch_count(int32_t reset);

/* ---- building-block ops, exposed for unit parity tests (tests/test_ops_gpu.py) ---- */
/* y[M,N] = act(x[M,K] @ W[N,K]^T (+bias)); act: 0 none, 1 GELU-tanh (gpt_t2i.py:171), 2 GELU-erf. */
int car_op_linear(int32_t dtype, const void* x, const void* w, const void* bias, void* y, int32_t M, int32_t N,
                  int32_t K, int32_t act, void* stream);
/* y[M,N] = act(x[M,K] w[N,K]^T) (+ resid[M,N]) on the dense tensor-core path of the prefill (bf16, fp32 accumulate; act 1 = GELU-tanh),
 * through gemm() (csrc/gemm.cu): K a multiple of 8, x and w 16-byte aligned.  Unit-test / micro-benchmark hook. */
int car_op_dense_linear(const void* x, const void* w, const void* resid, void* y, int32_t M, int32_t N, int32_t K, int32_t act,
                        void* stream);

/* The dense GEMM front end (csrc/gemm.h), exposed for conformance tests.  CarGemmDesc mirrors gemm.h's DenseP field for field
 * (pointers are device pointers; bf16 operands, fp32 bias_f / resid_f); the contract, the epilogue order and the routes are
 * documented there.
 * car_op_gemm_route: the route gemm() takes for (desc, batch): 0 wgmma plain, 1 wgmma 3x3 convolution, 2 mma.sync, 3 mma.sync
 *   window; < 0 (CAR_ERR_ARG, message in car_last_error) when the descriptor is refused.  Host only: never touches the device.
 * car_op_gemm: gemm() itself, the code path every library caller takes.
 * car_op_gemm_f32 / car_op_gemm_f32_conv3: gemm.h's gemm_f32 and gemm_f32_conv3 (fp32 output over split-bf16 operands). */
typedef struct CarGemmDesc {
    const void *A, *B;
    int32_t M, N, K;
    int32_t lda, ldb;
    int64_t sA, sB, sC, sR;
    int32_t amode, Hs, Ws, Cin, Ho, Wo, ups;
    float alpha;
    const void* bias; int32_t bias_along_m;
    const float* bias_f;
    const float* resid_f;
    int32_t act;
    const void* scale;
    const void* resid; int32_t ldr;
    void* C; int32_t ldc;
    int32_t out_mode;
    int32_t kh, kw, ws;
    int32_t osy, osx, oay, oax, oH, oW;
} CarGemmDesc;
int car_op_gemm_route(const CarGemmDesc* desc, int32_t batch);
int car_op_gemm(const CarGemmDesc* desc, int32_t batch, void* stream);
int car_op_gemm_f32(const void* A, const void* B, int32_t M, int32_t N, int32_t K, const float* bias, const float* resid, float* out,
                    int32_t ldc, void* stream);
int car_op_gemm_f32_conv3(const void* src, int32_t fh, int32_t fw, const void* B, int32_t nimg, int32_t H, int32_t W, int32_t cin,
                          int32_t N, const float* bias, const float* resid, float* out, void* stream);

/* RMSNorm.forward (gpt_t2i.py:193-198). */
int car_op_rmsnorm(int32_t dtype, const void* x, const void* w, void* y, int32_t M, int32_t K, float eps,
                   void* stream);

/* KV-cache attention (csrc/attention.cuh), launched exactly as the model chains launch it.  k_cache, v_cache: [B, H, S, 64] in dtype,
 * 16-byte aligned.  Mask (generate.py:184-193): key s is visible to query position i iff s <= i and (s >= Tpre or emb_mask[b][s] != 0
 * or s == i); emb_mask int32 [B][mask_ld], mask_ld >= Tpre, or NULL (all ones).  Scale 1/8, fp32 arithmetic, output rounded to dtype.
 * car_op_attn_decode: the decode step's attn_decode_kernel.  q [B, H*64] -> out [B, H*64], the query at position pos = *pos_dev
 * (device int32; Tpre <= pos < S, read back to check it, which synchronises the stream) against keys [0, pos].  nsplit in [0, 16]
 * CTAs per (b, h), 0 = the choice car_state_create makes.  part: fp32 scratch of B * H * nsplit * 68 floats (B * H * 16 * 68 always
 * suffices); tickets: int32 [B * H], zero before the call and left zero by it.
 * car_op_attn_prefill: the prefix rows.  q [B * Tq, H*64] (rows b * Tq + i) -> out [B * Tq, H*64], queries at positions i < Tq
 * (1 <= Tq <= 256, Tpre <= Tq <= S) against keys [0, i].  impl 0: attn_prefill_kernel (one warp per query row; bf16 or fp32);
 * impl 1: attn_prefill_mma_kernel (bf16 tensor cores, probabilities rounded to bf16 before the value product). */
int car_op_attn_decode(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, const int32_t* emb_mask, int32_t mask_ld,
                       const int32_t* pos_dev, int32_t B, int32_t H, int32_t S, int32_t Tpre, int32_t nsplit, float* part,
                       int32_t* tickets, void* out, void* stream);
int car_op_attn_prefill(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, const int32_t* emb_mask,
                        int32_t mask_ld, int32_t B, int32_t H, int32_t S, int32_t Tq, int32_t Tpre, int32_t impl, void* out,
                        void* stream);

/* =====================================================================================================
 * Control encoder: Dinov2_Adapter.forward (autoregressive/models/dinov2_adapter.py:16-29) = resize to multiples
 * of 14 -> HF Dinov2Model (third-party: transformers, unpinned in requirements.txt:19; 5.5.0 restated) -> drop CLS,
 * optionally followed by adapter_mlp (generate.py:138).  Arithmetic: bf16 tensor-core operands, fp32 accumulate.
 * ===================================================================================================== */
typedef struct CarDino CarDino;
typedef struct CarDinoDesc {
    int32_t dtype;            /* dtype of the borrowed weights and of the input image (CAR_BF16 | CAR_F32) */
    int32_t hidden, heads, layers;
    int32_t patch;            /* 14 (DINOv2) | 16 (HF ViT-S/16 of the legacy c2i class: unit LayerScale, resize_mode 0) */
    int32_t pos_grid;         /* 37 (image_size 518 / 14) | 14 (224 / 16) */
    int32_t resize_mode;      /* 0 nearest (canny, seg) ; 1 bicubic align_corners=True (others) */
    int32_t adapter_out_dim;  /* d of adapter_mlp, 0 = no adapter_mlp registered */
    float   eps;              /* layer_norm_eps 1e-6 */
} CarDinoDesc;
typedef struct CarDinoWeights {   /* HF state-dict tensors, in `dtype`; arrays have `layers` entries */
    const void *cls_token, *pos_emb, *patch_w, *patch_b, *ln_w, *ln_b;
    const void *const *n1_w, *const *n1_b, *const *q_w, *const *q_b, *const *k_w, *const *k_b, *const *v_w, *const *v_b,
               *const *o_w, *const *o_b, *const *ls1, *const *n2_w, *const *n2_b, *const *fc1_w, *const *fc1_b,
               *const *fc2_w, *const *fc2_b, *const *ls2;
    const void *adapter_fc1, *adapter_fc2;   /* adapter_mlp.fc{1,2}.weight or NULL */
} CarDinoWeights;
int car_dino_create(const CarDinoDesc* desc, const CarDinoWeights* w, void* stream, CarDino** out);
/* image [B,3,H,W] in `dtype`, values in [-1,1]; out bf16 [B, (H/16)(W/16), hidden] or, with apply_mlp, [.., adapter_out_dim] */
int car_dino_forward(CarDino* m, const void* image, int32_t B, int32_t H, int32_t W, void* out_bf16, int32_t apply_mlp,
                     void* stream);
int car_dino_destroy(CarDino* m);

/* Trainable control encoder: the same module (Dinov2_Adapter.forward / ViT_Adapter.forward) with fp32 parameters under the train
 * loop's bf16 autocast (fp32 residual stream, LayerNorm, LayerScale and position embeddings; bf16 patch projection, nn.Linear,
 * attention and GELU), and its backward.  `w` holds the fp32 master weights (desc->dtype = CAR_F32), BORROWED: they must stay
 * valid and in place for the handle's life; every forward re-casts them.  ls1 / ls2 NULL: no LayerScale (ViT); adapter_fc* are
 * not read.  Forward: image fp32 [B,3,H,W] -> feat fp32 [B, (H/16)(W/16), hidden].  Backward of the LAST forward on the handle:
 * d_feat fp32 of feat's shape -> fp32 gradients, OVERWRITTEN, through the non-NULL pointers of `g` (same layout as the weights;
 * NULL fields and array entries are skipped). */
typedef struct CarDinoTrain CarDinoTrain;
int car_dino_train_create(const CarDinoDesc* desc, const CarDinoWeights* w, void* stream, CarDinoTrain** out);
int car_dino_train_forward(CarDinoTrain* m, const float* image, int32_t B, int32_t H, int32_t W, float* feat, void* stream);
int car_dino_train_backward(CarDinoTrain* m, const float* d_feat, const CarDinoWeights* g, void* stream);
int car_dino_train_destroy(CarDinoTrain* m);

/* =====================================================================================================
 * Image tokenizer: VQModel.decode_code / encode (tokenizer/tokenizer_image/vq_model.py:41-56).
 * tensors: the fp32 state-dict tensors in canonical order = encoder, decoder, quantize.embedding.weight,
 * quant_conv, post_quant_conv, each module as (weight, bias) in definition order (controlar_b200/vision.py
 * `vq_tensor_order`).  Arithmetic: NHWC bf16 activations/weights on tensor cores, fp32 accumulate and statistics.
 * ===================================================================================================== */
typedef struct CarVQ CarVQ;
typedef struct CarVQDesc {
    int32_t codebook_size, embed_dim, ch, z_channels, n_levels, num_res_blocks;
    int32_t ch_mult[8];
} CarVQDesc;
int car_vq_create(const CarVQDesc* desc, const void* const* tensors, int32_t n_tensors, void* stream, CarVQ** out);
int car_vq_decode_code(CarVQ* m, const int32_t* codes, int32_t B, int32_t h, int32_t w, float* out_nchw, void* stream);
/* VQModel.decode (vq_model.py:48-51): quant fp32 [B, e, h, w] */
int car_vq_decode(CarVQ* m, const float* quant_nchw, int32_t B, int32_t h, int32_t w, float* out_nchw, void* stream);
int car_vq_encode(CarVQ* m, const float* img_nchw, int32_t B, int32_t H, int32_t W, int32_t* idx_out, float* quant_out,
                  void* stream);
int car_vq_destroy(CarVQ* m);

/* =====================================================================================================
 * Training forward (SURVEY.md row f1): Transformer.forward(idx, cond_idx, targets, mask, valid, condition) with the module
 * in train mode (autoregressive/models/gpt_t2i.py:420-431,451-484) as the train scripts run it — fp32 parameters under bf16
 * autocast (autoregressive/train/train_t2i_canny.py:166-167, train_c2i_canny.py:200-201).  The CFG drop decision
 * (gpt_t2i.py:83,116,148: torch.rand(B) < class_dropout_prob) is drawn by the caller and passed in.  Token, residual and
 * feed-forward dropout and stochastic depth (drop path) run inside the forward and backward kernels when car_train_set_dropout
 * turns them on; their keep decisions come from a counter-based generator keyed by a device seed (car_dropout_keep_mask), so the
 * backward regenerates the forward's masks instead of storing them.  Attention-probability dropout is not supported.
 * car_train_backward gives the gradients of every parameter on this path and of the control tokens.
 * ===================================================================================================== */
typedef struct CarTrain CarTrain;
typedef struct CarTrainWeights {
    CarWeights  w;             /* the transformer's fp32 master tensors (same keys as above; desc.dtype = CAR_F32) */
    const void* adapter_fc1;   /* adapter_mlp.fc1.weight [d, adapter_dim] fp32 */
    const void* adapter_fc2;   /* adapter_mlp.fc2.weight [d, d]           fp32 */
    const void* cap_uncond;    /* cls_embedding.uncond_embedding [T, caption_dim] fp32 (t2i), else NULL */
    int32_t     adapter_dim;   /* 384 (DINOv2-small / ViT-S) | 768 (DINOv2-base) */
    int32_t     num_classes;   /* c2i: row of the dropped label in cls_embedding.embedding_table */
    const void* cond_uncond;   /* condition_mlp.uncond_embedding [>= n_img, d] fp32 (a buffer: rows given to dropped samples,
                                  gpt_t2i.py:107,120); NULL = zeros, which is what the released checkpoints hold */
} CarTrainWeights;
/* Workspaces are sized for max_batch sequences of cls_token_num + max_img_tokens - 1 rows.  Weights and rope_table
 * (fp32 [T + block_size, 32, 2], as for car_state_create) are borrowed until car_train_destroy. */
int car_train_create(const CarModelDesc* desc, const CarTrainWeights* weights, int32_t max_batch, int32_t max_img_tokens,
                     const float* rope_table, void* stream, CarTrain** out);
/* idx int32 [B, n_img - 1] (the scripts pass z[:, :-1]); cond: t2i fp32 [B, T, caption_dim] | c2i int32 [B];
 * feat: control-encoder output tokens bf16 [B, n_img, adapter_dim] (= self.adapter(condition)) or NULL;
 * drop_ids uint8 [B]; mask uint8 [B, S, S] with S = T + n_img - 1 (1 = attend) or NULL = causal (is_causal=True);
 * targets int32 [B, n_img] (with loss_out, else both NULL); valid fp32 [B] or NULL (plain mean);
 * logits_out fp32 [B, n_img, V] or NULL; loss_out fp32 [1]. */
int car_train_forward(CarTrain* t, int32_t B, int32_t n_img, const int32_t* idx, const void* cond, const void* feat,
                      const uint8_t* drop_ids, const uint8_t* mask, const int32_t* targets, const float* valid,
                      float* logits_out, float* loss_out, void* stream);
/* Backward of the LAST car_train_forward(targets != NULL) on this handle (in the reference: autograd, train_c2i_canny.py:200-211
 * `scaler.scale(loss).backward()`), recomputing each block from the fp32 stream saved at its input.  `grads` is a CarTrainWeights
 * whose pointers address fp32 GRADIENT buffers of the parameters' shapes (every non-NULL one is overwritten with d loss / d param;
 * cap_uncond / cond_uncond / the two int fields are ignored); d_feat: bf16 [B, n_img, adapter_dim] or NULL (the hand-over to the
 * control encoder's own backward); loss_grad: device fp32 [1] multiplying every gradient (d / d loss, e.g. a GradScaler factor) or
 * NULL = 1.  The tensors passed to that car_train_forward must still be alive.  Gradients are bf16-rounded where autograd under
 * bf16 autocast rounds them (tests/test_zz_train_backward_gpu.py: <= 3e-2 rel-L2 per tensor against autograd over the oracle,
 * itself pinned to gradients the reference produced).  Needs dim, ffn_dim, vocab_size multiples of 64. */
int car_train_backward(CarTrain* t, const CarTrainWeights* grads, void* d_feat, const float* loss_grad, void* stream);
int car_train_destroy(CarTrain* t);
/* Dropout of the training path, applied the way nn.Dropout / DropPath apply it on CUDA under bf16 autocast:
 *   token_p  tok_dropout on the fp32 stream rows (prefix rows and image tokens) before the first control add (gpt_t2i.py:430);
 *   resid_p  resid_dropout on wo's bf16 output (gpt_t2i.py:290);  ffn_p  ffn_dropout on w2's bf16 output (gpt_t2i.py:217);
 *            a kept element becomes x * fp32(1 / keep) rounded once to the tensor's dtype, a dropped one 0 (keep = 1 - p);
 *   drop_path  per-layer DropPath rates (host fp32 [n_layer], the reference's torch.linspace(0, rate, n_layer) values) or NULL:
 *            after the branch's dropout, the bf16 branch is multiplied by bf16(bernoulli(keep) / keep), one draw per sample and
 *            branch (gpt_t2i.py:305-306, utils/drop_path.py);
 *   seed     DEVICE uint64 [1], read by the kernels (no host synchronisation); required when any site is on.
 * Every p and rate must lie in [0, 1); 0 turns a site off and the path is then bit for bit the dropout-free one.  The settings
 * (copied, except the seed, which is borrowed) apply from the next car_train_forward on; car_train_backward uses the settings and
 * seed of the forward it differentiates, so the seed must stay unchanged until then.  cfg NULL turns every site off. */
typedef struct CarTrainDropout {
    float           token_p, resid_p, ffn_p;
    int32_t         n_layer;        /* entries of drop_path (the model's n_layer), 0 when drop_path is NULL */
    const float*    drop_path;
    const uint64_t* seed;
} CarTrainDropout;
int car_train_set_dropout(CarTrain* t, const CarTrainDropout* cfg);
/* Conformance entry point for the dropout generator: out uint8 [B, rows, cols] = 1 where the training kernels keep element
 * (row, col) of sample b at `site` (0 token, 1 resid, 2 ffn, 3 drop path of the attention branch, 4 drop path of the feed-forward
 * branch) of `layer` (0 for the token site) with drop probability p.  The drop-path sites decide per sample: every (row, col) of a
 * sample holds that sample's decision.  Same device function as the training kernels; oracle/dropout_masks.py restates it. */
int car_dropout_keep_mask(const uint64_t* seed_dev, int32_t site, int32_t layer, int32_t B, int32_t rows, int32_t cols, float p,
                          uint8_t* out, void* stream);

/* ---- antialiased bilinear resize in front of the online VQ encode of the multi-resolution training scripts (SURVEY.md row f2):
 * F.interpolate(x.float(), size=(OH, OW), mode='bilinear', align_corners=False, antialias=True),
 * autoregressive/train/train_t2i_depth_multiscale.py:44-56.  in fp32 [B, C, H, W] -> out fp32 [B, C, OH, OW];
 * tmp: caller-provided fp32 scratch [B, C, H, OW]. ---- */
int car_resize_bilinear_aa(const float* in, int32_t B, int32_t C, int32_t H, int32_t W, float* out, int32_t OH, int32_t OW,
                           float* tmp, void* stream);

/* ---- control-map / prompt front-end (SURVEY.md row f3) ----
 * car_canny_u8: condition/canny.py:14 `cv2.Canny(img, low, high)` (OpenCV 4.x, aperture 3, L1 gradient) — integer arithmetic,
 * bit-exact against OpenCV.  img uint8 [H][W][C] (C <= 4) -> edges uint8 [H][W] in {0, 255}; `work`: car_canny_workspace_bytes(H, W)
 * bytes of device scratch.  restart != 0 computes gradients / non-maximum suppression / thresholds and runs `sweeps` hysteresis
 * sweeps; restart == 0 runs `sweeps` more on the state in `work`.  *changed_dev (int32, device) ends 1 iff the last sweep still grew
 * an edge: repeat with restart = 0 until it is 0 (the only host-visible check; the reference's call is synchronous host code).
 * car_left_pad_captions: autoregressive/sample/sample_t2i.py:146-156 — valid caption tokens (a prefix) rotated to the END of the
 * sequence, mask flipped; embs [B][L][row_bytes] of any dtype (row_bytes % 16 == 0), masks int64 [B][L]. */
int64_t car_canny_workspace_bytes(int32_t H, int32_t W);
int car_canny_u8(const uint8_t* img, int32_t H, int32_t W, int32_t C, int32_t low, int32_t high, uint8_t* edges_out, void* work,
                 int32_t sweeps, int32_t restart, int32_t* changed_dev, void* stream);
int car_left_pad_captions(const void* embs, const int64_t* masks, int32_t B, int32_t L, int32_t row_bytes, void* embs_out,
                          int64_t* masks_out, void* stream);

/* HED soft-edge detector: condition/hed.py:17-84 (ControlNetHED_Apache2 + the arithmetic of HEDdetector.__call__), fp32 in the
 * reference => fp32-grade split-bf16 convolutions here.  car_hed_create: 37 fp32 device tensors in state-dict order — norm [3];
 * per block b = 1..5: convs.{i}.weight [Cout][Cin][3][3], convs.{i}.bias (2, 2, 3, 3, 3 convolutions), projection.weight [C],
 * projection.bias [1] — copied / packed (nothing borrowed).  car_hed_forward: image fp32 NCHW [B][3][H][W] in 0..255 ->
 * edge fp32 [B][H][W] in [0, 255]; proj_out (optional) receives the five projection maps back to back ([B][H >> k][W >> k]). */
typedef struct CarHED CarHED;
int car_hed_create(const void* const* tensors, int32_t n_tensors, void* stream, CarHED** out);
int car_hed_forward(CarHED* m, const float* img, int32_t B, int32_t H, int32_t W, float* edge_out, float* proj_out, void* stream);
int car_hed_destroy(CarHED* m);

/* LineArt detector: condition/lineart.py:8-86 (LineArt.forward), fp32 in the reference => fp32-grade split-bf16 convolutions here.
 * car_lineart_create: 24 fp32 device tensors in state-dict order — model0.1, model1.0, model1.3, model2.{0,1,2}.conv_block.{1,5},
 * model3.0 (ConvTranspose2d, [Cin][Cout][3][3]), model3.3, model4.1, each .weight then .bias — copied / packed (nothing borrowed).
 * car_lineart_forward: image fp32 NCHW [B][3][H][W] in 0..255 (H, W > 4) -> map fp32 [B][1][Ho][Wo] in [0, 1] with
 * Ho = 4 * ceil(ceil(H / 2) / 2), Wo likewise (70 x 90 in -> 72 x 92 out, as in the reference). */
typedef struct CarLineArt CarLineArt;
int car_lineart_create(const void* const* tensors, int32_t n_tensors, void* stream, CarLineArt** out);
int car_lineart_forward(CarLineArt* m, const float* img, int32_t B, int32_t H, int32_t W, float* out, void* stream);
int car_lineart_destroy(CarLineArt* m);

/* DPT depth detector: transformers DPTForDepthEstimation (Intel/dpt-large, non-hybrid ViT backbone, readout "project",
 * reassemble factors 4, 2, 1, 0.5, 64-dim heads, exact GELU, no fusion batch norm), fp32 in the reference => fp32-grade here: every
 * GEMM and 3x3 convolution on split-bf16 operands with fp32 accumulation, attention fused.  car_dpt_create: n fp32 device tensors
 * in state-dict order (4 + 16 * n_layers + 74 of them, dpt.layernorm included and unused) — copied / packed (nothing borrowed).
 * Sizes: hidden % 64 == 0 (heads of 64), mlp % 8 == 0, neck sizes and fusion / 2 multiples of 64.
 * car_dpt_forward: pixel_values fp32 NCHW [B][3][H][W] with H == W, H % 32 == 0, H >= 64 -> predicted_depth fp32 [B][H][W]. */
typedef struct {
    int32_t hidden, n_layers, n_heads, mlp;
    int32_t out_indices[4];         /* encoder layers whose outputs feed the neck, ascending */
    int32_t neck[4];                /* neck_hidden_sizes */
    int32_t fusion;                 /* fusion_hidden_size */
    int32_t pos_grid;               /* side of the stored position-embedding grid (image_size / 16) */
    float ln_eps;
} CarDptDesc;
typedef struct CarDpt CarDpt;
int car_dpt_create(const CarDptDesc* desc, const void* const* tensors, int32_t n_tensors, void* stream, CarDpt** out);
int car_dpt_forward(CarDpt* m, const float* pixel_values, int32_t B, int32_t H, int32_t W, float* depth, void* stream);
int car_dpt_destroy(CarDpt* m);

/* MiDaS DPT-Hybrid depth detector (reference condition/midas: DPTDepthModel, backbone vitb_rn50_384, features 256, readout
 * "project", non_negative): a weight-standardised GroupNorm ResNet-50 trunk (stages 3, 4, 9, TF "SAME" padding) whose stage-2 map
 * is the token grid of a ViT-B/16, then the DPT neck, fusion and head.  fp32 in the reference => fp32-grade here.  The network is
 * fixed, so there is no descriptor.  car_midas_create: 368 fp32 device tensors in the state-dict order of
 * controlar_b200.condition.midas.DPTDepthModel (the ViT's final norm and classifier included and unused) — copied / packed, the
 * convolution weights standardised once (fp64 statistics).
 * car_midas_forward: x fp32 NCHW [B][3][H][W], H % 32 == 0, W % 32 == 0, H, W >= 64 -> depth fp32 [B][H][W].  No host sync. */
typedef struct CarMidas CarMidas;
int car_midas_create(const void* const* tensors, int32_t n_tensors, void* stream, CarMidas** out);
int car_midas_forward(CarMidas* m, const float* x, int32_t B, int32_t H, int32_t W, float* depth, void* stream);
int car_midas_destroy(CarMidas* m);

/* Fused multi-tensor AdamW step (row f1: autoregressive/train/train_c2i.py:28-50 builds torch.optim.AdamW(fused=True)).
 * tensors_dev: device array of { float* param; const float* grad; float* exp_avg; float* exp_avg_sq; int64 numel; float weight_decay;
 * int32 pad } (48 bytes each); chunks_dev: device array of int32 pairs { tensor index, chunk index } — chunk = 65536 elements;
 * step is 1-based (bias corrections 1 - beta^step).  fp32 state, ATen's fused arithmetic. */
int car_adamw_step(const void* tensors_dev, const void* chunks_dev, int32_t n_chunks, float lr, float beta1, float beta2, float eps,
                   int32_t step, void* stream);

/* T5 text encoder (SURVEY.md row f3): language/t5.py:58-79 — HF T5EncoderModel(input_ids, attention_mask).last_hidden_state in
 * bf16 (v1.1 / flan architecture: gated gelu_new feed-forward, no biases, RMS layer norm, relative position bias of block 0 shared
 * by all blocks, no 1/sqrt(d) scaling).  Weights ([out, in] row-major bf16, HF state-dict tensors) are borrowed until
 * car_t5_destroy; workspaces hold max_rows = B * L token rows. */
typedef struct CarT5 CarT5;
typedef struct CarT5Desc {
    int32_t dtype;             /* CAR_BF16 */
    int32_t d_model, d_kv, n_heads, d_ff, n_layers, vocab;
    int32_t num_buckets, max_distance;   /* relative_attention_num_buckets (32), relative_attention_max_distance (128) */
    float   eps;               /* layer_norm_epsilon (1e-6) */
} CarT5Desc;
typedef struct CarT5Weights {
    const void* embed;         /* shared.weight [vocab, d_model] */
    const void* rel_bias;      /* encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight [num_buckets, n_heads] */
    const void* final_norm;    /* encoder.final_layer_norm.weight [d_model] */
    const void* const* ln1;    /* per block: layer.0.layer_norm.weight */
    const void* const* q; const void* const* k; const void* const* v; const void* const* o;   /* layer.0.SelfAttention.{q,k,v,o}.weight */
    const void* const* ln2;    /* layer.1.layer_norm.weight */
    const void* const* wi_0; const void* const* wi_1; const void* const* wo;                  /* layer.1.DenseReluDense.{wi_0,wi_1,wo}.weight */
} CarT5Weights;
int car_t5_create(const CarT5Desc* desc, const CarT5Weights* weights, int32_t max_rows, void* stream, CarT5** out);
/* ids int32 [B, L], mask int32 [B, L] (1 = token) -> out bf16 [B, L, d_model] */
int car_t5_forward(CarT5* t, const int32_t* ids, const int32_t* mask, int32_t B, int32_t L, void* out, void* stream);
int car_t5_destroy(CarT5* t);

#ifdef __cplusplus
}
#endif
#endif /* CONTROLAR_B200_H_ */
