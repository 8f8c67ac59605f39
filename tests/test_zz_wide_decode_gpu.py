"""GPU: the wide decode route (bf16, 32 < B_eff <= 64): every decode-step GEMM through gemm_wide (csrc/gemm.cu, one wgmma weight
pass per step, split-K partials summed in a fixed order), in car_generate (CUDA-graph replay), car_decode_step and car_generate_forced.
B_eff 18 and 32 run the same teacher-forced loop on the skinny chain (the route starts above 32 rows).

  * against the reference at the benchmarked shape: the reference-made GPT-XL fixture (8 images, CFG 4) tiled 2x and 4x into one
    batch (B_eff 32 and 64), teacher-forced, every row at the XL bar of tests/test_zz_xl_parity_gpu.py;
  * row independence: the copies of one sequence get bit-identical logits and sampled grids;
  * against the reference's small-model fixtures at B_eff 18, 34, 50 and 64 (t2i with masks and control strength, c2i) at the
    small-model bar of tests/test_ar_gpu.py;
  * loop = replay at B_eff 64, determinism, and one end-to-end run at the config-2 shape with 32 images."""
import pytest
import torch

from oracle.ar_oracle import cfg_combine
from oracle.inputs import text_inputs, xl_ctrl_in
from oracle.weights import GPTSpec
from tests.helpers import (load_golden, build_product_gpt, rel_l2, near_tie_bound, assert_mismatches_are_near_ties)

pytestmark = pytest.mark.gpu

TOL_XL = 3e-2          # worst per-row rel-L2 of XL bf16 logits vs the reference (DESIGN §2)
TOL_SMALL = 2e-2       # the small models' bf16 bar
_XL = {}


def _xl(g):
    if "m" not in _XL:
        spec = GPTSpec(**g["spec"])
        _XL["m"] = (spec, build_product_gpt(spec, g["seed"], torch.bfloat16)[0])
    return _XL["m"]


def _xl_prefill(g, reps):
    """The fixture's 8 images, each repeated `reps` times (image b of copy k at row k * 8 + b), prefilled on a fresh state."""
    spec, model = _xl(g)
    dev, dt = "cuda", torch.bfloat16
    B0, N_img, T = g["B"], g["N_img"], spec.cls_token_num
    cond, masks = text_inputs(T, spec.caption_dim, B0, g["seed"] + 1, dt)
    ctrl_in = xl_ctrl_in(B0, N_img, spec.dim, g["seed"] + 7, dt).to(dev)
    c, masks, ctrl_in = cond.to(dev).repeat(reps, 1, 1), masks.to(dev).repeat(reps, 1), ctrl_in.repeat(reps, 1, 1)
    cc = torch.cat([c, torch.zeros_like(c) + model.cls_embedding.uncond_embedding])
    model.setup_caches(2 * B0 * reps, T + N_img, dt, n_img_tokens=N_img)
    st = model._car_state
    st.set_emb_mask(torch.cat([masks, masks]))
    st.prefill(cc, torch.cat([ctrl_in, torch.zeros_like(ctrl_in)]), g["control_strength"], all_rows=False)
    return st


@pytest.mark.parametrize("reps", [2, 4])
def test_xl_tiled_fixture_teacher_forced(reps):
    """B = 8 reps images (B_eff 32: skinny chain, 64: wide route), teacher-forced along the fixture's grid: every row of every stored step
    against the reference's row of the same sequence, greedy disagreements only at the reference's near-ties, and the copies of one
    sequence bit-identical."""
    from controlar_b200 import engine
    g = load_golden("xl_b8_short")
    B0, n = g["B"], g["n_tokens"]
    st = _xl_prefill(g, reps)
    sp = engine.make_sampling(temperature=1.0, top_k=0, top_p=1.0, sample_logits=False, cfg_scale=g["cfg_scale"])
    choice, trace = st.generate_forced(sp, g["forced_tokens"].cuda().repeat(reps, 1))
    torch.cuda.synchronize()
    assert bool(torch.isfinite(trace).all())
    B = B0 * reps
    src = torch.tensor([r % B0 for r in range(B)] + [B0 + r % B0 for r in range(B)])      # fixture row of each batch row
    worst = 0.0
    for j, s in enumerate(g["full_steps"]):
        got, ref = trace[s].float().cpu(), g["full_logits"][:, j].float()
        worst = max(worst, max(rel_l2(got[r], ref[src[r]]) for r in range(2 * B)))
    assert worst < TOL_XL, f"worst full-row rel-L2 {worst:.3e}"
    cols = g["cols"]
    got_cols = trace[torch.tensor(g["col_steps"], device=trace.device)][:, :, cols.to(trace.device)].float().cpu()
    ref_cols = g["col_logits"].float().permute(1, 0, 2)[:, src]
    worst_col = float(((got_cols - ref_cols).double().norm(dim=-1) / ref_cols.double().norm(dim=-1)).max())
    assert worst_col < 2.5 * TOL_XL, f"worst 256-column probe rel-L2 {worst_col:.3e}"
    ref_arg = g["argmax_cfg"].long()
    ch = choice.cpu().long()
    for b, i in (ch != ref_arg.repeat(reps, 1)).nonzero().tolist():
        bound = 2.0 * near_tie_bound(float(g["raw_absmax"][i]), g["cfg_scale"])
        assert float(g["margin_cfg"][b % B0, i]) <= bound, f"step {i} image {b}: not a near-tie in the reference"
    # row independence: every copy equals copy 0, bit for bit
    tr = trace.view(n, 2, reps, B0, -1)
    for k in range(1, reps):
        assert torch.equal(tr[:, :, k], tr[:, :, 0]), f"copy {k}: logits differ from copy 0"
        assert torch.equal(ch[k * B0:(k + 1) * B0], ch[:B0])


def test_xl_b32_sampled_grids_copies_and_determinism():
    """B = 32 (B_eff 64), car_generate with top-k 2000 and explicit noise repeated per copy: the four copies of an image sample the
    same grid, and two runs give identical grids."""
    from controlar_b200 import engine
    g = load_golden("xl_b8_short")
    B0, n, V = g["B"], g["n_tokens"], 16384
    gen = torch.Generator().manual_seed(3)
    noise = torch.empty(n, B0, V).exponential_(1.0, generator=gen).cuda().repeat(1, 4, 1)
    sp = engine.make_sampling(temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True, cfg_scale=g["cfg_scale"])
    grids = []
    for _ in range(2):
        st = _xl_prefill(g, 4)
        grids.append(st.generate(sp, n, noise, "cuda").cpu())
    assert torch.equal(grids[0], grids[1]), "two runs differ"
    gr = grids[0].view(4, B0, n)
    for k in range(1, 4):
        assert torch.equal(gr[k], gr[0]), f"copy {k} sampled a different grid"
    assert not torch.equal(gr[0, 0], gr[0, 1])


def _small(name, nB):
    """Fixture `name`'s images cycled to nB images, prefilled; returns (state, fixture, row map of the b_eff rows, spec)."""
    from tests.test_ar_gpu import _setup
    g, spec, dt, model, sd, cond, masks = _setup(name)
    dev = "cuda"
    B0, N, T = g["B"], g["greedy_tokens"].shape[1], spec.cls_token_num
    pick = torch.tensor([b % B0 for b in range(nB)])
    c, ctrl_in = cond.to(dev)[pick], g["ctrl_in"].to(dev)[pick]
    if spec.model_type == "t2i":
        cc = torch.cat([c, torch.zeros_like(c) + model.cls_embedding.uncond_embedding])
    else:
        cc = torch.cat([c, torch.full_like(c, spec.num_classes)])
    model.setup_caches(2 * nB, T + N, dt, n_img_tokens=N)
    st = model._car_state
    st.set_emb_mask(None if masks is None else torch.cat([masks[pick], masks[pick]]).to(dev))
    st.prefill(cc, torch.cat([ctrl_in, torch.zeros_like(ctrl_in)]), g["control_strength"], all_rows=False)
    return st, g, torch.cat([pick, B0 + pick])


@pytest.mark.parametrize("name", ["t2i_small_bf16", "c2i_small_bf16"])
@pytest.mark.parametrize("b_eff", [18, 34, 50, 64])
def test_small_models_teacher_forced_vs_reference(name, b_eff):
    """Teacher-forced logits of every step at odd batch sizes against the reference's fixture rows of the same sequences."""
    from controlar_b200 import engine
    st, g, rows = _small(name, b_eff // 2)
    assert g["cfg_scale"] > 1.0
    sp = engine.make_sampling(temperature=1.0, top_k=0, top_p=1.0, sample_logits=False, cfg_scale=g["cfg_scale"])
    choice, trace = st.generate_forced(sp, g["greedy_tokens"].cuda()[rows[: b_eff // 2]])
    got = trace.permute(1, 0, 2).float().cpu()                       # [b_eff, N, V]
    assert bool(torch.isfinite(got).all())
    ref_all = g["raw_logits_all"].float()[rows]
    N = got.shape[1]
    worst = max(rel_l2(got[:, i], ref_all[:, i]) for i in range(N))
    assert worst < TOL_SMALL, f"{name} B_eff {b_eff}: worst per-step rel-L2 {worst:.3e}"
    zr = cfg_combine(ref_all, g["cfg_scale"])
    rate = assert_mismatches_are_near_ties(zr, ref_all, g["greedy_tokens"].long()[rows[: b_eff // 2]], choice.cpu().long(), g["cfg_scale"], name)
    assert rate < 0.25


@pytest.mark.parametrize("explicit", [True, False])
def test_graph_loop_replays_through_decode_step_b_eff_64(explicit):
    """B = 32 with CFG: the generate grid equals decode_step + car_sample step by step (explicit noise and Philox noise)."""
    from controlar_b200 import engine
    from tests.test_sampler_gpu import _model, _prefill, SPEC, N_TOK
    model = _model("plain")
    B, V = 32, SPEC.vocab_size
    gen = torch.Generator().manual_seed(43)
    noise = torch.empty(N_TOK, B, V).exponential_(1.0, generator=gen).cuda() if explicit else None
    sp = engine.make_sampling(1.0, 2000, 1.0, sample_logits=True, cfg_scale=4.0, seed=78)
    st, _ = _prefill(model, B, True)
    assert st.b_eff == 64
    grid = st.generate(sp, N_TOK, noise, "cuda").cpu().long()
    st, _ = _prefill(model, B, True)
    again = st.generate(sp, N_TOK, noise, "cuda").cpu().long()
    assert torch.equal(grid, again), "two runs differ"
    st, logits = _prefill(model, B, True)
    for s in range(N_TOK):
        idx = engine.sample(logits, sp, step=s, noise=None if noise is None else noise[s]).cpu().long()
        assert torch.equal(idx, grid[:, s]), f"step {s}: replay differs from the loop"
        if s + 1 < N_TOK:
            t = grid[:, s].cuda()
            logits = st.decode_step(torch.cat([t, t]), SPEC.cls_token_num + s)


def test_config2_shape_b32_end_to_end():
    """GPT-XL t2i + DINOv2-small canny at 512 x 512, 32 images: generate + decode_code give finite images; the serving engine runs
    32 control requests as one batch."""
    from controlar_b200.autoregressive.models.gpt_t2i import GPT_models
    from controlar_b200.autoregressive.models.generate import generate
    from controlar_b200.autoregressive.serve.llm import LLM, SamplingParams
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    from controlar_b200.synthetic import text_inputs as syn_text, control_map
    _XL.clear()
    torch.manual_seed(0)
    gpt = GPT_models["GPT-XL"](block_size=32 * 32, cls_token_num=120, model_type="t2i", condition_type="canny", adapter_size="small").eval()
    gpt.output.weight.data.normal_(0, 0.02)
    for blk in gpt.adapter.model.encoder.layer:
        blk.layer_scale1.lambda1.data.fill_(1.0); blk.layer_scale2.lambda1.data.fill_(1.0)
    gpt = gpt.to("cuda", torch.bfloat16)
    vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    B = 32
    cond, masks = syn_text(120, 2048, B, 11, torch.bfloat16)
    cmap = control_map(B, 512, 512, 12, "canny", torch.bfloat16)
    toks = generate(gpt, cond.cuda(), 1024, emb_masks=masks.cuda(), condition=cmap.cuda(), cfg_scale=4.0, temperature=1.0, top_k=2000,
                    top_p=1.0, sample_logits=True, seed=5)
    assert toks.shape == (B, 1024) and int(toks.min()) >= 0 and int(toks.max()) < 16384
    img = vq.decode_code(toks, [B, 8, 32, 32])
    assert img.shape == (B, 3, 512, 512) and bool(torch.isfinite(img).all())
    llm = LLM(model=gpt, vq=vq, cfg_scale=4.0, max_images_per_batch=32, seed=2)
    prompts = [dict(cond=cond[i], emb_mask=masks[i], control=cmap[i], control_strength=1.0) for i in range(B)]
    outs = llm.generate(prompts=prompts, sampling_params=SamplingParams(temperature=1.0, top_k=2000, max_tokens=1024))
    assert len(outs) == B and all(o.image is not None and bool(torch.isfinite(o.image).all()) for o in outs)
    assert llm._launches == 1, "32 requests of one configuration run as one batch"
