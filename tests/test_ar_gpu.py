"""GPU parity of the AR path (prefill, KV-cache decode, device-side generate) against the oracle and the golden
fixtures made by the reference itself.  All calls go through the C ABI (ctypes)."""
import pytest
import torch

from oracle.weights import GPTSpec
from oracle.ar_oracle import AROracle, oracle_generate, cfg_combine
from oracle.inputs import text_inputs, class_inputs
from tests.helpers import (log_measurement, load_golden, dtype_of, build_product_gpt, rel_l2, near_tie_bound,
                           assert_mismatches_are_near_ties)

pytestmark = pytest.mark.gpu

# Tolerances.  fp32: two fp32 implementations differ only by summation order.  bf16: every rounding point turns an
# fp32-level difference eps into an rms error ~sqrt(eps*ulp); measured spread between two *reference* configurations
# (math vs fused SDPA, tests/test_oracle_golden.py::test_reference_own_spread) is ~7e-3 on the 6-layer model.
TOL = {torch.float32: 2e-5, torch.bfloat16: 2e-2}


def _inputs(g, spec):
    seed, B = g["seed"], g["B"]
    dt = dtype_of(g)
    if spec.model_type == "t2i":
        cond, masks = text_inputs(spec.cls_token_num, spec.caption_dim, B, seed + 1, dt)
    else:
        cond, masks = class_inputs(spec.num_classes, B, seed + 1), None
    return cond, masks


def _setup(name):
    g = load_golden(name)
    spec = GPTSpec(**g["spec"])
    dt = dtype_of(g)
    model, sd = build_product_gpt(spec, g["seed"], dt)
    cond, masks = _inputs(g, spec)
    return g, spec, dt, model, sd, cond, masks


CASES = ["t2i_small_fp32", "t2i_small_bf16", "c2i_small_fp32", "c2i_small_bf16", "t2i_mr_bf16", "t2i_mr_tall_bf16"]


@pytest.mark.parametrize("name", CASES)
def test_teacher_forced_logits_vs_golden_and_oracle(name):
    """prefill + every decode step along the reference's greedy trajectory: raw model logits [B_eff, N, V]."""
    g, spec, dt, model, sd, cond, masks = _setup(name)
    dev = "cuda"
    B, N, T = g["B"], g["greedy_tokens"].shape[1], spec.cls_token_num
    use_cfg = g["cfg_scale"] > 1.0
    b_eff = 2 * B if use_cfg else B
    ctrl_in = g["ctrl_in"].to(dev)
    if spec.model_type == "t2i":
        c = cond.to(dev)
        cc = torch.cat([c, torch.zeros_like(c) + model.cls_embedding.uncond_embedding]) if use_cfg else c
    else:
        c = cond.to(dev)
        cc = torch.cat([c, torch.full_like(c, spec.num_classes)]) if use_cfg else c
    cond_comb = torch.cat([ctrl_in, torch.zeros_like(ctrl_in)]) if use_cfg else ctrl_in
    model.setup_caches(b_eff, T + N, dt, n_img_tokens=N)
    st = model._car_state
    if masks is not None:
        st.set_emb_mask(torch.cat([masks, masks]).to(dev) if use_cfg else masks.to(dev))
    cs = g["control_strength"] if use_cfg else 1.0
    ref_all = g["raw_logits_all"].float()
    toks = g["greedy_tokens"].to(dev)
    got = [st.prefill(cc, cond_comb, cs, all_rows=False)]
    for i in range(N - 1):
        t = toks[:, i]
        got.append(st.decode_step(torch.cat([t, t]) if use_cfg else t, T + i))
    got = torch.stack(got, dim=1).cpu()
    worst = max(rel_l2(got[:, i], ref_all[:, i]) for i in range(N))
    assert worst < TOL[dt], f"{name}: worst per-step rel-L2 vs reference golden {worst:.3e}"
    # arg-max agreement of the CFG-combined logits with the reference's greedy choice
    z = cfg_combine(got, g["cfg_scale"]) if use_cfg else got
    mine = z.argmax(-1)
    ref_tok = g["greedy_tokens"].long()
    mism = (mine != ref_tok)
    if dt == torch.float32:
        assert not mism.any(), f"{name}: fp32 teacher-forced arg-max differs at {mism.nonzero()[:4].tolist()}"
    else:
        # bf16: any disagreement must be a rounding-level near-tie in the reference's own logits
        zr = cfg_combine(ref_all, g["cfg_scale"]) if use_cfg else ref_all
        rate = assert_mismatches_are_near_ties(zr, ref_all, ref_tok, mine, g["cfg_scale"], name)
        assert rate < 0.25, f"{name}: {rate:.3f} of teacher-forced arg-maxes differ"


@pytest.mark.parametrize("name", ["t2i_small_bf16", "c2i_small_bf16", "t2i_mr_bf16", "t2i_mr_tall_bf16"])
def test_persistent_kernel_teacher_forced_every_step(name):
    """The PRODUCT bf16 decode path (the persistent kernel behind car_generate), teacher-forced along the reference's greedy
    trajectory through car_generate_forced: raw logits of EVERY step vs the reference golden (not only up to the first
    divergence of a free-running comparison)."""
    import json
    from controlar_b200 import engine
    g, spec, dt, model, sd, cond, masks = _setup(name)
    dev = "cuda"
    B, N, T = g["B"], g["greedy_tokens"].shape[1], spec.cls_token_num
    use_cfg = g["cfg_scale"] > 1.0
    b_eff = 2 * B if use_cfg else B
    ctrl_in = g["ctrl_in"].to(dev)
    c = cond.to(dev)
    if spec.model_type == "t2i":
        cc = torch.cat([c, torch.zeros_like(c) + model.cls_embedding.uncond_embedding]) if use_cfg else c
    else:
        cc = torch.cat([c, torch.full_like(c, spec.num_classes)]) if use_cfg else c
    cond_comb = torch.cat([ctrl_in, torch.zeros_like(ctrl_in)]) if use_cfg else ctrl_in
    model.setup_caches(b_eff, T + N, dt, n_img_tokens=N)
    st = model._car_state
    st.set_emb_mask(None if masks is None else (torch.cat([masks, masks]).to(dev) if use_cfg else masks.to(dev)))
    cs = g["control_strength"] if use_cfg else 1.0
    st.prefill(cc, cond_comb, cs, all_rows=False)
    sp = engine.make_sampling(temperature=1.0, top_k=0, top_p=1.0, sample_logits=False, cfg_scale=g["cfg_scale"])
    choice, trace = st.generate_forced(sp, g["greedy_tokens"].to(dev))
    got = trace.permute(1, 0, 2).float().cpu()          # [b_eff, N, V]
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite logits at steps {sorted(set((~torch.isfinite(got)).nonzero()[:, 1].tolist()))[:8]}"
    ref_all = g["raw_logits_all"].float()
    worst = max(rel_l2(got[:, i], ref_all[:, i]) for i in range(N))
    log_measurement("small_parity.jsonl", json.dumps({"case": name, "worst_step_rel_l2": worst}) + "\n")
    assert worst < TOL[dt], f"{name}: worst per-step rel-L2 vs reference golden {worst:.3e}"
    zr = cfg_combine(ref_all, g["cfg_scale"]) if use_cfg else ref_all
    rate = assert_mismatches_are_near_ties(zr, ref_all, g["greedy_tokens"].long(), choice.cpu().long(), g["cfg_scale"], name)
    assert rate < 0.25, f"{name}: {rate:.3f} of teacher-forced choices differ"


@pytest.mark.parametrize("name", ["t2i_small_fp32", "c2i_small_fp32"])
def test_generate_greedy_bit_exact_fp32(name):
    """Free-running device-side loop (car_prefill + car_generate): greedy token grid == reference golden."""
    g, spec, dt, model, sd, cond, masks = _setup(name)
    from controlar_b200.autoregressive.models.generate import generate
    dev = "cuda"
    N = g["greedy_tokens"].shape[1]
    # feed the reference's adapter_mlp output directly (control-encoder parity is tested separately)
    model.adapter.forward = lambda x: x
    model.adapter_mlp.forward = lambda x: x
    out = generate(model, cond.to(dev), N, emb_masks=None if masks is None else masks.to(dev), cfg_scale=g["cfg_scale"],
                   condition=g["ctrl_in"].to(dev), control_strength=g["control_strength"], temperature=1.0, top_k=0,
                   top_p=1.0, sample_logits=False)
    assert out.dtype == torch.int32 and tuple(out.shape) == tuple(g["greedy_tokens"].shape)
    assert torch.equal(out.cpu(), g["greedy_tokens"]), (out.cpu()[0, :16], g["greedy_tokens"][0, :16])


@pytest.mark.parametrize("name", ["t2i_small_bf16", "c2i_small_bf16", "t2i_mr_bf16"])
def test_generate_greedy_bf16_vs_oracle(name):
    """bf16 free-running greedy: report agreement with the reference golden; require the prefix up to the first
    divergence to be a near-tie in the oracle's logits (bit-exactness is not defined for bf16 across GEMM
    implementations, SURVEY.md §7 hard-part 3)."""
    g, spec, dt, model, sd, cond, masks = _setup(name)
    from controlar_b200.autoregressive.models.generate import generate
    dev = "cuda"
    N = g["greedy_tokens"].shape[1]
    model.adapter.forward = lambda x: x
    model.adapter_mlp.forward = lambda x: x
    out = generate(model, cond.to(dev), N, emb_masks=None if masks is None else masks.to(dev), cfg_scale=g["cfg_scale"],
                   condition=g["ctrl_in"].to(dev), control_strength=g["control_strength"], temperature=1.0, top_k=0,
                   top_p=1.0, sample_logits=False).cpu()
    ref = g["greedy_tokens"]
    zr_all = g["raw_logits_all"].float()
    zc = cfg_combine(zr_all, g["cfg_scale"]) if g["cfg_scale"] > 1.0 else zr_all
    for b in range(ref.shape[0]):
        diff = (out[b] != ref[b]).nonzero()
        if len(diff) == 0:
            continue
        i = int(diff[0])          # first divergence: until here both runs saw identical prefixes
        margin = float(zc[b, i, ref[b, i]] - zc[b, i, out[b, i]])
        bound = near_tie_bound(float(zr_all[:, i].abs().max()), g["cfg_scale"])
        assert margin <= bound, (name, b, i, margin, bound)
    # determinism: a second run reproduces the grid bit-for-bit
    out2 = generate(model, cond.to(dev), N, emb_masks=None if masks is None else masks.to(dev), cfg_scale=g["cfg_scale"],
                    condition=g["ctrl_in"].to(dev), control_strength=g["control_strength"], temperature=1.0, top_k=0,
                    top_p=1.0, sample_logits=False).cpu()
    assert torch.equal(out, out2)


def test_prefill_all_rows_matches_oracle_fp32():
    g, spec, dt, model, sd, cond, masks = _setup("t2i_small_fp32")
    dev = "cuda"
    B, N, T = g["B"], 64, spec.cls_token_num
    orc = AROracle(spec, sd, dt)
    c = cond.float()
    cc = torch.cat([c, torch.zeros_like(c) + orc.w["cls_embedding.uncond_embedding"]])
    ci = g["ctrl_in"].float()
    cic = torch.cat([ci, torch.zeros_like(ci)])
    em = torch.cat([masks, masks])
    orc.setup_caches(2 * B, T + N)
    orc.apply_emb_masks(em)
    want = orc.prefill(cc, cic, 0.6)
    model.setup_caches(2 * B, T + N, dt, n_img_tokens=N)
    model._car_state.set_emb_mask(em.to(dev))
    got = model._car_state.prefill(cc.to(dev), cic.to(dev), 0.6, all_rows=True).cpu()
    # rows whose text token is masked out still produce logits (they only see themselves); compare all rows
    assert rel_l2(got, want) < 2e-5
    # KV cache contents of layer 0 (reference KVCache layout) for the prefix rows
    k0 = model.layers[0].attention.kv_cache.k_cache[:, :, :T].float().cpu()
    v0 = model.layers[0].attention.kv_cache.v_cache[:, :, :T].float().cpu()
    assert k0.abs().max() == 0.0                      # zero RoPE rows for the prefix => K == 0 (gpt_t2i.py:518)
    assert rel_l2(v0, orc.v_cache[0][:, :, :T]) < 2e-5


def _torch_multinomial_noise(seed, n_steps, B, V):
    """The Exp(1) draws torch.multinomial(probs, 1) consumes on the reference's CPU run: one `empty_like(probs).exponential_(1)` of
    shape [B, V] per sampled token, in call order, from the default generator seeded like make_golden.py
    (ATen multinomial with num_samples == 1: argmax(probs / q); SURVEY.md section 7 hard-part 4)."""
    torch.manual_seed(seed)
    return torch.stack([torch.empty(B, V).exponential_(1) for _ in range(n_steps)])


def test_sampled_grid_bit_exact_with_torch_noise_fp32():
    """generate.py:59-74 with sample_logits=True: replaying the reference's own Exp(1) draws through `noise=` reproduces the
    reference's SAMPLED token grid bit for bit (fp32 checkpoint, top-k 100, CFG 4, masks, control_strength 0.6)."""
    g, spec, dt, model, sd, cond, masks = _setup("t2i_small_fp32")
    from controlar_b200.autoregressive.models.generate import generate
    dev = "cuda"
    ref = g["sampled_tokens"]
    B, N = ref.shape
    noise = _torch_multinomial_noise(g["sampled_seed"], N, B, spec.vocab_size).to(dev)
    model.adapter.forward = lambda x: x
    model.adapter_mlp.forward = lambda x: x
    out = generate(model, cond.to(dev), N, emb_masks=masks.to(dev), cfg_scale=g["cfg_scale"], condition=g["ctrl_in"].to(dev),
                   control_strength=g["control_strength"], temperature=1.0, top_k=g["sampled_top_k"], top_p=1.0, sample_logits=True,
                   noise=noise).cpu()
    assert torch.equal(out, ref), f"first difference at {(out != ref).nonzero()[:3].tolist()}"


def test_sampled_choices_with_torch_noise_bf16_persistent_kernel():
    """The `noise=` path of the persistent decode kernel: teacher-forced along the reference's SAMPLED trajectory (bf16), with the
    reference's Exp(1) draws, the in-kernel sampler must pick the reference's token at (nearly) every step — a flip needs a
    bf16-level logit difference to reorder two race candidates."""
    from controlar_b200 import engine
    g, spec, dt, model, sd, cond, masks = _setup("t2i_small_bf16")
    dev = "cuda"
    ref = g["sampled_tokens"]
    B, N = ref.shape
    T = spec.cls_token_num
    noise = _torch_multinomial_noise(g["sampled_seed"], N, B, spec.vocab_size).to(dev)
    ctrl_in = g["ctrl_in"].to(dev)
    c = cond.to(dev)
    cc = torch.cat([c, torch.zeros_like(c) + model.cls_embedding.uncond_embedding])
    cond_comb = torch.cat([ctrl_in, torch.zeros_like(ctrl_in)])
    model.setup_caches(2 * B, T + N, dt, n_img_tokens=N)
    st = model._car_state
    st.set_emb_mask(torch.cat([masks, masks]).to(dev))
    st.prefill(cc, cond_comb, g["control_strength"], all_rows=False)
    sp = engine.make_sampling(temperature=1.0, top_k=g["sampled_top_k"], top_p=1.0, sample_logits=True, cfg_scale=g["cfg_scale"])
    choice, _ = st.generate_forced(sp, ref.to(dev), trace=False, noise=noise)
    agree = float((choice.cpu() == ref).float().mean())
    assert agree >= 0.9, f"only {agree:.3f} of the sampled choices match the reference"


# the smoke test's model: bf16 decodes on the persistent kernel, fp32 on the per-kernel graph chain
SMALL = GPTSpec(dim=256, n_layer=6, n_head=4, vocab_size=2048, cls_token_num=120, block_size=64, model_type="t2i")


def _greedy_grid(model):
    """generate()'s greedy token grid on fixed inputs (CFG, masks, control tokens given as the control encoder's output)."""
    from controlar_b200.autoregressive.models.generate import generate
    dt = model.tok_embeddings.weight.dtype
    cond, masks = text_inputs(SMALL.cls_token_num, SMALL.caption_dim, 2, 1, dt)
    ctrl = torch.randn(2, 16, SMALL.dim, generator=torch.Generator().manual_seed(3)) * 0.5
    model.adapter.forward = lambda x: x
    model.adapter_mlp.forward = lambda x: x
    return generate(model, cond.cuda(), 16, emb_masks=masks.cuda(), cfg_scale=4.0, condition=ctrl.to(dt).cuda(), control_strength=0.7,
                    temperature=1.0, top_k=0, top_p=1.0, sample_logits=False).cpu()


def test_weight_update_repacks_the_model():
    """load_state_dict between two generate() calls: the packed copies are rewritten in place (car_model_repack) and the grid is that
    of a model built with the new weights."""
    model, _ = build_product_gpt(SMALL, 0, torch.bfloat16)
    g0 = _greedy_grid(model)
    generation = model._car_model.generation
    fresh, sd5 = build_product_gpt(SMALL, 5, torch.bfloat16)
    missing, unexpected = model.load_state_dict(sd5, strict=False)
    assert not unexpected and all(".kv_cache." in k for k in missing)     # the caches setup_caches added are buffers too
    g5 = _greedy_grid(model)
    assert model._car_model.generation == generation               # same layout: repacked, not re-created
    assert torch.equal(g5, _greedy_grid(fresh)) and not torch.equal(g0, g5)


def test_replaced_parameter_data_is_picked_up():
    """`p.data = t` on any weight the library borrows (it changes data_ptr, not _version) takes effect at the next generate()."""
    model, _ = build_product_gpt(SMALL, 0, torch.bfloat16)
    fresh, _ = build_product_gpt(SMALL, 0, torch.bfloat16)
    g0 = _greedy_grid(model)
    w = model.layers[1].attention.wo.weight
    new = (torch.randn(w.shape, generator=torch.Generator().manual_seed(7)) * 0.05).to(device=w.device, dtype=w.dtype)
    w.data = new.clone()
    fresh.layers[1].attention.wo.weight.data.copy_(new)
    g1 = _greedy_grid(model)
    assert torch.equal(g1, _greedy_grid(fresh)) and not torch.equal(g0, g1)


def test_failed_model_recreate_leaves_no_stale_handle(monkeypatch):
    """A new layout (bf16 -> fp32) whose CarModel create is refused leaves no handle behind: the next call builds a new model and
    state, and every model and state the library created is destroyed exactly once."""
    import gc
    from controlar_b200 import _lib
    from tests.helpers import ObservedLib
    gc.collect()                                       # earlier tests' handles are destroyed by the library itself, not observed
    lib = ObservedLib(_lib.lib(), ["model", "state"])
    monkeypatch.setattr(_lib, "_lib", lib)
    model, _ = build_product_gpt(SMALL, 0, torch.bfloat16)
    _greedy_grid(model)
    model.to(torch.float32)
    lib.refuse = True
    with pytest.raises(RuntimeError, match="car_model_create"):
        _greedy_grid(model)
    assert not model._car_model.handle
    lib.refuse = False
    want = _greedy_grid(build_product_gpt(SMALL, 0, torch.bfloat16)[0].to(torch.float32))
    assert torch.equal(_greedy_grid(model), want)
    del model
    gc.collect()
    assert len(lib.created) == 6 and sorted(lib.destroyed) == sorted(lib.created), (lib.created, lib.destroyed)
