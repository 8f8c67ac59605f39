"""GPU: per-image sampling parameters and control strengths in one launch (car_state_set_row_sampling, car_sample_rows,
generate()'s per-image arguments, LLM(mixed_sampling=True)).  Procedural weights only.

The contract: row b of a mixed launch is bit-identical to row b of a uniform launch of the same size whose parameters are row b's.
  * the sampler's per-row build against the exact oracle (oracle/sampler_oracle.py), its uniform rows against car_sample, and
    the independence of an image's draws from its row when it has its own seed;
  * the persistent kernel's sampler (pk_sample) against car_sample_rows, step by step;
  * the whole decode loop on every route: the persistent kernel at B_eff 16 (a small model and a GPT-XL-shaped one), the per-kernel
    chain at 24 and the wide route at 50, teacher-forced with mixed control strengths and free-running with mixed sampling;
    mixed strengths also on an fp32 checkpoint (the chain at 24, teacher-forced through car_decode_step), where every control add
    reads its row's strength exactly as a uniform launch reads it, so the compiler's fused multiply-add is the same in both;
  * the serving engine in mixed mode: 8 configurations in one launch."""
import pytest
import torch

from oracle.inputs import class_inputs
from oracle.sampler_oracle import catalogue, cfg_temperature, oracle_sample
from oracle.weights import GPTSpec
from tests.helpers import build_product_gpt
from tests.test_sampler_gpu import _check, _identical, _model, _prefill, SPEC, N_TOK

pytestmark = pytest.mark.gpu

# (temperature, top_k, top_p, greedy): every selection path of the sampler (list, row, no threshold, nucleus)
CONFIGS = [(1.0, 2000, 1.0, False), (0.7, 100, 0.9, True), (1.3, 0, 0.5, False), (1.0, 2241, 0.999, False), (0.7, 8000, 1.0, True),
           (1.0, 1, 1.0, False), (2.0, 16384, 0.9, False), (0.5, 50, 1e-6, True)]


def _rows(n, seeds=None, strengths=None, configs=CONFIGS, flip=False):
    from controlar_b200 import engine
    out = []
    for b in range(n):
        T, k, p, greedy = configs[b % len(configs)]
        out.append(engine.make_row_sampling(T, k, p, greedy == flip, 0 if seeds is None else seeds[b], 0,
                                            1.0 if strengths is None else strengths[b]))
    return out


def _catalogue_rows():
    return torch.cat([r for r in catalogue().values()])                 # [14, 16384]


@pytest.mark.parametrize("cfg_on", [True, False, None])
def test_sample_rows_vs_oracle(cfg_on):
    """Every catalogue row with its own (temperature, top_k, top_p, greedy), explicit noise; with CFG (cfg_on True / False) and
    without (None).  Each row passes tests/test_sampler_gpu.py's acceptance rule; a second launch with every greedy flag flipped
    gives each row its other draw."""
    from controlar_b200 import engine
    cond = _catalogue_rows()
    B, V = cond.shape
    g = torch.Generator().manual_seed(61)
    noise = torch.empty(B, V).exponential_(1.0, generator=g)
    cfg_scale = 1.0 if cfg_on is None else 4.0
    lg = cond if cfg_on is None else torch.cat([cond, (torch.randn(B, V, generator=g) * 2.0).to(torch.bfloat16).float()])
    rows, flipped = _rows(B), _rows(B, flip=True)
    on = cfg_on is not False
    idx, probs, kept = engine.sample_rows(lg.cuda(), rows, cfg_scale, on, noise=noise.cuda(), return_probs=True, return_kept=True)
    idx2 = engine.sample_rows(lg.cuda(), flipped, cfg_scale, on, noise=noise.cuda())
    idx, idx2, probs, kept = idx.cpu().long(), idx2.cpu().long(), probs.cpu(), kept.cpu()
    for b in range(B):
        T, k, p, greedy = CONFIGS[b % len(CONFIGS)]
        z = cfg_temperature(lg[[b, B + b]] if cfg_on is not None else lg[b:b + 1], 1, cfg_scale, on, T)
        o1 = oracle_sample(z, k, 1.0, sample_logits=False)
        sampled, gidx = (idx2, idx) if greedy else (idx, idx2)
        _check(f"row {b} T={T} top_k={k} top_p={p} greedy={greedy} cfg={cfg_on}", z, k, p, o1, kept[b:b + 1], probs[b:b + 1],
               sampled[b:b + 1], noise[b:b + 1], gidx[b:b + 1])


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("cfg", [True, False])
def test_uniform_rows_reproduce_car_sample(explicit, cfg):
    """Uniform rows with the scalar seed rule (key = seed, counter word = image index) are car_sample, bit for bit."""
    from controlar_b200 import engine
    g = torch.Generator().manual_seed(62)
    B, V = 6, 16384
    lg = (torch.randn((2 if cfg else 1) * B, V, generator=g) * 2.0).cuda()
    noise = torch.empty(B, V).exponential_(1.0, generator=g).cuda() if explicit else None
    for step, (T, k, p, greedy) in enumerate(CONFIGS):
        sp = engine.make_sampling(T, k, p, not greedy, cfg_scale=4.0 if cfg else 1.0, seed=1000 + step)
        rows = [engine.make_row_sampling(T, k, p, not greedy, 1000 + step, b) for b in range(B)]
        for on in (True, False) if cfg else (True,):
            a = engine.sample(lg, sp, cfg_on=on, step=step, noise=noise, return_probs=True, return_kept=True)
            r = engine.sample_rows(lg, rows, sp.cfg_scale, on, step=step, noise=noise, return_probs=True, return_kept=True)
            _identical(tuple(x.cpu() for x in a), tuple(x.cpu() for x in r), f"T={T} top_k={k} top_p={p} greedy={greedy} cfg_on={on}")


@pytest.mark.parametrize("cfg", [True, False])
def test_own_seed_draws_do_not_depend_on_the_row(cfg):
    """Per-image seeds and in-kernel Philox: permuting the images (logits, unconditional partners and parameters) permutes the
    outputs bit for bit, at every step."""
    from controlar_b200 import engine
    g = torch.Generator().manual_seed(63)
    B, V = 8, 16384
    lg = torch.randn((2 if cfg else 1) * B, V, generator=g) * 2.0
    seeds = [int(x) for x in torch.randint(0, 2 ** 62, (B,), generator=g)]
    rows = _rows(B, seeds=seeds, configs=[(T, k, p, False) for T, k, p, _ in CONFIGS])
    perm = torch.randperm(B, generator=g)
    lp = lg[torch.cat([perm, B + perm])] if cfg else lg[perm]
    cs = 4.0 if cfg else 1.0
    for step in (0, 5, 200):
        a = engine.sample_rows(lg.cuda(), rows, cs, step=step, return_probs=True, return_kept=True)
        b = engine.sample_rows(lp.cuda(), [rows[i] for i in perm.tolist()], cs, step=step, return_probs=True, return_kept=True)
        _identical(tuple(x.cpu()[perm] for x in a), tuple(x.cpu() for x in b), f"step {step}")
    # the draws do follow the seed: the same logits under other seeds choose differently somewhere
    other = _rows(B, seeds=[s + 1 for s in seeds], configs=[(1.0, 0, 1.0, False)])
    same = _rows(B, seeds=seeds, configs=[(1.0, 0, 1.0, False)])
    assert not torch.equal(engine.sample_rows(lg.cuda(), same, cs), engine.sample_rows(lg.cuda(), other, cs))


@pytest.mark.parametrize("explicit", [True, False])
def test_persistent_build_matches_sample_rows(explicit):
    """car_generate_forced at B = 8 with CFG (the persistent kernel's pk_sample) with per-image parameters and seeds, replayed step
    by step through car_sample_rows: identical choices at every step; the free-running grid replays teacher-forced to itself."""
    from controlar_b200 import engine
    model = _model("plain")
    B, V = 8, SPEC.vocab_size
    g = torch.Generator().manual_seed(64)
    forced = torch.randint(0, V, (B, N_TOK), generator=g).cuda()
    noise = torch.empty(N_TOK, B, V).exponential_(1.0, generator=g).cuda() if explicit else None
    rows = _rows(B, seeds=[int(x) for x in torch.randint(0, 2 ** 62, (B,), generator=g)])
    for ci in (-1, 5):
        sp = engine.make_sampling(cfg_scale=4.0, cfg_interval=ci)
        st, _ = _prefill(model, B, True)
        st.set_row_sampling(rows)
        choice, trace = st.generate_forced(sp, forced, trace=True, noise=noise)
        choice = choice.cpu().long()
        for s in range(N_TOK):
            on = not (ci > -1 and s - 1 > ci)
            idx = engine.sample_rows(trace[s], rows, 4.0, on, step=s, noise=None if noise is None else noise[s]).cpu().long()
            assert torch.equal(idx, choice[:, s]), f"cfg_interval={ci} step {s}: persistent {choice[:, s].tolist()} vs {idx.tolist()}"
        st, _ = _prefill(model, B, True)
        st.set_row_sampling(rows)
        free = st.generate(sp, N_TOK, noise, "cuda")
        st, _ = _prefill(model, B, True)
        st.set_row_sampling(rows)
        again, _ = st.generate_forced(sp, free, trace=False, noise=noise)
        st.set_row_sampling(None)
        assert torch.equal(again, free), f"cfg_interval={ci}: teacher-forced replay of the free-running grid differs"


# ------------------------------------------------------------------------------------------------------------------------------
# the contract on every decode route
# ------------------------------------------------------------------------------------------------------------------------------
N_GEN = 16
SMALL = GPTSpec(dim=256, n_layer=6, n_head=4, vocab_size=16384, cls_token_num=1, block_size=N_GEN, model_type="c2i")
XL = GPTSpec(dim=1280, n_layer=36, n_head=20, vocab_size=16384, cls_token_num=1, block_size=N_GEN, model_type="c2i")
_MODELS = {}


def _ctl_model(spec, dtype=torch.bfloat16):
    key = (spec.dim, dtype)
    if key not in _MODELS:
        m, _ = build_product_gpt(spec, 8, dtype)
        m.adapter.forward = lambda x: x              # control tokens given directly
        m.adapter_mlp.forward = lambda x: x
        _MODELS[key] = m
    return _MODELS[key]


def _inputs(spec, B):
    g = torch.Generator().manual_seed(65 + B)
    cond = class_inputs(spec.num_classes, B, 9 + B).cuda()
    ctrl = (torch.randn(B, N_GEN, spec.dim, generator=g) * 0.5).to(torch.bfloat16).cuda()
    forced = torch.randint(0, spec.vocab_size, (B, N_GEN), generator=g).cuda()
    noise = torch.empty(N_GEN, B, spec.vocab_size).exponential_(1.0, generator=g).cuda()
    return cond, ctrl, forced, noise


STRENGTHS = (0.3, 0.6, 1.0)
ROUTES = [pytest.param(SMALL, 8, id="persistent-b16"), pytest.param(XL, 8, id="persistent-xl-b16"),
          pytest.param(SMALL, 12, id="chain-b24"), pytest.param(SMALL, 25, id="wide-b50")]


@pytest.mark.parametrize("spec,B,dtype", [pytest.param(*r.values, torch.bfloat16, id=r.id) for r in ROUTES] +
                         [pytest.param(SMALL, 12, torch.float32, id="chain-b24-fp32")])
def test_mixed_strengths_teacher_forced_equal_uniform_launches(spec, B, dtype):
    """car_generate_forced (fp32: car_decode_step per token) with strengths 0.3 / 0.6 / 1.0 cycling over the images: the logits
    trace of image b (its conditional and unconditional row) equals, bit for bit, the trace of a uniform launch at image b's
    strength."""
    from controlar_b200 import engine
    model = _ctl_model(spec, dtype)
    cond, ctrl, forced, _ = _inputs(spec, B)
    cc = torch.cat([cond, torch.full_like(cond, spec.num_classes)])
    ctl = torch.cat([ctrl, torch.zeros_like(ctrl)])
    sp = engine.make_sampling(sample_logits=False, top_k=0, cfg_scale=4.0)
    strength = [STRENGTHS[b % 3] for b in range(B)]

    def run(rows, cs):
        model.setup_caches(2 * B, 1 + N_GEN, dtype, n_img_tokens=N_GEN)
        st = model._car_state
        st.set_emb_mask(None)
        st.set_row_sampling(rows)
        logits = st.prefill(cc, ctl, cs, all_rows=False)
        if dtype == torch.bfloat16:
            _, trace = st.generate_forced(sp, forced)
        else:       # car_generate_forced is bf16 only: the same teacher-forced steps one at a time, the CFG pair sharing its token
            tok = torch.cat([forced, forced])
            trace = torch.stack([logits] + [st.decode_step(tok[:, i], st.T + i) for i in range(N_GEN - 1)])
        st.set_row_sampling(None)
        return trace.cpu()
    mixed = run([engine.make_row_sampling(sample_logits=False, control_strength=s) for s in strength], 1.0)
    assert bool(torch.isfinite(mixed).all())
    for s in STRENGTHS:
        uni = run(None, s)
        for b in [b for b in range(B) if strength[b] == s]:
            for r in (b, B + b):
                assert torch.equal(mixed[:, r], uni[:, r]), f"strength {s}, image {b}, row {r}: logits differ from the uniform launch"
    assert not torch.equal(run(None, 0.3)[:, 1], mixed[:, 1]), "the strength must reach the logits"


# (temperature, top_k, top_p, greedy, strength) of the free-running launches
GEN_CONFIGS = [(1.0, 2000, 1.0, False, 1.0), (0.7, 100, 0.9, False, 0.6), (1.3, 0, 1.0, True, 0.3), (1.0, 9000, 0.95, False, 0.6)]


@pytest.mark.parametrize("spec,B", ROUTES)
def test_mixed_sampling_generate_equals_uniform_launches(spec, B):
    """generate() with per-image temperature, top_k, top_p, sample_logits and control_strength, explicit noise: image b's grid equals,
    bit for bit, its grid in a uniform launch (scalar arguments) at image b's parameters."""
    from controlar_b200.autoregressive.models.generate import generate
    model = _ctl_model(spec)
    cond, ctrl, _, noise = _inputs(spec, B)
    cfgs = [GEN_CONFIGS[b % len(GEN_CONFIGS)] for b in range(B)]
    kw = dict(cfg_scale=4.0, condition=ctrl, noise=noise)
    mixed = generate(model, cond, N_GEN, temperature=[c[0] for c in cfgs], top_k=[c[1] for c in cfgs], top_p=[c[2] for c in cfgs],
                     sample_logits=[not c[3] for c in cfgs], control_strength=[c[4] for c in cfgs], seed=3, **kw).cpu()
    for c in GEN_CONFIGS:
        uni = generate(model, cond, N_GEN, temperature=c[0], top_k=c[1], top_p=c[2], sample_logits=not c[3], control_strength=c[4],
                       seed=3, **kw).cpu()
        for b in [b for b in range(B) if cfgs[b] == c]:
            assert torch.equal(mixed[b], uni[b]), f"config {c}, image {b}: grid differs from the uniform launch"
    assert len({tuple(mixed[b].tolist()) for b in range(B)}) > 1


def test_engine_mixed_mode_runs_eight_configurations_in_one_launch():
    """LLM(mixed_sampling=True): 8 requests with 8 sampling configurations, strengths and seeds run as one launch, and every
    request's grid equals the direct per-image generate() call for that batch."""
    from controlar_b200.autoregressive.models.generate import generate
    from controlar_b200.autoregressive.serve.llm import LLM, SamplingParams, derived_seed
    model = _ctl_model(SMALL)
    B = 8
    cond, ctrl, _, _ = _inputs(SMALL, B)
    sps = [SamplingParams(temperature=T if not greedy else 0, top_k=k, top_p=p, max_tokens=N_GEN, seed=(None if b % 2 else 500 + b))
           for b, (T, k, p, greedy) in enumerate(CONFIGS)]
    strengths = [STRENGTHS[b % 3] for b in range(B)]
    llm = LLM(model=model, cfg_scale=4.0, max_images_per_batch=8, seed=9, mixed_sampling=True)
    outs = llm.generate(prompts=[dict(cond=int(cond[b]), control=ctrl[b], control_strength=strengths[b], sampling_params=sps[b])
                                 for b in range(B)])
    assert llm._launches == 1
    seeds = [sp.seed if sp.seed is not None else derived_seed(9, b) for b, sp in enumerate(sps)]
    want = generate(model, cond, N_GEN, cfg_scale=4.0, condition=ctrl, control_strength=strengths,
                    temperature=[1.0 if sp.temperature == 0 else sp.temperature for sp in sps], top_k=[max(sp.top_k, 0) for sp in sps],
                    top_p=[sp.top_p for sp in sps], sample_logits=[sp.temperature != 0 for sp in sps], seed=seeds).cpu()
    for b, o in enumerate(outs):
        assert o.outputs[0].token_ids == want[b].tolist(), f"request {b}"
