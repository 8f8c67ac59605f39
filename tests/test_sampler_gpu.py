"""GPU conformance of the fused top-k / top-p / CFG sampler (csrc/sampler.cuh) against the exact restatement of the reference in
oracle/sampler_oracle.py, in both of its builds: the standalone 1024-thread `sample_kernel` (car_sample, the CUDA-graph loop) and
the 512-thread copy inside the persistent decode kernel (car_generate / car_generate_forced).

Which test reaches which selection path of sample_body (checked with a counter-instrumented build of the kernel):
  * list path (0 < top_k <= 2240, exact ranks in the boundary bin): test_catalogue_vs_oracle (random, bf16, pm0_small, tie200 at
    top_k <= 2000, ...), test_cfg_batches_vs_oracle, test_path_identity_list_vs_row / _bisection, the persistent runs (100, 2000)
  * row path (2241 <= top_k < V): test_catalogue_vs_oracle (2241, 8000, V - 1), test_path_identity_*, the persistent runs (2241, 9000)
  * crowded boundary bin (> 1024 candidates, bisection): the outlier / all-equal / -inf / tie3000 / pm0 rows,
    test_path_identity_bisection, the persistent runs on the "zero" model (8192-way tie at 0)
  * tie overflow (> 2304 kept on the list path after exact ranks): tie200 at top_k 2240, test_path_identity_tie_overflow, the
    persistent runs on the "tieovf" model at top_k 2000 (steps where the one-direction logits are positive)
  * no threshold (top_k <= 0 or >= V): top_k -1, 0, V, V + 5
  * nucleus: every top_p < 1
"""
import numpy as np
import pytest
import torch

from oracle.sampler_oracle import (catalogue, cfg_temperature, choice_ok, oracle_sample, small_v_rows)
from oracle.weights import GPTSpec
from oracle.inputs import class_inputs
from tests.helpers import build_product_gpt

pytestmark = pytest.mark.gpu

TOP_K = (-1, 0, 1, 100, 2000, 2240, 2241, 8000, "V-1", "V", "V+5")
TOP_P = (1.0, 0.999, 0.9, 0.5, 1e-6, 0.0)
TEMPS = (1.0, 0.7, 1.3, 0.0)


def _k(k, V):
    return {"V-1": V - 1, "V": V, "V+5": V + 5}[k] if isinstance(k, str) else k


def _run(logits, sp, cfg_on=True, step=0, noise=None):
    from controlar_b200 import engine
    idx, probs, kept = engine.sample(logits, sp, cfg_on=cfg_on, step=step, noise=noise, return_probs=True, return_kept=True)
    return idx.cpu().long(), probs.cpu(), kept.cpu()


def _check(what, z, top_k, top_p, o1, got_kept, got_probs, got_idx, noise, greedy_idx):
    """kept set, probabilities and both draws of one car_sample call against the oracle.  o1: the oracle at top_p = 1."""
    o = oracle_sample(z, top_k, top_p, noise=noise)
    out = ~o.band
    bad = (got_kept != o.kept) & out
    assert not bool(bad.any()), f"{what}: kept set differs at {bad.nonzero()[:6].tolist()} (kernel kept {int(got_kept.sum())}, " \
                                f"oracle {int(o.kept.sum())})"
    # the oracle's soft-max over the set the kernel kept (identical to o.probs unless a band token went the other way)
    p = o1.probs * got_kept
    p = p / p.sum(-1, keepdim=True)
    assert torch.allclose(got_probs.double(), p, atol=1e-7, rtol=2e-5), \
        f"{what}: probabilities, max err {float((got_probs.double() - p).abs().max()):.3e}"
    # probs > 0 == the oracle's kept tokens whose fp32 probability is non-zero
    nz = got_kept & (p.float() > 0)
    assert torch.equal(got_probs > 0, nz), f"{what}: probs > 0 differs from the kept tokens with a non-zero fp32 probability"
    for r in range(z.shape[0]):
        if bool((got_kept[r] == o.kept[r]).all()):
            assert choice_ok(int(got_idx[r]), o, r), f"{what} row {r}: race chose {int(got_idx[r])}, oracle {int(o.choice[r])} " \
                                                   f"(second {int(o.second[r])}, gap {float(o.gap[r]):.2e})"
    og = oracle_sample(z, top_k, top_p, noise=None, sample_logits=False)
    for r in range(z.shape[0]):
        if bool((got_kept[r] == og.kept[r]).all()):
            assert choice_ok(int(greedy_idx[r]), og, r), f"{what} row {r}: greedy chose {int(greedy_idx[r])}, oracle {int(og.choice[r])}"


def _rowsets():
    out = [(n, r) for n, r in catalogue().items()]
    out += [(f"v{V}", r) for V, r in small_v_rows().items()]
    return out


ROWSETS = _rowsets()


@pytest.mark.parametrize("name", [n for n, _ in ROWSETS])
def test_catalogue_vs_oracle(name):
    """Every row of the catalogue x top_k x top_p x temperature, explicit noise and greedy."""
    from controlar_b200 import engine
    rows = dict(ROWSETS)[name]
    R, V = rows.shape
    g = torch.Generator().manual_seed(17)
    noise = torch.empty(R, V).exponential_(1.0, generator=g)
    dev = rows.cuda()
    for T in TEMPS:
        # the temperature the reference applies on the GPU: torch's `tensor / python_float` (pins reciprocal-multiply vs divide)
        zt = (dev / max(T, 1e-5)).cpu()
        z = cfg_temperature(rows, R, 1.0, True, T)
        assert torch.equal(zt, z), f"{name} T={T}: torch's CUDA division differs from the reciprocal multiply"
        for kk in TOP_K:
            k = _k(kk, V)
            o1 = oracle_sample(z, k, 1.0, sample_logits=False)
            for p in TOP_P:
                sp = engine.make_sampling(T, k, p, sample_logits=True, cfg_scale=1.0)
                idx, probs, kept = _run(dev, sp, noise=noise.cuda())
                spg = engine.make_sampling(T, k, p, sample_logits=False, cfg_scale=1.0)
                gidx = engine.sample(dev, spg).cpu().long()
                _check(f"{name} T={T} top_k={kk} top_p={p}", z, k, p, o1, kept, probs, idx, noise, gidx)


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("kind", ["normal", "bf16"])
def test_cfg_batches_vs_oracle(B, kind):
    """CFG at scale 4 on and off, batches of 1, 3 and 8 images; bf16-valued rows give the production tie structure."""
    from controlar_b200 import engine
    V = 16384
    g = torch.Generator().manual_seed(100 + B)
    lg = torch.randn(2 * B, V, generator=g) * 2.0
    if kind == "bf16":
        lg = lg.to(torch.bfloat16).float()
    noise = torch.empty(B, V).exponential_(1.0, generator=g)
    for cfg_on in (True, False):
        for T, k, p in ((1.0, 2000, 1.0), (0.7, 100, 0.9), (1.3, 0, 0.5), (1.0, 2241, 0.999), (0.7, 8000, 1.0)):
            z = cfg_temperature(lg, B, 4.0, cfg_on, T)
            o1 = oracle_sample(z, k, 1.0, sample_logits=False)
            sp = engine.make_sampling(T, k, p, sample_logits=True, cfg_scale=4.0)
            idx, probs, kept = _run(lg.cuda(), sp, cfg_on=cfg_on, noise=noise.cuda())
            gidx = engine.sample(lg.cuda(), engine.make_sampling(T, k, p, sample_logits=False, cfg_scale=4.0), cfg_on=cfg_on).cpu().long()
            _check(f"B={B} {kind} cfg_on={cfg_on} T={T} top_k={k} top_p={p}", z, k, p, o1, kept, probs, idx, noise, gidx)


def test_negative_zero_ties_positive_zero_at_threshold():
    """The k-th largest value is +0: the reference keeps every -0 entry (-0 < +0 is false), so the kernel must too."""
    from controlar_b200 import engine
    cat = catalogue()
    # pm0: 3000 zeros crowd the boundary bin (bisection); pm0_small: 200 zeros, resolved by the exact-rank comparison
    for name, ks, n_zero, n_keep in (("pm0", (1000, 1500, 2000), 3000, 3100), ("pm0_small", (1950, 2000), 200, 2100)):
        rows = cat[name]
        zero = rows[0] == 0
        assert int(zero.sum()) == n_zero
        for k in ks:
            sp = engine.make_sampling(1.0, k, 1.0, sample_logits=False)
            _, probs = engine.sample(rows.cuda(), sp, return_probs=True)
            kept = probs.cpu()[0] > 0                              # (no kept token underflows on these rows)
            assert bool(kept[zero].all()), f"{name} top_k={k}: {int((~kept[zero]).sum())} of the {n_zero} +-0 entries dropped"
            assert int(kept.sum()) == n_keep


def test_dropin_filtering_keeps_underflowing_tokens():
    """top_k_top_p_filtering (drop-in) keeps exactly the reference's set: kept tokens more than ~100 below the row maximum have a
    probability that underflows to 0, yet keep their logit."""
    from controlar_b200.autoregressive.models.generate import top_k_top_p_filtering
    g = torch.Generator().manual_seed(9)
    lg = torch.randn(3, 4096, generator=g) * 60.0                 # rows spanning several hundred
    for k, p in ((0, 1.0), (3000, 1.0), (100, 1.0), (0, 0.9), (2000, 0.5)):
        got = top_k_top_p_filtering(lg.clone().cuda(), top_k=k, top_p=p).cpu()
        o = oracle_sample(lg, k, p, sample_logits=False)
        out = ~o.band
        assert torch.equal(torch.isfinite(got)[out], o.kept[out]), f"top_k={k} top_p={p}: filtered set differs"
        assert torch.equal(got[o.kept & out], lg[o.kept & out]), f"top_k={k} top_p={p}: kept logits changed"
        if k == 0 and p == 1.0:
            assert torch.equal(got, lg)
        if k == 3000:
            assert bool((o.kept & (o.probs.float() == 0)).any()), "the case must hold kept tokens whose probability underflows"


def _identical(a, b, what):
    ia, pa, ka = a
    ib, pb, kb = b
    assert torch.equal(ka, kb), f"{what}: kept sets differ"
    assert torch.equal(pa.view(torch.int32), pb.view(torch.int32)), f"{what}: probabilities not bitwise identical"
    assert torch.equal(ia, ib), f"{what}: choices differ"


def test_path_identity_list_vs_row():
    """A tie spanning ranks 2200 .. 2300: top_k = 2240 takes the list path and 2241 the row path, with the same kept set."""
    from controlar_b200 import engine
    g = torch.Generator().manual_seed(21)
    V = 16384
    z = torch.randn(1, V, generator=g)
    order = torch.sort(z[0], descending=True).indices
    z[0, order[2199:2300]] = float(z[0, order[2199]])
    noise = torch.empty(1, V).exponential_(1.0, generator=g).cuda()
    for p in (1.0, 0.9):
        a = _run(z.cuda(), engine.make_sampling(1.0, 2240, p), noise=noise)
        b = _run(z.cuda(), engine.make_sampling(1.0, 2241, p), noise=noise)
        assert int(a[2].sum()) == 2300 or p < 1.0
        _identical(a, b, f"list vs row, top_p={p}")


def test_path_identity_bisection():
    """The same 100 tokens kept from a plain row (histogram + exact ranks) and from the row with its smallest entry set to -inf
    (bin scale 0: crowded boundary bin, bisection over the whole row)."""
    from controlar_b200 import engine
    g = torch.Generator().manual_seed(22)
    V = 16384
    z = torch.randn(1, V, generator=g)
    z2 = z.clone()
    z2[0, int(z[0].argmin())] = -float("inf")
    noise = torch.empty(1, V).exponential_(1.0, generator=g).cuda()
    for k, p in ((100, 1.0), (100, 0.7), (2000, 1.0)):
        a = _run(z.cuda(), engine.make_sampling(1.0, k, p), noise=noise)
        b = _run(z2.cuda(), engine.make_sampling(1.0, k, p), noise=noise)
        _identical(a, b, f"bisection top_k={k} top_p={p}")


def test_path_identity_tie_overflow():
    """2200 distinct values above a 200-way exact tie (ranks 2201 .. 2400).  The tie stays in one boundary bin of <= 1024
    candidates, so the threshold comes from the exact ranks; top_k = 2240 then takes the list path and overflows it (2400 kept
    > 2304), while 2241 and 2300 take the row path.  All keep the same 2400 tokens."""
    from controlar_b200 import engine
    g = torch.Generator().manual_seed(23)
    V = 16384
    z = torch.randn(1, V, generator=g)
    order = torch.sort(z[0], descending=True).indices
    z[0, order[2200:2400]] = float(z[0, order[2200]])
    noise = torch.empty(1, V).exponential_(1.0, generator=g).cuda()
    for p in (1.0, 0.9):
        a = _run(z.cuda(), engine.make_sampling(1.0, 2240, p), noise=noise)
        if p == 1.0:
            assert int(a[2].sum()) == 2400
        for k in (2241, 2300):
            _identical(a, _run(z.cuda(), engine.make_sampling(1.0, k, p), noise=noise), f"tie overflow vs row top_k={k}, top_p={p}")


# ------------------------------------------------------------------------------------------------------------------------------
# the persistent-kernel build (512 threads) against the standalone build, and the CUDA-graph loop
# ------------------------------------------------------------------------------------------------------------------------------
N_TOK = 16
# (the library's decode path needs n_layer to be a multiple of 3: the control tokens are added every n_layer / 3 layers,
#  gpt_t2i.py:320,457)
SPEC = GPTSpec(dim=256, n_layer=3, n_head=4, vocab_size=16384, cls_token_num=1, block_size=N_TOK, model_type="c2i")


def _model(variant: str):
    model, _ = build_product_gpt(SPEC, 3, torch.bfloat16)
    with torch.no_grad():
        w = model.output.weight
        if variant == "zero":
            w[:8192] = 0                                   # an exact 8192-way tie at 0 after CFG: crowded boundary bin
        if variant == "tieovf":
            # every row along one hidden direction, so per step and image every logit is gain * a for one scalar a: 330 zero rows,
            # 1990 gains in [1, 2), the rest in [-2, -1).  When a > 0 the 330-way tie at 0 holds ranks 1991 .. 2320, alone in its
            # histogram bin; top_k = 2000 then resolves the threshold by exact ranks and overflows the kept list (2320 > 2304)
            g4 = torch.Generator().manual_seed(4)
            gain = torch.cat([torch.zeros(330), 1.0 + torch.rand(1990, generator=g4), -1.0 - torch.rand(SPEC.vocab_size - 2320, generator=g4)])
            w.zero_()
            w[:, 7] = gain.to(w.dtype).to(w.device)
    model.adapter.forward = lambda x: x
    model.adapter_mlp.forward = lambda x: x
    return model


def _prefill(model, B, cfg):
    cond = class_inputs(SPEC.num_classes, B, 5).cuda()
    cc = torch.cat([cond, torch.full_like(cond, SPEC.num_classes)]) if cfg else cond
    b_eff = cc.shape[0]
    model.setup_caches(b_eff, 1 + N_TOK, torch.bfloat16, n_img_tokens=N_TOK)
    st = model._car_state
    st.set_emb_mask(None)
    logits = st.prefill(cc, None, 1.0, all_rows=False)
    return st, logits


def _pk_matrix():
    out, i = [], 0
    for k in (0, 100, 2000, 2241, 9000):
        for p in (1.0, 0.9):
            for T in (1.0, 0.7):
                out.append((k, p, T, (-1, 0, 5)[i % 3], bool(i % 2)))
                i += 1
    return out


@pytest.mark.parametrize("variant", ["plain", "zero", "tieovf"])
@pytest.mark.parametrize("B", [1, 8])
def test_persistent_build_matches_standalone_bit_for_bit(variant, B):
    """car_generate_forced (512-thread sampler inside the persistent kernel) replayed step by step through car_sample
    (1024-thread build): identical choices at every step, and agreement with the oracle apart from its declared near-ties."""
    from controlar_b200 import engine
    model = _model(variant)
    V, cfg_scale = SPEC.vocab_size, 4.0
    g = torch.Generator().manual_seed(31 + B)
    forced = torch.randint(0, V, (B, N_TOK), generator=g).cuda()
    for (k, p, T, ci, explicit) in _pk_matrix():
        noise = torch.empty(N_TOK, B, V).exponential_(1.0, generator=g).cuda() if explicit else None
        sp = engine.make_sampling(T, k, p, sample_logits=True, cfg_scale=cfg_scale, cfg_interval=ci, seed=1234 + k)
        st, _ = _prefill(model, B, True)
        choice, trace = st.generate_forced(sp, forced, trace=True, noise=noise)       # raises unless the persistent kernel runs
        choice = choice.cpu().long()
        what = f"{variant} B={B} top_k={k} top_p={p} T={T} cfg_interval={ci} noise={'explicit' if explicit else 'philox'}"
        for s in range(N_TOK):
            cfg_on = not (ci > -1 and s - 1 > ci)
            idx = engine.sample(trace[s], sp, cfg_on=cfg_on, step=s, noise=None if noise is None else noise[s]).cpu().long()
            assert torch.equal(idx, choice[:, s]), f"{what} step {s}: persistent {choice[:, s].tolist()} vs standalone {idx.tolist()}"
            if explicit:
                z = cfg_temperature(trace[s], B, cfg_scale, cfg_on, T)
                o = oracle_sample(z, k, p, noise=noise[s].cpu())
                for b in range(B):
                    if bool(o.band[b].any()):
                        continue                                   # a nucleus-band token may legitimately go either way
                    assert choice_ok(int(choice[b, s]), o, b), f"{what} step {s} image {b}: {int(choice[b, s])} vs oracle " \
                                                               f"{int(o.choice[b])} (gap {float(o.gap[b]):.2e})"
        # a free-running generate() re-run teacher-forced along its own output returns that output as its choices
        st, _ = _prefill(model, B, True)
        free = st.generate(sp, N_TOK, noise, "cuda")
        st, _ = _prefill(model, B, True)
        again, _ = st.generate_forced(sp, free, trace=False, noise=noise)
        assert torch.equal(again, free), f"{what}: teacher-forced replay of the free-running grid differs"


@pytest.mark.parametrize("explicit", [True, False])
def test_graph_loop_replays_through_car_sample(explicit):
    """B = 9 with CFG (b_eff = 18 > 16: no persistent kernel): the CUDA-graph loop with the fused next-step embedding, the
    device-side position and done_ctr.  Teacher-forcing decode_step along its tokens and replaying each step's logits through
    car_sample reproduces the grid; cfg_interval and top_p are exercised too."""
    from controlar_b200 import engine
    model = _model("plain")
    B, V = 9, SPEC.vocab_size
    g = torch.Generator().manual_seed(41)
    for (k, p, T, ci) in ((2000, 1.0, 1.0, -1), (100, 0.9, 0.7, 3), (0, 0.5, 1.0, 0)):
        noise = torch.empty(N_TOK, B, V).exponential_(1.0, generator=g).cuda() if explicit else None
        sp = engine.make_sampling(T, k, p, sample_logits=True, cfg_scale=4.0, cfg_interval=ci, seed=77)
        st, _ = _prefill(model, B, True)
        grid = st.generate(sp, N_TOK, noise, "cuda").cpu().long()
        st, logits = _prefill(model, B, True)
        for s in range(N_TOK):
            cfg_on = not (ci > -1 and s - 1 > ci)
            idx = engine.sample(logits, sp, cfg_on=cfg_on, step=s, noise=None if noise is None else noise[s]).cpu().long()
            assert torch.equal(idx, grid[:, s]), f"top_k={k} top_p={p} cfg_interval={ci} step {s}: replay {idx.tolist()} vs " \
                                                 f"loop {grid[:, s].tolist()}"
            if s + 1 < N_TOK:
                t = grid[:, s].cuda()
                logits = st.decode_step(torch.cat([t, t]), SPEC.cls_token_num + s)


# ------------------------------------------------------------------------------------------------------------------------------
# distribution of the in-kernel Philox race
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,k,p", [(64, 0, 1.0), (64, 10, 1.0), (64, 0, 0.8), (4096, 100, 1.0), (4096, 0, 0.9)])
def test_philox_race_distribution(V, k, p):
    """~50 000 seeded draws (500 rows x 100 steps) from one distribution: chi-square goodness of fit against the oracle's kept
    distribution, no draw outside the kept set, and no dependence between consecutive steps of a row or between rows."""
    from scipy import stats
    from controlar_b200 import engine
    R, S = 500, 100
    g = torch.Generator().manual_seed(V + k)
    row = torch.randn(1, V, generator=g) * (1.0 if V == 64 else 1.5)
    o = oracle_sample(row, k, p, sample_logits=False)
    prob = o.probs[0].numpy()
    sp = engine.make_sampling(1.0, k, p, sample_logits=True, seed=2024)
    lg = row.repeat(R, 1).cuda()
    draws = torch.stack([engine.sample(lg, sp, step=s) for s in range(S)], dim=1).cpu().numpy()   # [R, S]
    kept = o.kept[0].numpy()
    assert kept[draws].all(), f"{int((~kept[draws]).sum())} draws outside the kept set"
    counts = np.bincount(draws.ravel(), minlength=V).astype(np.float64)
    n = draws.size
    exp = prob * n
    big = exp >= 5
    obs_c = np.append(counts[big], counts[~big].sum())
    exp_c = np.append(exp[big], exp[~big].sum())
    if exp_c[-1] == 0:
        obs_c, exp_c = obs_c[:-1], exp_c[:-1]
    pv = stats.chisquare(obs_c, exp_c).pvalue
    assert pv > 1e-6, f"goodness of fit p = {pv:.2e}"

    def indep(a, b):
        cats = np.argsort(-prob)[:8]                          # the 8 likeliest tokens, the rest pooled
        lut = np.full(V, 8)
        lut[cats] = np.arange(8)
        tab = np.zeros((9, 9))
        np.add.at(tab, (lut[a], lut[b]), 1)
        tab = tab[tab.sum(1) > 0][:, tab.sum(0) > 0]
        return stats.chi2_contingency(tab).pvalue
    pv_step = indep(draws[:, :-1].ravel(), draws[:, 1:].ravel())
    pv_row = indep(draws[:-1].ravel(), draws[1:].ravel())
    assert pv_step > 1e-6 and pv_row > 1e-6, f"dependence: consecutive steps p = {pv_step:.2e}, neighbouring rows p = {pv_row:.2e}"
