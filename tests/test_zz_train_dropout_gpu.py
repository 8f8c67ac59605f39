"""GPU: dropout in the training forward and backward (token / residual / feed-forward dropout and drop path,
controlar_b200/csrc/dropout.cuh).  The generator against its CPU restatement bit for bit, the rounding rules against torch's own CUDA
dropout, the library's loss and gradients against autograd over the oracle with the same masks (and against the reference's
gradient probes, tests/golden/train_*_dropout.pt), reproducibility, and the reference's training recipe with ModelArgs defaults."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import dropout_masks as DM
from oracle.weights import GPTSpec, make_gpt_state_dict
from oracle.train_dropout_oracle import DropoutTrainOracle
from oracle.inputs import text_inputs, class_inputs, train_attn_mask, code_inputs
from tests import dropout_fixture as DF
from tests.helpers import log_measurement, load_golden, rel_l2

pytestmark = pytest.mark.gpu


def _seed_tensor(seed):
    return torch.tensor([int(seed) & 0xFFFFFFFFFFFFFFFF], dtype=torch.uint64).view(torch.int64).cuda()


def _build(spec, seed, dropout):
    from controlar_b200.autoregressive.models.gpt_t2i import Transformer, ModelArgs
    d = dropout or {}
    rates = d.get("drop_path")
    m = Transformer(ModelArgs(dim=spec.dim, n_layer=spec.n_layer, n_head=spec.n_head, multiple_of=spec.multiple_of,
                              vocab_size=spec.vocab_size, cls_token_num=spec.cls_token_num, block_size=spec.block_size,
                              caption_dim=spec.caption_dim, num_classes=spec.num_classes, model_type=spec.model_type,
                              adapter_size=spec.adapter_size, condition_type=spec.condition_type,
                              token_dropout_p=d.get("token_p", 0.0), resid_dropout_p=d.get("resid_p", 0.0),
                              ffn_dropout_p=d.get("ffn_p", 0.0), drop_path_rate=rates[-1] if rates else 0.0, class_dropout_prob=0.5))
    m.load_state_dict(make_gpt_state_dict(spec, seed), strict=True)
    return m.to("cuda").train()


def _inputs(g, spec):
    B, N = g["B"], (g["H"] // 16) * (g["W"] // 16)
    if spec.model_type == "t2i":
        cond, masks = text_inputs(spec.cls_token_num, spec.caption_dim, B, g["seed"] + 1, torch.float32)
    else:
        cond, masks = class_inputs(spec.num_classes, B, g["seed"] + 1), None
    z = code_inputs(spec.vocab_size, B, N, g["seed"] + 4)
    mask = train_attn_mask(masks, N) if g["use_mask"] else None
    valid = None if g["valid"] is None else torch.tensor(g["valid"])
    return cond, z, mask, valid


def _step(m, g, cond, z, mask, valid, feat_src):
    with torch.enable_grad():
        feat = feat_src.cuda().clone().requires_grad_(True)
        m.adapter.forward = lambda x: feat
        logits, loss = m(idx=z[:, :-1].cuda(), cond_idx=cond.cuda(), targets=z.cuda(), mask=None if mask is None else mask.cuda(),
                         valid=None if valid is None else valid.cuda(), condition=torch.zeros(g["B"], 3, g["H"], g["W"], device="cuda"))
        loss.backward()
    torch.cuda.synchronize()
    return feat, loss


def _run_cuda(g, dropout, seed=None):
    spec, cond, z, mask, valid, feat0 = DF.inputs(g)
    m = _build(spec, g["seed"], dropout)
    m._force_drop_ids = g["drop_ids"]
    if seed is not None:
        m._force_dropout_seed = seed
    with torch.enable_grad():
        feat = feat0.cuda().requires_grad_(True)
        m.adapter.forward = lambda x: feat
        logits, loss = m(idx=z[:, :-1].cuda(), cond_idx=cond.cuda(), targets=z.cuda(), mask=None if mask is None else mask.cuda(),
                         valid=None if valid is None else valid.cuda(), condition=torch.zeros(g["B"], 3, g["H"], g["W"], device="cuda"))
        loss.backward()
    torch.cuda.synchronize()
    return m, feat, logits.detach(), float(loss)


def _dense_grads(m):
    return {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None and "embedding" not in k}


# ---- 1. the generator ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["train_t2i_small_ac", "train_c2i_small_ac", "train_t2i_mr_ac"])
def test_keep_mask_matches_cpu_restatement(name):
    from controlar_b200 import _lib
    lib = _lib.lib()
    g = load_golden(name)
    spec = GPTSpec(**g["spec"])
    B, S, d = g["B"], spec.cls_token_num + (g["H"] // 16) * (g["W"] // 16) - 1, spec.dim
    for seed in (0, 0x5EED0001, 0xFEDCBA9876543210):
        sd = _seed_tensor(seed)
        for site, layer, p in [(DM.TOKEN, 0, 0.1), (DM.RESID, 0, 0.1), (DM.RESID, spec.n_layer - 1, 0.5), (DM.FFN, 3, 0.1),
                               (DM.PATH_ATTN, 2, 0.3), (DM.PATH_FFN, 5, 0.5)]:
            out = torch.empty(B, S, d, dtype=torch.uint8, device="cuda")
            rc = lib.car_dropout_keep_mask(sd.data_ptr(), site, layer, B, S, d, C.c_float(p), out.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream)
            assert rc == 0, lib.car_last_error()
            torch.cuda.synchronize()
            want = DM.keep_mask(seed, site, layer, B, S, d, p)
            assert torch.equal(out.cpu().bool(), want), (seed, site, layer)


# ---- 2. rounding rules -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("p", [0.1, 0.3])
def test_torch_cuda_dropout_scales_in_fp32_and_rounds_once(dtype, p):
    x = (torch.randn(1 << 16, generator=torch.Generator().manual_seed(3)) * 3).to(dtype).cuda()
    y = F.dropout(x, p, training=True)
    kept = y != 0
    assert 0.5 < float(kept.float().mean()) < 1.0
    want = (x.float() * DM.elem_scale(p)).to(dtype)
    assert torch.equal(y[kept], want[kept])
    assert torch.equal(DM.apply_dropout(x.cpu(), kept.cpu(), p).cuda()[kept], y[kept])


def test_drop_path_multiplier_is_bf16_of_inverse_keep():
    for rate in (0.1, 0.25, 0.5, DM.drop_path_rates(0.1, 24)[7]):
        keep = 1 - rate
        rt = torch.ones(4, 1, 1, dtype=torch.bfloat16, device="cuda").div_(keep)         # utils/drop_path.py on a kept sample
        assert float(rt[0]) == DM.path_mult(rate), rate
    assert DM.path_mult(0.1) == 1.109375


# ---- 3. forward and backward against autograd over the oracle and the reference's own probes ---------------------------------
@pytest.mark.parametrize("name", DF.CASES)
def test_dropout_train_step_vs_autograd_oracle(name):
    g = load_golden(name)
    dr = g["dropout"]
    spec, cond, z, mask, valid, feat0 = DF.inputs(g)
    orc = DropoutTrainOracle(spec, make_gpt_state_dict(spec, g["seed"]), torch.bfloat16)
    ofeat = feat0.clone().requires_grad_(True)
    with torch.enable_grad():
        _, oloss = orc.forward(z[:, :-1], cond, ofeat, g["drop_ids"], mask, z, valid, dropout=dr)
        oloss.backward()
    ref = {k: p.grad for k, p in orc.p.items() if p.grad is not None}
    if dr["drop_path"]:
        assert g["dropped_paths"] > 0
    m, feat, logits, loss = _run_cuda(g, dr, seed=dr["seed"])
    n = g["probe_sizes"]
    el, _, _ = DF.probe_err("logits", logits, g["logits"], n["logits"])
    rows, bad = ["loss %.6f oracle %.6f reference %.6f  logits-vs-reference %.3e" % (loss, float(oloss), float(g["loss"]), el)], []
    if not (abs(loss - float(oloss)) < 2e-3 * float(oloss) and el < 1e-2):
        bad.append(rows[0])
    got = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert set(got) == set(ref), sorted(set(got) ^ set(ref))
    for k in sorted(ref):                                             # every gradient against autograd over the oracle
        e = rel_l2(got[k].float().cpu(), ref[k])
        rows.append("%-48s rel_l2 %.3e" % (k, e))
        if not e < 3e-2:
            bad.append(rows[-1])
    prow, pbad = DF.grad_rows(g, got, 2e-2, 3e-2)                     # and the reference's probes of it
    ef = rel_l2(feat.grad.float().cpu(), ofeat.grad.float())
    er, _, _ = DF.probe_err("feat", feat.grad, g["feat_grad"], n["feat"])
    rows += prow + ["%-48s rel_l2 %.3e  probe-vs-reference %.3e" % ("d loss / d feat", ef, er)]
    bad += pbad
    if not (ef < 3e-2 and er < 3e-2):
        bad.append(rows[-1])
    log_measurement("train_dropout_%s.txt" % name, "\n".join(rows) + "\n", mode="w")
    assert not bad, "\n" + "\n".join(bad)


# ---- 4. reproducibility ----------------------------------------------------------------------------------------------------
def test_seeded_steps_reproduce_and_consecutive_steps_differ():
    g = load_golden("train_c2i_small_ac_dropout")
    spec, cond, z, mask, valid, feat0 = DF.inputs(g)
    dr = dict(g["dropout"], drop_path=DM.drop_path_rates(0.2, spec.n_layer))
    runs = []
    for _ in range(2):
        m = _build(spec, g["seed"], dr)
        torch.manual_seed(1234)
        f, l1 = _step(m, g, cond, z, mask, valid, feat0)
        runs.append((float(l1), _dense_grads(m), f.grad.clone()))
        for p in m.parameters():
            p.grad = None
        _, l2 = _step(m, g, cond, z, mask, valid, feat0)              # no reseed: fresh masks (and CFG draw)
        assert float(l2) != float(l1)
    (la, ga, fa), (lb, gb, fb) = runs
    assert la == lb
    assert torch.equal(fa, fb)
    for k in ga:
        assert torch.equal(ga[k], gb[k]), k


def test_all_sites_off_is_the_dropout_free_path_bit_for_bit():
    """p = 0 everywhere: no seed is drawn (the CUDA generator is left where the dropout-free path leaves it), and handing the
    library an explicit all-off setting with a seed changes nothing either."""
    from controlar_b200.engine import ARTrainHandle
    g = load_golden("train_t2i_small_ac")
    spec = GPTSpec(**g["spec"])
    cond, z, mask, valid = _inputs(g, spec)
    m = _build(spec, g["seed"], None)
    m._force_drop_ids = g["drop_ids"]
    st0 = torch.cuda.get_rng_state()
    f0, l0 = _step(m, g, cond, z, mask, valid, g["feat"])
    assert torch.equal(torch.cuda.get_rng_state(), st0)
    g0 = _dense_grads(m)
    h = m._car_train
    args = (z[:, :-1].cuda(), cond.cuda(), g["feat"].cuda(), g["drop_ids"].cuda(), mask.cuda(), z.cuda(), valid.cuda())
    lg_a, la = h.forward(*args)
    lg_b, lb = h.forward(*args, dropout=(0.0, 0.0, 0.0, [0.0] * spec.n_layer, _seed_tensor(5)))
    torch.cuda.synchronize()
    assert torch.equal(lg_a, lg_b) and float(la) == float(lb) == float(l0)
    G, _ = h.backward(m)
    for k in g0:
        assert torch.equal(G[k], g0[k]), k
    assert isinstance(h, ARTrainHandle)


# ---- 5. the reference's recipe with ModelArgs defaults --------------------------------------------------------------------
@pytest.mark.parametrize("cls", ["gpt_t2i", "gpt"])
def test_reference_recipe_with_default_dropout(cls):
    import importlib
    from controlar_b200.optim import AdamW
    mod = importlib.import_module("controlar_b200.autoregressive.models." + cls)
    if cls == "gpt_t2i":
        m = mod.GPT_models["GPT-B"](vocab_size=4096, block_size=64, cls_token_num=120, model_type="t2i")
    else:
        m = mod.GPT_models["GPT-B"](vocab_size=4096, block_size=64, num_classes=10, cls_token_num=1, model_type="c2i",
                                    condition_token_num=0, image_size=128)
    cfg = m.config
    assert (cfg.token_dropout_p, cfg.resid_dropout_p, cfg.ffn_dropout_p, cfg.attn_dropout_p) == (0.1, 0.1, 0.1, 0.0)
    torch.nn.init.normal_(m.output.weight, std=0.02)
    m = m.cuda().train()
    B, n = 2, 64
    gen = torch.Generator().manual_seed(11)
    z = torch.randint(0, 4096, (B, n), generator=gen).cuda()
    cond = (torch.randn(B, 120, cfg.caption_dim, generator=gen) * 0.5).cuda() if cls == "gpt_t2i" else torch.tensor([3, 7]).cuda()
    feat = (torch.randn(B, n, m.adapter_mlp.fc1.weight.shape[1], generator=gen) * 0.5).to(torch.bfloat16).cuda()
    m.adapter.forward = lambda x: feat
    cmap = torch.zeros(B, 3, 128, 128, device="cuda")
    trained = [p for _, p in __import__("controlar_b200.engine", fromlist=["x"]).ARTrainHandle.grad_params(m)]
    opt = AdamW(trained, lr=1e-4, betas=(0.9, 0.95), weight_decay=0.05)

    def loss_at(seed, backward):
        torch.manual_seed(seed)
        with torch.enable_grad():
            _, loss = m(cond_idx=cond, idx=z[:, :-1], targets=z, condition=cmap)
            if backward:
                loss.backward()
        return float(loss)
    l0 = loss_at(21, True)
    assert m.output.weight.grad is not None and m.layers[0].attention.wqkv.weight.grad.norm() > 0
    opt.step()
    opt.zero_grad(set_to_none=True)
    with torch.no_grad():
        l1 = loss_at(21, False)
    assert l1 < l0, (l0, l1)
    if cls == "gpt_t2i":
        m2 = mod.GPT_models["GPT-B"](vocab_size=4096, block_size=64, cls_token_num=120, model_type="t2i", attn_dropout_p=0.1)
    else:
        m2 = mod.GPT_models["GPT-B"](vocab_size=4096, block_size=64, num_classes=10, cls_token_num=1, model_type="c2i",
                                     condition_token_num=0, image_size=128, attn_dropout_p=0.1)
    m2 = m2.cuda().train()
    with pytest.raises(NotImplementedError):
        m2(cond_idx=cond, idx=z[:, :-1], targets=z, condition=cmap)


def test_dropout_keeps_valid_semantics_and_is_fixed_at_construction():
    """With dropout on, a valid = 0 sample still contributes nothing; the probabilities are those the model was built with
    (the reference builds its dropout layers from ModelArgs once), so editing model.config afterwards is refused, and
    attention-probability dropout is refused at any time."""
    g = load_golden("train_t2i_small_ac")
    spec = GPTSpec(**g["spec"])
    m = _build(spec, g["seed"], {"resid_p": 0.1, "ffn_p": 0.1, "token_p": 0.1})
    B, N = g["B"], 64
    cond, masks = text_inputs(spec.cls_token_num, spec.caption_dim, B, g["seed"] + 1, torch.float32)
    z = code_inputs(spec.vocab_size, B, N, g["seed"] + 4).cuda()
    mask = train_attn_mask(masks, N).cuda()
    feat = g["feat"].cuda()
    m.adapter.forward = lambda x: feat
    m._force_drop_ids = torch.zeros(B, dtype=torch.bool)
    m._force_dropout_seed = 77
    cmap = torch.zeros(B, 3, 128, 128, device="cuda")
    valid = torch.tensor([1, 0, 1]).cuda()
    z2 = z.clone(); z2[1] = (z2[1] + 7) % spec.vocab_size
    _, l0 = m(idx=z[:, :-1], cond_idx=cond.cuda(), targets=z, mask=mask, valid=valid, condition=cmap)
    _, l1 = m(idx=z2[:, :-1], cond_idx=cond.cuda(), targets=z2, mask=mask, valid=valid, condition=cmap)
    assert float(l0) == float(l1)
    m.config.resid_dropout_p = 0.2
    with pytest.raises(NotImplementedError):
        m(idx=z[:, :-1], cond_idx=cond.cuda(), targets=z, mask=mask, valid=valid, condition=cmap)
    m.config.resid_dropout_p = 0.1
    _, l2 = m(idx=z[:, :-1], cond_idx=cond.cuda(), targets=z, mask=mask, valid=valid, condition=cmap)
    assert float(l2) == float(l0)
