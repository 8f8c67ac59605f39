"""GPU: the trainable control encoder (car_dino_train_*, csrc/dino_train.cuh) behind `loss.backward()` of the drop-in modules —
gpt_t2i with DINOv2 (small / base, canny / depth, square / non-square) and the legacy gpt.py with ViT-S/16 — against autograd over
oracle/train_encoder_oracle.py + oracle/train_oracle.py on the same inputs, and against the reference's own probes
(tests/golden/train_enc_*.pt).
Bars: per-tensor rel-L2 of every encoder gradient against the oracle <= 3e-2, the transformer backward's bar (both sides round at
the same places; fp32 summation order inside GEMMs, attention and column sums differs).  The key bias is compared in absolute
terms: softmax is invariant to it, its gradient is zero up to rounding on both sides.  Probes against the reference: <= 6e-2,
the oracle's own measured gap to the reference (<= 3.1e-2, tests/test_train_encoder_cpu.py) plus the bar above."""
import pytest
import torch

from oracle.train_oracle import TrainOracle
from oracle.train_encoder_oracle import encoder_forward, encoder_params
from tests.helpers import load_golden, log_measurement, rel_l2
from tests.test_train_encoder_cpu import CASES, case_setup, probe_gap

pytestmark = pytest.mark.gpu
GRAD_BAR, PROBE_BAR, FEAT_BAR = 3e-2, 6e-2, 1e-2
ENC = "adapter.model."


def _model(g, spec, sd, vit):
    if vit:
        from controlar_b200.autoregressive.models.gpt import Transformer, ModelArgs
        from controlar_b200.autoregressive.models.vit_adapter import ViT_Adapter
        m = Transformer(ModelArgs(dim=spec.dim, n_layer=spec.n_layer, n_head=spec.n_head, multiple_of=spec.multiple_of,
                                  vocab_size=spec.vocab_size, cls_token_num=1, block_size=spec.block_size, num_classes=spec.num_classes,
                                  model_type="c2i", condition_token_num=0, image_size=g["H"], token_dropout_p=0.0, resid_dropout_p=0.0,
                                  ffn_dropout_p=0.0, class_dropout_prob=0.5))
        m.adapter = ViT_Adapter(layers=g["vit_layers"])
    else:
        from controlar_b200.autoregressive.models.gpt_t2i import Transformer, ModelArgs
        m = Transformer(ModelArgs(dim=spec.dim, n_layer=spec.n_layer, n_head=spec.n_head, multiple_of=spec.multiple_of,
                                  vocab_size=spec.vocab_size, cls_token_num=spec.cls_token_num, block_size=spec.block_size,
                                  caption_dim=spec.caption_dim, num_classes=spec.num_classes, model_type=spec.model_type,
                                  adapter_size=spec.adapter_size, condition_type=spec.condition_type, token_dropout_p=0.0,
                                  resid_dropout_p=0.0, ffn_dropout_p=0.0, class_dropout_prob=0.5))
    m.load_state_dict(sd, strict=True)
    m = m.to("cuda").train()
    m._force_drop_ids = g["drop_ids"]
    return m


def _step(m, inputs):
    cond, cmap, z, mask, valid = inputs
    with torch.enable_grad():
        _, loss = m(idx=z[:, :-1].cuda(), cond_idx=cond.cuda(), targets=z.cuda(), mask=None if mask is None else mask.cuda(),
                    valid=None if valid is None else valid.cuda(), condition=cmap.cuda())
        loss.backward()
    torch.cuda.synchronize()
    return float(loss)


def _oracle(g, spec, sd, vit, inputs):
    cond, cmap, z, mask, valid = inputs
    p = encoder_params(sd)
    if vit:
        sd = dict(sd, **{"condition_mlp.uncond_embedding": torch.zeros_like(sd["condition_mlp.uncond_embedding"])})
    heads = p["layernorm.weight"].shape[0] // 64
    with torch.enable_grad():
        feat = encoder_forward(p, cmap, vit, spec.condition_type, heads, 1e-12 if vit else 1e-6)
        _, loss = TrainOracle(spec, sd, torch.bfloat16).forward(z[:, :-1], cond, feat, g["drop_ids"], mask, z, valid)
        loss.backward()
    return feat.detach(), float(loss.detach()), {ENC + k: t.grad for k, t in p.items()}


@pytest.mark.parametrize("name", CASES)
def test_encoder_gradients_vs_oracle_and_reference(name):
    g = load_golden(name)
    spec, sd, vit, inputs = case_setup(g)
    m = _model(g, spec, sd, vit)
    loss = _step(m, inputs)
    ofeat, oloss, ref = _oracle(g, spec, sd, vit, inputs)
    assert abs(loss - oloss) < 2e-3 * oloss
    got = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    # the set of parameters with a gradient is the reference's
    assert sorted(got) == sorted(g["params_with_grad"]), sorted(set(got) ^ set(g["params_with_grad"]))
    rows, bad = [], []
    eg = g["enc_grads"]
    for i, k in enumerate(eg["keys"]):
        a = got[k].float().cpu()
        if k.endswith("key.bias"):
            kw = float(ref[k.replace("key.bias", "key.weight")].norm())
            e = float(a.norm()) / kw
            if e > 1e-2:
                bad.append((k, e))
            continue
        e = rel_l2(a, ref[k])
        ep = probe_gap(k, a, {"val": eg["val"][i], "norm": eg["norm"][i]}, g["probe_sizes"]["grad"])
        rows.append((e, ep, k))
        if e > GRAD_BAR or ep > PROBE_BAR:
            bad.append((k, e, ep))
    rows.sort(reverse=True)
    log_measurement("train_encoder_gpu.txt", f"{name}: loss {loss:.6f} vs oracle {oloss:.6f}; worst rel-L2 vs oracle / probe vs reference: "
                    + "; ".join(f"{k} {e:.2e} {ep:.2e}" for e, ep, k in rows[:4]) + "\n")
    assert not bad, bad[:8]
    # feat: the trainable forward against the oracle
    with torch.enable_grad():
        feat = m.adapter(inputs[1].cuda())
    assert feat.requires_grad and feat.dtype == torch.float32
    assert rel_l2(feat.detach().cpu(), ofeat) < FEAT_BAR


def test_two_identical_steps_give_bit_identical_gradients():
    g = load_golden("train_enc_dinov2s_mr_t2i_128x192")
    spec, sd, vit, inputs = case_setup(g)
    m = _model(g, spec, sd, vit)
    _step(m, inputs)
    first = {k: p.grad.clone() for k, p in m.named_parameters() if k.startswith(ENC) and p.grad is not None}
    for p in m.parameters():
        p.grad = None
    _step(m, inputs)
    for k, t in first.items():
        assert torch.equal(t, dict(m.named_parameters())[k].grad), k


@pytest.mark.parametrize("name", ["train_enc_dinov2s_canny_c2i_128", "train_enc_dinov2b_depth_t2i_128", "train_enc_vit_gptpy_c2i_64"])
def test_frozen_encoder_is_the_inference_encoder(name):
    """requires_grad off (or no_grad / eval) keeps today's inference encoder, bit for bit"""
    g = load_golden(name)
    spec, sd, vit, inputs = case_setup(g)
    m = _model(g, spec, sd, vit)
    x = inputs[1].cuda()
    with torch.no_grad():
        want = m.adapter(x)
    for p in m.adapter.parameters():
        p.requires_grad_(False)
    with torch.enable_grad():
        frozen = m.adapter(x)
    assert not frozen.requires_grad and torch.equal(frozen, want)
    assert getattr(m.adapter, "_car_dino_train", None) is None
    _step(m, inputs)                                            # a training step with the encoder frozen leaves it without grads
    assert all(p.grad is None for p in m.adapter.parameters())


def test_reference_style_step_updates_the_encoder():
    """One train-script step (train_t2i_canny.py: AdamW over model.parameters(), autocast forward, loss.backward(), step) changes the
    encoder's weights, and the next forward runs on the new values (the handle re-casts its borrowed masters)."""
    g = load_golden("train_enc_dinov2s_canny_c2i_128")
    spec, sd, vit, inputs = case_setup(g)
    m = _model(g, spec, sd, vit)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3, weight_decay=0.05, betas=(0.9, 0.95))
    x = inputs[1].cuda()
    with torch.no_grad():
        before_inf = m.adapter(x).clone()
    w0 = m.adapter.model.encoder.layer[0].mlp.fc1.weight.detach().clone()
    h0 = None
    for _ in range(2):
        opt.zero_grad(set_to_none=True)
        _step(m, inputs)
        h0 = h0 or m.adapter._car_dino_train
        opt.step()
    assert m.adapter._car_dino_train is h0                    # an optimizer step does not rebuild the handle
    assert not torch.equal(w0, m.adapter.model.encoder.layer[0].mlp.fc1.weight.detach())
    # the trainable forward after the steps equals the oracle on the stepped weights
    p = {k[len("model."):]: t.detach().cpu().float() for k, t in m.adapter.state_dict().items() if not k.startswith("model.embeddings.mask")}
    want = encoder_forward(p, inputs[1], False, spec.condition_type, 6, 1e-6)
    with torch.enable_grad():
        feat = m.adapter(x)
    assert rel_l2(feat.detach().cpu(), want) < FEAT_BAR
    with torch.no_grad():
        after_inf = m.adapter(x)
    assert not torch.equal(before_inf, after_inf)
