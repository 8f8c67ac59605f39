#!/usr/bin/env python
"""Generate tests/golden/train_enc_*.pt by running the REFERENCE ITSELF with its control encoder trainable: the teacher-forced
training forward + backward of autoregressive/models/gpt_t2i.py (HF Dinov2Model adapter) and of the legacy
autoregressive/models/gpt.py (HF ViTModel ViT-S/16 adapter), read-only import from $CONTROLAR_REFERENCE (default ../reference next
to this repository), on the CPU: fp32 master weights under bf16 autocast, math SDPA, dropout p = 0, the condition map cast to bf16
as the train scripts do (train_t2i_canny.py:167).  Run from the repo root:

    python tests/golden/make_train_encoder_golden.py [case ...]

Stored, kept small: loss, the CFG drop decision, a probe (oracle.train_oracle.grad_probe: norm, sum, values at positions drawn from
the key; the tests redraw the positions) of the encoder output `feat` and of the gradient of every encoder tensor, and the names of
every parameter whose .grad is not None after loss.backward().  Weights are procedural (oracle/weights.py), as in make_golden.py.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG     # noqa: E402  (puts the reference and this repository on sys.path)
import torch                 # noqa: E402

from oracle.weights import GPTSpec, make_gpt_state_dict, vit_shapes, _fill   # noqa: E402
from oracle.inputs import text_inputs, class_inputs, control_map, code_inputs, train_attn_mask   # noqa: E402
from oracle.train_oracle import grad_probe   # noqa: E402

N_GRAD, N_FEAT = 128, 4096
ENC = "adapter.model."


def _summary(key, t, n):
    """grad_probe without the positions (the tests redraw them from the key)"""
    pr = grad_probe(key, t, n)
    return {"norm": pr["norm"], "sum": pr["sum"], "val": pr["val"]}


def _probes(m):
    keys = sorted(k for k, p in m.named_parameters() if k.startswith(ENC) and p.grad is not None)
    pg = dict(m.named_parameters())
    per = [_summary(k, pg[k].grad, N_GRAD) for k in keys]
    return {"keys": keys, "norm": torch.stack([x["norm"] for x in per]), "sum": torch.stack([x["sum"] for x in per]),
            "val": torch.nn.utils.rnn.pad_sequence([x["val"] for x in per], batch_first=True)}


def _run(m, name, spec, B, H, W, seed, use_mask, valid, kind, extra):
    m.train()
    N = (H // 16) * (W // 16)
    T = spec.cls_token_num
    if spec.model_type == "t2i":
        cond, masks = text_inputs(T, spec.caption_dim, B, seed + 1, torch.float32)
    else:
        cond, masks = class_inputs(spec.num_classes, B, seed + 1), None
    cmap = control_map(B, H, W, seed + 2, kind, torch.float32)
    z = code_inputs(spec.vocab_size, B, N, seed + 4)
    mask = train_attn_mask(masks, N) if (use_mask and masks is not None) else None
    seen = {}
    orig_drop = m.cls_embedding.token_drop

    def spy_drop(*a, **k):
        out = orig_drop(*a, **k)
        seen["drop_ids"] = out[1].clone()
        return out
    m.cls_embedding.token_drop = spy_drop
    hook = m.adapter.register_forward_hook(lambda mod, inp, out: seen.__setitem__("feat", out.detach().clone()))
    torch.manual_seed(1)
    kw = {} if mask is None else {"mask": mask}
    if valid is not None:
        kw["valid"] = torch.tensor(valid)
    torch.set_grad_enabled(True)
    with torch.autocast("cpu", dtype=torch.bfloat16), MG.math_sdpa():
        _, loss = m(cond_idx=cond, idx=z[:, :-1], targets=z, condition=cmap.to(torch.bfloat16), **kw)
    loss.backward()
    hook.remove()
    out = {"header": {**MG.header(), "generator": "tests/golden/make_train_encoder_golden.py"}, "spec": spec.__dict__, "seed": seed,
           "B": B, "H": H, "W": W, "autocast": "torch.bfloat16", "sdpa": "math", "use_mask": bool(mask is not None), "valid": valid,
           "kind": kind, "inputs": "oracle.inputs: text_inputs/class_inputs(seed+1), control_map(seed+2, kind) cast to bf16, "
                                   "code_inputs(seed+4), train_attn_mask; class_dropout_prob 0.5, torch.manual_seed(1)",
           "drop_ids": seen["drop_ids"], "loss": loss.detach().clone(), "feat": _summary("feat", seen["feat"], N_FEAT),
           "probe_sizes": {"grad": N_GRAD, "feat": N_FEAT}, "enc_grads": _probes(m),
           "params_with_grad": sorted(k for k, p in m.named_parameters() if p.grad is not None), **extra}
    torch.save(out, os.path.join(MG.OUT, name + ".pt"))
    torch.set_grad_enabled(False)
    print(name, "loss %.6f" % float(loss), "drop", seen["drop_ids"].tolist(), "encoder grads", len(out["enc_grads"]["keys"]), flush=True)


def t2i_case(name, spec, B, H, W, use_mask, valid, seed=0):
    m = MG.build_ref_gpt(spec, seed, torch.float32, token_dropout_p=0.0, resid_dropout_p=0.0, ffn_dropout_p=0.0, class_dropout_prob=0.5)
    kind = "canny" if spec.condition_type in ("canny", "seg") else "depth"
    _run(m, name, spec, B, H, W, seed, use_mask, valid, kind, {"class": "autoregressive/models/gpt_t2i.py Transformer"})


def gptpy_case(name, B, H, W, vit_layers=12, seed=0):
    """The legacy class autoregressive/models/gpt.py as train_c2i_canny.py builds it (cls_token_num 1, condition_token_num 0)."""
    from autoregressive.models.gpt import Transformer as RefLegacy, ModelArgs as RefArgs
    spec = GPTSpec(**MG.SMALL, cls_token_num=1, block_size=(H // 16) * (W // 16), model_type="c2i")
    with MG.fake_vit_cwd(vit_layers), contextlib.redirect_stdout(io.StringIO()):
        m = RefLegacy(RefArgs(dim=spec.dim, n_layer=spec.n_layer, n_head=spec.n_head, multiple_of=spec.multiple_of, vocab_size=spec.vocab_size,
                              cls_token_num=1, block_size=spec.block_size, num_classes=spec.num_classes, model_type="c2i",
                              condition_token_num=0, image_size=H, token_dropout_p=0.0, resid_dropout_p=0.0, ffn_dropout_p=0.0,
                              class_dropout_prob=0.5))
    full = dict(make_gpt_state_dict(spec, seed, with_adapter=False))
    full.update(_fill(vit_shapes(384, layers=vit_layers, prefix=ENC), seed, 0.02))
    full["condition_norm.weight"] = torch.ones(spec.dim)
    m.load_state_dict(full, strict=True)
    m = m.float()
    _run(m, name, spec, B, H, W, seed, False, None, "canny",
         {"class": "autoregressive/models/gpt.py Transformer (legacy c2i class)", "vit_layers": vit_layers})


SMALL = MG.SMALL
C2I = dict(SMALL, cls_token_num=1, model_type="c2i")
T2I = dict(SMALL, cls_token_num=120, model_type="t2i")

CASES = {
    "train_enc_dinov2s_canny_c2i_128": lambda: t2i_case("train_enc_dinov2s_canny_c2i_128", GPTSpec(**C2I, block_size=64), 2, 128, 128, False, None),
    "train_enc_dinov2s_canny_c2i_256": lambda: t2i_case("train_enc_dinov2s_canny_c2i_256", GPTSpec(**C2I, block_size=256), 2, 256, 256, False, None),
    "train_enc_dinov2b_depth_t2i_128": lambda: t2i_case("train_enc_dinov2b_depth_t2i_128",
                                                        GPTSpec(**T2I, block_size=64, adapter_size="base", condition_type="depth"),
                                                        2, 128, 128, True, [1, 1]),
    "train_enc_dinov2s_mr_t2i_128x192": lambda: t2i_case("train_enc_dinov2s_mr_t2i_128x192", GPTSpec(**T2I, block_size=144),
                                                         2, 128, 192, True, [1, 0]),
    "train_enc_vit_gptpy_c2i_64": lambda: gptpy_case("train_enc_vit_gptpy_c2i_64", 2, 64, 64),
}

if __name__ == "__main__":
    for c in sys.argv[1:] or list(CASES):
        CASES[c]()
