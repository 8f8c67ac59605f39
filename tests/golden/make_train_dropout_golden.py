#!/usr/bin/env python
"""Generate tests/golden/train_*_dropout.pt by running the REFERENCE ITSELF in train mode with its dropout layers on: the
teacher-forced training forward + backward of autoregressive/models/gpt_t2i.py (read-only import from $CONTROLAR_REFERENCE,
default ../reference next to this repository) on the CPU, fp32 master weights under bf16 autocast, as
tests/golden/make_golden.py::train_case runs it at p = 0.  Run from the repo root:

    python tests/golden/make_train_dropout_golden.py [case ...]

torch's own dropout bit stream cannot be reproduced elsewhere, so the reference's `tok_dropout`, every block's `resid_dropout` /
`ffn_dropout` and every `DropPath` are replaced by stand-ins that draw their keep decisions from oracle/dropout_masks.py (the
library's generator) and apply them with the rounding of torch's CUDA kernels.  Everything else — which tensor each module
receives, in which order, the prefix rows inside tok_dropout's input and the control adds after it — is the reference's graph.
The control encoder is replaced by procedural tokens (oracle.train_dropout_oracle.control_tokens: it has its own parity tests), so
the fixtures need not carry its output.  Stored, kept small: loss, the CFG drop decision, the dropout settings and seed, and
summaries (norm, sum, values at the positions oracle.train_oracle.grad_probe draws for the key) of the logits, of every parameter
gradient and of d loss / d control tokens; the first block's and the final norm weights' gradients in full.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as MG     # noqa: E402  (puts the reference and this repository on sys.path)
import torch                 # noqa: E402

from oracle import dropout_masks as DM                      # noqa: E402
from oracle.weights import GPTSpec                          # noqa: E402
from oracle.inputs import text_inputs, class_inputs, train_attn_mask, code_inputs   # noqa: E402
from oracle.train_oracle import grad_probe                  # noqa: E402
from oracle.train_dropout_oracle import control_tokens      # noqa: E402

N_LOGITS, N_GRAD, N_FEAT = 4096, 128, 1024                  # probe sizes


def summary(key, t, n):
    """grad_probe without the positions (the tests redraw them from the key)"""
    pr = grad_probe(key, t, n)
    return {"norm": pr["norm"], "sum": pr["sum"], "val": pr["val"]}


class Tokens(torch.nn.Module):
    """stand-in for the control encoder: returns the procedural tokens as a leaf whose gradient is kept"""

    def __init__(self, feat):
        super().__init__()
        self.feat = feat

    def forward(self, condition):
        return self.feat


class ElemDropout(torch.nn.Module):
    """nn.Dropout(p) in train mode with the generator's mask for (site, layer)"""

    def __init__(self, seed, site, layer, p):
        super().__init__()
        self.seed, self.site, self.layer, self.p = seed, site, layer, p

    def forward(self, x):
        B, S, d = x.shape
        return DM.apply_dropout(x, DM.keep_mask(self.seed, self.site, self.layer, B, S, d, self.p), self.p)


class PathDropout(torch.nn.Module):
    """DropPath(rate) of one block: TransformerBlock.forward calls it on the attention branch, then on the feed-forward branch"""

    def __init__(self, seed, layer, rate, log):
        super().__init__()
        self.seed, self.layer, self.rate, self.calls, self.log = seed, layer, rate, 0, log

    def forward(self, x):
        site = DM.PATH_ATTN if self.calls % 2 == 0 else DM.PATH_FFN
        self.calls += 1
        keep = DM.path_keep(self.seed, site, self.layer, x.shape[0], self.rate)
        self.log.append((site, self.layer, keep.clone()))
        return DM.apply_drop_path(x, keep, self.rate)


def dropout_case(name: str, spec: GPTSpec, B: int, H: int, W: int, use_mask: bool, valid, dseed: int, p: float = 0.0,
                 token_p: float = 0.0, drop_path_rate: float = 0.0, seed: int = 0, drop_prob: float = 0.5, rand_seed: int = 1):
    torch.set_grad_enabled(True)
    autocast = torch.bfloat16
    m = MG.build_ref_gpt(spec, seed, torch.float32, token_dropout_p=token_p, resid_dropout_p=p, ffn_dropout_p=p,
                         drop_path_rate=drop_path_rate, class_dropout_prob=drop_prob)
    m.train()
    rates = DM.drop_path_rates(drop_path_rate, spec.n_layer) if drop_path_rate > 0 else None
    path_log = []
    N = (H // 16) * (W // 16)
    feat = control_tokens(B, N, m.adapter_mlp.fc1.weight.shape[1], seed + 3).requires_grad_(True)
    m.adapter = Tokens(feat)
    m.tok_dropout = ElemDropout(dseed, DM.TOKEN, 0, token_p)
    for i, layer in enumerate(m.layers):
        layer.attention.resid_dropout = ElemDropout(dseed, DM.RESID, i, p)
        layer.feed_forward.ffn_dropout = ElemDropout(dseed, DM.FFN, i, p)
        if rates is not None and rates[i] > 0:
            assert abs(layer.drop_path.drop_prob - rates[i]) == 0.0, (i, layer.drop_path.drop_prob, rates[i])
            layer.drop_path = PathDropout(dseed, i, rates[i], path_log)
        else:
            assert isinstance(layer.drop_path, torch.nn.Identity)
    T = spec.cls_token_num
    if spec.model_type == "t2i":
        cond, masks = text_inputs(T, spec.caption_dim, B, seed + 1, torch.float32)
    else:
        cond, masks = class_inputs(spec.num_classes, B, seed + 1), None
    z = code_inputs(spec.vocab_size, B, N, seed + 4)
    mask = train_attn_mask(masks, N) if (use_mask and masks is not None) else None
    seen = {}
    orig_drop = m.cls_embedding.token_drop

    def spy_drop(*a, **k):
        out = orig_drop(*a, **k)
        seen["drop_ids"] = out[1].clone()
        return out
    m.cls_embedding.token_drop = spy_drop
    torch.manual_seed(rand_seed)
    kw = {} if mask is None else {"mask": mask}
    if valid is not None:
        kw["valid"] = torch.tensor(valid)
    with torch.autocast("cpu", dtype=autocast), MG.math_sdpa():
        logits, loss = m(cond_idx=cond, idx=z[:, :-1], targets=z, condition=torch.zeros(B, 3, H, W, dtype=autocast), **kw)
    loss.backward()
    dropped_paths = sum(int((~k).sum()) for _, _, k in path_log)
    if rates is not None:
        assert dropped_paths > 0, "choose a seed that drops at least one (sample, layer) branch"
    keys = sorted(k for k, q in m.named_parameters() if q.grad is not None)
    pg = dict(m.named_parameters())
    per = [summary(k, pg[k].grad, N_GRAD) for k in keys]
    grads = {"keys": keys, "norm": torch.stack([x["norm"] for x in per]), "sum": torch.stack([x["sum"] for x in per]),
             "val": torch.stack([x["val"] for x in per])}                    # one tensor per field keeps the file small
    full_keys = [k for k in keys if k.endswith("norm.weight") and ("layers.0." in k or k == "norm.weight")]
    small = {"keys": full_keys, "grad": torch.stack([pg[k].grad for k in full_keys])}
    out = {"header": {**MG.header(), "generator": "tests/golden/make_train_dropout_golden.py"}, "spec": spec.__dict__, "seed": seed,
           "B": B, "H": H, "W": W, "autocast": str(autocast), "sdpa": "math", "use_mask": bool(mask is not None), "valid": valid,
           "dropout": {"seed": dseed, "token_p": token_p, "resid_p": p, "ffn_p": p, "drop_path": rates},
           "dropped_paths": dropped_paths,
           "inputs": "oracle.inputs: text_inputs/class_inputs(seed+1), code_inputs(seed+4), train_attn_mask; control_tokens(seed+3); "
                     "class_dropout_prob = %g, torch.manual_seed(%d)" % (drop_prob, rand_seed),
           "probe_sizes": {"logits": N_LOGITS, "grad": N_GRAD, "feat": N_FEAT},
           "drop_ids": seen["drop_ids"], "feat_grad": summary("feat", feat.grad, N_FEAT),
           "logits": summary("logits", logits.detach().to(autocast).float(), N_LOGITS), "loss": loss.detach().clone(),
           "grads": grads, "grads_full": small}
    torch.save(out, os.path.join(MG.OUT, name + ".pt"))
    torch.set_grad_enabled(False)
    print(name, "loss %.6f" % float(loss), "drop", seen["drop_ids"].tolist(), "dropped paths", dropped_paths, flush=True)


SMALL = MG.SMALL
T2I = dict(SMALL, cls_token_num=120, block_size=64, model_type="t2i")
C2I = dict(SMALL, cls_token_num=1, block_size=64, model_type="c2i")
MR = dict(SMALL, cls_token_num=120, block_size=144, model_type="t2i", condition_type="depth")

CASES = {
    "train_t2i_small_ac_dropout": lambda: dropout_case("train_t2i_small_ac_dropout", GPTSpec(**T2I), B=3, H=128, W=128, use_mask=True,
                                                       valid=[1, 0, 1], dseed=0x5EED0001, p=0.1, token_p=0.1),
    "train_c2i_small_ac_dropout": lambda: dropout_case("train_c2i_small_ac_dropout", GPTSpec(**C2I), B=4, H=128, W=128, use_mask=False,
                                                       valid=None, dseed=0x5EED0002, p=0.1, token_p=0.1),
    "train_t2i_mr_ac_dropout": lambda: dropout_case("train_t2i_mr_ac_dropout", GPTSpec(**MR), B=2, H=128, W=192, use_mask=True,
                                                    valid=[1, 1], dseed=0x5EED0003, p=0.1, token_p=0.1),
    # the c2i scripts' --drop-path-rate recipe: stochastic depth instead of dropout (train_c2i_canny.py:98-112)
    "train_c2i_small_ac_droppath_dropout": lambda: dropout_case("train_c2i_small_ac_droppath_dropout", GPTSpec(**C2I), B=4, H=128, W=128,
                                                                use_mask=False, valid=None, dseed=0x5EED0004, drop_path_rate=0.5),
}

if __name__ == "__main__":
    for c in sys.argv[1:] or list(CASES):
        CASES[c]()
