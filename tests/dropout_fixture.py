"""Inputs and comparisons shared by the CPU and GPU tests of the training path's dropout against the fixtures
tests/golden/train_*_dropout.pt (tests/golden/make_train_dropout_golden.py)."""
import math

import torch

from oracle.weights import GPTSpec
from oracle.inputs import text_inputs, class_inputs, train_attn_mask, code_inputs
from oracle.train_dropout_oracle import control_tokens
from oracle.train_oracle import grad_probe
from tests.helpers import rel_l2

CASES = ["train_t2i_small_ac_dropout", "train_c2i_small_ac_dropout", "train_t2i_mr_ac_dropout", "train_c2i_small_ac_droppath_dropout"]


def inputs(g):
    """(spec, cond, z, mask, valid, feat) the fixture was made with"""
    spec = GPTSpec(**g["spec"])
    B, N = g["B"], (g["H"] // 16) * (g["W"] // 16)
    if spec.model_type == "t2i":
        cond, masks = text_inputs(spec.cls_token_num, spec.caption_dim, B, g["seed"] + 1, torch.float32)
    else:
        cond, masks = class_inputs(spec.num_classes, B, g["seed"] + 1), None
    z = code_inputs(spec.vocab_size, B, N, g["seed"] + 4)
    mask = train_attn_mask(masks, N) if g["use_mask"] else None
    valid = None if g["valid"] is None else torch.tensor(g["valid"])
    feat = control_tokens(B, N, 384 if spec.adapter_size == "small" else 768, g["seed"] + 3)
    return spec, cond, z, mask, valid, feat


def probe_err(key, got, ref, n):
    """relative L2 distance of `got` at the fixture's probe positions of `key`, and of its norm"""
    pm = grad_probe(key, got.detach().float().cpu(), n)
    ev = float((pm["val"] - ref["val"]).norm()) / max(float(ref["val"].norm()), 1e-30)
    en = abs(float(pm["norm"]) - float(ref["norm"])) / float(ref["norm"])
    return ev, en, pm


def grad_rows(g, grads, tol_n, tol_v):
    """(rows, failures) for every parameter gradient: norm within tol_n, probed values within tol_v (the rule of
    tests/test_train_oracle_golden.py: the value error is measured against the probe's norm plus the gradient's RMS per entry)"""
    G, n = g["grads"], g["probe_sizes"]["grad"]
    rows, bad = [], []
    assert sorted(grads) == list(G["keys"]), sorted(set(grads) ^ set(G["keys"]))
    for i, k in enumerate(G["keys"]):
        ref = {"norm": G["norm"][i], "val": G["val"][i]}
        _, en, pm = probe_err(k, grads[k], ref, n)
        nr = float(ref["norm"])
        scale = nr / max(grads[k].numel(), 1) ** 0.5
        ev = float((pm["val"] - ref["val"]).norm()) / (float(ref["val"].norm()) + scale * math.sqrt(n))
        rows.append("%-48s norm %.3e  probe %.3e" % (k, en, ev))
        if not (en <= tol_n and ev <= tol_v):
            bad.append(rows[-1])
    F = g["grads_full"]
    for i, k in enumerate(F["keys"]):
        e = rel_l2(grads[k].float().cpu(), F["grad"][i])
        rows.append("%-48s full %.3e" % (k, e))
        if not e < tol_v:
            bad.append(rows[-1])
    return rows, bad
