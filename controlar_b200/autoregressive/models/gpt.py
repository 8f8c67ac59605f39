"""Drop-in for the reference ``autoregressive/models/gpt.py`` — the LEGACY class-conditional model (``sample_c2i.py``,
``train_c2i_*.py`` import it): ViT-S/16 control encoder (vit_adapter.py), ``adapter_mlp`` 384 -> d, ``condition_mlp``,
three ``condition_layers`` applied to the control token of the current position at layers 0, L/3, 2L/3 (gpt.py:444-448),
no ``control_strength``.

Its inference arithmetic is the ``gpt_t2i`` chain with T = cls_token_num = 1 and strength 1 (the per-step
``condition_layers[j](condition_token[:, pos])`` equals the row of the MLP applied to all positions once) — pinned on the CPU
by tests/golden/c2i_gptpy_bf16.pt, produced by running the reference's gpt.py — so this module is a thin shell over
``gpt_t2i.Transformer`` with gpt.py's constructor surface, state-dict keys (``adapter.model.*`` = HF ViT keys,
``condition_norm.weight``) and ``forward`` signature.  Differences kept on purpose: CFG works here (the reference raises
TypeError for gpt.py + cfg_scale > 1, generate.py:87 vs gpt.py:400-409); fp32 models work (gpt.py:427 hard-casts to bf16).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from . import gpt_t2i as _t
from .vit_adapter import ViT_Adapter


@dataclass
class ModelArgs:                      # field-for-field the constructor surface of reference gpt.py:31-60
    dim: int = 4096
    n_layer: int = 32
    n_head: int = 32
    n_kv_head: Optional[int] = None
    multiple_of: int = 256
    ffn_dim_multiplier: Optional[float] = None
    rope_base: float = 10000
    norm_eps: float = 1e-5
    initializer_range: float = 0.02
    token_dropout_p: float = 0.1
    attn_dropout_p: float = 0.0
    resid_dropout_p: float = 0.1
    ffn_dropout_p: float = 0.1
    drop_path_rate: float = 0.0
    num_classes: int = 1000
    caption_dim: int = 2048
    class_dropout_prob: float = 0.1
    model_type: str = "c2i"
    vocab_size: int = 16384
    cls_token_num: int = 1
    block_size: int = 256
    max_batch_size: int = 32
    max_seq_len: int = 2048
    condition_token_num: int = 256
    image_size: int = 256


class Transformer(_t.Transformer):
    # training branch (gpt.py:410-421,440-449): with cls_token_num = 1 and condition_token_num = 0 it is gpt_t2i's branch (control
    # tokens added to every row, logits from row 0) except that ConditionEmbedder.token_drop hands dropped samples literal zeros
    # (gpt.py:118-119) instead of the `uncond_embedding` buffer — pinned against the reference's gpt.py in train mode by
    # tests/test_train_oracle_golden.py::test_legacy_gptpy_train_branch_is_the_same_arithmetic; forward / backward are inherited.
    zero_uncond_on_drop = True
    has_control_strength = False      # generate() refuses per-image strengths other than 1, as forward() does below

    def __init__(self, config: ModelArgs):
        if config.condition_token_num != 0:
            # the reference's own generate() cannot use condition_token_num > 0 (T = 1 + n at generate.py:154 while the
            # prefill emits cls_token_num rows, gpt.py:424-425 — SURVEY.md §7 hard-part 5); only 0 is ever passed
            raise NotImplementedError("condition_token_num must be 0 (the only value the reference's sampling scripts pass)")
        if (config.image_size // 16) ** 2 != config.block_size:
            raise NotImplementedError("gpt.py sizes condition_mlp by (image_size // 16) ** 2; it must equal block_size")
        base = _t.ModelArgs(**{k: getattr(config, k) for k in (
            "dim", "n_layer", "n_head", "n_kv_head", "multiple_of", "ffn_dim_multiplier", "rope_base", "norm_eps",
            "initializer_range", "token_dropout_p", "attn_dropout_p", "resid_dropout_p", "ffn_dropout_p", "drop_path_rate",
            "num_classes", "caption_dim", "class_dropout_prob", "model_type", "vocab_size", "cls_token_num", "block_size",
            "max_batch_size", "max_seq_len")}, adapter_size="small", condition_type="canny")
        super().__init__(base)
        self.config = base
        self.condition_token_num = config.condition_token_num
        self.condition_norm = _t.RMSNorm(config.dim, eps=config.norm_eps)      # gpt.py:352 — in the checkpoint, unused by forward

    def _make_adapter(self, config) -> nn.Module:
        return ViT_Adapter()                                                  # gpt.py:322

    def forward(self, idx, cond_idx, input_pos=None, targets=None, mask=None, valid=None, condition=None, control_strength=1):
        """gpt.py:400-470.  (``control_strength`` is accepted and must be 1: gpt.py has no such argument.)"""
        if control_strength != 1:
            raise TypeError("the legacy c2i class has no control_strength (gpt.py:400-409)")
        return super().forward(idx, cond_idx, input_pos, targets, mask, valid, condition, 1)


def _factory(n_layer, n_head, dim):
    def make(**kwargs):
        return Transformer(ModelArgs(n_layer=n_layer, n_head=n_head, dim=dim, **kwargs))
    return make


GPT_7B, GPT_3B, GPT_1B = _factory(32, 32, 4096), _factory(24, 32, 3200), _factory(22, 32, 2048)
GPT_XXXL, GPT_XXL, GPT_XL = _factory(48, 40, 2560), _factory(48, 24, 1536), _factory(36, 20, 1280)
GPT_L, GPT_B = _factory(24, 16, 1024), _factory(12, 12, 768)

GPT_models = {"GPT-B": GPT_B, "GPT-L": GPT_L, "GPT-XL": GPT_XL, "GPT-XXL": GPT_XXL, "GPT-XXXL": GPT_XXXL,
              "GPT-1B": GPT_1B, "GPT-3B": GPT_3B, "GPT-7B": GPT_7B}
