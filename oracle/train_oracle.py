"""TEST INFRASTRUCTURE — CPU restatement of ControlAR's teacher-forced *training* forward (SURVEY.md §8 row f1).

Checker for the (round-2) CUDA training forward / backward; never shipped or called by the product.  Every function cites the
reference lines it restates (paths relative to the reference checkout).  Pinned against the reference itself (loss, logits, gradients)
by tests/golden/make_golden.py::train_case -> tests/golden/train_*.pt, checked in tests/test_train_oracle_golden.py.

Scope: `Transformer.forward` with both ``idx`` and ``cond_idx`` given, module in train mode
(autoregressive/models/gpt_t2i.py:420-431,451-484), from the control encoder's OUTPUT tokens (``feat`` = `self.adapter(condition)`,
the DINOv2 forward is restated in vision_oracle.py) to ``(logits, loss)``; gradients come from autograd over this restatement.
Random draws are inputs, not state: the CFG drop decision ``drop_ids`` (gpt_t2i.py:83,116,148) is an argument, and the
dropout layers (token / residual / FFN, gpt_t2i.py:214,255,338) are restated for p = 0 only (a dropout mask of another RNG
cannot be compared bit-wise; p = 0 is `--dropout-p 0 --token-dropout-p 0` of the train scripts).

Numerics model: the train scripts keep fp32 parameters and run the forward under bf16 autocast
(train_t2i_canny.py:166-167, train_c2i_canny.py:200-201).  The autocast rules are written out as explicit casts:
`nn.Linear` and SDPA take bf16 operands and return bf16 (``lc``); embeddings, RMSNorm (fp32 in, fp32 weight) and every residual
add stay fp32 because fp32 + bf16 promotes to fp32; GELU / SiLU / the SwiGLU product run on the bf16 tensors they receive;
cross-entropy is fp32.  ``autocast=None`` restates the plain fp32 forward.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from .weights import GPTSpec
from .ar_oracle import rope_table_2d

_BUFFERS = ("cls_embedding.uncond_embedding", "condition_mlp.uncond_embedding")


class TrainOracle:
    def __init__(self, spec: GPTSpec, sd: Dict[str, torch.Tensor], autocast: Optional[torch.dtype] = torch.bfloat16):
        self.spec = spec
        self.ac = autocast
        self.p: Dict[str, torch.Tensor] = {}
        for k, v in sd.items():
            if k.startswith("adapter.model."):
                continue
            t = v.detach().clone().float()
            self.p[k] = t if k in _BUFFERS else t.requires_grad_(True)
        grid = int(round(spec.block_size ** 0.5))
        self.freqs = rope_table_2d(grid, spec.head_dim, spec.rope_base, spec.cls_token_num)   # gpt_t2i.py:405

    # ---- primitives --------------------------------------------------------------------------------------------
    def lc(self, x: torch.Tensor) -> torch.Tensor:
        """autocast's operand cast for 'lower precision' ops"""
        return x.to(self.ac) if self.ac is not None else x

    def linear(self, x: torch.Tensor, key: str) -> torch.Tensor:
        return F.linear(self.lc(x), self.lc(self.p[key]))

    def mlp(self, x: torch.Tensor, prefix: str) -> torch.Tensor:
        """MLP.forward gpt_t2i.py:177-181 (no bias, GELU-tanh on the tensor fc1 returned)"""
        return self.linear(F.gelu(self.linear(x, prefix + ".fc1.weight"), approximate="tanh"), prefix + ".fc2.weight")

    def rmsnorm(self, x: torch.Tensor, key: str) -> torch.Tensor:
        """RMSNorm.forward gpt_t2i.py:193-198: x is the fp32 residual stream in training, so both casts are no-ops"""
        xf = x.float()
        n = (xf * torch.rsqrt(torch.mean(xf * xf, dim=-1, keepdim=True) + self.spec.norm_eps)).type_as(x)
        return n * self.p[key]

    @staticmethod
    def rope(x: torch.Tensor, fr: torch.Tensor) -> torch.Tensor:
        """apply_rotary_emb gpt_t2i.py:522-532: fp32 rotation, cast back to the dtype of x.  x [B,S,H,Dh], fr [S,Dh/2,2]"""
        xs = x.float().reshape(*x.shape[:-1], -1, 2)
        c, s = fr[None, :, None, :, 0], fr[None, :, None, :, 1]
        o = torch.stack([xs[..., 0] * c - xs[..., 1] * s, xs[..., 1] * c + xs[..., 0] * s], dim=-1)
        return o.flatten(3).type_as(x)

    def attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
        """F.scaled_dot_product_attention gpt_t2i.py:282-286, math semantics: fp32 scores, fp32 soft-max, result cast to the
        operand dtype.  mask None -> causal (is_causal=True); bool mask [B,1,S,S] -> True = attend."""
        S = q.shape[-2]
        s = (q.float() @ k.float().transpose(-1, -2)) * (1.0 / math.sqrt(q.shape[-1]))
        keep = torch.tril(torch.ones(S, S, dtype=torch.bool)) if mask is None else mask
        s = s.masked_fill(~keep, float("-inf"))
        return (torch.softmax(s, dim=-1) @ v.float()).to(q.dtype)

    # ---- forward -----------------------------------------------------------------------------------------------
    def forward(self, idx: torch.Tensor, cond: torch.Tensor, feat: Optional[torch.Tensor], drop_ids: torch.Tensor,
                mask: Optional[torch.Tensor] = None, targets: Optional[torch.Tensor] = None,
                valid: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """idx [B, n] int64 (the train scripts pass z[:, :-1]); cond: t2i [B, T, caption_dim] fp32 | c2i [B] int64;
        feat [B, n+1, C_adapter] control-encoder output or None; drop_ids [B] bool; mask [B,1,T+n,T+n] bool or None;
        targets [B, n+1]; valid [B].  Returns (logits fp32 [B, n+1, V], loss)."""
        sp, P = self.spec, self.p
        T = sp.cls_token_num
        drop = drop_ids.bool()
        if sp.model_type == "t2i":      # CaptionEmbedder gpt_t2i.py:145-162 (train: token_drop then cap_proj)
            cap = torch.where(drop[:, None, None], P["cls_embedding.uncond_embedding"], cond.float())
            ce = self.mlp(cap, "cls_embedding.cap_proj")[:, :T]
        else:                           # LabelEmbedder gpt_t2i.py:78-97
            lab = torch.where(drop, torch.full_like(cond, sp.num_classes), cond)
            ce = F.embedding(lab, P["cls_embedding.embedding_table.weight"]).unsqueeze(1)[:, :T]
        te = F.embedding(idx, P["tok_embeddings.weight"])                           # :423
        ctok = None
        if feat is not None:                                                        # :424-427
            c = self.mlp(feat, "adapter_mlp")
            c = torch.where(drop[:, None, None], P["condition_mlp.uncond_embedding"][: c.shape[1]], c)   # :110-120
            ctok = self.mlp(c, "condition_mlp.cap_proj")
        h = torch.cat((ce, te), dim=1)                                              # :428 (promotes to fp32); tok_dropout p=0
        fr = self.freqs[: h.shape[1]]                                               # :452
        B, S, d = h.shape
        step = sp.n_layer // 3
        for l in range(sp.n_layer):
            if l % step == 0 and ctok is not None:                                  # :458-460
                add = self.mlp(ctok, f"condition_layers.{l // step}")
                h = torch.cat((h[:, : T - 1], h[:, T - 1:] + add), dim=1)
            pre = f"layers.{l}."
            x = self.rmsnorm(h, pre + "attention_norm.weight")                      # TransformerBlock :303-307
            q, k, v = self.linear(x, pre + "attention.wqkv.weight").split([d, d, d], dim=-1)   # Attention :257-291
            q = self.rope(q.view(B, S, sp.n_head, sp.head_dim), fr).transpose(1, 2)
            k = self.rope(k.view(B, S, sp.n_head, sp.head_dim), fr).transpose(1, 2)
            v = v.view(B, S, sp.n_head, sp.head_dim).transpose(1, 2)
            a = self.attention(q, k, v, mask).transpose(1, 2).reshape(B, S, d)
            h = h + self.linear(a, pre + "attention.wo.weight")
            y = self.rmsnorm(h, pre + "ffn_norm.weight")                            # FeedForward :216-217
            act = F.silu(self.linear(y, pre + "feed_forward.w1.weight")) * self.linear(y, pre + "feed_forward.w3.weight")
            h = h + self.linear(act, pre + "feed_forward.w2.weight")
        logits = self.linear(self.rmsnorm(h, "norm.weight"), "output.weight").float()[:, T - 1:]   # :469-473
        loss = None
        if valid is not None:                                                       # :476-479
            la = F.cross_entropy(logits.reshape(-1, logits.size(-1)), targets.reshape(-1), reduction="none")
            va = valid[:, None].repeat(1, targets.shape[1]).reshape(-1)
            loss = (la * va).sum() / max(va.sum(), 1)
        elif targets is not None:                                                   # :480-481
            loss = F.cross_entropy(logits.reshape(-1, logits.size(-1)), targets.reshape(-1))
        return logits, loss


def grad_probe(key: str, g: torch.Tensor, n: int = 256) -> Dict[str, torch.Tensor]:
    """Fixture-sized summary of one gradient tensor: L2 norm, sum, and n entries at positions drawn from a generator keyed by
    the parameter name (same positions in make_golden.py and in the tests)."""
    import zlib
    gen = torch.Generator().manual_seed(zlib.crc32(key.encode()) & 0x7FFFFFFF)
    flat = g.detach().float().reshape(-1)
    pos = torch.randint(0, flat.numel(), (min(n, flat.numel()),), generator=gen)
    return {"norm": flat.norm(), "sum": flat.double().sum().float(), "pos": pos, "val": flat[pos].clone()}
