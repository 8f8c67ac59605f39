"""TEST INFRASTRUCTURE — the teacher-forced training forward of oracle/train_oracle.py with the dropout layers on.

`DropoutTrainOracle.forward(..., dropout=...)` restates `Transformer.forward` in train mode (autoregressive/models/gpt_t2i.py:420-484)
like `TrainOracle.forward`, plus the token, residual and feed-forward dropout (gpt_t2i.py:430,290,217) and the per-sample DropPath of
each block (gpt_t2i.py:305-306, utils/drop_path.py).  The keep decisions are the library's generator (oracle/dropout_masks.py; torch's
own dropout bit stream depends on its launch geometry and is not restated), applied with the rounding of torch's CUDA kernels: a kept
element is x * fp32(1 / keep) rounded once to x's dtype, a drop-path branch is multiplied by bf16(1 / keep).  Without ``dropout=``
it is `TrainOracle.forward`.  Where the masks act in the reference's graph is pinned by tests/golden/make_train_dropout_golden.py ->
tests/golden/train_*_dropout.pt.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from . import dropout_masks as DM
from .train_oracle import TrainOracle


def control_tokens(B: int, n_img: int, channels: int, seed: int) -> torch.Tensor:
    """The control-encoder output the dropout fixtures feed to adapter_mlp (bf16 [B, n_img, channels]); the encoder itself has its
    own parity tests"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, n_img, channels, generator=g) * 0.5).to(torch.bfloat16)


class DropoutTrainOracle(TrainOracle):
    def forward(self, idx: torch.Tensor, cond: torch.Tensor, feat: Optional[torch.Tensor], drop_ids: torch.Tensor,
                mask: Optional[torch.Tensor] = None, targets: Optional[torch.Tensor] = None,
                valid: Optional[torch.Tensor] = None, dropout: Optional[dict] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """Arguments and result of TrainOracle.forward, plus dropout: None (every p = 0) or {"seed": int, "token_p", "resid_p",
        "ffn_p": float, "drop_path": per-layer rates or None} (missing keys = 0 / None)."""
        if not dropout:
            return super().forward(idx, cond, feat, drop_ids, mask, targets, valid)
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
        h = torch.cat((ce, te), dim=1)                                              # :428 (promotes to fp32)
        fr = self.freqs[: h.shape[1]]                                               # :452
        B, S, d = h.shape
        seed = dropout["seed"]
        rates = dropout.get("drop_path") or [0.0] * sp.n_layer

        def elem(x, site, layer, p):                                                # nn.Dropout(p) in train mode
            return DM.apply_dropout(x, DM.keep_mask(seed, site, layer, B, S, d, p), p) if p else x

        def path(x, site, layer):                                                   # DropPath(rates[layer]); rate 0 = nn.Identity
            r = rates[layer]
            return DM.apply_drop_path(x, DM.path_keep(seed, site, layer, B, r), r) if r > 0 else x
        h = elem(h, DM.TOKEN, 0, dropout.get("token_p", 0.0))                       # tok_dropout :430, before the control adds
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
            o = elem(self.linear(a, pre + "attention.wo.weight"), DM.RESID, l, dropout.get("resid_p", 0.0))      # resid_dropout :290
            h = h + path(o, DM.PATH_ATTN, l)                                        # :305
            y = self.rmsnorm(h, pre + "ffn_norm.weight")                            # FeedForward :216-217
            act = F.silu(self.linear(y, pre + "feed_forward.w1.weight")) * self.linear(y, pre + "feed_forward.w3.weight")
            o = elem(self.linear(act, pre + "feed_forward.w2.weight"), DM.FFN, l, dropout.get("ffn_p", 0.0))     # ffn_dropout :217
            h = h + path(o, DM.PATH_FFN, l)                                         # :306
        logits = self.linear(self.rmsnorm(h, "norm.weight"), "output.weight").float()[:, T - 1:]   # :469-473
        loss = None
        if valid is not None:                                                       # :476-479
            la = F.cross_entropy(logits.reshape(-1, logits.size(-1)), targets.reshape(-1), reduction="none")
            va = valid[:, None].repeat(1, targets.shape[1]).reshape(-1)
            loss = (la * va).sum() / max(va.sum(), 1)
        elif targets is not None:                                                   # :480-481
            loss = F.cross_entropy(logits.reshape(-1, logits.size(-1)), targets.reshape(-1))
        return logits, loss
