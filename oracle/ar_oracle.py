"""TEST INFRASTRUCTURE — CPU restatement of ControlAR's conditional-decoding transformer path.

This is the checker for the CUDA path (and the timed CPU baseline of bench.py); it is never shipped or called
by the product.  Every function cites the reference lines it restates (paths relative to the reference checkout).
It is pinned against the reference itself by tests/golden/make_golden.py -> tests/golden/*.pt
(tests/test_oracle_golden.py); the reference has no golden vectors of its own (SURVEY.md §4).

Numerics model ("rounding points", SURVEY.md §8 a-notes): tensors are carried as fp32 holding values that are
exactly representable in the model dtype (bf16 by default); every place where eager PyTorch would materialise a
model-dtype tensor is an explicit ``r()`` here; GEMMs accumulate in fp32 and round once; RMSNorm, RoPE and the
attention soft-max run in fp32 exactly as the reference does.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from .weights import GPTSpec


def rope_table_2d(grid: int, head_dim: int, base: float, n_prefix: int) -> torch.Tensor:
    """[n_prefix + grid*grid, head_dim/2, 2] fp32 (cos, sin); the first n_prefix rows are all-zero.
    Restates precompute_freqs_cis_2d, autoregressive/models/gpt_t2i.py:506-519."""
    half = head_dim // 2
    k = torch.arange(0, half, 2)[: half // 2].float()
    theta = 1.0 / (base ** (k / half))                    # half/2 frequencies
    t = torch.arange(grid)
    ang = torch.outer(t, theta)                           # [grid, half/2]
    rows = ang[:, None, :].expand(grid, grid, half // 2)  # pairs 0..half/2-1  <- row index i
    cols = ang[None, :, :].expand(grid, grid, half // 2)  # pairs half/2..half-1 <- col index j
    g = torch.cat([rows, cols], dim=-1).reshape(grid * grid, half)
    tab = torch.stack([torch.cos(g), torch.sin(g)], dim=-1)
    return torch.cat([torch.zeros(n_prefix, half, 2), tab], dim=0)


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    """nn.GELU(approximate='tanh') — gpt_t2i.py:171."""
    return F.gelu(x, approximate="tanh")


class AROracle:
    """Restatement of gpt_t2i.Transformer's *inference* branches (prefill + KV-cache decode),
    autoregressive/models/gpt_t2i.py:409-470, for model_type 't2i' and 'c2i'."""

    def __init__(self, spec: GPTSpec, sd: Dict[str, torch.Tensor], dtype: torch.dtype = torch.bfloat16):
        self.spec = spec
        self.dtype = dtype
        # weights: fp32 tensors holding dtype-rounded values (== model.to(dtype))
        self.w = {k: v.to(dtype).float() for k, v in sd.items() if not k.startswith("adapter.model.")}
        grid = int(round(spec.block_size ** 0.5))
        assert grid * grid == spec.block_size
        self.freqs = rope_table_2d(grid, spec.head_dim, spec.rope_base, spec.cls_token_num)  # gpt_t2i.py:405
        self.k_cache: List[torch.Tensor] = []
        self.v_cache: List[torch.Tensor] = []
        self.ctrl: Optional[List[torch.Tensor]] = None
        self.cs = 1.0

    # ---- primitives ------------------------------------------------------------------------------------
    def r(self, x: torch.Tensor) -> torch.Tensor:
        return x.to(self.dtype).float()

    def linear(self, x: torch.Tensor, key: str) -> torch.Tensor:
        """bias-free nn.Linear in model dtype: fp32 accumulate, one rounding."""
        return self.r(x @ self.w[key].t())

    def mlp(self, x: torch.Tensor, prefix: str) -> torch.Tensor:
        """MLP.forward, gpt_t2i.py:177-181: fc2(gelu_tanh(fc1(x)))."""
        h = self.linear(x, prefix + ".fc1.weight")
        h = self.r(gelu_tanh(h))
        return self.linear(h, prefix + ".fc2.weight")

    def rmsnorm(self, x: torch.Tensor, key: str) -> torch.Tensor:
        """RMSNorm.forward, gpt_t2i.py:193-198: fp32 normalise -> cast -> * weight (model dtype)."""
        n = x * torch.rsqrt(torch.mean(x * x, dim=-1, keepdim=True) + self.spec.norm_eps)
        return self.r(self.r(n) * self.w[key])

    def rope(self, x: torch.Tensor, fr: torch.Tensor) -> torch.Tensor:
        """apply_rotary_emb, gpt_t2i.py:522-532.  x [B, S, H, Dh], fr [S, Dh/2, 2]."""
        xs = x.reshape(*x.shape[:-1], -1, 2)
        c = fr[None, :, None, :, 0]
        s = fr[None, :, None, :, 1]
        o = torch.stack([xs[..., 0] * c - xs[..., 1] * s, xs[..., 1] * c + xs[..., 0] * s], dim=-1)
        return self.r(o.flatten(3))

    # ---- state -----------------------------------------------------------------------------------------
    def setup_caches(self, b_eff: int, max_seq: int) -> None:
        """Transformer.setup_caches, gpt_t2i.py:391-405 (S rounded up to a multiple of 8)."""
        sp = self.spec
        S = max_seq if max_seq % 8 == 0 else max_seq + 8 - max_seq % 8
        self.S = S
        self.b_eff = b_eff
        self.k_cache = [torch.zeros(b_eff, sp.n_head, S, sp.head_dim) for _ in range(sp.n_layer)]
        self.v_cache = [torch.zeros(b_eff, sp.n_head, S, sp.head_dim) for _ in range(sp.n_layer)]
        self.mask = torch.tril(torch.ones(S, S, dtype=torch.bool)).unsqueeze(0).repeat(b_eff, 1, 1)

    def apply_emb_masks(self, emb_masks: torch.Tensor) -> None:
        """generate.py:184-193: text columns gated by emb_masks, diagonal forced on."""
        T = emb_masks.shape[-1]
        self.mask[:, :, :T] = self.mask[:, :, :T] & (emb_masks != 0).unsqueeze(1)
        eye = torch.eye(self.S, dtype=torch.bool)
        self.mask = self.mask | eye

    # ---- one transformer block -------------------------------------------------------------------------
    def _block(self, l: int, h: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
        """TransformerBlock.forward gpt_t2i.py:303-307 + Attention.forward :257-291 + FeedForward :216-217."""
        sp = self.spec
        B, S_q, d = h.shape
        p = f"layers.{l}."
        x = self.rmsnorm(h, p + "attention_norm.weight")
        qkv = self.linear(x, p + "attention.wqkv.weight")
        q, k, v = qkv.split([d, d, d], dim=-1)
        q = q.view(B, S_q, sp.n_head, sp.head_dim)
        k = k.view(B, S_q, sp.n_head, sp.head_dim)
        v = v.view(B, S_q, sp.n_head, sp.head_dim)
        fr = self.freqs[pos]
        q = self.rope(q, fr).transpose(1, 2)
        k = self.rope(k, fr).transpose(1, 2)
        v = v.transpose(1, 2)
        self.k_cache[l][:, :, pos] = k          # KVCache.update gpt_t2i.py:227-235
        self.v_cache[l][:, :, pos] = v
        m = self.mask[:B, None, pos]            # [B,1,S_q,S]   gpt_t2i.py:448
        # F.scaled_dot_product_attention, math backend (generate.py:120): fp32 up-cast, soft-max fp32, cast out
        s = (q @ self.k_cache[l].transpose(-1, -2)) * (1.0 / math.sqrt(sp.head_dim))
        s = s.masked_fill(~m, float("-inf"))
        a = torch.softmax(s, dim=-1) @ self.v_cache[l]
        a = self.r(a).transpose(1, 2).reshape(B, S_q, d)
        h = self.r(h + self.linear(a, p + "attention.wo.weight"))
        y = self.rmsnorm(h, p + "ffn_norm.weight")
        g = self.linear(y, p + "feed_forward.w1.weight")
        u = self.linear(y, p + "feed_forward.w3.weight")
        act = self.r(self.r(F.silu(g)) * u)
        return self.r(h + self.linear(act, p + "feed_forward.w2.weight"))

    def _head(self, h: torch.Tensor) -> torch.Tensor:
        """gpt_t2i.py:469-470: norm -> output -> .float()"""
        return self.linear(self.rmsnorm(h, "norm.weight"), "output.weight")

    # ---- prefill ---------------------------------------------------------------------------------------
    def prefill(self, cond: torch.Tensor, condition: Optional[torch.Tensor], control_strength: float = 1.0
                ) -> torch.Tensor:
        """Inference prefill branch gpt_t2i.py:433-442,455-470.
        cond: t2i [B_eff, T, caption_dim] float (dtype-representable) | c2i [B_eff] int64 class ids.
        condition: [B_eff, N, dim] adapter_mlp output (rows of the un-conditional half are zero) or None.
        Returns logits fp32 [B_eff, T, V]."""
        sp = self.spec
        T = sp.cls_token_num
        self.cs = control_strength
        if sp.model_type == "t2i":
            h = self.mlp(self.r(cond.float()), "cls_embedding.cap_proj")[:, :T]      # CaptionEmbedder :156-162
        else:
            h = self.w["cls_embedding.embedding_table.weight"][cond].unsqueeze(1)[:, :T]  # LabelEmbedder :89-97
        if condition is not None:
            c = self.mlp(self.r(condition.float()), "condition_mlp.cap_proj")        # ConditionEmbedder :123-128
            self.ctrl = [self.mlp(c, f"condition_layers.{j}") for j in range(3)]     # :440-442
        else:
            self.ctrl = None
        pos = torch.arange(T)
        step = sp.n_layer // 3
        for l in range(sp.n_layer):
            if l % step == 0 and self.ctrl is not None:
                # gpt_t2i.py:463 — only the last prefix row receives control token 0
                add = self.r(self.cs * self.ctrl[l // step][:, 0:1])
                h = h.clone()
                h[:, -1:] = self.r(h[:, -1:] + add)
            h = self._block(l, h, pos)
        return self._head(h)

    # ---- decode ----------------------------------------------------------------------------------------
    def decode(self, tok: torch.Tensor, pos: int) -> torch.Tensor:
        """KV-cache decode branch gpt_t2i.py:444-470 for one position.  tok [B_eff] int; returns [B_eff, V]."""
        sp = self.spec
        T = sp.cls_token_num
        h = self.w["tok_embeddings.weight"][tok.long()].unsqueeze(1)
        p = torch.tensor([pos])
        step = sp.n_layer // 3
        for l in range(sp.n_layer):
            if l % step == 0 and self.ctrl is not None:
                # gpt_t2i.py:466 — control token of the position about to be predicted (one ahead)
                add = self.r(self.cs * self.ctrl[l // step][:, pos - T + 1: pos - T + 2])
                h = self.r(h + add)
            h = self._block(l, h, p)
        return self._head(h)[:, 0]


# ------------------------------------------------------------------------------------------------------------
# sampling (generate.py:17-74) and the generation driver (generate.py:85-204)
# ------------------------------------------------------------------------------------------------------------

def cfg_combine(logits: torch.Tensor, cfg_scale: float, cfg_on: bool = True) -> torch.Tensor:
    """generate.py:89-90,103-107: cond/uncond halves -> u + (c-u)*s; cond only when cfg_on is False."""
    c, u = torch.split(logits, logits.shape[0] // 2, dim=0)
    return u + (c - u) * cfg_scale if cfg_on else c


def filter_logits(z: torch.Tensor, top_k: int, top_p: float) -> torch.Tensor:
    """top_k_top_p_filtering generate.py:17-56 on [B, V] fp32 (returns a new tensor)."""
    z = z.clone()
    V = z.shape[-1]
    if top_k > 0:
        k = min(max(top_k, 1), V)
        thr = torch.topk(z, k)[0][..., -1, None]
        z[z < thr] = float("-inf")            # ties at the threshold are kept
    if top_p < 1.0:
        sl, si = torch.sort(z, descending=True)
        cp = torch.cumsum(torch.softmax(sl, dim=-1), dim=-1)
        rm = cp > top_p
        rm[..., 1:] = rm[..., :-1].clone()
        rm[..., 0] = False
        z[rm.scatter(1, si, rm)] = float("-inf")
    return z


def sample_from_logits(z: torch.Tensor, temperature: float = 1.0, top_k: int = 2000, top_p: float = 1.0,
                       sample_logits: bool = True, noise: Optional[torch.Tensor] = None
                       ) -> Tuple[torch.Tensor, torch.Tensor]:
    """sample() generate.py:59-74 on the last-position logits [B, V].
    noise=None  -> torch.multinomial (reference-identical RNG use on CPU);
    noise=[B,V] -> argmax(p / noise) with noise ~ Exp(1): the same draw torch.multinomial makes internally
                   (SURVEY.md §7 hard-part 4), used to compare with the CUDA sampler on identical noise."""
    z = z / max(temperature, 1e-5)
    if top_k > 0 or top_p < 1.0:
        z = filter_logits(z, top_k, top_p)
    p = torch.softmax(z, dim=-1)
    if not sample_logits:
        idx = torch.argmax(p, dim=-1, keepdim=True)      # lowest index among ties (topk(1) is unspecified)
    elif noise is None:
        idx = torch.multinomial(p, num_samples=1)
    else:
        idx = torch.argmax(p / noise, dim=-1, keepdim=True)
    return idx, p


def oracle_generate(orc: AROracle, cond: torch.Tensor, max_new_tokens: int, emb_masks: Optional[torch.Tensor],
                    cfg_scale: float, condition: Optional[torch.Tensor], control_strength: float = 1.0,
                    cfg_interval: int = -1, temperature: float = 1.0, top_k: int = 2000, top_p: float = 1.0,
                    sample_logits: bool = True, noise: Optional[torch.Tensor] = None,
                    return_logits: bool = False):
    """generate() generate.py:134-204 given the *adapter_mlp output* ``condition`` [B, N, dim] (or None).
    noise: optional [max_new_tokens, B, V] Exp(1) draws consumed one slice per step."""
    sp = orc.spec
    B = cond.shape[0]
    use_cfg = cfg_scale > 1.0
    if sp.model_type == "t2i":
        T = cond.shape[1]
        if use_cfg:
            null = torch.zeros_like(cond) + orc.w["cls_embedding.uncond_embedding"]     # generate.py:156
            cond_c = torch.cat([cond, null])
        else:
            cond_c = cond
    else:
        T = 1
        cond_c = torch.cat([cond, torch.full_like(cond, sp.num_classes)]) if use_cfg else cond  # :141-142
    cond_comb = None
    if condition is not None:
        cond_comb = torch.cat([condition, torch.zeros_like(condition)]) if use_cfg else condition  # :145,161
    b_eff = 2 * B if use_cfg else B
    orc.setup_caches(b_eff, T + max_new_tokens)
    if emb_masks is not None:
        orc.apply_emb_masks(torch.cat([emb_masks, emb_masks]) if use_cfg else emb_masks)
    # generate.py:92 does not forward control_strength when cfg_scale <= 1 (it is then reset to 1, gpt_t2i.py:434)
    cs = control_strength if use_cfg else 1.0
    logits = orc.prefill(cond_c, cond_comb, cs)
    all_logits = []
    z = cfg_combine(logits, cfg_scale)[:, -1] if use_cfg else logits[:, -1]
    all_logits.append(z)
    kw = dict(temperature=temperature, top_k=top_k, top_p=top_p, sample_logits=sample_logits)
    tok, _ = sample_from_logits(z, noise=None if noise is None else noise[0], **kw)
    toks = [tok]
    cfg_on = True
    for i in range(max_new_tokens - 1):
        if cfg_interval > -1 and i > cfg_interval:
            cfg_on = False
        t = tok.view(-1)
        lg = orc.decode(torch.cat([t, t]) if use_cfg else t, T + i)
        z = cfg_combine(lg, cfg_scale, cfg_on) if use_cfg else lg
        all_logits.append(z)
        tok, _ = sample_from_logits(z, noise=None if noise is None else noise[i + 1], **kw)
        toks.append(tok)
    seq = torch.cat(toks, dim=1).to(torch.int32)
    if return_logits:
        return seq, torch.stack(all_logits, dim=1)
    return seq
