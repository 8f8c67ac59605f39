"""fp64 reference of the KV-cache attention of the LlamaGen block (csrc/attention.cuh), with the reference's mask semantics.

The reference attends through F.scaled_dot_product_attention with the bool mask `causal_mask[:, None, input_pos]`
(gpt_t2i.py:282-286,447-448), where generate.py:184-193 has edited causal_mask: lower-triangular, text columns s < T multiplied by
emb_masks (so any non-zero value attends), then the diagonal forced on.  Scale 1/sqrt(64) = 1/8.

Optional rounding points:
  * p_dtype: the probabilities of the tensor-core prefill, exp(s - max) rounded to p_dtype and normalised by the sum of the
    rounded values (attn_prefill_mma_kernel rounds them before the value product);
  * out_dtype: the output cast to the model dtype.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

SCALE = 0.125


def attention_mask(B: int, S: int, emb_mask: Optional[torch.Tensor] = None, device=None) -> torch.Tensor:
    """bool [B, S, S], True = query row i may attend key column s: s <= i, and for text columns s < T (T = emb_mask.shape[-1])
    emb_mask[b][s] != 0, and always s == i."""
    m = torch.tril(torch.ones(S, S, dtype=torch.bool, device=device)).unsqueeze(0).repeat(B, 1, 1)
    if emb_mask is not None:
        T = emb_mask.shape[-1]
        m[:, :, :T] &= (emb_mask.to(device) != 0).unsqueeze(1)
        m |= torch.eye(S, dtype=torch.bool, device=device)
    return m


def masked_sdpa(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, positions: Sequence[int], emb_mask: Optional[torch.Tensor] = None,
                p_dtype: Optional[torch.dtype] = None, out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """q [B, H, R, 64]: the queries at sequence positions `positions` (R of them); k, v [B, H, n, 64]: the cache rows 0 .. n-1, with
    n > max(positions) (rows past the live range are not passed, so their contents never matter).  emb_mask [B, T] or None.
    Returns fp64 [B, H, R, 64], rounded through out_dtype when given."""
    B, _, _, _ = q.shape
    n = k.shape[2]
    pos = torch.as_tensor(list(positions), dtype=torch.long, device=q.device)
    assert int(pos.max()) < n
    m = attention_mask(B, n, emb_mask, q.device)[:, pos][:, None]            # [B, 1, R, n]
    s = (q.double() @ k.double().transpose(-1, -2)) * SCALE
    s = s.masked_fill(~m, float("-inf"))
    if p_dtype is None:
        p = torch.softmax(s, dim=-1)
    else:
        e = torch.exp(s - s.amax(dim=-1, keepdim=True)).to(p_dtype).double()
        p = e / e.sum(dim=-1, keepdim=True)
    o = p @ v.double()
    return o.to(out_dtype).double() if out_dtype is not None else o
