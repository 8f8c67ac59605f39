"""Seeded synthetic inputs (no arithmetic of the path itself): shared by bench.py, tests/golden/make_golden.py and the tests
(oracle/inputs.py re-exports this module).

Shapes follow SURVEY.md §8(d): T5 embeddings left-padded and zeroed like
autoregressive/sample/sample_t2i.py:146-160; control maps in [-1, 1] with three identical
channels like sample_t2i.py:119-141 (`2*(x/255-0.5)`, `.repeat(1,3,1,1)`).
"""
from __future__ import annotations

import torch


def text_inputs(T: int, caption_dim: int, B: int, seed: int, dtype=torch.float32, min_valid: int = 3):
    g = torch.Generator().manual_seed(seed)
    emb = torch.randn(B, T, caption_dim, generator=g)
    valid = torch.randint(min_valid, T + 1, (B,), generator=g)
    masks = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        masks[b, T - int(valid[b]):] = 1          # left padding: valid tokens at the end
    emb = emb * masks[:, :, None]
    return emb.to(dtype), masks


def class_inputs(num_classes: int, B: int, seed: int):
    return torch.randint(0, num_classes, (B,), generator=torch.Generator().manual_seed(seed))


def control_map(B: int, H: int, W: int, seed: int, kind: str, dtype=torch.float32):
    """kind 'canny': Bernoulli(0.1) edges in {-1,+1}; otherwise a smooth random field in [-1,1]."""
    g = torch.Generator().manual_seed(seed)
    if kind == "canny":
        m = (torch.rand(B, 1, H, W, generator=g) < 0.1).float()
    else:
        lo = torch.rand(B, 1, max(H // 16, 1), max(W // 16, 1), generator=g)
        m = torch.nn.functional.interpolate(lo, size=(H, W), mode="bilinear", align_corners=False)
    return (2 * (m - 0.5)).repeat(1, 3, 1, 1).to(dtype)


def xl_ctrl_in(B: int, N: int, dim: int, seed: int, dtype=torch.float32):
    """Procedural adapter_mlp output [B, N, dim] for the XL-shape teacher-forced fixtures (never stored; the control encoder has
    its own goldens)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, N, dim, generator=g) * 0.5).to(dtype)


def train_attn_mask(emb_masks: torch.Tensor, n_img: int) -> torch.Tensor:
    """Per-sample training mask of the t2i datasets, dataset/t2i_control.py:134-139 followed by the slicing of
    train_t2i_canny.py:165-167: causal [S,S] with S = T + n_img, padded text COLUMNS switched off, diagonal forced on,
    then [..., :-1, :-1].  Returns bool [B, 1, S-1, S-1]."""
    B, T = emb_masks.shape
    S = T + n_img
    out = []
    for b in range(B):
        a = torch.tril(torch.ones(S, S))
        a[:, :T] = a[:, :T] * emb_masks[b].float().unsqueeze(0)
        eye = torch.eye(S)
        out.append((a * (1 - eye) + eye).bool())
    return torch.stack(out).unsqueeze(1)[:, :, :-1, :-1]


def code_inputs(vocab: int, B: int, n_img: int, seed: int) -> torch.Tensor:
    """VQ code grid z_indices [B, n_img] int64 (what dataset['code'] holds)."""
    return torch.randint(0, vocab, (B, n_img), generator=torch.Generator().manual_seed(seed))
