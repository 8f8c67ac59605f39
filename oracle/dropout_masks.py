"""TEST INFRASTRUCTURE — CPU restatement of the training path's dropout generator (controlar_b200/csrc/dropout.cuh).

Philox4x32-10 (Salmon et al., SC 2011) in numpy integer arithmetic.  Key = the 64-bit seed (low word first), counter =
(column // 4, row, sample, site << 16 | layer); output word column % 4 decides column `column`.  Keep iff
(word >> 8) * 2^-24 < keep, keep = fp32(1 - p).  Drop path decides once per sample from word 0 of (row 0, column 0) of its own
site.  Also the rounding rules the kernels apply the decisions with (the ones torch's CUDA `nn.Dropout` and the reference's
`utils/drop_path.py` apply), and the reference's per-layer drop-path rates.
"""
from __future__ import annotations

from typing import List

import numpy as np
import torch

TOKEN, RESID, FFN, PATH_ATTN, PATH_FFN = 0, 1, 2, 3, 4
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_U32 = 0xFFFFFFFF


def philox4x32_10(c0, c1, c2, c3, seed: int):
    """Philox4x32-10 on broadcastable uint64 arrays holding 32-bit counters; returns the four output words (uint64 arrays)."""
    c = [np.asarray(x, dtype=np.uint64) & _U32 for x in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c = [x.copy() for x in c]
    k0, k1 = seed & _U32, (seed >> 32) & _U32
    for i in range(10):
        if i:
            k0, k1 = (k0 + _W0) & _U32, (k1 + _W1) & _U32
        p0 = c[0] * np.uint64(_M0)
        p1 = c[2] * np.uint64(_M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_U32)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_U32)
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return c


def keep_prob(p: float) -> np.float32:
    """keep = fp32(1 - p) (p as the fp32 the ABI carries)"""
    return np.float32(1.0 - float(np.float32(p)))


def elem_scale(p: float) -> float:
    """fp32(1 / keep): the scale ATen's CUDA dropout multiplies kept elements by"""
    return float(np.float32(1.0 / float(keep_prob(p))))


def path_mult(rate: float) -> float:
    """bf16(1 / keep): `bernoulli_(keep).div_(keep)` on a bf16 tensor (utils/drop_path.py), for a kept sample"""
    k = keep_prob(rate)
    return float(torch.tensor(float(np.float32(1.0) / k), dtype=torch.float32).to(torch.bfloat16).float())


def _keep(words, p: float) -> np.ndarray:
    u = (words >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return u < keep_prob(p)


def keep_mask(seed: int, site: int, layer: int, B: int, rows: int, cols: int, p: float) -> torch.Tensor:
    """bool [B, rows, cols]: what car_dropout_keep_mask returns.  Drop-path sites repeat each sample's decision."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    tag = (site << 16) | layer
    if site in (PATH_ATTN, PATH_FFN):
        w = philox4x32_10(0, 0, np.arange(B, dtype=np.uint64), tag, seed)[0]
        k = _keep(w, p)[:, None, None]
        return torch.from_numpy(np.broadcast_to(k, (B, rows, cols)).copy())
    b = np.arange(B, dtype=np.uint64)[:, None, None]
    r = np.arange(rows, dtype=np.uint64)[None, :, None]
    c = np.arange(cols, dtype=np.uint64)[None, None, :]
    words = philox4x32_10(c >> np.uint64(2), r, b, tag, seed)
    lane = (c & np.uint64(3)).astype(np.int64)
    w = np.where(lane == 0, words[0], np.where(lane == 1, words[1], np.where(lane == 2, words[2], words[3])))
    return torch.from_numpy(_keep(w, p))


def path_keep(seed: int, site: int, layer: int, B: int, rate: float) -> torch.Tensor:
    """bool [B]: the per-sample drop-path decisions of one branch"""
    return keep_mask(seed, site, layer, B, 1, 1, rate)[:, 0, 0]


def drop_path_rates(rate: float, n_layer: int) -> List[float]:
    """the reference's per-layer rates: [x.item() for x in torch.linspace(0, drop_path_rate, n_layer)] (gpt_t2i.py:347)"""
    return [x.item() for x in torch.linspace(0, rate, n_layer)]


def apply_dropout(x: torch.Tensor, keep: torch.Tensor, p: float) -> torch.Tensor:
    """nn.Dropout as ATen's CUDA kernel computes it: x * mask * fp32(1 / keep) in fp32, rounded once to x's dtype"""
    return (x.float() * keep.float() * elem_scale(p)).to(x.dtype)


def apply_drop_path(x: torch.Tensor, keep: torch.Tensor, rate: float) -> torch.Tensor:
    """utils/drop_path.py: x * random_tensor, random_tensor = bernoulli(keep).div_(keep) in x's dtype, one per sample"""
    rt = (keep.float() * path_mult(rate)).to(x.dtype).view(-1, *([1] * (x.dim() - 1)))
    return x * rt
