"""TEST INFRASTRUCTURE — CPU restatement of the antialiased bilinear resize in front of the online VQ encode of the
multi-resolution training scripts (SURVEY.md §8 row f2): `F.interpolate(x.float(), size, mode='bilinear', align_corners=False,
antialias=True)`, autoregressive/train/train_t2i_depth_multiscale.py:44-56 (image and control map, then
`2*(image/255-0.5)` and `vq_model.encode`, :216-223; the encode itself is oracle/vision_oracle.py:vq_encode_oracle).

The arithmetic lives in a third-party dependency, PyTorch (ATen `_upsample_bilinear2d_aa`, UpSampleKernel.cpp
`HelperInterpBase::_compute_indices_min_size_weights_aa`, unpinned in the reference's requirements; installed here: 2.11).
Published algorithm (same as Pillow's): separable triangle filter whose support is stretched by the down-scale factor,
    scale = in / out, support = max(scale, 1), centre_i = scale * (i + 0.5),
    taps j in [max(int(c - support + 0.5), 0), min(int(c + support + 0.5), in)),  w_j = max(0, 1 - |(j - c + 0.5) / max(scale, 1)|),
weights normalised to sum 1, width pass first, then height, fp32.  Pinned against `F.interpolate` itself in
tests/test_train_oracle_golden.py::test_resize_oracle_matches_torch (no fixture needed: torch is the dependency the reference calls).
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch


def aa_weights(n_in: int, n_out: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Per output index: first tap, tap count, weights [n_out, max_taps] (zero padded).  ATen does the weight arithmetic in the
    tensor's scalar type (fp32: scale, centre, tap distance, normalisation) — fp64 weights differ from it by 4e-6 relative,
    fp32 weights reproduce it to the last bits, so every step below is an explicit float32 operation."""
    f = np.float32
    scale = f(n_in) / f(n_out)
    support = scale if scale >= 1.0 else f(1.0)
    inv = f(1.0) / scale if scale >= 1.0 else f(1.0)
    taps = int(np.ceil(support)) * 2 + 1
    xmin = torch.zeros(n_out, dtype=torch.long)
    xsize = torch.zeros(n_out, dtype=torch.long)
    w = torch.zeros(n_out, taps, dtype=torch.float32)
    for i in range(n_out):
        c = scale * (f(i) + f(0.5))
        lo = max(int(c - support + f(0.5)), 0)
        hi = min(int(c + support + f(0.5)), n_in)
        ws = [max(f(0.0), f(1.0) - abs((f(j + lo) - c + f(0.5)) * inv)) for j in range(hi - lo)]
        tot = f(0.0)
        for v in ws:
            tot = tot + v
        xmin[i], xsize[i] = lo, hi - lo
        w[i, : hi - lo] = torch.tensor(np.array([v / tot for v in ws], dtype=np.float32))
    return xmin, xsize, w


def _resize_last(x: torch.Tensor, n_out: int) -> torch.Tensor:
    n_in = x.shape[-1]
    xmin, xsize, w = aa_weights(n_in, n_out)
    out = torch.zeros(*x.shape[:-1], n_out, dtype=torch.float32)
    for i in range(n_out):
        k = int(xsize[i])
        out[..., i] = (x[..., int(xmin[i]): int(xmin[i]) + k] * w[i, :k]).sum(-1)
    return out


def bilinear_aa_resize(x: torch.Tensor, size: Tuple[int, int]) -> torch.Tensor:
    """x [B, C, H, W] -> [B, C, size[0], size[1]] fp32."""
    y = _resize_last(x.float(), size[1])
    return _resize_last(y.transpose(-1, -2), size[0]).transpose(-1, -2).contiguous()
