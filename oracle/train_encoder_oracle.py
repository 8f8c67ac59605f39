"""TEST INFRASTRUCTURE — CPU restatement of the control encoder in TRAINING: Dinov2_Adapter.forward
(autoregressive/models/dinov2_adapter.py:16-29 over HF modeling_dinov2.py 5.5.0) or ViT_Adapter.forward (vit_adapter.py:13-15 over
HF modeling_vit.py 5.5.0) with fp32 parameters inside the train loop's bf16 autocast (train_t2i_canny.py:166-167,
train_c2i_canny.py:200-201).  Written with explicit casts, so autograd over it gives the gradients at autograd's rounding points.
Checker for csrc/dino_train.cuh; never shipped or called by the product.  Pinned against the reference itself by
tests/golden/make_train_encoder_golden.py -> tests/golden/train_enc_*.pt (tests/test_train_encoder_cpu.py).

Autocast rules, as they apply to this module (the input map arrives in bf16, `condition_img.to(ptdtype)`, train_t2i_canny.py:167):
  * input resize (DINOv2 only): nearest for canny / seg, bicubic align_corners=True otherwise; the value reaches the convolution as
    one bf16 rounding of the fp32 interpolation (bf16 resize output, `.to(fp32)` in Dinov2Embeddings, autocast's bf16 cast).
    The map is data: no gradient.
  * patch projection: conv2d on bf16 operands, bf16 result (autocast lower-precision op).
  * position embeddings: fp32 bicubic (align_corners=False) of the pos_grid^2 table to (h, w), skipped when the grid already
    matches and the map is square; the CLS token and CLS position row stay fp32.  torch.cat(fp32 CLS, bf16 tokens) -> fp32.
  * residual stream: fp32 (fp32 + bf16 promotes to fp32).  LayerNorm: fp32 in, fp32 out.
  * q / k / v / o, fc1, fc2: bf16 operands (weights and biases cast), bf16 results.
  * attention: SDPA on bf16 q, k, v, scale 1/8, no mask; the math backend computes in fp32 and rounds the output to bf16.
  * GELU: erf form on the bf16 tensor fc1 returned.
  * LayerScale: bf16 x fp32 lambda -> fp32 (type promotion).  ViT has none.
  * output: final LayerNorm (fp32), CLS row dropped.
CPU and CUDA autocast: conv2d, linear and scaled_dot_product_attention are lower-precision ops on both; layer_norm is an fp32 op
on CUDA and runs in fp32 here anyway because its input (the stream) is fp32; upsample_* are not cast on either, so the resize
runs in the dtype of the map.  This module therefore has the same arithmetic under both; the golden was made on the CPU.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

BF = torch.bfloat16


def _lc(t: torch.Tensor) -> torch.Tensor:
    """autocast's operand cast"""
    return t.to(BF)


def _linear(x, w, b):
    return F.linear(_lc(x), _lc(w), _lc(b))


def encoder_forward(p: Dict[str, torch.Tensor], x: torch.Tensor, vit: bool, condition_type: str = "canny", heads: int = 6,
                    eps: float = 1e-6) -> torch.Tensor:
    """p: backbone parameters by HF key (without the `model.` prefix), fp32; x [B,3,H,W] (any float dtype).  -> feat fp32
    [B, (H/16)(W/16), C]"""
    B, _, H, W = x.shape
    patch = p["embeddings.patch_embeddings.projection.weight"].shape[-1]
    with torch.no_grad():
        xi = x.float()
        if not vit:                                                           # dinov2_adapter.py:16-24 (to_patch14)
            size = ((H // 16) * 14, (W // 16) * 14)
            if condition_type in ("canny", "seg"):
                xi = F.interpolate(xi, size=size, mode="nearest")
            else:
                xi = F.interpolate(xi, size=size, mode="bicubic", align_corners=True)
    e = F.conv2d(_lc(xi), _lc(p["embeddings.patch_embeddings.projection.weight"]), _lc(p["embeddings.patch_embeddings.projection.bias"]),
                 stride=patch).flatten(2).transpose(1, 2)
    C = e.shape[-1]
    h, w = xi.shape[2] // patch, xi.shape[3] // patch
    pos = p["embeddings.position_embeddings"]
    G = int(round((pos.shape[1] - 1) ** 0.5))
    if not (h * w == G * G and h == w):                                         # interpolate_pos_encoding
        pp = pos[:, 1:].reshape(1, G, G, C).permute(0, 3, 1, 2)
        pp = F.interpolate(pp, size=(h, w), mode="bicubic", align_corners=False)
        pos = torch.cat([pos[:, :1], pp.permute(0, 2, 3, 1).reshape(1, -1, C)], dim=1)
    hs = torch.cat([p["embeddings.cls_token"].expand(B, -1, -1), e.float()], dim=1) + pos
    L = 1 + max(int(k.split(".")[2]) for k in p if k.startswith("encoder.layer."))
    n1, n2 = ("layernorm_before", "layernorm_after") if vit else ("norm1", "norm2")
    for l in range(L):
        q = f"encoder.layer.{l}."
        y = F.layer_norm(hs, (C,), p[q + n1 + ".weight"], p[q + n1 + ".bias"], eps)
        a = [_linear(y, p[q + f"attention.attention.{n}.weight"], p[q + f"attention.attention.{n}.bias"]) for n in ("query", "key", "value")]
        sh = lambda t: t.view(B, -1, heads, C // heads).transpose(1, 2)
        att = F.scaled_dot_product_attention(sh(a[0]), sh(a[1]), sh(a[2]), scale=0.125).transpose(1, 2).reshape(B, -1, C)
        o = _linear(att, p[q + "attention.output.dense.weight"], p[q + "attention.output.dense.bias"])
        hs = (o if vit else o * p[q + "layer_scale1.lambda1"]) + hs
        y = F.layer_norm(hs, (C,), p[q + n2 + ".weight"], p[q + n2 + ".bias"], eps)
        if vit:
            f = _linear(F.gelu(_linear(y, p[q + "intermediate.dense.weight"], p[q + "intermediate.dense.bias"])),
                        p[q + "output.dense.weight"], p[q + "output.dense.bias"])
        else:
            f = _linear(F.gelu(_linear(y, p[q + "mlp.fc1.weight"], p[q + "mlp.fc1.bias"])), p[q + "mlp.fc2.weight"], p[q + "mlp.fc2.bias"])
        hs = (f if vit else f * p[q + "layer_scale2.lambda1"]) + hs
    hs = F.layer_norm(hs, (C,), p["layernorm.weight"], p["layernorm.bias"], eps)
    return hs[:, 1:]


ON_PATH_EXCLUDED = ("embeddings.mask_token", "pooler.")


def encoder_params(sd: Dict[str, torch.Tensor], prefix: str = "adapter.model.") -> Dict[str, torch.Tensor]:
    """fp32 leaf copies (requires_grad) of the backbone parameters of a state dict, keyed without `prefix`; the ones off the forward
    path (mask_token, ViT's pooler) are left out, as they get no gradient in the reference."""
    out = {}
    for k, v in sd.items():
        if k.startswith(prefix):
            n = k[len(prefix):]
            if not n.startswith(ON_PATH_EXCLUDED):
                out[n] = v.detach().clone().float().requires_grad_(True)
    return out
