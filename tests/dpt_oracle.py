"""DPT depth detector (transformers DPTForDepthEstimation, Intel/dpt-large): configurations, procedural weights, seeded inputs and
an fp64 torch restatement of the decomposition the CUDA kernels implement (csrc/dpt.cuh, car_vision.cu: car_dpt_forward):
  - the 16x16/16 patch convolution as a GEMM over (c, ky, kx) patches, position embeddings resized bilinearly (align_corners=False),
  - attention with q scaled by 1/8 before the product,
  - the readout projection over the materialised concatenation cat(token, [CLS]),
  - ConvTranspose2d(k = s = f) as one GEMM with N = f^2 Cout followed by a pixel shuffle.
It runs on the CPU or on CUDA, in fp64 by default, and pins the decomposition against HF's own output (tests/golden/dpt.pt)."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

DPT_LARGE = dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096, image_size=384, patch_size=16,
                 backbone_out_indices=[5, 11, 17, 23], neck_hidden_sizes=[256, 512, 1024, 1024], fusion_hidden_size=256,
                 readout_type="project", reassemble_factors=[4, 2, 1, 0.5], layer_norm_eps=1e-12, hidden_act="gelu", qkv_bias=True)
# small network: every stage of DPT-Large, and a 6 x 6 position grid that the 128 x 128 input resizes to 8 x 8
DPT_SMALL = dict(DPT_LARGE, hidden_size=256, num_hidden_layers=4, num_attention_heads=4, intermediate_size=1024, image_size=96,
                 backbone_out_indices=[0, 1, 2, 3], neck_hidden_sizes=[64, 64, 128, 128], fusion_hidden_size=128)


def dpt_keys_and_shapes(config):
    from controlar_b200.condition.depth import DPTForDepthEstimation
    with torch.device("meta"):
        m = DPTForDepthEstimation(config)
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def dpt_input(B: int, side: int, seed: int) -> torch.Tensor:
    """Seeded pixel_values in [-1, 1] (DPTImageProcessor's range): smooth structure plus pixel noise."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(B, 3, side // 16 + 2, side // 16 + 2, generator=g)
    up = F.interpolate(base, size=(side, side), mode="bicubic", align_corners=False)
    return ((up + torch.randn(B, 3, side, side, generator=g) * 0.02) * 2 - 1).clamp(-1, 1)


def make_dpt_state_dict(config, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Fan-in-scaled weights, LayerNorm gains 1 +- 0.1, biases N(0, 0.05), cls and position embeddings N(0, 0.5).  HF's own N(0, 0.02)
    init leaves almost the whole map at 0 after the final ReLU, so head.head.4.bias is re-centred on the median plus half the standard
    deviation of the pre-ReLU map of a 64 x 64 input: about a quarter of the output is then exactly 0, the rest spread out."""
    sd: Dict[str, torch.Tensor] = {}
    for i, (k, shape) in enumerate(dpt_keys_and_shapes(config)):
        g = torch.Generator().manual_seed(seed * 100003 + i)
        if k.endswith(("cls_token", "position_embeddings")):
            v = torch.randn(shape, generator=g) * 0.5
        elif ("layernorm" in k) and k.endswith(".weight"):
            v = 1 + torch.randn(shape, generator=g) * 0.1
        elif len(shape) == 1:
            v = torch.randn(shape, generator=g) * 0.05
        else:
            fan_in = shape[0] if k.endswith("resize.weight") and len(shape) == 4 and "layers.3." not in k else \
                shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1)
            v = torch.randn(shape, generator=g) / fan_in ** 0.5
        sd[k] = v.float()
    sd["head.head.4.bias"] = torch.zeros(1)
    pre = dpt_oracle(sd, config, dpt_input(1, 64, 1000 + seed), pre_relu=True).flatten()
    sd["head.head.4.bias"] = (-(pre.median() + 0.5 * pre.std())).reshape(1).float()
    return sd


def golden_windows(side: int):
    """(y0, x0, h, w) windows of a side x side map kept in tests/golden/dpt.pt for the DPT-Large cases: the four 32 x 32 corners,
    the four 32 x 32 edge middles and the 64 x 64 centre (the whole maps stay out of the fixture to keep it small; the GPU test
    compares the whole 512 x 512 map with this oracle instead)."""
    e, m = side - 32, side // 2 - 16
    return [(0, 0, 32, 32), (0, e, 32, 32), (e, 0, 32, 32), (e, e, 32, 32), (0, m, 32, 32), (m, 0, 32, 32), (m, e, 32, 32),
            (e, m, 32, 32), (side // 2 - 32, side // 2 - 32, 64, 64)]


def windows(y: torch.Tensor):
    return [y[..., y0:y0 + h, x0:x0 + w].clone() for (y0, x0, h, w) in golden_windows(y.shape[-1])]


@torch.no_grad()
def dpt_oracle(sd: Dict[str, torch.Tensor], config, x: torch.Tensor, dtype=torch.float64, pre_relu: bool = False) -> torch.Tensor:
    """pixel_values (B, 3, H, W) -> predicted_depth (B, H, W) in `dtype`, on x's device."""
    from controlar_b200.condition.depth import _Cfg
    c = _Cfg(config)
    p = {k: v.to(device=x.device, dtype=dtype) for k, v in sd.items()}
    x = x.to(dtype)
    B, _, H, _ = x.shape
    h, C, g, nh = H // 16, c.hidden_size, c.image_size // 16, c.num_attention_heads
    lin = lambda t, k: F.linear(t, p[k + ".weight"], p[k + ".bias"])          # noqa: E731
    # embeddings
    patches = x.reshape(B, 3, h, 16, h, 16).permute(0, 2, 4, 1, 3, 5).reshape(B, h * h, 768)
    pe = "dpt.embeddings."
    t = patches @ p[pe + "patch_embeddings.projection.weight"].reshape(C, 768).T + p[pe + "patch_embeddings.projection.bias"]
    pos = p[pe + "position_embeddings"]
    grid = F.interpolate(pos[0, 1:].reshape(1, g, g, C).permute(0, 3, 1, 2), size=(h, h), mode="bilinear", align_corners=False)
    pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, h * h, C)], 1)
    X = torch.cat([p[pe + "cls_token"].expand(B, 1, C), t], 1) + pos
    T = X.shape[1]
    outs = []
    for l in range(max(c.backbone_out_indices) + 1):
        q = f"dpt.encoder.layer.{l}."
        y = F.layer_norm(X, (C,), p[q + "layernorm_before.weight"], p[q + "layernorm_before.bias"], c.layer_norm_eps)
        heads = lambda t: t.reshape(B, T, nh, 64).transpose(1, 2)             # noqa: E731
        qq = heads(lin(y, q + "attention.attention.query")) * 0.125
        kk, vv = heads(lin(y, q + "attention.attention.key")), heads(lin(y, q + "attention.attention.value"))
        ctx = (torch.softmax(qq @ kk.transpose(-1, -2), -1) @ vv).transpose(1, 2).reshape(B, T, C)
        X = lin(ctx, q + "attention.output.dense") + X
        y = F.layer_norm(X, (C,), p[q + "layernorm_after.weight"], p[q + "layernorm_after.bias"], c.layer_norm_eps)
        X = lin(F.gelu(lin(y, q + "intermediate.dense")), q + "output.dense") + X
        if l in c.backbone_out_indices:
            outs.append(X)
    # reassemble + neck convolutions
    feats = []
    for i, (Xi, f) in enumerate(zip(outs, (4, 2, 1, 0))):
        r = "neck.reassemble_stage."
        tok = Xi[:, 1:]
        z = F.gelu(lin(torch.cat([tok, Xi[:, :1].expand_as(tok)], -1), r + f"readout_projects.{i}.0"))
        w = p[r + f"layers.{i}.projection.weight"]
        Cn = w.shape[0]
        z = F.linear(z, w.reshape(Cn, C), p[r + f"layers.{i}.projection.bias"])                 # [B, h^2, Cn]
        if f > 1:
            wt = p[r + f"layers.{i}.resize.weight"]                                               # [Cin][Cout][f][f]
            zz = z @ wt.permute(0, 2, 3, 1).reshape(Cn, f * f * Cn) + p[r + f"layers.{i}.resize.bias"].repeat(f * f)
            z = zz.reshape(B, h, h, f, f, Cn).permute(0, 5, 1, 3, 2, 4).reshape(B, Cn, f * h, f * h)
        else:
            z = z.reshape(B, h, h, Cn).permute(0, 3, 1, 2)
            if f == 0:
                z = F.conv2d(z, p[r + f"layers.{i}.resize.weight"], p[r + f"layers.{i}.resize.bias"], stride=2, padding=1)
        feats.append(F.conv2d(z, p[f"neck.convs.{i}.weight"], padding=1))

    def rcu(t, k):
        u = F.conv2d(torch.relu(t), p[k + ".convolution1.weight"], p[k + ".convolution1.bias"], padding=1)
        return F.conv2d(torch.relu(u), p[k + ".convolution2.weight"], p[k + ".convolution2.bias"], padding=1) + t
    prev = None
    for j in range(4):
        k = f"neck.fusion_stage.layers.{j}"
        t = feats[3 - j] if prev is None else prev + rcu(feats[3 - j], k + ".residual_layer1")
        t = F.interpolate(rcu(t, k + ".residual_layer2"), scale_factor=2, mode="bilinear", align_corners=True)
        prev = F.conv2d(t, p[k + ".projection.weight"], p[k + ".projection.bias"])
    y = F.conv2d(prev, p["head.head.0.weight"], p["head.head.0.bias"], padding=1)
    y = F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=True)
    y = torch.relu(F.conv2d(y, p["head.head.2.weight"], p["head.head.2.bias"], padding=1))
    y = F.conv2d(y, p["head.head.4.weight"], p["head.head.4.bias"]).squeeze(1)
    return y if pre_relu else torch.relu(y)
