"""MiDaS DPT-Hybrid depth detector (reference condition/midas, DPTDepthModel with backbone vitb_rn50_384): procedural weights, seeded
inputs and an fp64 torch restatement of the decomposition the CUDA kernels implement (csrc/midas.cuh, dpt.cuh, car_vision.cu:
car_midas_forward):
  - weight standardisation per output channel with biased variance and eps 1e-8,
  - TF "SAME" padding written out: 7x7/2 stem (2 before, 3 after), 3x3/2 convolutions and the max-pool (0 before, 1 after), none
    for the 1x1/2 downsample,
  - GroupNorm(32, eps 1e-5) with the downsample shortcut normalised before the residual add,
  - position embeddings resized bilinearly (align_corners=False) to a non-square h x w grid, q scaled by 1/8 before the product,
  - the readout projection over cat(token, [CLS]).
It runs on the CPU or on CUDA, in fp64 by default, and pins the decomposition against the reference's own output
(tests/golden/midas.pt)."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

DEPTHS, WIDTHS = (3, 4, 9), (256, 512, 1024)


def midas_keys_and_shapes():
    from controlar_b200.condition.midas import DPTDepthModel
    with torch.device("meta"):
        m = DPTDepthModel()
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


def midas_image(H: int, W: int, seed: int, uint8: bool = True) -> torch.Tensor:
    """Seeded (H, W, 3) image in 0..255 (uint8, or float32 with fractions): smooth structure plus pixel noise."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(1, 3, H // 16 + 2, W // 16 + 2, generator=g)
    up = F.interpolate(base, size=(H, W), mode="bicubic", align_corners=False)[0].permute(1, 2, 0)
    img = ((up + torch.randn(H, W, 3, generator=g) * 0.03) * 255).clamp(0, 255)
    return img.round().to(torch.uint8) if uint8 else img.float()


def midas_input(image: torch.Tensor) -> torch.Tensor:
    """MidasDetector's pre-processing: (H, W, 3) in 0..255 -> (1, 3, H, W) in [-1, 1]."""
    return (image / 127.5 - 1.0).permute(2, 0, 1).unsqueeze(0)


def make_midas_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Fan-in-scaled weights, norm gains 1 +- 0.1, biases N(0, 0.05), cls and position embeddings N(0, 0.5).  scratch.output_conv.4.bias
    is re-centred on the median plus half the standard deviation of the pre-ReLU map of a 64 x 96 input, so that about a quarter of
    the map is exactly 0 and the rest is spread out."""
    sd: Dict[str, torch.Tensor] = {}
    for i, (k, shape) in enumerate(midas_keys_and_shapes()):
        g = torch.Generator().manual_seed(seed * 100003 + i)
        if k.endswith(("cls_token", "pos_embed")):
            v = torch.randn(shape, generator=g) * 0.5
        elif "norm" in k and k.endswith(".weight"):
            v = 1 + torch.randn(shape, generator=g) * 0.1
        elif len(shape) == 1:
            v = torch.randn(shape, generator=g) * 0.05
        else:
            fan_in = shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1)
            v = torch.randn(shape, generator=g) / fan_in ** 0.5
        sd[k] = v.float()
    sd["scratch.output_conv.4.bias"] = torch.zeros(1)
    pre = midas_oracle(sd, midas_input(midas_image(64, 96, 1000 + seed)), pre_relu=True).flatten()
    sd["scratch.output_conv.4.bias"] = (-(pre.median() + 0.5 * pre.std())).reshape(1).float()
    return sd


def windows(y: torch.Tensor):
    """(y0, x0) 32 x 32 windows of an H x W map kept in tests/golden/midas.pt: the four corners and the centre."""
    H, W = y.shape[-2:]
    at = [(0, 0), (0, W - 32), (H - 32, 0), (H - 32, W - 32), (H // 2 - 16, W // 2 - 16)]
    return [y[..., a:a + 32, b:b + 32].clone() for a, b in at]


@torch.no_grad()
def midas_oracle(sd: Dict[str, torch.Tensor], x: torch.Tensor, dtype=torch.float64, pre_relu: bool = False) -> torch.Tensor:
    """x (B, 3, H, W) in [-1, 1] -> depth (B, H, W) in `dtype`, on x's device."""
    p = {k: v.to(device=x.device, dtype=dtype) for k, v in sd.items()}
    x = x.to(dtype)
    B, _, H, W = x.shape
    h, w, C = H // 16, W // 16, 768

    def ws(k):
        wt = p[k]
        f = wt.reshape(wt.shape[0], -1)
        m = f.mean(1, keepdim=True)
        return ((f - m) / torch.sqrt(((f - m) ** 2).mean(1, keepdim=True) + 1e-8)).reshape_as(wt)

    def gn(t, k, relu=True):
        t = F.group_norm(t, 32, p[k + ".weight"], p[k + ".bias"], 1e-5)
        return torch.relu(t) if relu else t

    bb = "pretrained.model.patch_embed.backbone."
    t = F.conv2d(F.pad(x, (2, 3, 2, 3)), ws(bb + "stem.conv.weight"), stride=2)
    t = F.max_pool2d(F.pad(gn(t, bb + "stem.norm"), (0, 1, 0, 1)), 3, 2)
    feats = []
    for s, d in enumerate(DEPTHS):
        for b in range(d):
            q = bb + f"stages.{s}.blocks.{b}."
            stride = 2 if (s and b == 0) else 1
            if b == 0:
                sc = gn(F.conv2d(t, ws(q + "downsample.conv.weight"), stride=stride), q + "downsample.norm", relu=False)
            else:
                sc = t
            u = gn(F.conv2d(t, ws(q + "conv1.weight")), q + "norm1")
            u = F.conv2d(u, ws(q + "conv2.weight"), padding=1) if stride == 1 else F.conv2d(F.pad(u, (0, 1, 0, 1)), ws(q + "conv2.weight"), stride=2)
            u = gn(F.conv2d(gn(u, q + "norm2"), ws(q + "conv3.weight")), q + "norm3", relu=False)
            t = torch.relu(u + sc)
        if s < 2:
            feats.append(t)
    # ViT-B/16 over the stage-2 map
    pm = "pretrained.model."
    tok = F.conv2d(t, p[pm + "patch_embed.proj.weight"], p[pm + "patch_embed.proj.bias"]).flatten(2).transpose(1, 2)
    pos = p[pm + "pos_embed"]
    grid = F.interpolate(pos[0, 1:].reshape(1, 24, 24, C).permute(0, 3, 1, 2), size=(h, w), mode="bilinear", align_corners=False)
    pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, h * w, C)], 1)
    X = torch.cat([p[pm + "cls_token"].expand(B, 1, C), tok], 1) + pos
    T = X.shape[1]
    lin = lambda t, k: F.linear(t, p[k + ".weight"], p[k + ".bias"])          # noqa: E731
    outs = []
    for l in range(12):
        q = pm + f"blocks.{l}."
        y = F.layer_norm(X, (C,), p[q + "norm1.weight"], p[q + "norm1.bias"], 1e-6)
        qq, kk, vv = lin(y, q + "attn.qkv").reshape(B, T, 3, 12, 64).permute(2, 0, 3, 1, 4)
        ctx = (torch.softmax((qq * 0.125) @ kk.transpose(-1, -2), -1) @ vv).transpose(1, 2).reshape(B, T, C)
        X = lin(ctx, q + "attn.proj") + X
        y = F.layer_norm(X, (C,), p[q + "norm2.weight"], p[q + "norm2.bias"], 1e-6)
        X = lin(F.gelu(lin(y, q + "mlp.fc1")), q + "mlp.fc2") + X
        if l in (8, 11):
            outs.append(X)
    for i, Xi in enumerate(outs):
        a = f"pretrained.act_postprocess{3 + i}."
        tk = Xi[:, 1:]
        z = F.gelu(lin(torch.cat([tk, Xi[:, :1].expand_as(tk)], -1), a + "0.project.0"))
        z = F.conv2d(z.transpose(1, 2).reshape(B, C, h, w), p[a + "3.weight"], p[a + "3.bias"])
        if i == 1:
            z = F.conv2d(z, p[a + "4.weight"], p[a + "4.bias"], stride=2, padding=1)
        feats.append(z)
    rn = [F.conv2d(f, p[f"scratch.layer{i + 1}_rn.weight"], padding=1) for i, f in enumerate(feats)]

    def rcu(t, k):
        u = F.conv2d(torch.relu(t), p[k + ".conv1.weight"], p[k + ".conv1.bias"], padding=1)
        return F.conv2d(torch.relu(u), p[k + ".conv2.weight"], p[k + ".conv2.bias"], padding=1) + t
    prev = None
    for r in (4, 3, 2, 1):
        k = f"scratch.refinenet{r}"
        t = rn[r - 1] if prev is None else prev + rcu(rn[r - 1], k + ".resConfUnit1")
        t = F.interpolate(rcu(t, k + ".resConfUnit2"), scale_factor=2, mode="bilinear", align_corners=True)
        prev = F.conv2d(t, p[k + ".out_conv.weight"], p[k + ".out_conv.bias"])
    o = "scratch.output_conv."
    y = F.conv2d(prev, p[o + "0.weight"], p[o + "0.bias"], padding=1)
    y = F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=True)
    y = torch.relu(F.conv2d(y, p[o + "2.weight"], p[o + "2.bias"], padding=1))
    y = F.conv2d(y, p[o + "4.weight"], p[o + "4.bias"]).squeeze(1)
    return y if pre_relu else torch.relu(y)
