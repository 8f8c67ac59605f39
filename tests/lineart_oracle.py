"""LineArt (reference condition/lineart.py:8-86): procedural weights, seeded inputs and a CPU restatement of the decomposition the
CUDA kernels implement (csrc/lineart.cuh, car_vision.cu: car_lineart_forward):
  - padding materialised by index (reflection / zeros) before every convolution,
  - every convolution a window convolution over the pre-padded tensor (no padding inside the convolution),
  - ConvTranspose2d(3, stride 2, pad 1, output_padding 1) as four sub-pixel stride-1 convolutions over the input with one zero row /
    column appended at the bottom / right, with the weights repacked per parity class,
  - instance-norm statistics in two passes (mean, then centred squares), eps 1e-5.
It runs in fp64, so it pins the decomposition itself against the reference's fp32 output (tests/golden/lineart.pt)."""
from __future__ import annotations

from typing import Dict, List

import torch

# (key, shape) in state-dict order; model3.* are ConvTranspose2d weights [Cin][Cout][3][3]
LINEART_SHAPES = [("model0.1", (64, 3, 7, 7)), ("model1.0", (128, 64, 3, 3)), ("model1.3", (256, 128, 3, 3))] + \
    [(f"model2.{r}.conv_block.{i}", (256, 256, 3, 3)) for r in range(3) for i in (1, 5)] + \
    [("model3.0", (256, 128, 3, 3)), ("model3.3", (128, 64, 3, 3)), ("model4.1", (1, 64, 7, 7))]


def make_lineart_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """He-scaled convolution weights and small biases (4 290 945 parameters, regenerated from the seed, never stored).  The head is
    scaled up so that the pre-sigmoid map spreads over roughly +-4: the comparison is then not made in saturated sigmoid tails."""
    sd: Dict[str, torch.Tensor] = {}
    for i, (key, shape) in enumerate(LINEART_SHAPES):
        g = torch.Generator().manual_seed(seed * 1000 + i)
        fan_in = (shape[0] if key.startswith("model3.") else shape[1]) * shape[2] * shape[3]
        std = (2.0 / fan_in) ** 0.5 * (2.0 if key == "model4.1" else 1.0)
        cout = shape[1] if key.startswith("model3.") else shape[0]
        sd[key + ".weight"] = torch.randn(shape, generator=g) * std
        sd[key + ".bias"] = torch.randn(cout, generator=g) * 0.1
    return sd


def lineart_inputs() -> Dict[str, torch.Tensor]:
    """Seeded (B, 3, H, W) float images in 0..255: a batch, an odd size (70 x 90 -> 72 x 92 out), the smallest accepted size
    (5 x 7 -> 8 x 8) and one image at the size the product runs (512 x 512)."""
    g = torch.Generator().manual_seed(29)

    def img(B, H, W):
        base = torch.rand(B, 3, H // 4 + 2, W // 4 + 2, generator=g)
        up = torch.nn.functional.interpolate(base, size=(H, W), mode="bicubic", align_corners=False)
        return (up * 255 + torch.randn(B, 3, H, W, generator=g) * 4).clamp(0, 255).round()
    return {"b2_96x128": img(2, 96, 128), "b1_70x90": img(1, 70, 90), "b1_5x7": img(1, 5, 7), "b1_512x512": img(1, 512, 512)}


# (y0, x0, h, w) windows of the 512 x 512 output map kept in tests/golden/lineart.pt: the four corners (reflection borders of the stem
# and the head), the four edge middles and the centre
GOLDEN_WINDOWS_512 = [(0, 0, 64, 64), (0, 448, 64, 64), (448, 0, 64, 64), (448, 448, 64, 64),
                      (0, 224, 64, 64), (224, 0, 64, 64), (224, 448, 64, 64), (448, 224, 64, 64), (192, 192, 128, 128)]


def golden_max_abs(g, name: str, y: torch.Tensor) -> float:
    """Max-abs of an output map y (B, 1, Ho, Wo) against the reference's fp32 output stored for input `name` in
    tests/golden/lineart.pt: the whole map, or for the 512 x 512 input the stored windows of it."""
    assert tuple(y.shape) == tuple(g[name + "_shape"]), (name, tuple(y.shape), g[name + "_shape"])
    y = y.detach().cpu().to(torch.float64)
    if name in g:
        return (y - g[name].to(torch.float64)).abs().max().item()
    return max((y[..., y0:y0 + h, x0:x0 + w] - t.to(torch.float64)).abs().max().item() for (y0, x0, h, w), t in g[name + "_windows"])


def _reflect_idx(n: int, pad: int) -> torch.Tensor:
    i = torch.arange(-pad, n + pad)
    return torch.where(i < 0, -i, torch.where(i >= n, 2 * n - 2 - i, i))


def pad_reflect(x: torch.Tensor, p: int) -> torch.Tensor:
    return x[:, :, _reflect_idx(x.shape[2], p)][:, :, :, _reflect_idx(x.shape[3], p)]


def pad_zero(x: torch.Tensor, top: int, left: int, bottom: int, right: int) -> torch.Tensor:
    B, C, H, W = x.shape
    y = x.new_zeros(B, C, H + top + bottom, W + left + right)
    y[:, :, top:top + H, left:left + W] = x
    return y


def window_conv(xp: torch.Tensor, w: torch.Tensor, b: torch.Tensor, stride: int, Ho: int, Wo: int) -> torch.Tensor:
    """out[b, o, y, x] = bias[o] + sum_{c, ky, kx} w[o, c, ky, kx] * xp[b, c, stride*y + ky, stride*x + kx] (xp already padded)."""
    kh, kw = w.shape[2], w.shape[3]
    out = b.view(1, -1, 1, 1).expand(xp.shape[0], -1, Ho, Wo).clone()
    for ky in range(kh):
        for kx in range(kw):
            win = xp[:, :, ky: ky + stride * (Ho - 1) + 1: stride, kx: kx + stride * (Wo - 1) + 1: stride]
            out += torch.einsum("bchw,oc->bohw", win, w[:, :, ky, kx])
    return out


def convT_class_weights(w: torch.Tensor) -> List[torch.Tensor]:
    """[Cin][Cout][3][3] -> per parity class (a, b) in the order (0,0) (0,1) (1,0) (1,1) a [Cout][Cin][1+a][1+b] window weight: even
    outputs 2i take tap 1 of input i; odd outputs 2i+1 take tap 2 of input i (window tap 0) and tap 0 of input i+1 (window tap 1)."""
    taps = {0: [1], 1: [2, 0]}
    return [w[:, :, taps[a]][:, :, :, taps[b]].permute(1, 0, 2, 3).contiguous() for a in (0, 1) for b in (0, 1)]


def conv_transpose_subpixel(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    B, _, H, W = x.shape
    xp = pad_zero(x, 0, 0, 1, 1)
    out = x.new_empty(B, w.shape[1], 2 * H, 2 * W)
    for cls, wc in enumerate(convT_class_weights(w)):
        a, bb = cls >> 1, cls & 1
        out[:, :, a::2, bb::2] = window_conv(xp, wc, b, 1, H, W)
    return out


def instance_norm(x: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    mean = x.mean(dim=(2, 3), keepdim=True)
    var = ((x - mean) ** 2).mean(dim=(2, 3), keepdim=True)
    return (x - mean) / torch.sqrt(var + eps)


@torch.no_grad()
def lineart_oracle(sd: Dict[str, torch.Tensor], x: torch.Tensor, dtype=torch.float64, cast: bool = True) -> torch.Tensor:
    """(B, 3, H, W) in 0..255 -> (B, 1, 4 ceil(H/4), 4 ceil(W/4)) in [0, 1], returned as fp32 (as `dtype` when cast is False)."""
    p = {k: v.to(dtype) for k, v in sd.items()}
    W_ = lambda k: (p[k + ".weight"], p[k + ".bias"])      # noqa: E731
    h = x.to(dtype)
    H, Wd = h.shape[2], h.shape[3]
    h = torch.relu(instance_norm(window_conv(pad_reflect(h, 3), *W_("model0.1"), 1, H, Wd)))
    for k in ("model1.0", "model1.3"):
        H, Wd = (H + 1) // 2, (Wd + 1) // 2
        h = torch.relu(instance_norm(window_conv(pad_zero(h, 1, 1, 1, 1), *W_(k), 2, H, Wd)))
    for r in range(3):
        t = torch.relu(instance_norm(window_conv(pad_reflect(h, 1), *W_(f"model2.{r}.conv_block.1"), 1, H, Wd)))
        h = h + instance_norm(window_conv(pad_reflect(t, 1), *W_(f"model2.{r}.conv_block.5"), 1, H, Wd))
    for k in ("model3.0", "model3.3"):
        h = torch.relu(instance_norm(conv_transpose_subpixel(h, *W_(k))))
    H, Wd = h.shape[2], h.shape[3]
    y = torch.sigmoid(window_conv(pad_reflect(h, 3), *W_("model4.1"), 1, H, Wd))
    return y.float() if cast else y
