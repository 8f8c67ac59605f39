"""HED soft-edge control-map detector on the GPU — same surface as the reference's `condition/hed.py`: `ControlNetHED_Apache2` (an
nn.Module with the reference's state-dict keys: `norm`, `block{1..5}.convs.{i}.{weight,bias}`, `block{k}.projection.{weight,bias}`)
and `HEDdetector()(input_image)` (tensor (B, C, H, W) in 0..255 -> tensor (B, H, W) in [0, 255]).  The reference runs fp32; the
13 ReLU convolutions here run on the fp32-grade split-bf16 tensor-core path (csrc/split3.cuh "x3"), pooling / projections / resize /
sigmoid in fp32 (csrc/frontend.cuh).  Weights come from the caller (`load_state_dict`) — there is no network to download
ControlNetHED.pth from; `HEDdetector(modelpath=...)` loads a local copy like the reference does."""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.nn as nn

from .. import _lib
from .._lib import check, cur_stream, _ptr, _ptr_array

BLOCKS = ((3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3))


class DoubleConvBlock(nn.Module):
    def __init__(self, input_channel, output_channel, layer_number):
        super().__init__()
        self.convs = nn.Sequential()
        self.convs.append(nn.Conv2d(input_channel, output_channel, (3, 3), (1, 1), padding=1))
        for _ in range(1, layer_number):
            self.convs.append(nn.Conv2d(output_channel, output_channel, (3, 3), (1, 1), padding=1))
        self.projection = nn.Conv2d(output_channel, 1, (1, 1), (1, 1), padding=0)


class ControlNetHED_Apache2(nn.Module):
    """Parameter container with the reference's keys (condition/hed.py:37-45); `__call__` returns the five projections (:47-53)."""

    def __init__(self):
        super().__init__()
        self.norm = nn.Parameter(torch.zeros(size=(1, 3, 1, 1)))
        for b, (cin, cout, n) in enumerate(BLOCKS, start=1):
            setattr(self, f"block{b}", DoubleConvBlock(cin, cout, n))
        self._car_hed = None

    def _tensors(self):
        ts = [self.norm.detach().reshape(3)]
        for b in range(1, 6):
            blk = getattr(self, f"block{b}")
            for conv in blk.convs:
                ts += [conv.weight.detach(), conv.bias.detach()]
            ts += [blk.projection.weight.detach().reshape(-1), blk.projection.bias.detach()]
        return [t.to(torch.float32).contiguous() for t in ts]

    def _create(self, out):
        ts = self._tensors()
        arr = _ptr_array(ts)
        check(_lib.lib().car_hed_create(C.cast(arr, C.POINTER(C.c_void_p)), len(ts), cur_stream(), C.byref(out)), "car_hed_create")

    def _handle(self):
        if self._car_hed is None:
            object.__setattr__(self, "_car_hed", _lib.ModuleHandle("car_hed_destroy"))
        return self._car_hed.get(list(self.parameters()), self._create)

    def run(self, x: torch.Tensor, want_projections: bool = False):
        if x.device.type != "cuda":
            raise RuntimeError("controlar_b200 HED needs CUDA tensors (no CPU path)")
        x = x.to(torch.float32).contiguous()
        B, Cc, H, W = x.shape
        assert Cc == 3, "HED takes RGB images (B, 3, H, W)"
        edge = torch.empty(B, H, W, dtype=torch.float32, device=x.device)
        sizes, h, w = [], H, W
        for _ in range(5):
            sizes.append((h, w)); h //= 2; w //= 2
        proj = torch.empty(sum(B * a * b for a, b in sizes), dtype=torch.float32, device=x.device) if want_projections else None
        with torch.cuda.device(x.device):
            check(_lib.lib().car_hed_forward(self._handle(), _ptr(x), B, H, W, _ptr(edge), None if proj is None else _ptr(proj), cur_stream()),
                  "car_hed_forward")
        if proj is None:
            return edge, None
        out, off = [], 0
        for a, b in sizes:
            out.append(proj[off: off + B * a * b].view(B, 1, a, b)); off += B * a * b
        return edge, tuple(out)

    def __call__(self, x):
        return self.run(x, want_projections=True)[1]


class HEDdetector(nn.Module):
    def __init__(self, modelpath: str | None = None):
        super().__init__()
        self.netNetwork = ControlNetHED_Apache2().float()
        if modelpath is None:
            modelpath = os.path.join(os.path.dirname(__file__), "ckpts", "ControlNetHED.pth")     # the reference's annotator_ckpts_path
        if os.path.exists(modelpath):
            self.netNetwork.load_state_dict(torch.load(modelpath))
        # (the reference downloads the checkpoint here; without a network the caller loads it: det.netNetwork.load_state_dict(...))

    def __call__(self, input_image):
        """input: tensor (B,C,H,W); output: tensor (B,H,W) — reference condition/hed.py:69-84."""
        return self.netNetwork.run(input_image)[0]
