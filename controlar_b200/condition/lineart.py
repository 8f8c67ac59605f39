"""LineArt control-map detector on the GPU — same surface as the reference's `condition/lineart.py`: `ResidualBlock` and
`LineArt(input_nc=3, output_nc=1, n_residual_blocks=3, sigmoid=True)`, nn.Modules with the reference's `nn.Sequential` structure and
state-dict keys (`model0.1`, `model1.{0,3}`, `model2.{0,1,2}.conv_block.{1,5}`, `model3.{0,3}`, `model4.1`, each `.weight` / `.bias`),
so `load_state_dict(torch.load('condition/ckpts/model.pth'))` of the released checkpoint works unchanged.  `forward(x)` takes
(B, 3, H, W) pixels in 0..255 and returns (B, 1, Ho, Wo) in [0, 1], Ho = 4 * ceil(ceil(H / 2) / 2) (likewise Wo).  The reference runs
fp32; here every convolution but the head runs on the fp32-grade split-bf16 tensor-core path (csrc/split3.cuh "x3", csrc/lineart.cuh)
with instance norm, padding and the head in fp32.  No autograd: the reference calls it under no_grad."""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from .. import _lib
from .._lib import check, cur_stream, _ptr, _ptr_array

norm_layer = nn.InstanceNorm2d


class ResidualBlock(nn.Module):
    def __init__(self, in_features):
        super().__init__()
        self.conv_block = nn.Sequential(nn.ReflectionPad2d(1), nn.Conv2d(in_features, in_features, 3), norm_layer(in_features),
                                        nn.ReLU(inplace=True), nn.ReflectionPad2d(1), nn.Conv2d(in_features, in_features, 3),
                                        norm_layer(in_features))


class LineArt(nn.Module):
    """Parameter container with the reference's structure (condition/lineart.py:26-72); forward runs `car_lineart_forward`."""

    def __init__(self, input_nc=3, output_nc=1, n_residual_blocks=3, sigmoid=True):
        super().__init__()
        if (input_nc, output_nc, n_residual_blocks, sigmoid) != (3, 1, 3, True):
            raise NotImplementedError("controlar_b200 LineArt implements the reference's default network only "
                                      "(input_nc=3, output_nc=1, n_residual_blocks=3, sigmoid=True)")
        self.model0 = nn.Sequential(nn.ReflectionPad2d(3), nn.Conv2d(input_nc, 64, 7), norm_layer(64), nn.ReLU(inplace=True))
        model1, cin = [], 64
        for _ in range(2):
            model1 += [nn.Conv2d(cin, cin * 2, 3, stride=2, padding=1), norm_layer(cin * 2), nn.ReLU(inplace=True)]
            cin *= 2
        self.model1 = nn.Sequential(*model1)
        self.model2 = nn.Sequential(*[ResidualBlock(cin) for _ in range(n_residual_blocks)])
        model3 = []
        for _ in range(2):
            model3 += [nn.ConvTranspose2d(cin, cin // 2, 3, stride=2, padding=1, output_padding=1), norm_layer(cin // 2),
                       nn.ReLU(inplace=True)]
            cin //= 2
        self.model3 = nn.Sequential(*model3)
        self.model4 = nn.Sequential(nn.ReflectionPad2d(3), nn.Conv2d(64, output_nc, 7), nn.Sigmoid())
        self._car_lineart = None

    def _create(self, out):
        ts = [p.detach().to(torch.float32).contiguous() for p in self.parameters()]   # state-dict order, 24 tensors
        arr = _ptr_array(ts)
        check(_lib.lib().car_lineart_create(C.cast(arr, C.POINTER(C.c_void_p)), len(ts), cur_stream(), C.byref(out)), "car_lineart_create")

    def _handle(self):
        if self._car_lineart is None:
            object.__setattr__(self, "_car_lineart", _lib.ModuleHandle("car_lineart_destroy"))
        return self._car_lineart.get(list(self.parameters()), self._create)

    @staticmethod
    def output_size(H: int, W: int):
        return 4 * ((H + 3) // 4), 4 * ((W + 3) // 4)

    def forward(self, x, cond=None):
        """input: tensor (B, 3, H, W) in 0..255; output: tensor (B, 1, Ho, Wo) in [0, 1] — reference condition/lineart.py:74-86."""
        if x.device.type != "cuda":
            raise RuntimeError("controlar_b200 LineArt needs CUDA tensors (no CPU path)")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("LineArt takes RGB images (B, 3, H, W)")
        x = x.detach().to(torch.float32).contiguous()
        B, _, H, W = x.shape
        Ho, Wo = self.output_size(H, W)
        out = torch.empty(B, 1, Ho, Wo, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(_lib.lib().car_lineart_forward(self._handle(), _ptr(x), B, H, W, _ptr(out), cur_stream()), "car_lineart_forward")
        return out
