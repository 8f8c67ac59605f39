"""MiDaS DPT-Hybrid depth detector on the GPU — the reference's `condition.midas.depth.MidasDetector` (model_type "dpt_hybrid"),
which the multi-resolution sampler calls for every non-square depth input, plus its `DPTDepthModel(backbone="vitb_rn50_384",
non_negative=True)`.  `DPTDepthModel` is a parameter container with the reference's state-dict keys and order (timm's
`vit_base_resnet50_384` under `pretrained.model`); its forward runs `car_midas_forward` (csrc/midas.cuh, dpt.cuh, car_vision.cu).
The reference runs this network in fp32; here every convolution and GEMM runs on the fp32-grade split-bf16 tensor-core path with
GroupNorm, LayerNorm, soft-max, resampling and the head in fp32.  The convolution weights are standardised once per handle (fp64
statistics) where the reference re-standardises them in fp32 on every call.  No autograd, no CPU path, and no download: a missing
checkpoint raises.  Inputs: H and W multiples of 32 and at least 64, not necessarily equal."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch
import torch.nn as nn

from .. import _lib
from .._lib import check, cur_stream, _ptr, _ptr_array

CKPT_NAME = "dpt_hybrid-midas-501f0c75.pt"
DEPTHS, WIDTHS = (3, 4, 9), (256, 512, 1024)


class _Module(nn.Module):
    pass


def _wsconv(cin, cout, k, stride=1):
    return nn.Conv2d(cin, cout, k, stride=stride, bias=False)


def _bottleneck(cin, cout, stride, first):
    b = _Module()
    mid = cout // 4
    if first:
        b.downsample = _Module()
        b.downsample.conv = _wsconv(cin, cout, 1, stride)
        b.downsample.norm = nn.GroupNorm(32, cout, eps=1e-5)
    b.conv1, b.norm1 = _wsconv(cin, mid, 1), nn.GroupNorm(32, mid, eps=1e-5)
    b.conv2, b.norm2 = _wsconv(mid, mid, 3, stride), nn.GroupNorm(32, mid, eps=1e-5)
    b.conv3, b.norm3 = _wsconv(mid, cout, 1), nn.GroupNorm(32, cout, eps=1e-5)
    return b


def _readout(c):
    r = _Module()
    r.project = nn.Sequential(nn.Linear(2 * c, c), nn.GELU())
    return r


def _rcu(f):
    u = _Module()
    u.conv1 = nn.Conv2d(f, f, 3, padding=1)
    u.conv2 = nn.Conv2d(f, f, 3, padding=1)
    return u


class DPTDepthModel(nn.Module):
    """Parameter container with the keys of the reference's `DPTDepthModel(backbone="vitb_rn50_384", non_negative=True)` (features
    256, readout "project"); forward(x (B, 3, H, W)) -> (B, H, W) fp32 on `car_midas_forward`."""

    def __init__(self):
        super().__init__()
        Cd, F = 768, 256
        self.pretrained = _Module()
        m = self.pretrained.model = _Module()
        m.cls_token = nn.Parameter(torch.zeros(1, 1, Cd))
        m.pos_embed = nn.Parameter(torch.zeros(1, 1 + 24 * 24, Cd))
        m.patch_embed = _Module()
        bb = m.patch_embed.backbone = _Module()
        bb.stem = _Module()
        bb.stem.conv = _wsconv(3, 64, 7, 2)
        bb.stem.norm = nn.GroupNorm(32, 64, eps=1e-5)
        stages, cin = [], 64
        for s, (d, w) in enumerate(zip(DEPTHS, WIDTHS)):
            st = _Module()
            st.blocks = nn.ModuleList([_bottleneck(cin if b == 0 else w, w, 2 if (s and b == 0) else 1, b == 0) for b in range(d)])
            stages.append(st)
            cin = w
        bb.stages = nn.ModuleList(stages)
        m.patch_embed.proj = nn.Conv2d(1024, Cd, 1)
        blocks = []
        for _ in range(12):
            b = _Module()
            b.norm1 = nn.LayerNorm(Cd, eps=1e-6)
            b.attn = _Module()
            b.attn.qkv = nn.Linear(Cd, 3 * Cd)
            b.attn.proj = nn.Linear(Cd, Cd)
            b.norm2 = nn.LayerNorm(Cd, eps=1e-6)
            b.mlp = _Module()
            b.mlp.fc1 = nn.Linear(Cd, 4 * Cd)
            b.mlp.fc2 = nn.Linear(4 * Cd, Cd)
            blocks.append(b)
        m.blocks = nn.ModuleList(blocks)
        m.norm = nn.LayerNorm(Cd, eps=1e-6)                # loaded, unused: the features are taken before it
        m.head = nn.Linear(Cd, 1000)                       # timm's classifier: loaded, unused
        self.pretrained.act_postprocess3 = nn.Sequential(_readout(Cd), nn.Identity(), nn.Identity(), nn.Conv2d(Cd, Cd, 1))
        self.pretrained.act_postprocess4 = nn.Sequential(_readout(Cd), nn.Identity(), nn.Identity(), nn.Conv2d(Cd, Cd, 1),
                                                         nn.Conv2d(Cd, Cd, 3, stride=2, padding=1))
        sc = self.scratch = _Module()
        for i, cin in enumerate((256, 512, Cd, Cd)):
            setattr(sc, f"layer{i + 1}_rn", nn.Conv2d(cin, F, 3, padding=1, bias=False))
        for i in range(1, 5):
            r = _Module()
            r.out_conv = nn.Conv2d(F, F, 1)
            r.resConfUnit1 = _rcu(F)
            r.resConfUnit2 = _rcu(F)
            setattr(sc, f"refinenet{i}", r)
        sc.output_conv = nn.Sequential(nn.Conv2d(F, F // 2, 3, padding=1), nn.Identity(), nn.Conv2d(F // 2, 32, 3, padding=1), nn.ReLU(True),
                                       nn.Conv2d(32, 1, 1), nn.ReLU(True), nn.Identity())
        self._car_midas = None

    def _create(self, out):
        ts = [p.detach().contiguous() for p in self.parameters()]     # state-dict order
        arr = _ptr_array(ts)
        check(_lib.lib().car_midas_create(C.cast(arr, C.POINTER(C.c_void_p)), len(ts), cur_stream(), C.byref(out)), "car_midas_create")

    def _handle(self):
        ps = list(self.parameters())
        bad = {p.dtype for p in ps} - {torch.float32}
        if bad:
            raise RuntimeError(f"controlar_b200 DPTDepthModel runs in fp32, as the reference does; parameters are {sorted(map(str, bad))}")
        if self._car_midas is None:
            object.__setattr__(self, "_car_midas", _lib.ModuleHandle("car_midas_destroy"))
        return self._car_midas.get(ps, self._create)

    def forward(self, x):
        """x (B, 3, H, W), H and W multiples of 32 and at least 64 -> depth (B, H, W) fp32."""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"DPTDepthModel takes x (B, 3, H, W), got {tuple(x.shape)}")
        B, _, H, W = x.shape
        if H % 32 or W % 32 or H < 64 or W < 64:
            raise ValueError(f"x must have H and W multiples of 32 and at least 64, got {H} x {W}")
        if x.device.type != "cuda":
            raise RuntimeError("controlar_b200 DPTDepthModel needs CUDA tensors (no CPU path)")
        x = x.detach().to(torch.float32).contiguous()
        out = torch.empty(B, H, W, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(_lib.lib().car_midas_forward(self._handle(), _ptr(x), B, H, W, _ptr(out), cur_stream()), "car_midas_forward")
        return out


def load_state_dict_file(path):
    """A checkpoint as `BaseModel.load` reads it: a state dict, or {"model": state dict, ...} (weights_only=True)."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if "optimizer" in sd or ("model" in sd and isinstance(sd["model"], dict)):
        sd = sd["model"]
    return sd


class MidasDetector:
    """`MidasDetector(device, model_type="dpt_hybrid")` of the reference (condition/midas/depth.py:176-206): an (H, W, 3) uint8 or
    float tensor in 0..255 -> an (H, W) uint8 numpy depth map.  The checkpoint is read from `model_path`, by default
    condition/ckpts/dpt_hybrid-midas-501f0c75.pt under the working directory (the reference's path when its scripts run from its
    root); it is never downloaded."""

    def __init__(self, device=torch.device("cuda:0"), model_type="dpt_hybrid", model_path=None):
        if model_type != "dpt_hybrid":
            raise NotImplementedError(f"controlar_b200 MidasDetector: model_type {model_type!r} is not supported ('dpt_hybrid' only)")
        path = model_path or os.path.join(os.getcwd(), "condition", "ckpts", CKPT_NAME)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"{path}: MiDaS DPT-Hybrid checkpoint not found (controlar_b200 never downloads checkpoints)")
        self.device = device
        model = DPTDepthModel()
        model.load_state_dict(load_state_dict_file(path), strict=True)
        self.model = model.to(device).eval()

    def __call__(self, input_image, a=np.pi * 2.0, bg_th=0.1):
        if input_image.ndim != 3:
            raise ValueError(f"MidasDetector takes an (H, W, 3) image, got {tuple(input_image.shape)}")
        with torch.no_grad():
            image_depth = input_image / 127.5 - 1.0
            image_depth = image_depth.permute(2, 0, 1).unsqueeze(0)           # rearrange 'h w c -> 1 c h w'
            depth = self.model(image_depth)[0]
            depth_pt = depth.clone()
            depth_pt -= torch.min(depth_pt)
            depth_pt /= torch.max(depth_pt)
            depth_pt = depth_pt.cpu().numpy()
            return (depth_pt * 255.0).clip(0, 255).astype(np.uint8)
