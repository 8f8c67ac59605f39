"""DPT depth detector on the GPU — the surface of transformers' `DPTForDepthEstimation` (Intel/dpt-large) that the reference's
sampling scripts use (`model = DPTForDepthEstimation.from_pretrained(dir)`, `model(**processor(...))`, `outputs.predicted_depth`),
without importing transformers.  The module is a parameter container with HF's state-dict keys and shapes; the forward runs
`car_dpt_forward` (csrc/dpt.cuh, car_vision.cu): the reference runs this network in fp32, and here every GEMM and convolution runs
on the fp32-grade split-bf16 tensor-core path with activations, LayerNorm, soft-max, resampling and the head in fp32.  No autograd
and no CPU path.

Supported: the non-hybrid ViT DPT with readout "project", reassemble factors [4, 2, 1, 0.5], 64-dimensional heads, exact GELU,
qkv bias, four backbone out indices, no batch norm in the fusion residual units, no head projection, head_in_index -1 and no ignored
neck stages; neck sizes and half the fusion size multiples of 64.  Inputs are square, the side a multiple of 32 and at least 64
(HF's reassemble stage assumes a square token grid; the sampling scripts pass multiples of 32, and an even token grid lines the
stride-2 stage up with the next fusion stage)."""
from __future__ import annotations

import ctypes as C
import json
import os

import torch
import torch.nn as nn

from .. import _lib
from .._lib import check, cur_stream, _ptr, _ptr_array

# transformers DPTConfig defaults for the fields read here (a config.json written by transformers lists them all)
_DEFAULTS = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
                 layer_norm_eps=1e-12, image_size=384, patch_size=16, num_channels=3, is_hybrid=False, qkv_bias=True,
                 backbone_out_indices=[2, 5, 8, 11], readout_type="project", reassemble_factors=[4, 2, 1, 0.5],
                 neck_hidden_sizes=[96, 192, 384, 768], fusion_hidden_size=256, head_in_index=-1,
                 use_batch_norm_in_fusion_residual=False, use_bias_in_fusion_residual=None, add_projection=False,
                 neck_ignore_stages=[], backbone_config=None, backbone=None)


class _Cfg:
    def __init__(self, config):
        get = (lambda k: config.get(k, _DEFAULTS[k])) if isinstance(config, dict) else (lambda k: getattr(config, k, _DEFAULTS[k]))
        for k in _DEFAULTS:
            setattr(self, k, get(k))

    def check(self):
        def need(ok, field, rule):
            if not ok:
                raise NotImplementedError(f"controlar_b200 DPTForDepthEstimation: {field}={getattr(self, field)!r} is not supported ({rule})")
        need(not self.is_hybrid, "is_hybrid", "the ViT backbone only")
        need(self.backbone_config is None, "backbone_config", "the built-in ViT backbone only")
        need(self.backbone is None, "backbone", "the built-in ViT backbone only")
        need(self.readout_type == "project", "readout_type", "'project' only")
        need([float(f) for f in self.reassemble_factors] == [4.0, 2.0, 1.0, 0.5], "reassemble_factors", "[4, 2, 1, 0.5] only")
        need(self.hidden_size == 64 * self.num_attention_heads, "num_attention_heads", "heads of 64 dimensions only")
        need(self.hidden_act == "gelu", "hidden_act", "'gelu' (erf) only")
        need(bool(self.qkv_bias), "qkv_bias", "True only")
        need(len(self.backbone_out_indices) == 4 and list(self.backbone_out_indices) == sorted(set(self.backbone_out_indices))
             and 0 <= min(self.backbone_out_indices) and max(self.backbone_out_indices) < self.num_hidden_layers,
             "backbone_out_indices", "four ascending encoder layers")
        need(not self.use_batch_norm_in_fusion_residual, "use_batch_norm_in_fusion_residual", "False only")
        need(self.use_bias_in_fusion_residual in (None, True), "use_bias_in_fusion_residual", "None or True only")
        need(not self.add_projection, "add_projection", "False only")
        need(self.head_in_index == -1, "head_in_index", "-1 only")
        need(len(self.neck_ignore_stages) == 0, "neck_ignore_stages", "empty only")
        need(self.num_channels == 3, "num_channels", "3 only")
        need(self.patch_size == 16, "patch_size", "16 only")
        need(self.image_size % 16 == 0, "image_size", "a multiple of the patch size")
        need(self.intermediate_size % 8 == 0, "intermediate_size", "a multiple of 8")
        need(len(self.neck_hidden_sizes) == 4 and all(n > 0 and n % 64 == 0 for n in self.neck_hidden_sizes), "neck_hidden_sizes",
             "four multiples of 64")
        need(self.fusion_hidden_size > 0 and self.fusion_hidden_size % 128 == 0, "fusion_hidden_size", "a multiple of 128")


def _conv(cin, cout, k, stride=1, padding=0, bias=True):
    return nn.Conv2d(cin, cout, k, stride=stride, padding=padding, bias=bias)


class _Module(nn.Module):
    pass


class DepthEstimatorOutput(dict):
    """`outputs.predicted_depth`, `outputs["predicted_depth"]` and `outputs[0]`, as transformers' ModelOutput offers them."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None

    def __getitem__(self, k):
        return list(self.values())[k] if isinstance(k, int) else super().__getitem__(k)


class DPTForDepthEstimation(nn.Module):
    """Parameter container with transformers' `DPTForDepthEstimation` keys; forward runs `car_dpt_forward`."""

    def __init__(self, config):
        super().__init__()
        cfg = _Cfg(config)
        cfg.check()
        self.config = cfg
        Cd, L, mlp, eps, g = cfg.hidden_size, cfg.num_hidden_layers, cfg.intermediate_size, cfg.layer_norm_eps, cfg.image_size // 16
        self.dpt = _Module()
        emb = self.dpt.embeddings = _Module()
        emb.cls_token = nn.Parameter(torch.zeros(1, 1, Cd))
        emb.position_embeddings = nn.Parameter(torch.zeros(1, g * g + 1, Cd))
        emb.patch_embeddings = _Module()
        emb.patch_embeddings.projection = _conv(3, Cd, 16, stride=16)
        self.dpt.encoder = _Module()
        layers = []
        for _ in range(L):
            ly = _Module()
            ly.attention = _Module()
            ly.attention.attention = _Module()
            for k in ("query", "key", "value"):
                setattr(ly.attention.attention, k, nn.Linear(Cd, Cd))
            ly.attention.output = _Module()
            ly.attention.output.dense = nn.Linear(Cd, Cd)
            ly.intermediate = _Module()
            ly.intermediate.dense = nn.Linear(Cd, mlp)
            ly.output = _Module()
            ly.output.dense = nn.Linear(mlp, Cd)
            ly.layernorm_before = nn.LayerNorm(Cd, eps=eps)
            ly.layernorm_after = nn.LayerNorm(Cd, eps=eps)
            layers.append(ly)
        self.dpt.encoder.layer = nn.ModuleList(layers)
        self.dpt.layernorm = nn.LayerNorm(Cd, eps=eps)
        self.neck = _Module()
        rs = self.neck.reassemble_stage = _Module()
        rl = []
        for n, f in zip(cfg.neck_hidden_sizes, (4, 2, 1, 0.5)):
            m = _Module()
            m.projection = _conv(Cd, n, 1)
            if f > 1:
                m.resize = nn.ConvTranspose2d(n, n, kernel_size=f, stride=f)
            elif f < 1:
                m.resize = _conv(n, n, 3, stride=2, padding=1)
            rl.append(m)
        rs.layers = nn.ModuleList(rl)
        rs.readout_projects = nn.ModuleList([nn.Sequential(nn.Linear(2 * Cd, Cd), nn.GELU()) for _ in range(4)])
        F = cfg.fusion_hidden_size
        self.neck.convs = nn.ModuleList([_conv(n, F, 3, padding=1, bias=False) for n in cfg.neck_hidden_sizes])
        fs = self.neck.fusion_stage = _Module()
        fl = []
        for _ in range(4):
            m = _Module()
            m.projection = _conv(F, F, 1)
            for r in ("residual_layer1", "residual_layer2"):
                u = _Module()
                u.convolution1 = _conv(F, F, 3, padding=1)
                u.convolution2 = _conv(F, F, 3, padding=1)
                setattr(m, r, u)
            fl.append(m)
        fs.layers = nn.ModuleList(fl)
        self.head = _Module()
        self.head.head = nn.Sequential(_conv(F, F // 2, 3, padding=1), nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True),
                                       _conv(F // 2, 32, 3, padding=1), nn.ReLU(), _conv(32, 1, 1), nn.ReLU())
        self._car_dpt = None

    # ---- constructors
    @classmethod
    def from_pretrained(cls, local_dir, **unused):
        """`config.json` + `model.safetensors` (or `pytorch_model.bin`, loaded with weights_only=True) from a local directory."""
        if not os.path.isdir(local_dir):
            raise FileNotFoundError(f"{local_dir} is not a local directory (controlar_b200 never downloads checkpoints)")
        with open(os.path.join(local_dir, "config.json")) as fh:
            m = cls(json.load(fh))
        st = os.path.join(local_dir, "model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(local_dir, "pytorch_model.bin"), map_location="cpu", weights_only=True)
        missing = [k for k in m.load_state_dict(sd, strict=False).missing_keys if not k.startswith("dpt.layernorm.")]
        if missing:
            raise RuntimeError(f"{local_dir}: checkpoint lacks {len(missing)} parameters, e.g. {missing[:4]}")
        return m.eval()

    @classmethod
    def from_hf(cls, model):
        """Copy of a transformers DPTForDepthEstimation (config and state dict)."""
        m = cls(model.config)
        m.load_state_dict(model.state_dict(), strict=True)
        return m.to(next(model.parameters()).device).eval()

    # ---- native handle
    def _desc(self):
        c = self.config
        d = _lib.CarDptDesc()
        d.hidden, d.n_layers, d.n_heads, d.mlp = c.hidden_size, c.num_hidden_layers, c.num_attention_heads, c.intermediate_size
        for i in range(4):
            d.out_indices[i] = c.backbone_out_indices[i]
            d.neck[i] = c.neck_hidden_sizes[i]
        d.fusion, d.pos_grid, d.ln_eps = c.fusion_hidden_size, c.image_size // 16, c.layer_norm_eps
        return d

    def _create(self, out):
        ts = [p.detach().contiguous() for p in self.parameters()]     # state-dict order
        arr = _ptr_array(ts)
        desc = self._desc()
        check(_lib.lib().car_dpt_create(C.byref(desc), C.cast(arr, C.POINTER(C.c_void_p)), len(ts), cur_stream(), C.byref(out)),
              "car_dpt_create")

    def _handle(self):
        ps = list(self.parameters())
        bad = {p.dtype for p in ps} - {torch.float32}
        if bad:
            raise RuntimeError(f"controlar_b200 DPTForDepthEstimation runs in fp32, as the reference does; parameters are {sorted(map(str, bad))}")
        if self._car_dpt is None:
            object.__setattr__(self, "_car_dpt", _lib.ModuleHandle("car_dpt_destroy"))
        return self._car_dpt.get(ps, self._create)

    def forward(self, pixel_values, labels=None, **unused):
        """pixel_values (B, 3, H, W), H == W, H % 32 == 0, H >= 64 -> DepthEstimatorOutput(predicted_depth=(B, H, W) fp32)."""
        if labels is not None:
            raise NotImplementedError("Training is not implemented yet")
        if pixel_values.dim() != 4 or pixel_values.shape[1] != 3:
            raise ValueError("DPTForDepthEstimation takes pixel_values (B, 3, H, W)")
        B, _, H, W = pixel_values.shape
        if H != W or H % 32 or H < 64:
            raise ValueError(f"pixel_values must be square with a side that is a multiple of 32 and at least 64, got {H} x {W}")
        if pixel_values.device.type != "cuda":
            raise RuntimeError("controlar_b200 DPTForDepthEstimation needs CUDA tensors (no CPU path)")
        x = pixel_values.detach().to(torch.float32).contiguous()
        out = torch.empty(B, H, W, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(_lib.lib().car_dpt_forward(self._handle(), _ptr(x), B, H, W, _ptr(out), cur_stream()), "car_dpt_forward")
        return DepthEstimatorOutput(predicted_depth=out)
