"""Host-side handles for the control encoder (car_dino_*) and the VQGAN tokenizer (car_vq_*)."""
from __future__ import annotations

import ctypes as C
from typing import List

import torch

from . import _lib
from ._lib import check, cur_stream, dtype_code, on_own_device, param_signature, _ptr, _ptr_array


class CarDinoDesc(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("hidden", C.c_int32), ("heads", C.c_int32), ("layers", C.c_int32),
                ("patch", C.c_int32), ("pos_grid", C.c_int32), ("resize_mode", C.c_int32),
                ("adapter_out_dim", C.c_int32), ("eps", C.c_float)]


_DINO_ARRAYS = ["n1_w", "n1_b", "q_w", "q_b", "k_w", "k_b", "v_w", "v_b", "o_w", "o_b", "ls1", "n2_w", "n2_b",
                "fc1_w", "fc1_b", "fc2_w", "fc2_b", "ls2"]


class CarDinoWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ["cls_token", "pos_emb", "patch_w", "patch_b", "ln_w", "ln_b"]] + \
               [(n, C.POINTER(C.c_void_p)) for n in _DINO_ARRAYS] + \
               [("adapter_fc1", C.c_void_p), ("adapter_fc2", C.c_void_p)]


class CarVQDesc(C.Structure):
    _fields_ = [("codebook_size", C.c_int32), ("embed_dim", C.c_int32), ("ch", C.c_int32), ("z_channels", C.c_int32),
                ("n_levels", C.c_int32), ("num_res_blocks", C.c_int32), ("ch_mult", C.c_int32 * 8)]


_PROTOS = {
    "car_dino_create": (C.c_int, [C.POINTER(CarDinoDesc), C.POINTER(CarDinoWeights), C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_dino_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "car_dino_destroy": (C.c_int, [C.c_void_p]),
    "car_vq_create": (C.c_int, [C.POINTER(CarVQDesc), C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "car_vq_decode_code": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_vq_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "car_resize_bilinear_aa": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                         C.c_void_p, C.c_void_p]),
    "car_vq_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "car_vq_destroy": (C.c_int, [C.c_void_p]),
}
_lib.PROTOTYPES.update(_PROTOS)


# ---------------------------------------------------------------------------------------------------------------
# DINOv2
# ---------------------------------------------------------------------------------------------------------------
def _dev_of(module):
    return next(module.parameters()).device


class DinoHandle(_lib.ModuleHandle):
    def __init__(self, adapter, adapter_mlp=None):
        super().__init__("car_dino_destroy")
        self.lib = _lib.lib()
        self.adapter, self.adapter_mlp = adapter, adapter_mlp
        self._build()

    @property
    def device(self):
        return _dev_of(self.adapter)

    def _params(self):
        ps = list(self.adapter.model.parameters())
        if self.adapter_mlp is not None:
            ps += list(self.adapter_mlp.parameters())
        return ps

    @on_own_device
    def _build(self):
        m = self.adapter.model
        dt = m.layernorm.weight.dtype
        keep = []

        def P(t):
            t = t.detach().contiguous()
            keep.append(t)
            return _ptr(t)
        w = CarDinoWeights()
        e = m.embeddings
        w.cls_token, w.pos_emb = P(e.cls_token), P(e.position_embeddings)
        w.patch_w, w.patch_b = P(e.patch_embeddings.projection.weight), P(e.patch_embeddings.projection.bias)
        w.ln_w, w.ln_b = P(m.layernorm.weight), P(m.layernorm.bias)
        layers = list(m.encoder.layer)
        is_vit = hasattr(layers[0], "layernorm_before")      # HF ViTModel key names (vit_adapter.py) vs Dinov2Model
        if is_vit:
            ones = torch.ones(m.hidden, dtype=dt, device=m.layernorm.weight.device)     # no LayerScale in ViT: x 1 is exact
            keep.append(ones)
            get = {
                "n1_w": lambda b: b.layernorm_before.weight, "n1_b": lambda b: b.layernorm_before.bias,
                "q_w": lambda b: b.attention.attention.query.weight, "q_b": lambda b: b.attention.attention.query.bias,
                "k_w": lambda b: b.attention.attention.key.weight, "k_b": lambda b: b.attention.attention.key.bias,
                "v_w": lambda b: b.attention.attention.value.weight, "v_b": lambda b: b.attention.attention.value.bias,
                "o_w": lambda b: b.attention.output.dense.weight, "o_b": lambda b: b.attention.output.dense.bias,
                "ls1": lambda b: ones, "n2_w": lambda b: b.layernorm_after.weight, "n2_b": lambda b: b.layernorm_after.bias,
                "fc1_w": lambda b: b.intermediate.dense.weight, "fc1_b": lambda b: b.intermediate.dense.bias,
                "fc2_w": lambda b: b.output.dense.weight, "fc2_b": lambda b: b.output.dense.bias, "ls2": lambda b: ones,
            }
        else:
          get = {
            "n1_w": lambda b: b.norm1.weight, "n1_b": lambda b: b.norm1.bias,
            "q_w": lambda b: b.attention.attention.query.weight, "q_b": lambda b: b.attention.attention.query.bias,
            "k_w": lambda b: b.attention.attention.key.weight, "k_b": lambda b: b.attention.attention.key.bias,
            "v_w": lambda b: b.attention.attention.value.weight, "v_b": lambda b: b.attention.attention.value.bias,
            "o_w": lambda b: b.attention.output.dense.weight, "o_b": lambda b: b.attention.output.dense.bias,
            "ls1": lambda b: b.layer_scale1.lambda1, "n2_w": lambda b: b.norm2.weight, "n2_b": lambda b: b.norm2.bias,
            "fc1_w": lambda b: b.mlp.fc1.weight, "fc1_b": lambda b: b.mlp.fc1.bias,
            "fc2_w": lambda b: b.mlp.fc2.weight, "fc2_b": lambda b: b.mlp.fc2.bias, "ls2": lambda b: b.layer_scale2.lambda1,
          }
        for name in _DINO_ARRAYS:
            ts = [get[name](b).detach().contiguous() for b in layers]
            arr = _ptr_array(ts)
            keep.extend(ts)
            keep.append(arr)
            setattr(w, name, C.cast(arr, C.POINTER(C.c_void_p)))
        out_dim = 0
        if self.adapter_mlp is not None:
            w.adapter_fc1, w.adapter_fc2 = P(self.adapter_mlp.fc1.weight), P(self.adapter_mlp.fc2.weight)
            out_dim = self.adapter_mlp.fc2.weight.shape[0]
        # dinov2_adapter.py:20-24: nearest for canny / seg, bicubic otherwise; ViT_Adapter does not resize (nearest at P = 16 is the identity)
        mode = 0 if (is_vit or self.adapter.condition_type in ("canny", "seg")) else 1
        d = CarDinoDesc(dtype=dtype_code(dt), hidden=m.hidden, heads=m.heads, layers=m.n_layers, patch=m.patch,
                        pos_grid=m.pos_grid, resize_mode=mode, adapter_out_dim=out_dim, eps=m.eps)
        self.close()
        check(self.lib.car_dino_create(C.byref(d), C.byref(w), cur_stream(), C.byref(self.handle)), "car_dino_create")
        torch.cuda.current_stream().synchronize()     # conversions read `keep` tensors; safe to drop afterwards
        self.dtype, self.hidden, self.out_dim = dt, m.hidden, out_dim
        self.sig = param_signature(self._params())

    @on_own_device
    def forward(self, x: torch.Tensor, apply_mlp: bool) -> torch.Tensor:
        if param_signature(self._params()) != self.sig:
            self._build()
        B, _, H, W = x.shape
        x = x.to(self.dtype).contiguous()
        n = (H // 16) * (W // 16)
        out = torch.empty((B, n, self.out_dim if apply_mlp else self.hidden), dtype=torch.bfloat16, device=x.device)
        check(self.lib.car_dino_forward(self.handle, _ptr(x), B, H, W, _ptr(out), 1 if apply_mlp else 0, cur_stream()),
              "car_dino_forward")
        self._keep = x
        return out.to(self.dtype)


def dinov2_forward(adapter, x: torch.Tensor) -> torch.Tensor:
    """Dinov2_Adapter.forward: [B,3,H,W] -> [B,(H/16)(W/16),C] (reference dinov2_adapter.py:26-29)."""
    h = getattr(adapter, "_car_dino", None)
    if h is None:
        h = DinoHandle(adapter)
        object.__setattr__(adapter, "_car_dino", h)
    return h.forward(x, apply_mlp=False)


# ---------------------------------------------------------------------------------------------------------------
# VQGAN
# ---------------------------------------------------------------------------------------------------------------
def vq_tensor_order(vq) -> List[torch.Tensor]:
    """Canonical order consumed by car_vq_create (csrc/car_vision.cu: car_vq_create)."""
    out: List[torch.Tensor] = []

    def conv(c): out.extend([c.weight, c.bias])
    def norm(n): out.extend([n.weight, n.bias])

    def res(r):
        norm(r.norm1); conv(r.conv1); norm(r.norm2); conv(r.conv2)
        if r.in_channels != r.out_channels:
            conv(r.nin_shortcut)

    def attn(a):
        norm(a.norm); conv(a.q); conv(a.k); conv(a.v); conv(a.proj_out)
    enc, dec = vq.encoder, vq.decoder
    conv(enc.conv_in)
    for lvl, blk in enumerate(enc.conv_blocks):
        for i, r in enumerate(blk.res):
            res(r)
            if len(blk.attn) > 0:
                attn(blk.attn[i])
        if hasattr(blk, "downsample"):
            conv(blk.downsample.conv)
    res(enc.mid[0]); attn(enc.mid[1]); res(enc.mid[2])
    norm(enc.norm_out); conv(enc.conv_out)
    conv(dec.conv_in)
    res(dec.mid[0]); attn(dec.mid[1]); res(dec.mid[2])
    for blk in dec.conv_blocks:
        for i, r in enumerate(blk.res):
            res(r)
            if len(blk.attn) > 0:
                attn(blk.attn[i])
        if hasattr(blk, "upsample"):
            conv(blk.upsample.conv)
    norm(dec.norm_out); conv(dec.conv_out)
    out.append(vq.quantize.embedding.weight)
    conv(vq.quant_conv); conv(vq.post_quant_conv)
    return out


class VQHandle(_lib.ModuleHandle):
    def __init__(self, vq):
        super().__init__("car_vq_destroy")
        self.lib = _lib.lib()
        self.vq = vq
        self._build()

    @property
    def device(self):
        return _dev_of(self.vq)

    @on_own_device
    def _build(self):
        vq = self.vq
        cfg = vq.config
        ts = [t.detach().to(torch.float32).contiguous() for t in vq_tensor_order(vq)]
        arr = _ptr_array(ts)
        d = CarVQDesc(codebook_size=cfg.codebook_size, embed_dim=cfg.codebook_embed_dim, ch=128, z_channels=cfg.z_channels,
                      n_levels=len(cfg.decoder_ch_mult), num_res_blocks=2)
        assert list(cfg.encoder_ch_mult) == list(cfg.decoder_ch_mult)
        for i, v in enumerate(cfg.decoder_ch_mult):
            d.ch_mult[i] = int(v)
        self.close()
        check(self.lib.car_vq_create(C.byref(d), C.cast(arr, C.POINTER(C.c_void_p)), len(ts), cur_stream(), C.byref(self.handle)),
              "car_vq_create")
        torch.cuda.current_stream().synchronize()
        self.sig = param_signature(vq_tensor_order(vq))
        self.down = 2 ** (len(cfg.decoder_ch_mult) - 1)
        self.e_dim = cfg.codebook_embed_dim

    def _fresh(self):
        if param_signature(vq_tensor_order(self.vq)) != self.sig:
            self._build()

    @on_own_device
    def decode_code(self, codes: torch.Tensor, B: int, h: int, w: int) -> torch.Tensor:
        self._fresh()
        codes = codes.reshape(B, h * w).to(torch.int32).contiguous()
        out = torch.empty((B, 3, h * self.down, w * self.down), dtype=torch.float32, device=codes.device)
        check(self.lib.car_vq_decode_code(self.handle, _ptr(codes), B, h, w, _ptr(out), cur_stream()), "car_vq_decode_code")
        self._keep = codes
        return out

    @on_own_device
    def decode(self, quant: torch.Tensor) -> torch.Tensor:
        self._fresh()
        B, e, h, w = quant.shape
        quant = quant.to(torch.float32).contiguous()
        out = torch.empty((B, 3, h * self.down, w * self.down), dtype=torch.float32, device=quant.device)
        check(self.lib.car_vq_decode(self.handle, _ptr(quant), B, h, w, _ptr(out), cur_stream()), "car_vq_decode")
        self._keep = quant
        return out

    @on_own_device
    def encode(self, img: torch.Tensor):
        self._fresh()
        B, _, H, W = img.shape
        img = img.to(torch.float32).contiguous()
        h, w = H // self.down, W // self.down
        idx = torch.empty((B * h * w,), dtype=torch.int32, device=img.device)
        quant = torch.empty((B, self.e_dim, h, w), dtype=torch.float32, device=img.device)
        check(self.lib.car_vq_encode(self.handle, _ptr(img), B, H, W, _ptr(idx), _ptr(quant), cur_stream()), "car_vq_encode")
        self._keep = img
        return quant, idx


def resize_bilinear_aa(x: torch.Tensor, size) -> torch.Tensor:
    """`F.interpolate(x.float(), size=size, mode='bilinear', align_corners=False, antialias=True)` — the multi-resolution training
    scripts' `random_sample_scale` (reference autoregressive/train/train_t2i_depth_multiscale.py:44-56) — on the GPU library."""
    x = x.to(torch.float32).contiguous()
    B, Cc, H, W = x.shape
    OH, OW = int(size[0]), int(size[1])
    out = torch.empty(B, Cc, OH, OW, device=x.device, dtype=torch.float32)
    tmp = torch.empty(B, Cc, H, OW, device=x.device, dtype=torch.float32)
    check(_lib.lib().car_resize_bilinear_aa(_ptr(x), B, Cc, H, W, _ptr(out), OH, OW, _ptr(tmp), cur_stream()), "car_resize_bilinear_aa")
    return out
