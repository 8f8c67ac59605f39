"""Host-side handles for the control encoder (car_dino_*) and the VQGAN tokenizer (car_vq_*)."""
from __future__ import annotations

import ctypes as C
from typing import List

import torch

from . import _lib
from ._lib import CarDinoDesc, CarDinoWeights, CarVQDesc, check, cur_stream, dtype_code, on_own_device, _ptr, _ptr_array
from ._lib import _DINO_ARRAYS  # noqa: F401  (callers that fill a CarDinoWeights by hand find its array names here)


# ---------------------------------------------------------------------------------------------------------------
# DINOv2
# ---------------------------------------------------------------------------------------------------------------
def _dev_of(module):
    return next(module.parameters()).device


def _block_tensors(b, is_vit: bool):
    """One encoder block's tensors by CarDinoWeights array name: HF ViTModel key names (vit_adapter.py) or Dinov2Model's.  ViT has
    no LayerScale: ls1 / ls2 are None."""
    att = b.attention
    t = {"q_w": att.attention.query.weight, "q_b": att.attention.query.bias, "k_w": att.attention.key.weight,
         "k_b": att.attention.key.bias, "v_w": att.attention.value.weight, "v_b": att.attention.value.bias,
         "o_w": att.output.dense.weight, "o_b": att.output.dense.bias}
    if is_vit:
        t.update(n1_w=b.layernorm_before.weight, n1_b=b.layernorm_before.bias, n2_w=b.layernorm_after.weight, n2_b=b.layernorm_after.bias,
                 fc1_w=b.intermediate.dense.weight, fc1_b=b.intermediate.dense.bias, fc2_w=b.output.dense.weight,
                 fc2_b=b.output.dense.bias, ls1=None, ls2=None)
    else:
        t.update(n1_w=b.norm1.weight, n1_b=b.norm1.bias, n2_w=b.norm2.weight, n2_b=b.norm2.bias, fc1_w=b.mlp.fc1.weight,
                 fc1_b=b.mlp.fc1.bias, fc2_w=b.mlp.fc2.weight, fc2_b=b.mlp.fc2.bias, ls1=b.layer_scale1.lambda1,
                 ls2=b.layer_scale2.lambda1)
    return t


def _is_vit(m) -> bool:
    return hasattr(m.encoder.layer[0], "layernorm_before")      # HF ViTModel key names (vit_adapter.py) vs Dinov2Model


def _dino_desc(adapter, dtype: int, adapter_out_dim: int) -> CarDinoDesc:
    m = adapter.model
    # dinov2_adapter.py:20-24: nearest for canny / seg, bicubic otherwise; ViT_Adapter does not resize (nearest at P = 16 is the identity)
    mode = 0 if (_is_vit(m) or adapter.condition_type in ("canny", "seg")) else 1
    return CarDinoDesc(dtype=dtype, hidden=m.hidden, heads=m.heads, layers=m.n_layers, patch=m.patch, pos_grid=m.pos_grid,
                       resize_mode=mode, adapter_out_dim=adapter_out_dim, eps=m.eps)


class DinoHandle(_lib.ModuleHandle):
    def __init__(self, adapter, adapter_mlp=None):
        super().__init__("car_dino_destroy")
        self.lib = _lib.lib()
        self.adapter, self.adapter_mlp = adapter, adapter_mlp
        self._get()

    @property
    def device(self):
        return _dev_of(self.adapter)

    def _get(self):
        ps = list(self.adapter.model.parameters())
        if self.adapter_mlp is not None:
            ps += list(self.adapter_mlp.parameters())
        return self.get(ps, self._create)

    def _create(self, out):
        m, mlp = self.adapter.model, self.adapter_mlp
        dt = m.layernorm.weight.dtype
        entries = encoder_train_params(m)
        if _is_vit(m):
            ones = torch.ones(m.hidden, dtype=dt, device=m.layernorm.weight.device)     # no LayerScale in ViT: x 1 is exact
            entries += [(f, i, ones) for f in ("ls1", "ls2") for i in range(m.n_layers)]
        out_dim = 0
        if mlp is not None:
            entries += [("adapter_fc1", None, mlp.fc1.weight), ("adapter_fc2", None, mlp.fc2.weight)]
            out_dim = mlp.fc2.weight.shape[0]
        w, keep = _lib.fill_struct(CarDinoWeights, [(f, i, t.detach().contiguous()) for f, i, t in entries], m.n_layers)
        check(self.lib.car_dino_create(C.byref(_dino_desc(self.adapter, dtype_code(dt), out_dim)), C.byref(w), cur_stream(), C.byref(out)),
              "car_dino_create")
        self.dtype, self.hidden, self.out_dim = dt, m.hidden, out_dim

    @on_own_device
    def forward(self, x: torch.Tensor, apply_mlp: bool) -> torch.Tensor:
        self._get()
        B, _, H, W = x.shape
        x = x.to(self.dtype).contiguous()
        n = (H // 16) * (W // 16)
        out = torch.empty((B, n, self.out_dim if apply_mlp else self.hidden), dtype=torch.bfloat16, device=x.device)
        check(self.lib.car_dino_forward(self.handle, _ptr(x), B, H, W, _ptr(out), 1 if apply_mlp else 0, cur_stream()),
              "car_dino_forward")
        self._keep = x
        return out.to(self.dtype)


_TOP = [("cls_token", "embeddings.cls_token"), ("pos_emb", "embeddings.position_embeddings"),
        ("patch_w", "embeddings.patch_embeddings.projection.weight"), ("patch_b", "embeddings.patch_embeddings.projection.bias"),
        ("ln_w", "layernorm.weight"), ("ln_b", "layernorm.bias")]


def encoder_train_params(m):
    """The backbone parameters on the path of Dinov2_Adapter.forward / ViT_Adapter.forward, as (CarDinoWeights field, layer or None,
    parameter).  embeddings.mask_token and ViT's pooler.dense.* are not on it (the reference gives them no gradient)."""
    names = dict(m.named_parameters())
    out = [(f, None, names[k]) for f, k in _TOP]
    is_vit = _is_vit(m)
    for i, b in enumerate(m.encoder.layer):
        out += [(f, i, t) for f, t in _block_tensors(b, is_vit).items() if t is not None]
    return out


class DinoTrainHandle(_lib.NativeHandle):
    """CarDinoTrain: the control encoder's forward with fp32 parameters under bf16-autocast numerics, and its backward.  The fp32
    parameters are borrowed (re-cast to bf16 inside every forward), so an optimizer step needs no rebuild; replacing a parameter
    tensor (new storage) does, and `key` tells."""

    def __init__(self, adapter):
        super().__init__("car_dino_train_destroy")
        self.lib = _lib.lib()
        m = adapter.model
        self.params = encoder_train_params(m)
        self.key = self.key_of(adapter)
        self.device = m.layernorm.weight.device
        self.hidden, self.layers = m.hidden, m.n_layers
        self.generation = 0          # a backward belongs to the forward that produced its feat
        self._create(adapter)

    @staticmethod
    def key_of(adapter):
        return tuple(p.data_ptr() for _, _, p in encoder_train_params(adapter.model))

    @on_own_device
    def _create(self, adapter):
        w, keep = _lib.fill_struct(CarDinoWeights, [(f, i, p.detach()) for f, i, p in self.params], self.layers)
        check(self.lib.car_dino_train_create(C.byref(_dino_desc(adapter, _lib.CAR_F32, 0)), C.byref(w), cur_stream(), C.byref(self.handle)),
              "car_dino_train_create")

    @on_own_device
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        B, _, H, W = x.shape
        x = x.to(torch.float32).contiguous()
        feat = torch.empty((B, (H // 16) * (W // 16), self.hidden), dtype=torch.float32, device=x.device)
        check(self.lib.car_dino_train_forward(self.handle, _ptr(x), B, H, W, _ptr(feat), cur_stream()), "car_dino_train_forward")
        self._keep = x
        self.generation += 1
        return feat

    @on_own_device
    def backward(self, dfeat: torch.Tensor, want):
        """fp32 gradients of the last forward for the parameters flagged in `want` (parallel to self.params; None elsewhere)"""
        grads = [torch.empty_like(p, dtype=torch.float32) if wnt else None for (_, _, p), wnt in zip(self.params, want)]
        g, keep = _lib.fill_struct(CarDinoWeights, [(f, i, t) for (f, i, _), t in zip(self.params, grads)], self.layers)
        dfeat = dfeat.to(torch.float32).contiguous()
        check(self.lib.car_dino_train_backward(self.handle, _ptr(dfeat), C.byref(g), cur_stream()), "car_dino_train_backward")
        return grads


class _EncoderStep(torch.autograd.Function):
    """feat = car_dino_train_forward(x); backward = car_dino_train_backward.  The input map is data: it gets no gradient."""

    @staticmethod
    def forward(ctx, handle, x, *params):
        feat = handle.forward(x)
        ctx.handle, ctx.generation = handle, handle.generation
        return feat

    @staticmethod
    def backward(ctx, dfeat):
        if ctx.handle.generation != ctx.generation:
            raise RuntimeError("controlar_b200: the control encoder ran another trainable forward since this output was computed; its "
                               "backward recomputes from the LAST forward (call backward before the next forward)")
        want = [ctx.needs_input_grad[2 + i] for i in range(len(ctx.handle.params))]
        return (None, None, *ctx.handle.backward(dfeat, want))


def _trains(adapter) -> bool:
    """The trainable path runs when autograd records and the backbone is an fp32 module with a parameter that wants a gradient;
    every other call (generate(), eval, no_grad, a frozen or bf16 encoder) runs the inference encoder."""
    if not torch.is_grad_enabled():
        return False
    ps = [p for _, _, p in encoder_train_params(adapter.model)]
    return all(p.dtype == torch.float32 for p in ps) and any(p.requires_grad for p in ps)


def dinov2_forward(adapter, x: torch.Tensor) -> torch.Tensor:
    """Dinov2_Adapter.forward: [B,3,H,W] -> [B,(H/16)(W/16),C] (reference dinov2_adapter.py:26-29)."""
    if _trains(adapter):
        h = getattr(adapter, "_car_dino_train", None)
        if h is None or h.key != DinoTrainHandle.key_of(adapter):
            if h is not None:
                h.close()
            h = DinoTrainHandle(adapter)
            object.__setattr__(adapter, "_car_dino_train", h)
        return _EncoderStep.apply(h, x, *[p for _, _, p in h.params])
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
        cfg = vq.config
        self.down = 2 ** (len(cfg.decoder_ch_mult) - 1)
        self.e_dim = cfg.codebook_embed_dim
        self._get()

    @property
    def device(self):
        return _dev_of(self.vq)

    def _get(self):
        return self.get(vq_tensor_order(self.vq), self._create)

    def _create(self, out):
        cfg = self.vq.config
        ts = [t.detach().to(torch.float32).contiguous() for t in vq_tensor_order(self.vq)]
        arr = _ptr_array(ts)
        d = CarVQDesc(codebook_size=cfg.codebook_size, embed_dim=cfg.codebook_embed_dim, ch=128, z_channels=cfg.z_channels,
                      n_levels=len(cfg.decoder_ch_mult), num_res_blocks=2)
        assert list(cfg.encoder_ch_mult) == list(cfg.decoder_ch_mult)
        for i, v in enumerate(cfg.decoder_ch_mult):
            d.ch_mult[i] = int(v)
        check(self.lib.car_vq_create(C.byref(d), C.cast(arr, C.POINTER(C.c_void_p)), len(ts), cur_stream(), C.byref(out)), "car_vq_create")

    @on_own_device
    def decode_code(self, codes: torch.Tensor, B: int, h: int, w: int) -> torch.Tensor:
        self._get()
        codes = codes.reshape(B, h * w).to(torch.int32).contiguous()
        out = torch.empty((B, 3, h * self.down, w * self.down), dtype=torch.float32, device=codes.device)
        check(self.lib.car_vq_decode_code(self.handle, _ptr(codes), B, h, w, _ptr(out), cur_stream()), "car_vq_decode_code")
        self._keep = codes
        return out

    @on_own_device
    def decode(self, quant: torch.Tensor) -> torch.Tensor:
        self._get()
        B, e, h, w = quant.shape
        quant = quant.to(torch.float32).contiguous()
        out = torch.empty((B, 3, h * self.down, w * self.down), dtype=torch.float32, device=quant.device)
        check(self.lib.car_vq_decode(self.handle, _ptr(quant), B, h, w, _ptr(out), cur_stream()), "car_vq_decode")
        self._keep = quant
        return out

    @on_own_device
    def encode(self, img: torch.Tensor):
        self._get()
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
