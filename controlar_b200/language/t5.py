"""T5 text encoder on the GPU library — the `self.model(input_ids=..., attention_mask=...)['last_hidden_state']` call of the
reference's `language/t5.py:69-75` (HF `T5EncoderModel`, bf16 by default, `language/t5.py:22`).

    embedder = T5Embedder(device, ...)                       # the reference's class, unchanged (tokenizer, text cleaning)
    embedder.model = T5EncoderB200.from_hf(embedder.model)   # swap the encoder forward for the CUDA one

`T5EncoderB200(...)(input_ids=ids, attention_mask=mask)` returns a dict with `last_hidden_state` like the HF output the reference
indexes.  Architecture covered: T5 v1.1 / flan (gated gelu_new feed-forward, d_kv = 64).  bf16 only; no CPU path."""
from __future__ import annotations

import ctypes as C

import torch

from .. import _lib
from .._lib import CAR_BF16, CarT5Desc, CarT5Weights, check, cur_stream, on_own_device, _ptr


class T5EncoderB200:
    def __init__(self, state_dict, *, d_model, d_kv, num_heads, d_ff, num_layers, vocab_size, num_buckets=32, max_distance=128,
                 eps=1e-6, device="cuda", max_rows=8 * 120):
        if d_kv != 64:
            raise NotImplementedError("controlar_b200 T5 encoder: d_kv must be 64 (t5-v1_1 / flan-t5 have 64)")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("controlar_b200 T5 encoder needs a CUDA device (no CPU path)")
        self.device = dev
        sd = state_dict

        def W(key):
            t = sd[key]
            if t.dtype not in (torch.bfloat16, torch.float32):
                raise NotImplementedError("controlar_b200 T5 encoder: bf16 (or fp32, cast to bf16) checkpoints only")
            return t.detach().to(device=dev, dtype=torch.bfloat16).contiguous()
        emb_key = "shared.weight" if "shared.weight" in sd else "encoder.embed_tokens.weight"
        # the library borrows these: they live as long as the encoder (a deep copy gets its own)
        self._weights = [("embed", None, W(emb_key)),
                         ("rel_bias", None, W("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight")),
                         ("final_norm", None, W("encoder.final_layer_norm.weight"))]
        names = {"ln1": "layer.0.layer_norm", "q": "layer.0.SelfAttention.q", "k": "layer.0.SelfAttention.k", "v": "layer.0.SelfAttention.v",
                 "o": "layer.0.SelfAttention.o", "ln2": "layer.1.layer_norm", "wi_0": "layer.1.DenseReluDense.wi_0",
                 "wi_1": "layer.1.DenseReluDense.wi_1", "wo": "layer.1.DenseReluDense.wo"}
        for field, sub in names.items():
            self._weights += [(field, i, W(f"encoder.block.{i}.{sub}.weight")) for i in range(num_layers)]
        self.d_model = d_model
        self.max_rows = max_rows
        self._desc = CarT5Desc(CAR_BF16, d_model, d_kv, num_heads, d_ff, num_layers, vocab_size, num_buckets, max_distance, eps)
        self._h = _lib.NativeHandle("car_t5_destroy")
        self._handle(max_rows)

    @on_own_device
    def _handle(self, rows):
        """The CarT5, created first (after a copy dropped it) or again when `rows` exceeds the capacity it was created for."""
        if self._h is None:
            self._h = _lib.NativeHandle("car_t5_destroy")
        if not self._h.handle or rows > self.max_rows:
            self._h.close()
            max_rows = max(rows, self.max_rows)
            w, _ = _lib.fill_struct(CarT5Weights, self._weights, self._desc.n_layers)
            check(_lib.lib().car_t5_create(C.byref(self._desc), C.byref(w), max_rows, cur_stream(), C.byref(self._h.handle)), "car_t5_create")
            self.max_rows = max_rows
        return self._h.handle

    @classmethod
    def from_hf(cls, model, device=None, max_rows=8 * 120):
        """model: transformers.T5EncoderModel (the reference's `T5Embedder.model`)."""
        cfg = model.config
        if not getattr(cfg, "is_gated_act", False) or cfg.dense_act_fn != "gelu_new":
            raise NotImplementedError("controlar_b200 T5 encoder: gated gelu_new feed-forward (t5-v1_1 / flan-t5) only")
        dev = device or next(model.parameters()).device
        if torch.device(dev).type != "cuda":
            dev = "cuda"
        return cls(model.state_dict(), d_model=cfg.d_model, d_kv=cfg.d_kv, num_heads=cfg.num_heads, d_ff=cfg.d_ff, num_layers=cfg.num_layers,
                   vocab_size=cfg.vocab_size, num_buckets=cfg.relative_attention_num_buckets, max_distance=cfg.relative_attention_max_distance,
                   eps=cfg.layer_norm_epsilon, device=dev, max_rows=max_rows)

    @on_own_device
    def __call__(self, input_ids=None, attention_mask=None, **unused):
        ids = input_ids.to(device=self.device, dtype=torch.int32).contiguous()
        B, L = ids.shape
        mask = (torch.ones_like(ids) if attention_mask is None else attention_mask.to(device=self.device, dtype=torch.int32)).contiguous()
        h = self._handle(B * L)
        out = torch.empty(B, L, self.d_model, dtype=torch.bfloat16, device=self.device)
        check(_lib.lib().car_t5_forward(h, _ptr(ids), _ptr(mask), B, L, _ptr(out), cur_stream()), "car_t5_forward")
        return {"last_hidden_state": out}

    def eval(self):
        return self
