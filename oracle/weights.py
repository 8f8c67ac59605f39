"""TEST INFRASTRUCTURE — procedural (seeded) checkpoints with the reference's state-dict keys and shapes.

The reference ships no weights and there is no network, so every parity test uses random weights.  To keep the
committed fixtures small, weights are never stored: they are regenerated from (key name, seed) by the same
function in the golden-generation script (which loads them into the *reference* modules) and in the tests
(which load them into the oracle and into the CUDA path).  torch's CPU generator is platform independent for a
fixed torch version, which the fixture header records.

Key names / shapes follow the checkpoint contract in SURVEY.md §8(b):
  gpt_t2i.Transformer  : autoregressive/models/gpt_t2i.py:310-389
  HF Dinov2Model       : transformers/models/dinov2/modeling_dinov2.py (installed 5.5.0)
  VQModel              : tokenizer/tokenizer_image/vq_model.py:28-61
"""
from __future__ import annotations

import zlib
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch


def _gen(key: str, seed: int) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((zlib.crc32(key.encode()) + 1000003 * seed) & 0x7FFFFFFF)
    return g


def _randn(key: str, shape, std: float, seed: int, mean: float = 0.0) -> torch.Tensor:
    return torch.randn(*shape, generator=_gen(key, seed), dtype=torch.float32) * std + mean


def find_multiple(n: int, k: int) -> int:
    return n if n % k == 0 else n + k - (n % k)


@dataclass
class GPTSpec:
    """Mirror of the fields of gpt_t2i.ModelArgs that shape the checkpoint (gpt_t2i.py:31-61)."""
    dim: int = 768
    n_layer: int = 12
    n_head: int = 12
    multiple_of: int = 256
    vocab_size: int = 16384
    cls_token_num: int = 120
    block_size: int = 256
    caption_dim: int = 2048
    num_classes: int = 1000
    class_dropout_prob: float = 0.1
    model_type: str = "t2i"
    adapter_size: str = "small"
    condition_type: str = "canny"
    norm_eps: float = 1e-5
    rope_base: float = 10000.0

    @property
    def ffn_dim(self) -> int:  # gpt_t2i.py:204-209
        return find_multiple(int(2 * 4 * self.dim / 3), self.multiple_of)

    @property
    def head_dim(self) -> int:
        return self.dim // self.n_head

    @property
    def adapter_dim(self) -> int:
        return 384 if self.adapter_size == "small" else 768


def dinov2_shapes(hidden: int, layers: int = 12, mlp_ratio: int = 4, patch: int = 14, image: int = 518,
                  prefix: str = "") -> Dict[str, Tuple[int, ...]]:
    n_pos = (image // patch) ** 2 + 1
    s: Dict[str, Tuple[int, ...]] = {
        "embeddings.cls_token": (1, 1, hidden),
        "embeddings.mask_token": (1, hidden),
        "embeddings.position_embeddings": (1, n_pos, hidden),
        "embeddings.patch_embeddings.projection.weight": (hidden, 3, patch, patch),
        "embeddings.patch_embeddings.projection.bias": (hidden,),
        "layernorm.weight": (hidden,),
        "layernorm.bias": (hidden,),
    }
    for i in range(layers):
        p = f"encoder.layer.{i}."
        for n in ("norm1", "norm2"):
            s[p + n + ".weight"] = (hidden,)
            s[p + n + ".bias"] = (hidden,)
        for n in ("query", "key", "value"):
            s[p + f"attention.attention.{n}.weight"] = (hidden, hidden)
            s[p + f"attention.attention.{n}.bias"] = (hidden,)
        s[p + "attention.output.dense.weight"] = (hidden, hidden)
        s[p + "attention.output.dense.bias"] = (hidden,)
        s[p + "layer_scale1.lambda1"] = (hidden,)
        s[p + "layer_scale2.lambda1"] = (hidden,)
        s[p + "mlp.fc1.weight"] = (hidden * mlp_ratio, hidden)
        s[p + "mlp.fc1.bias"] = (hidden * mlp_ratio,)
        s[p + "mlp.fc2.weight"] = (hidden, hidden * mlp_ratio)
        s[p + "mlp.fc2.bias"] = (hidden,)
    return {prefix + k: v for k, v in s.items()}


def vit_shapes(hidden: int = 384, layers: int = 12, intermediate: int = 1536, patch: int = 16, image: int = 224,
               prefix: str = "", pooler: bool = True) -> Dict[str, Tuple[int, ...]]:
    """HF ViTModel keys (transformers/models/vit/modeling_vit.py, installed 5.5.0) — the encoder behind the legacy c2i class's
    ViT_Adapter (autoregressive/models/vit_adapter.py:11)."""
    n_pos = (image // patch) ** 2 + 1
    s: Dict[str, Tuple[int, ...]] = {
        "embeddings.cls_token": (1, 1, hidden),
        "embeddings.position_embeddings": (1, n_pos, hidden),
        "embeddings.patch_embeddings.projection.weight": (hidden, 3, patch, patch),
        "embeddings.patch_embeddings.projection.bias": (hidden,),
        "layernorm.weight": (hidden,),
        "layernorm.bias": (hidden,),
    }
    if pooler:
        s["pooler.dense.weight"] = (hidden, hidden)
        s["pooler.dense.bias"] = (hidden,)
    for i in range(layers):
        q = f"encoder.layer.{i}."
        for n in ("layernorm_before", "layernorm_after"):
            s[q + n + ".weight"] = (hidden,)
            s[q + n + ".bias"] = (hidden,)
        for n in ("query", "key", "value"):
            s[q + f"attention.attention.{n}.weight"] = (hidden, hidden)
            s[q + f"attention.attention.{n}.bias"] = (hidden,)
        s[q + "attention.output.dense.weight"] = (hidden, hidden)
        s[q + "attention.output.dense.bias"] = (hidden,)
        s[q + "intermediate.dense.weight"] = (intermediate, hidden)
        s[q + "intermediate.dense.bias"] = (intermediate,)
        s[q + "output.dense.weight"] = (hidden, intermediate)
        s[q + "output.dense.bias"] = (hidden,)
    return {prefix + k: v for k, v in s.items()}


def gpt_shapes(spec: GPTSpec, with_adapter: bool = True, dino_layers: int = 12) -> Dict[str, Tuple[int, ...]]:
    d, F, V = spec.dim, spec.ffn_dim, spec.vocab_size
    s: Dict[str, Tuple[int, ...]] = {}
    if with_adapter:
        s.update(dinov2_shapes(spec.adapter_dim, layers=dino_layers, prefix="adapter.model."))
    s["adapter_mlp.fc1.weight"] = (d, spec.adapter_dim)
    s["adapter_mlp.fc2.weight"] = (d, d)
    if spec.model_type == "t2i":
        s["cls_embedding.uncond_embedding"] = (120, spec.caption_dim)   # CaptionEmbedder token_num default, gpt_t2i.py:137
        s["cls_embedding.cap_proj.fc1.weight"] = (d, spec.caption_dim)
        s["cls_embedding.cap_proj.fc2.weight"] = (d, d)
    else:
        s["cls_embedding.embedding_table.weight"] = (spec.num_classes + (1 if spec.class_dropout_prob > 0 else 0), d)
    s["tok_embeddings.weight"] = (V, d)
    s["condition_embeddings.weight"] = (V, d)
    s["condition_mlp.uncond_embedding"] = (spec.block_size, d)
    s["condition_mlp.cap_proj.fc1.weight"] = (d, d)
    s["condition_mlp.cap_proj.fc2.weight"] = (d, d)
    for j in range(3):
        s[f"condition_layers.{j}.fc1.weight"] = (d, d)
        s[f"condition_layers.{j}.fc2.weight"] = (d, d)
    for i in range(spec.n_layer):
        p = f"layers.{i}."
        s[p + "attention.wqkv.weight"] = (3 * d, d)
        s[p + "attention.wo.weight"] = (d, d)
        s[p + "feed_forward.w1.weight"] = (F, d)
        s[p + "feed_forward.w3.weight"] = (F, d)
        s[p + "feed_forward.w2.weight"] = (d, F)
        s[p + "attention_norm.weight"] = (d,)
        s[p + "ffn_norm.weight"] = (d,)
    s["norm.weight"] = (d,)
    s["output.weight"] = (V, d)
    return s


def _fill(shapes: Dict[str, Tuple[int, ...]], seed: int, linear_std: float) -> Dict[str, torch.Tensor]:
    out: Dict[str, torch.Tensor] = {}
    for k, shp in shapes.items():
        if k.endswith("norm.weight") or k.endswith("norm1.weight") or k.endswith("norm2.weight") \
                or k.endswith("norm_out.weight") or k.endswith("layernorm.weight") or k.endswith("layernorm_before.weight") \
                or k.endswith("layernorm_after.weight"):
            out[k] = _randn(k, shp, 0.1, seed, mean=1.0)
        elif k.endswith("lambda1"):
            out[k] = _randn(k, shp, 0.2, seed, mean=1.0)
        elif k.endswith(".bias"):
            out[k] = _randn(k, shp, 0.02, seed)
        elif k.endswith("uncond_embedding"):
            out[k] = _randn(k, shp, 1.0 / (shp[-1] ** 0.5), seed)
        elif k.endswith("cls_token") or k.endswith("mask_token") or k.endswith("position_embeddings"):
            out[k] = _randn(k, shp, 0.02, seed)
        else:
            out[k] = _randn(k, shp, linear_std, seed)
    return out


def make_gpt_state_dict(spec: GPTSpec, seed: int = 0, with_adapter: bool = True, dino_layers: int = 12,
                        linear_std: float = 0.02) -> Dict[str, torch.Tensor]:
    """fp32 state dict; callers cast.  ``output.weight`` is random (the reference zero-inits it,
    gpt_t2i.py:377, which would make every logit 0)."""
    return _fill(gpt_shapes(spec, with_adapter, dino_layers), seed, linear_std)


# --------------------------------------------------------------------------------------------------------------
# VQ model (vq_model.py:28-61, 65-195, 280-397)
# --------------------------------------------------------------------------------------------------------------

def _res(s, p, cin, cout):
    s[p + "norm1.weight"] = (cin,); s[p + "norm1.bias"] = (cin,)
    s[p + "conv1.weight"] = (cout, cin, 3, 3); s[p + "conv1.bias"] = (cout,)
    s[p + "norm2.weight"] = (cout,); s[p + "norm2.bias"] = (cout,)
    s[p + "conv2.weight"] = (cout, cout, 3, 3); s[p + "conv2.bias"] = (cout,)
    if cin != cout:
        s[p + "nin_shortcut.weight"] = (cout, cin, 1, 1); s[p + "nin_shortcut.bias"] = (cout,)


def _attn(s, p, c):
    s[p + "norm.weight"] = (c,); s[p + "norm.bias"] = (c,)
    for n in ("q", "k", "v", "proj_out"):
        s[p + n + ".weight"] = (c, c, 1, 1); s[p + n + ".bias"] = (c,)


def vq_shapes(ch: int = 128, ch_mult=(1, 1, 2, 2, 4), z_channels: int = 256, codebook_size: int = 16384,
              codebook_embed_dim: int = 8, num_res_blocks: int = 2) -> Dict[str, Tuple[int, ...]]:
    s: Dict[str, Tuple[int, ...]] = {}
    nres = len(ch_mult)
    # encoder
    s["encoder.conv_in.weight"] = (ch, 3, 3, 3); s["encoder.conv_in.bias"] = (ch,)
    in_mult = (1,) + tuple(ch_mult)
    block_in = ch
    for lvl in range(nres):
        block_in = ch * in_mult[lvl]
        block_out = ch * ch_mult[lvl]
        for b in range(num_res_blocks):
            _res(s, f"encoder.conv_blocks.{lvl}.res.{b}.", block_in, block_out)
            block_in = block_out
            if lvl == nres - 1:
                _attn(s, f"encoder.conv_blocks.{lvl}.attn.{b}.", block_in)
        if lvl != nres - 1:
            s[f"encoder.conv_blocks.{lvl}.downsample.conv.weight"] = (block_in, block_in, 3, 3)
            s[f"encoder.conv_blocks.{lvl}.downsample.conv.bias"] = (block_in,)
    _res(s, "encoder.mid.0.", block_in, block_in)
    _attn(s, "encoder.mid.1.", block_in)
    _res(s, "encoder.mid.2.", block_in, block_in)
    s["encoder.norm_out.weight"] = (block_in,); s["encoder.norm_out.bias"] = (block_in,)
    s["encoder.conv_out.weight"] = (z_channels, block_in, 3, 3); s["encoder.conv_out.bias"] = (z_channels,)
    # decoder
    block_in = ch * ch_mult[nres - 1]
    s["decoder.conv_in.weight"] = (block_in, z_channels, 3, 3); s["decoder.conv_in.bias"] = (block_in,)
    _res(s, "decoder.mid.0.", block_in, block_in)
    _attn(s, "decoder.mid.1.", block_in)
    _res(s, "decoder.mid.2.", block_in, block_in)
    for idx, lvl in enumerate(reversed(range(nres))):
        block_out = ch * ch_mult[lvl]
        for b in range(num_res_blocks + 1):
            _res(s, f"decoder.conv_blocks.{idx}.res.{b}.", block_in, block_out)
            block_in = block_out
            if lvl == nres - 1:
                _attn(s, f"decoder.conv_blocks.{idx}.attn.{b}.", block_in)
        if lvl != 0:
            s[f"decoder.conv_blocks.{idx}.upsample.conv.weight"] = (block_in, block_in, 3, 3)
            s[f"decoder.conv_blocks.{idx}.upsample.conv.bias"] = (block_in,)
    s["decoder.norm_out.weight"] = (block_in,); s["decoder.norm_out.bias"] = (block_in,)
    s["decoder.conv_out.weight"] = (3, block_in, 3, 3); s["decoder.conv_out.bias"] = (3,)
    # quantizer + 1x1 convs
    s["quantize.embedding.weight"] = (codebook_size, codebook_embed_dim)
    s["quantize.codebook_used"] = (65536,)
    s["quant_conv.weight"] = (codebook_embed_dim, z_channels, 1, 1); s["quant_conv.bias"] = (codebook_embed_dim,)
    s["post_quant_conv.weight"] = (z_channels, codebook_embed_dim, 1, 1); s["post_quant_conv.bias"] = (z_channels,)
    return s


def make_vq_state_dict(seed: int = 0, **kw) -> Dict[str, torch.Tensor]:
    shapes = vq_shapes(**kw)
    out: Dict[str, torch.Tensor] = {}
    for k, shp in shapes.items():
        if k == "quantize.codebook_used":
            out[k] = torch.zeros(shp)
        elif k == "quantize.embedding.weight":
            out[k] = _randn(k, shp, 1.0, seed)
        elif k.endswith(".weight") and len(shp) == 4:
            fan_in = shp[1] * shp[2] * shp[3]
            out[k] = _randn(k, shp, 1.0 / (fan_in ** 0.5), seed)
        elif k.endswith(".weight"):
            out[k] = _randn(k, shp, 0.1, seed, mean=1.0)
        else:
            out[k] = _randn(k, shp, 0.02, seed)
    return out


# ---- HED control-map detector (condition/hed.py:17-52): procedural fp32 weights with the reference's state-dict keys ----
HED_BLOCKS = ((3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3))


def make_hed_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """He-scaled conv weights (activations keep their scale through the 13 ReLU convolutions), small biases, a per-channel `norm`
    like the mean the pretrained checkpoint subtracts.  14.7 M parameters: regenerated from the seed, never stored."""
    sd: Dict[str, torch.Tensor] = {"norm": _randn("hed.norm", (1, 3, 1, 1), 8.0, seed, mean=118.0)}
    for b, (cin, cout, n) in enumerate(HED_BLOCKS, start=1):
        c = cin
        for i in range(n):
            sd[f"block{b}.convs.{i}.weight"] = _randn(f"hed.b{b}.c{i}.w", (cout, c, 3, 3), (2.0 / (9 * c)) ** 0.5, seed)
            sd[f"block{b}.convs.{i}.bias"] = _randn(f"hed.b{b}.c{i}.b", (cout,), 0.05, seed)
            c = cout
        sd[f"block{b}.projection.weight"] = _randn(f"hed.b{b}.p.w", (1, cout, 1, 1), (1.0 / cout) ** 0.5 * 0.02, seed)
        sd[f"block{b}.projection.bias"] = _randn(f"hed.b{b}.p.b", (1,), 0.3, seed)
    return sd


# ---- T5 text encoder (language/t5.py:54 -> HF T5EncoderModel, v1.1 / flan architecture): procedural weights with the HF keys ----
def make_t5_state_dict(d_model: int, d_kv: int, num_heads: int, d_ff: int, num_layers: int, vocab: int, num_buckets: int = 32,
                       seed: int = 0) -> Dict[str, torch.Tensor]:
    inner = d_kv * num_heads
    sd: Dict[str, torch.Tensor] = {"shared.weight": _randn("t5.shared", (vocab, d_model), 1.0, seed)}
    sd["encoder.embed_tokens.weight"] = sd["shared.weight"]
    sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"] = _randn("t5.relbias", (num_buckets, num_heads), 0.5, seed)
    for i in range(num_layers):
        p = f"encoder.block.{i}."
        for n, shp, std in (("q", (inner, d_model), (d_model * d_kv) ** -0.5), ("k", (inner, d_model), d_model ** -0.5),
                            ("v", (inner, d_model), d_model ** -0.5), ("o", (d_model, inner), inner ** -0.5)):
            sd[p + f"layer.0.SelfAttention.{n}.weight"] = _randn(f"t5.{i}.{n}", shp, std * 1.5, seed)
        sd[p + "layer.0.layer_norm.weight"] = _randn(f"t5.{i}.ln1", (d_model,), 0.1, seed, mean=1.0)
        sd[p + "layer.1.DenseReluDense.wi_0.weight"] = _randn(f"t5.{i}.wi0", (d_ff, d_model), d_model ** -0.5, seed)
        sd[p + "layer.1.DenseReluDense.wi_1.weight"] = _randn(f"t5.{i}.wi1", (d_ff, d_model), d_model ** -0.5, seed)
        sd[p + "layer.1.DenseReluDense.wo.weight"] = _randn(f"t5.{i}.wo", (d_model, d_ff), d_ff ** -0.5, seed)
        sd[p + "layer.1.layer_norm.weight"] = _randn(f"t5.{i}.ln2", (d_model,), 0.1, seed, mean=1.0)
    sd["encoder.final_layer_norm.weight"] = _randn("t5.fn", (d_model,), 0.1, seed, mean=1.0)
    return sd
