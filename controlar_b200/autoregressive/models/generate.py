"""Drop-in for the reference ``autoregressive/models/generate.py``: same ``generate()`` signature and return
value (int32 [B, max_new_tokens]), but prefill, the N-1 decode steps, CFG, top-k/top-p and sampling all run on
the device behind ``car_prefill`` + ``car_generate`` (bf16: ONE persistent kernel launch for the whole decode loop;
fp32 / unsupported shapes: one CUDA-graph replay per token; no host sync in the loop either way).

Deviations, on purpose and documented in DESIGN.md:
  * sampled runs draw their exponential noise from an in-kernel Philox stream seeded from torch's generator
    (``torch.multinomial`` on CUDA uses its own Philox offsets, which cannot be replayed bit-for-bit from outside);
    greedy runs are deterministic.  Pass ``noise=`` ([N, B, V] Exp(1) draws) to fix the draws explicitly.
  * the per-step probability rows the reference keeps in Python lists (generate.py:127-128, never returned)
    are not materialised.

Extension: ``temperature``, ``top_k``, ``top_p``, ``sample_logits``, ``seed`` and ``control_strength`` also take one value per
image (a length-B sequence or tensor), all in one launch; see ``row_sampling``.  Scalars take the reference's path unchanged.
"""
from __future__ import annotations

from typing import Optional

import torch

from ... import engine as _engine


def top_k_top_p_filtering(logits, top_k: int = 0, top_p: float = 1.0, filter_value: float = -float("Inf"),
                          min_tokens_to_keep: int = 1):
    """Filters [B, V] logits IN PLACE and returns them, like the reference (generate.py:17-56: `logits[indices_to_remove] =
    filter_value; return logits`); the kept set comes from the fused sampler kernel.  It is the kernel's kept mask, not
    `probs > 0`: a kept token far below the row maximum has a probability that underflows to 0 and still keeps its logit."""
    if min_tokens_to_keep != 1:
        raise NotImplementedError("min_tokens_to_keep != 1 is never used by ControlAR")
    if top_k <= 0 and top_p >= 1.0:
        return logits
    sp = _engine.make_sampling(temperature=1.0, top_k=top_k, top_p=top_p, sample_logits=False, cfg_scale=1.0)
    _, kept = _engine.sample(logits, sp, return_kept=True)
    logits.masked_fill_(~kept, filter_value)
    return logits


def sample(logits, temperature: float = 1.0, top_k: int = 2000, top_p: float = 1.0, sample_logits=True,
           noise: Optional[torch.Tensor] = None, seed: Optional[int] = None):
    """(idx [B,1] int64, probs [B,V]) for the last position of [B, S, V] logits (reference generate.py:59-74)."""
    z = logits[:, -1, :]
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if sample_logits else 0
    sp = _engine.make_sampling(temperature, top_k, top_p, sample_logits, cfg_scale=1.0, seed=seed)
    idx, probs = _engine.sample(z, sp, noise=noise, return_probs=True)
    return idx.to(torch.int64).unsqueeze(-1), probs


def _per_image(name, v, B):
    if torch.is_tensor(v):
        v = v.tolist()
    if isinstance(v, (list, tuple)):
        if len(v) != B:
            raise ValueError(f"generate(): {name} has {len(v)} values for {B} images")
        return list(v)
    return [v] * B


def _is_seq(v) -> bool:
    return isinstance(v, (list, tuple)) or (torch.is_tensor(v) and v.dim() > 0)


def row_sampling(model, B: int, use_cfg: bool, control_strength=1, seed=None, **sampling_kwargs):
    """One CarRowSampling per image when any of temperature, top_k, top_p, sample_logits, seed or control_strength is a
    sequence; None when all are scalars (generate() then takes the reference's path).  Scalars apply to every image.

    A sequence of seeds gives image b the Philox key seed[b] and counter word 0, so its draws depend on its own seed alone, not on
    its row or its neighbours.  A scalar seed keeps the rule of one seed per launch: key = seed, counter word = b.  As in the
    scalar path, strengths are 1 without CFG (the reference's generate() does not pass them then), and the legacy gpt.py class,
    which has no control_strength, refuses any other value."""
    vals = {"temperature": sampling_kwargs.get("temperature", 1.0), "top_k": sampling_kwargs.get("top_k", 2000),
            "top_p": sampling_kwargs.get("top_p", 1.0), "sample_logits": sampling_kwargs.get("sample_logits", True),
            "control_strength": control_strength}
    if not any(_is_seq(v) for v in vals.values()) and not _is_seq(seed):
        return None
    col = {k: _per_image(k, v, B) for k, v in vals.items()}
    temps = [float(t) for t in col["temperature"]]
    top_k = [int(k or 0) for k in col["top_k"]]
    top_p = [float(p) for p in col["top_p"]]
    greedy = [not bool(x) for x in col["sample_logits"]]
    cs = [float(c) for c in col["control_strength"]] if use_cfg else [1.0] * B
    for b in range(B):
        if not (0.0 < temps[b] < float("inf")):
            raise ValueError(f"generate(): image {b}: temperature must be > 0, got {temps[b]}")
        if top_k[b] < 0:
            raise ValueError(f"generate(): image {b}: top_k must be >= 0, got {top_k[b]}")
        if not (0.0 < top_p[b] <= 1.0):
            raise ValueError(f"generate(): image {b}: top_p must be in (0, 1], got {top_p[b]}")
        if not (abs(cs[b]) < float("inf")):
            raise ValueError(f"generate(): image {b}: control_strength must be finite, got {cs[b]}")
    if not getattr(model, "has_control_strength", True) and any(c != 1.0 for c in cs):
        raise TypeError("the legacy c2i class has no control_strength (gpt.py:400-409)")
    if _is_seq(seed):
        seeds, rows = [int(x) for x in _per_image("seed", seed, B)], [0] * B
    else:
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if not all(greedy) else 0
        seeds, rows = [int(seed)] * B, list(range(B))
    return [_engine.make_row_sampling(temps[b], top_k[b], top_p[b], not greedy[b], seeds[b], rows[b], cs[b]) for b in range(B)]


def logits_to_probs(logits, temperature: float = 1.0, top_p: float = 1.0, top_k: int = None, **kwargs):
    sp = _engine.make_sampling(temperature, top_k or 0, top_p, False, cfg_scale=1.0)
    return _engine.sample(logits, sp, return_probs=True)[1]


@torch.no_grad()
def generate(model, cond, max_new_tokens, emb_masks=None, cfg_scale=1.0, cfg_interval=-1, condition=None,
             condition_null=None, condition_token_nums=0, control_strength=1, noise=None, seed=None,
             **sampling_kwargs):
    """Reference generate.py:134-204; per-image sampling parameters and strengths: `row_sampling`."""
    use_cfg = cfg_scale > 1.0
    rows = row_sampling(model, cond.shape[0], use_cfg, control_strength, seed, **sampling_kwargs)
    if condition is not None:
        if getattr(model.adapter, "forward", None) is not None and type(model.adapter).__name__ in ("Dinov2_Adapter", "ViT_Adapter") \
                and "forward" not in vars(model.adapter) and "forward" not in vars(model.adapter_mlp):
            # generate.py:137-138 as one library call: DINOv2 forward + adapter_mlp on the dense tensor-core path
            from ... import vision as _vision
            enc = getattr(model, "_car_encoder", None)
            if enc is None or enc.adapter is not model.adapter:
                enc = _vision.DinoHandle(model.adapter, model.adapter_mlp)
                object.__setattr__(model, "_car_encoder", enc)
            condition = enc.forward(condition, apply_mlp=True)
        else:
            condition = model.adapter(condition)                # generate.py:137
            condition = model.adapter_mlp(condition)            # generate.py:138
    if model.model_type == "c2i":
        cond_combined = torch.cat([cond, torch.ones_like(cond) * model.num_classes]) if use_cfg else cond
        T = 1 + condition_token_nums
    elif model.model_type == "t2i":
        if use_cfg:
            cond_null = torch.zeros_like(cond) + model.cls_embedding.uncond_embedding
            cond_combined = torch.cat([cond, cond_null])
        else:
            cond_combined = cond
        T = cond.shape[1]
    else:
        raise Exception("please check model type")
    condition_combined = None
    if condition is not None:
        condition_combined = torch.cat((condition, torch.zeros_like(condition)), dim=0) if use_cfg else condition

    B = cond.shape[0]
    b_eff = 2 * B if use_cfg else B
    model.setup_caches(max_batch_size=b_eff, max_seq_length=T + max_new_tokens, dtype=model.tok_embeddings.weight.dtype,
                       n_img_tokens=max_new_tokens)
    st = model._car_state
    if emb_masks is not None:
        assert emb_masks.shape[0] == B and emb_masks.shape[-1] == T
        em = torch.cat([emb_masks, emb_masks]) if use_cfg else emb_masks
        # keep the inspectable boolean mask consistent with the reference's in-place edit (generate.py:184-193)
        model.causal_mask[:, :, :T] = model.causal_mask[:, :, :T] & (em != 0).unsqueeze(1)
        idx = torch.arange(model.causal_mask.shape[1], device=model.causal_mask.device)
        model.causal_mask[:, idx, idx] = True
        st.set_emb_mask(em)
    else:
        st.set_emb_mask(None)
    model._mask_synced = True

    if rows is None:
        sample_logits = sampling_kwargs.get("sample_logits", True)
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if sample_logits else 0
        sp = _engine.make_sampling(temperature=sampling_kwargs.get("temperature", 1.0), top_k=sampling_kwargs.get("top_k", 2000),
                                   top_p=sampling_kwargs.get("top_p", 1.0), sample_logits=sample_logits,
                                   cfg_scale=cfg_scale, cfg_interval=cfg_interval, seed=seed)
        # generate.py:92 does not forward control_strength when cfg_scale <= 1; forward() then resets it to 1
        cs = float(control_strength) if use_cfg else 1.0
    else:       # per launch: cfg_scale and cfg_interval; sampling parameters and strengths come from `rows`
        sp, cs = _engine.make_sampling(cfg_scale=cfg_scale, cfg_interval=cfg_interval), 1.0
    st.set_row_sampling(rows)
    try:
        st.prefill(cond_combined, condition_combined, cs, all_rows=False)
        return st.generate(sp, max_new_tokens, noise, cond.device)
    finally:
        st.set_row_sampling(None)
