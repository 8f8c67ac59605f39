"""Shared test helpers: build the product modules / oracle from (spec, seed) and load golden fixtures."""
from __future__ import annotations

import os

import torch

from oracle.weights import GPTSpec, make_gpt_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def log_measurement(filename: str, text: str, mode: str = "a") -> None:
    """Record the values a test compares with its bars in $CAR_TEST_LOG_DIR/<filename>; nothing is written when it is unset."""
    d = os.environ.get("CAR_TEST_LOG_DIR")
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, filename), mode) as fh:
            fh.write(text)


def load_golden(name: str):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)


def dtype_of(g) -> torch.dtype:
    return {"torch.bfloat16": torch.bfloat16, "torch.float32": torch.float32}[g["dtype"]]


def build_product_gpt(spec: GPTSpec, seed: int, dtype, device="cuda"):
    from controlar_b200.autoregressive.models.gpt_t2i import Transformer, ModelArgs
    m = Transformer(ModelArgs(dim=spec.dim, n_layer=spec.n_layer, n_head=spec.n_head, multiple_of=spec.multiple_of,
                              vocab_size=spec.vocab_size, cls_token_num=spec.cls_token_num, block_size=spec.block_size,
                              caption_dim=spec.caption_dim, num_classes=spec.num_classes, model_type=spec.model_type,
                              adapter_size=spec.adapter_size, condition_type=spec.condition_type))
    sd = make_gpt_state_dict(spec, seed)
    missing, unexpected = m.load_state_dict(sd, strict=True)
    return m.to(device=device, dtype=dtype).eval(), sd


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def near_tie_bound(raw_absmax: float, cfg_scale: float) -> float:
    """Largest logit margin that two bf16 implementations can legitimately disagree on: each raw logit may land on
    either neighbouring bf16 value (1 ulp at the magnitude of the largest logits) and CFG combines
    u + (c - u) * s, i.e. amplifies c by s and u by (s - 1); both candidates can move, hence the factor 2."""
    import math
    ulp = 2.0 ** (math.floor(math.log2(max(raw_absmax, 1e-30))) - 7)
    amp = (2.0 * cfg_scale - 1.0) if cfg_scale > 1.0 else 1.0
    return 2.0 * amp * ulp


def assert_mismatches_are_near_ties(z_ref_combined, raw_ref, ref_tok, mine_tok, cfg_scale, what=""):
    """Every position where `mine_tok` differs from the reference's greedy token must be a near-tie in the
    REFERENCE's own (CFG-combined) logits."""
    mism = (mine_tok != ref_tok)
    for b, i in mism.nonzero().tolist():
        margin = float(z_ref_combined[b, i, ref_tok[b, i]] - z_ref_combined[b, i, mine_tok[b, i]])
        bound = near_tie_bound(float(raw_ref[:, i].abs().max()), cfg_scale)
        assert margin <= bound, f"{what}: token ({b},{i}) differs with margin {margin:.4f} > near-tie bound {bound:.4f}"
    return float(mism.float().mean())


class ObservedLib:
    """The library with the create / destroy entry points of `kinds` observed (e.g. "hed": car_hed_create / car_hed_destroy).
    `created` and `destroyed` list every handle; a destroy of a handle that is not live is recorded but never reaches the library;
    while `refuse` is set, creates fail before the library sees them.  Install with
    `monkeypatch.setattr(_lib, "_lib", ObservedLib(_lib.lib(), kinds))`."""

    def __init__(self, real, kinds):
        self.real, self.refuse = real, False
        self.created, self.destroyed, self.live = [], [], set()
        for k in kinds:
            setattr(self, f"car_{k}_create", self._create(getattr(real, f"car_{k}_create")))
            setattr(self, f"car_{k}_destroy", self._destroy(getattr(real, f"car_{k}_destroy")))

    def __getattr__(self, name):
        return getattr(self.real, name)

    def _create(self, fn):
        def create(*args):
            if self.refuse:
                return -1
            rc = fn(*args)
            h = args[-1]._obj.value                      # every create takes `out` last, as byref(c_void_p)
            self.created.append(h)
            self.live.add(h)
            return rc
        return create

    def _destroy(self, fn):
        def destroy(h):
            self.destroyed.append(h.value)
            if h.value not in self.live:
                return 0
            self.live.discard(h.value)
            return fn(h)
        return destroy
