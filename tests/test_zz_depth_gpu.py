"""GPU: the DPT depth detector (transformers DPTForDepthEstimation, fp32 in the reference) against HF's own fp32 output on
procedural weights (tests/golden/dpt.pt, tests/golden/make_dpt_golden.py), the whole 512 x 512 map against the fp64 oracle
(tests/dpt_oracle.py) run on the GPU, run-to-run and batch invariance, the handle rebuild on a weight update, and the reference's
sampling call sequence (autoregressive/sample/sample_t2i.py:114-116,133-141).  The bar is max-abs <= 3e-4 x the reference map's
maximum: 0.077 grey levels once the script scales the map by 255 / max, far below the bf16 quantum at which the map reaches the
control encoder.  The split-bf16 operands carry each fp32 value to about 2^-17 and drop the lo x lo term, so one product is good to
about 2^-18 where fp32 is good to 2^-24; through DPT-Large's 24 layers that leaves about 1.5e-4 x the maximum (the reference's own
fp32 map is 5e-6 x the maximum from its fp64 map).  Measured values are logged to depth.jsonl."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_MODELS = {}


def _model(cfg, seed):
    from controlar_b200.condition.depth import DPTForDepthEstimation
    from tests.dpt_oracle import make_dpt_state_dict
    m = DPTForDepthEstimation(cfg)
    m.load_state_dict(make_dpt_state_dict(cfg, seed), strict=True)
    return m.cuda().eval()


def _large():
    from tests.dpt_oracle import DPT_LARGE
    if "large" not in _MODELS:
        _MODELS["large"] = _model(DPT_LARGE, 0)
    return _MODELS["large"]


def test_depth_vs_reference_golden():
    from tests.helpers import load_golden, log_measurement
    from tests.dpt_oracle import DPT_LARGE, DPT_SMALL, dpt_input, dpt_oracle, make_dpt_state_dict, windows
    g = load_golden("dpt")
    assert g["large_keys"] == [(k, tuple(v.shape)) for k, v in _large().state_dict().items()]
    for name, cfg in (("small_b2_128", DPT_SMALL), ("large_b2_384", DPT_LARGE), ("large_b1_512", DPT_LARGE)):
        m = _large() if cfg is DPT_LARGE else _model(cfg, g["seed"])
        B, side = g[name + "_shape"][0], g[name + "_shape"][1]
        x = dpt_input(B, side, g[name + "_input_seed"]).cuda()
        with torch.no_grad():
            y = m(pixel_values=x).predicted_depth
        assert tuple(y.shape) == tuple(g[name + "_shape"])
        bar = 3e-4 * g[name + "_max"]
        yc = y.cpu().double()
        if name + "_windows" in g:
            err = max((a - b.double()).abs().max().item() for a, b in zip(windows(yc), g[name + "_windows"]))
        else:
            err = (yc - g[name].double()).abs().max().item()
        rec = {"case": name, "shape": list(y.shape), "ref_max": g[name + "_max"], "max_abs_vs_ref_fp32": err, "rel_to_max": err / g[name + "_max"],
               "ref_own_fp32_err": g[name + "_ref_fp32_err"]}
        if name == "large_b1_512":
            full = dpt_oracle(make_dpt_state_dict(DPT_LARGE, g["seed"]), DPT_LARGE, x)
            rec["max_abs_vs_oracle_fp64_full_map"] = (y.double() - full).abs().max().item()
        log_measurement("depth.jsonl", json.dumps(rec) + "\n")
        assert err <= bar, rec
        assert rec.get("max_abs_vs_oracle_fp64_full_map", 0.0) <= bar, rec


def test_depth_deterministic_and_batch_invariant():
    from tests.dpt_oracle import DPT_SMALL, dpt_input
    m = _model(DPT_SMALL, 2)
    x = dpt_input(2, 192, 5).cuda()
    with torch.no_grad():
        a = m(pixel_values=x)["predicted_depth"]
        b = m(pixel_values=x).predicted_depth
        singles = [m(pixel_values=x[i:i + 1]).predicted_depth for i in range(2)]
    assert torch.equal(a, b)
    for i, s in enumerate(singles):
        assert torch.equal(a[i:i + 1], s), i


def test_depth_weight_update_rebuilds_handle():
    from tests.dpt_oracle import DPT_SMALL, dpt_input, make_dpt_state_dict
    x = dpt_input(1, 64, 6).cuda()
    m = _model(DPT_SMALL, 0)
    with torch.no_grad():
        y0 = m(pixel_values=x).predicted_depth
        m.load_state_dict(make_dpt_state_dict(DPT_SMALL, 5))
        y5 = m(pixel_values=x).predicted_depth
        fresh = _model(DPT_SMALL, 5)(pixel_values=x).predicted_depth
    assert torch.equal(y5, fresh) and not torch.equal(y0, y5)


def test_depth_refusals_on_gpu():
    from tests.dpt_oracle import DPT_SMALL
    m = _model(DPT_SMALL, 0)
    with pytest.raises(ValueError, match="multiple of 32"):
        m(pixel_values=torch.zeros(1, 3, 96, 128, device="cuda"))
    with pytest.raises(NotImplementedError):
        m(pixel_values=torch.zeros(1, 3, 64, 64, device="cuda"), labels=torch.zeros(1, 64, 64, device="cuda"))
    with pytest.raises(RuntimeError, match="fp32"):
        m.to(torch.bfloat16)(pixel_values=torch.zeros(1, 3, 64, 64, device="cuda"))


CODE = r"""
import sys, torch
from controlar_b200.condition.depth import DPTForDepthEstimation     # INTEGRATION.md: after sample_t2i.py:33
from tokenizer.tokenizer_image.vq_model import VQ_models
from autoregressive.models.gpt_t2i import GPT_models
from autoregressive.models.generate import generate
from tests.dpt_oracle import DPT_SMALL, make_dpt_state_dict
device, precision = "cuda", torch.bfloat16
torch.manual_seed(0)
H = W = 128
model_large = DPTForDepthEstimation(DPT_SMALL)                          # sample_t2i.py:114-116 (from_pretrained of a local dir)
model_large.load_state_dict(make_dpt_state_dict(DPT_SMALL, 3))
model_large.to(device)
latent = H // 16
gpt_model = GPT_models["GPT-B"](block_size=latent ** 2, cls_token_num=120, model_type="t2i", condition_type="depth",
                                adapter_size="small").to(device=device, dtype=precision).eval()
gpt_model.output.weight.data.normal_(0, 0.02)
vq_model = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(device).eval()
inputs = {"pixel_values": torch.rand(1, 3, H, W) * 2 - 1}                # DPTImageProcessor output
with torch.no_grad():
    outputs = model_large(**{k: v.to(device) for k, v in inputs.items()})                  # :133-134
    predicted_depth = outputs.predicted_depth
    predicted_depth = predicted_depth.squeeze().cpu().numpy()                               # :135-138
    condition_img = torch.from_numpy(predicted_depth).unsqueeze(0).repeat(2, 3, 1, 1)
    condition_img = condition_img * 255 / condition_img.max()
    condition_img = condition_img.to(device)
    condition_img = 2 * (condition_img / 255 - 0.5)                                         # :141
    assert tuple(condition_img.shape) == (2, 3, H, W), condition_img.shape
    assert bool(torch.isfinite(condition_img).all()) and float(condition_img.max()) == 1.0
    caption_embs = torch.randn(2, 120, 2048, device=device, dtype=precision)
    emb_masks = torch.zeros(2, 120, dtype=torch.int64, device=device)
    emb_masks[:, -17:] = 1
    c_indices = caption_embs * emb_masks[:, :, None]
    index_sample = generate(gpt_model, c_indices, latent * latent, emb_masks, condition=condition_img.to(precision), cfg_scale=4.0,
                            temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True, control_strength=1.0)
    assert tuple(index_sample.shape) == (2, latent * latent)
    samples = vq_model.decode_code(index_sample, [2, 8, latent, latent])
    assert tuple(samples.shape) == (2, 3, H, W) and bool(torch.isfinite(samples).all())
assert "transformers" not in sys.modules
print("OK")
"""


def test_reference_depth_sampling_sequence(tmp_path):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT])
    r = subprocess.run([sys.executable, "-c", CODE], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-4000:]
