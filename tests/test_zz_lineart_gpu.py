"""GPU: the LineArt detector (reference condition/lineart.py:8-86, fp32) against the reference's own output on procedural weights
(tests/golden/lineart.pt, tests/golden/make_lineart_golden.py), run-to-run and batch invariance, and the reference's sampling call
sequence (autoregressive/sample/sample_t2i.py:109-113,129-132,141) through the drop-in names.  The bar on the [0, 1] map is 1e-4
max-abs (0.026 grey levels once the sample script scales it by 255), except for the smallest accepted input (5 x 7): there the
residual blocks normalise 2 x 2 maps, which amplifies rounding about 3.4 x (the reference's own fp32 output is 1.2e-5 from its fp64
evaluation there, 3.6e-6 at the other sizes), and the bar is 3e-4.  The fixture keeps windows of the 512 x 512 map; the whole
512 x 512 map is compared with the fp64 CPU oracle (tests/lineart_oracle.py, which tests/test_lineart_cpu.py holds to the
reference).  Measured values are logged to lineart.jsonl (tests/helpers.py: log_measurement)."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(seed):
    from controlar_b200.condition.lineart import LineArt
    from tests.lineart_oracle import make_lineart_state_dict
    m = LineArt()
    m.load_state_dict(make_lineart_state_dict(seed), strict=True)
    return m.cuda().eval()


def test_lineart_vs_reference_golden():
    from tests.helpers import load_golden, log_measurement
    from tests.lineart_oracle import lineart_inputs, golden_max_abs, lineart_oracle, make_lineart_state_dict
    g = load_golden("lineart")
    m = _model(g["seed"])
    for name, x in lineart_inputs().items():
        with torch.no_grad():
            y = m(x.cuda())
        bar = 3e-4 if name == "b1_5x7" else 1e-4
        err = golden_max_abs(g, name, y)
        rec = {"case": name, "shape_out": list(y.shape), "max_abs_vs_ref_fp32" + ("" if name in g else "_windows"): err}
        if name + "_fp64" in g:
            rec["max_abs_vs_ref_fp64"] = (y.cpu().double() - g[name + "_fp64"]).abs().max().item()
        if name not in g:
            full = (y.cpu().double() - lineart_oracle(make_lineart_state_dict(g["seed"]), x, cast=False)).abs().max().item()
            rec["max_abs_vs_oracle_fp64_full_map"] = full
        log_measurement("lineart.jsonl", json.dumps(rec) + "\n")
        assert err <= bar, (name, err)
        assert rec.get("max_abs_vs_oracle_fp64_full_map", 0.0) <= bar, (name, rec)


def test_lineart_deterministic_and_batch_invariant():
    from tests.lineart_oracle import lineart_inputs
    m = _model(2)
    x = lineart_inputs()["b2_96x128"].cuda()
    with torch.no_grad():
        a = m(x)
        b = m(x)
        singles = [m(x[i:i + 1]) for i in range(x.shape[0])]
    assert torch.equal(a, b)
    for i, s in enumerate(singles):
        assert torch.equal(a[i:i + 1], s), i


def test_lineart_rejects_tiny_images():
    m = _model(0)
    with pytest.raises(RuntimeError, match="4 x 4"):
        m(torch.zeros(1, 3, 4, 16, device="cuda"))


def test_lineart_weight_update_rebuilds_handle():
    from tests.lineart_oracle import lineart_inputs, make_lineart_state_dict
    x = lineart_inputs()["b1_70x90"].cuda()
    m = _model(0)
    with torch.no_grad():
        y0 = m(x)
        m.load_state_dict(make_lineart_state_dict(5))
        y5 = m(x)
    assert torch.equal(y5, _model(5)(x)) and not torch.equal(y0, y5)


CODE = r"""
import sys, torch
from condition.lineart import LineArt                                 # sample_t2i.py:31
from tokenizer.tokenizer_image.vq_model import VQ_models
from autoregressive.models.gpt_t2i import GPT_models
from autoregressive.models.generate import generate
from tests.lineart_oracle import make_lineart_state_dict
device, precision = "cuda", torch.bfloat16
torch.manual_seed(0)
H = W = 128
get_control = LineArt()                                               # sample_t2i.py:110-112
get_control.load_state_dict(make_lineart_state_dict(3))
get_control.to(device)
latent = H // 16
gpt_model = GPT_models["GPT-B"](block_size=latent ** 2, cls_token_num=120, model_type="t2i", condition_type="lineart",
                                adapter_size="small").to(device=device, dtype=precision).eval()
gpt_model.output.weight.data.normal_(0, 0.02)
vq_model = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(device).eval()
img = (torch.rand(H, W, 3) * 255).round().to(torch.uint8)            # np.array(Image.open(condition_path))
with torch.no_grad():
    condition_img = get_control(img.permute(2, 0, 1).unsqueeze(0).to(device).float())     # :129
    condition_img = 1 - condition_img                                                      # :130
    condition_img = condition_img.repeat(2, 3, 1, 1) * 255                                 # :131
    condition_img = condition_img.to(device)
    condition_img = 2 * (condition_img / 255 - 0.5)                                        # :141
    assert tuple(condition_img.shape) == (2, 3, H, W), condition_img.shape
    assert float(condition_img.min()) >= -1 and float(condition_img.max()) <= 1
    caption_embs = torch.randn(2, 120, 2048, device=device, dtype=precision)
    emb_masks = torch.zeros(2, 120, dtype=torch.int64, device=device)
    emb_masks[:, -17:] = 1
    c_indices = caption_embs * emb_masks[:, :, None]
    index_sample = generate(gpt_model, c_indices, latent * latent, emb_masks, condition=condition_img.to(precision), cfg_scale=4.0,
                            temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True, control_strength=1.0)
    assert tuple(index_sample.shape) == (2, latent * latent)
    samples = vq_model.decode_code(index_sample, [2, 8, latent, latent])
    assert tuple(samples.shape) == (2, 3, H, W) and bool(torch.isfinite(samples).all())
import condition.lineart as la
assert la.__file__.startswith(sys.argv[1]) and "controlnet_aux" not in sys.modules, la.__file__
print("OK")
"""


def test_reference_lineart_sampling_sequence_through_dropin_names(tmp_path):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT])
    r = subprocess.run([sys.executable, "-c", CODE, os.path.join(ROOT, "dropin")], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-4000:]
