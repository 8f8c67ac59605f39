"""GPU: antialiased bilinear resize (SURVEY.md §8 row f2; reference train_t2i_depth_multiscale.py:44-56 calls
F.interpolate(..., mode='bilinear', align_corners=False, antialias=True)) through the C ABI, against the CPU oracle
(oracle/resize_oracle.py, itself pinned to torch on the CPU) and against torch's own CUDA kernel.  fp32; tolerance 1e-3 of the
0..255 range (fp32 summation order and FMA contraction)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(64, 96, 48, 80), (50, 70, 64, 64), (96, 96, 24, 40), (33, 47, 33, 100), (512, 512, 384, 640)])
def test_resize_bilinear_aa(shape):
    from controlar_b200.vision import resize_bilinear_aa
    from oracle.resize_oracle import bilinear_aa_resize
    h, w, oh, ow = shape
    x = torch.rand(2, 3, h, w, generator=torch.Generator().manual_seed(h * 1000 + w)) * 255
    got = resize_bilinear_aa(x.cuda(), (oh, ow)).cpu()
    assert got.shape == (2, 3, oh, ow)
    ref_t = F.interpolate(x.cuda(), size=(oh, ow), mode="bilinear", align_corners=False, antialias=True).cpu()
    ref_c = F.interpolate(x, size=(oh, ow), mode="bilinear", align_corners=False, antialias=True)      # ATen's CPU kernel (the oracle's pin)
    e_cuda, e_cpu, cuda_vs_cpu = (float((got - ref_t).abs().max()), float((got - ref_c).abs().max()), float((ref_t - ref_c).abs().max()))
    import json
    from tests.helpers import log_measurement
    log_measurement("resize.jsonl", json.dumps({"shape": shape, "max_abs_vs_torch_cuda": e_cuda, "max_abs_vs_torch_cpu": e_cpu,
                                                "torch_cuda_vs_torch_cpu": cuda_vs_cpu}) + "\n")
    # bar: 1e-3 of the 0..255 range against ATen's CPU kernel (separable two-pass, what oracle/resize_oracle.py restates); ATen's CUDA
    # kernel is a one-pass 2-D gather with its own summation order — the product must be as close to it as ATen's two kernels are
    # to each other (+ 1e-3)
    assert e_cpu < 1e-3, (e_cpu, e_cuda, cuda_vs_cpu)
    assert e_cuda < cuda_vs_cpu + 1e-3, (e_cpu, e_cuda, cuda_vs_cpu)
    if h * w <= 96 * 96:
        assert float((got - bilinear_aa_resize(x, (oh, ow))).abs().max()) < 1e-3


def test_multiscale_preprocess_then_encode_runs():
    """random_sample_scale + `2*(image/255-0.5)` + vq_model.encode (train_t2i_depth_multiscale.py:216-223): shapes and code range."""
    from controlar_b200.vision import resize_bilinear_aa
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    from oracle.weights import make_vq_state_dict
    vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8)
    vq.load_state_dict(make_vq_state_dict(seed=3))
    vq = vq.cuda().eval()
    img = torch.rand(2, 3, 160, 128, generator=torch.Generator().manual_seed(5)).cuda() * 255
    x = resize_bilinear_aa(img, (96, 64))
    _, _, (_, _, idx) = vq.encode(2 * (x / 255 - 0.5))
    idx = idx.reshape(2, -1)
    assert idx.shape == (2, 6 * 4) and int(idx.min()) >= 0 and int(idx.max()) < 16384
