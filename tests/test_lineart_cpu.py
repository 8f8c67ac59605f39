"""CPU: the LineArt detector's module surface (reference condition/lineart.py:8-86), the drop-in import, and the CPU restatement of
the decomposition the CUDA kernels implement (tests/lineart_oracle.py) against the reference's own fp32 output (tests/golden/lineart.pt)."""
import os
import subprocess
import sys

import pytest
import torch

from tests.helpers import load_golden
from tests.lineart_oracle import (make_lineart_state_dict, lineart_inputs, lineart_oracle, conv_transpose_subpixel, window_conv,
                                  pad_reflect, pad_zero, golden_max_abs)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lineart_module_keys_and_shapes_match_reference():
    from controlar_b200.condition.lineart import LineArt
    g = load_golden("lineart")
    sd = LineArt().state_dict()
    assert list(sd) == g["keys"]
    assert {k: tuple(v.shape) for k, v in sd.items()} == g["shapes"]
    assert sum(v.numel() for v in sd.values()) == g["n_params"] == 4290945


def test_lineart_load_state_dict_strict():
    from controlar_b200.condition.lineart import LineArt
    m = LineArt()
    sd = make_lineart_state_dict(seed=1)
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.model3[0].weight, sd["model3.0.weight"]) and m.model3[0].weight.shape == (256, 128, 3, 3)


def test_lineart_cpu_input_raises():
    from controlar_b200.condition.lineart import LineArt
    m = LineArt()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 16, 16))


def test_lineart_non_default_constructor_raises():
    from controlar_b200.condition.lineart import LineArt
    for kw in ({"input_nc": 1}, {"output_nc": 3}, {"n_residual_blocks": 9}, {"sigmoid": False}):
        with pytest.raises(NotImplementedError):
            LineArt(**kw)


@pytest.mark.parametrize("H,W", [(70, 90), (5, 7), (96, 128), (9, 4 * 3)])
def test_lineart_output_size(H, W):
    from controlar_b200.condition.lineart import LineArt
    h, w = H, W
    for _ in range(2):
        h, w = (h + 1) // 2, (w + 1) // 2
    assert LineArt.output_size(H, W) == (4 * h, 4 * w)


def test_subpixel_transposed_conv_matches_conv_transpose2d():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 5, 6, 7, generator=g, dtype=torch.float64)
    w = torch.randn(5, 4, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(4, generator=g, dtype=torch.float64)
    want = torch.nn.functional.conv_transpose2d(x, w, b, stride=2, padding=1, output_padding=1)
    assert (conv_transpose_subpixel(x, w, b) - want).abs().max().item() < 1e-12


def test_window_conv_on_padded_input_matches_conv2d():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 3, 9, 11, generator=g, dtype=torch.float64)
    w = torch.randn(6, 3, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(6, generator=g, dtype=torch.float64)
    want = torch.nn.functional.conv2d(x, w, b, stride=2, padding=1)
    assert (window_conv(pad_zero(x, 1, 1, 1, 1), w, b, 2, 5, 6) - want).abs().max().item() < 1e-12
    want = torch.nn.functional.conv2d(torch.nn.functional.pad(x, (1, 1, 1, 1), mode="reflect"), w, b)
    assert (window_conv(pad_reflect(x, 1), w, b, 1, 9, 11) - want).abs().max().item() < 1e-12


def test_lineart_oracle_matches_reference_golden():
    """Against the reference's fp32 output (whole maps; windows of the 512 x 512 map): <= 1e-5 max-abs.  At 5 x 7 the residual
    blocks normalise 2 x 2 maps and the reference's own fp32 result is 1.2e-5 from its fp64 evaluation, so there (and at 70 x 90) the
    oracle is held to the reference's fp64 output instead, at 1e-9."""
    g = load_golden("lineart")
    sd = make_lineart_state_dict(g["seed"])
    for name, x in lineart_inputs().items():
        got64 = lineart_oracle(sd, x, cast=False)
        assert tuple(got64.shape) == tuple(g[name + "_shape"]), (name, got64.shape)
        if name + "_fp64" in g:
            assert (got64 - g[name + "_fp64"]).abs().max().item() <= 1e-9, name
        if name != "b1_5x7":
            err = golden_max_abs(g, name, got64)
            assert err <= 1e-5, (name, err)


CODE = r"""
import os, sys
from condition.lineart import LineArt, ResidualBlock                 # sample_t2i.py:31, train_t2i_lineart.py
import condition.lineart as la
root = sys.argv[1]
assert la.__file__.startswith(os.path.join(root, "dropin")), la.__file__
import controlar_b200.condition.lineart as impl
assert LineArt is impl.LineArt and ResidualBlock is impl.ResidualBlock
assert "controlnet_aux" not in sys.modules
print("OK")
"""


def test_dropin_resolves_condition_lineart(tmp_path):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT])
    r = subprocess.run([sys.executable, "-c", CODE, ROOT], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
