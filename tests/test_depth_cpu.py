"""CPU: the DPT depth detector's container and oracle.  The fp64 oracle (tests/dpt_oracle.py, the decomposition the kernels
implement) against transformers' own DPTForDepthEstimation output stored in tests/golden/dpt.pt; state-dict keys and shapes;
loading a local checkpoint directory; every refused configuration and input."""
import json

import pytest
import torch

from tests.dpt_oracle import DPT_LARGE, DPT_SMALL, dpt_input, dpt_keys_and_shapes, dpt_oracle, make_dpt_state_dict, windows


def _golden():
    from tests.helpers import load_golden
    return load_golden("dpt")


def test_oracle_matches_reference_small():
    g = _golden()
    x = dpt_input(2, 128, g["small_b2_128_input_seed"])
    y = dpt_oracle(make_dpt_state_dict(DPT_SMALL, g["seed"]), DPT_SMALL, x)
    assert (y[:1] - g["small_b2_128_fp64"]).abs().max().item() <= 1e-9
    assert (y - g["small_b2_128"].double()).abs().max().item() <= 1.01 * g["small_b2_128_ref_fp32_err"] + 1e-9


def test_oracle_matches_reference_large_384():
    g = _golden()
    x = dpt_input(2, 384, g["large_b2_384_input_seed"])
    y = dpt_oracle(make_dpt_state_dict(DPT_LARGE, g["seed"]), DPT_LARGE, x)
    err = max((a - b.double()).abs().max().item() for a, b in zip(windows(y), g["large_b2_384_windows"]))
    assert err <= 1.5 * g["large_b2_384_ref_fp32_err"], (err, g["large_b2_384_ref_fp32_err"])
    assert g["large_b2_384_zero_frac"] < 0.5 and g["large_b2_384_max"] > 1        # a non-degenerate map


def test_state_dict_keys_and_shapes():
    assert dpt_keys_and_shapes(DPT_LARGE) == [(k, tuple(s)) for k, s in _golden()["large_keys"]]
    transformers = pytest.importorskip("transformers")
    with torch.device("meta"):
        hf = transformers.DPTForDepthEstimation(transformers.DPTConfig(**DPT_SMALL))
    assert dpt_keys_and_shapes(DPT_SMALL) == [(k, tuple(v.shape)) for k, v in hf.state_dict().items()]


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
def test_from_pretrained_local_dir(tmp_path, fmt):
    from controlar_b200.condition.depth import DPTForDepthEstimation
    sd = make_dpt_state_dict(DPT_SMALL, 1)
    (tmp_path / "config.json").write_text(json.dumps(dict(DPT_SMALL, architectures=["DPTForDepthEstimation"])))
    if fmt == "safetensors":
        from safetensors.torch import save_file
        save_file(sd, str(tmp_path / "model.safetensors"))
    else:
        torch.save(sd, str(tmp_path / "pytorch_model.bin"))
    m = DPTForDepthEstimation.from_pretrained(str(tmp_path))
    got = m.state_dict()
    assert list(got) == list(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    assert not m.training


@pytest.mark.parametrize("field,value", [("is_hybrid", True), ("readout_type", "add"), ("reassemble_factors", [4, 2, 1, 1]),
                                         ("num_attention_heads", 8), ("hidden_act", "gelu_new"), ("qkv_bias", False),
                                         ("backbone_out_indices", [0, 1, 2]), ("use_batch_norm_in_fusion_residual", True),
                                         ("use_bias_in_fusion_residual", False), ("add_projection", True), ("head_in_index", 0),
                                         ("neck_ignore_stages", [0]), ("backbone_config", {"model_type": "bit"}), ("patch_size", 8),
                                         ("neck_hidden_sizes", [32, 64, 128, 128]), ("fusion_hidden_size", 96)])
def test_unsupported_config_raises(field, value):
    from controlar_b200.condition.depth import DPTForDepthEstimation
    with pytest.raises(NotImplementedError, match=field):
        DPTForDepthEstimation(dict(DPT_SMALL, **{field: value}))


def test_refused_inputs():
    from controlar_b200.condition.depth import DPTForDepthEstimation
    m = DPTForDepthEstimation(DPT_SMALL)
    for shape in [(1, 3, 64, 96), (1, 3, 80, 80), (1, 3, 32, 32), (1, 1, 64, 64), (3, 64, 64)]:
        with pytest.raises(ValueError, match="pixel_values"):
            m(pixel_values=torch.zeros(shape))
    with pytest.raises(NotImplementedError):
        m(pixel_values=torch.zeros(1, 3, 64, 64), labels=torch.zeros(1, 64, 64))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(pixel_values=torch.zeros(1, 3, 64, 64))
