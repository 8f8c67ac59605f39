"""CPU: the MiDaS DPT-Hybrid detector's container and oracle.  The fp64 oracle (tests/midas_oracle.py, the decomposition the kernels
implement) against the reference's own DPTDepthModel output stored in tests/golden/midas.pt; state-dict keys and shapes;
checkpoint loading; every refusal; the drop-in import without timm."""
import os
import subprocess
import sys

import pytest
import torch

from tests.midas_oracle import make_midas_state_dict, midas_image, midas_input, midas_keys_and_shapes, midas_oracle, windows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SD = {}


def _golden():
    from tests.helpers import load_golden
    return load_golden("midas")


def _sd(seed=0):
    if seed not in _SD:
        _SD[seed] = make_midas_state_dict(seed)
    return _SD[seed]


def test_oracle_matches_reference_small():
    g = _golden()
    H, W, iseed, u8 = g["small64_image"]
    y = midas_oracle(_sd(g["seed"]), midas_input(midas_image(H, W, iseed, u8)))[0]
    assert (y - g["small64_fp64"]).abs().max().item() <= 1e-9
    assert (y - g["small64"].double()).abs().max().item() <= 1.01 * g["small64_ref_fp32_err"] + 1e-9


@pytest.mark.parametrize("name", ["sq384", "land448", "port512"])
def test_oracle_matches_reference_windows(name):
    g = _golden()
    H, W, iseed, u8 = g[name + "_image"]
    y = midas_oracle(_sd(g["seed"]), midas_input(midas_image(H, W, iseed, u8)))[0]
    err = max((a - b.double()).abs().max().item() for a, b in zip(windows(y), g[name + "_windows"]))
    assert err <= 1.01 * g[name + "_ref_fp32_err"] + 1e-9, (err, g[name + "_ref_fp32_err"])
    assert g[name + "_zero_frac"] < 0.5 and g[name + "_max"] > 1                 # a non-degenerate map


def test_state_dict_keys_and_shapes():
    assert midas_keys_and_shapes() == [(k, tuple(s)) for k, s in _golden()["keys"]]
    assert len(midas_keys_and_shapes()) == 368


@pytest.mark.parametrize("wrap", [False, True])
def test_checkpoint_loading(tmp_path, monkeypatch, wrap):
    from controlar_b200.condition.midas import CKPT_NAME, DPTDepthModel, load_state_dict_file
    sd = _sd(0)
    path = tmp_path / "condition" / "ckpts" / CKPT_NAME
    path.parent.mkdir(parents=True)
    torch.save({"model": sd, "optimizer": {}} if wrap else sd, str(path))
    got = load_state_dict_file(str(path))
    assert list(got) == list(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    m = DPTDepthModel()
    m.load_state_dict(got, strict=True)
    with pytest.raises(RuntimeError, match="Unexpected|Missing"):
        DPTDepthModel().load_state_dict(dict(sd, extra=torch.zeros(1)), strict=True)


def test_refusals(tmp_path, monkeypatch):
    from controlar_b200.condition.midas import DPTDepthModel, MidasDetector
    with pytest.raises(NotImplementedError, match="dpt_large"):
        MidasDetector(device="cpu", model_type="dpt_large")
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError, match="dpt_hybrid-midas-501f0c75.pt"):
        MidasDetector(device="cpu")
    with pytest.raises(FileNotFoundError, match="nowhere.pt"):
        MidasDetector(device="cpu", model_path=str(tmp_path / "nowhere.pt"))
    m = DPTDepthModel()
    for shape in [(1, 3, 64, 80), (1, 3, 96, 32), (1, 3, 32, 64), (1, 1, 64, 64), (3, 64, 64)]:
        with pytest.raises(ValueError, match="x"):
            m(torch.zeros(shape))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 3, 64, 96))
    det = MidasDetector.__new__(MidasDetector)
    det.model = m
    with pytest.raises(ValueError, match="H, W, 3"):
        det(torch.zeros(64, 96))


CODE = r"""
import sys
from condition.midas.depth import MidasDetector          # sample_t2i_MR.py:34
import controlar_b200.condition.midas as m
assert MidasDetector is m.MidasDetector, MidasDetector
assert "timm" not in sys.modules
print("OK")
"""


def test_dropin_resolves_without_timm(tmp_path):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT])
    r = subprocess.run([sys.executable, "-c", CODE], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-4000:]
