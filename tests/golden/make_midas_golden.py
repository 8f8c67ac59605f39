"""Regenerate tests/golden/midas.pt: the reference's own MidasDetector and DPTDepthModel (condition/midas, model_type "dpt_hybrid"),
run on the CPU in fp32 and fp64 on the procedural weights of tests/midas_oracle.py (saved to a temporary checkpoint that
ISL_PATHS["dpt_hybrid"] points at), with tests/midas_timm_standin.py injected as `timm`.  Cases (B = 1, as the detector calls it):
  sq384      384 x 384 from a uint8 image (position grid 24 x 24, the identity resize)
  land448    448 x 768 from a uint8 image (the multi-resolution sampler's landscape size, grid 28 x 48)
  port512    512 x 320 from a float32 image (grid 32 x 20)
  small64    64 x 96 from a uint8 image (2 x 3 at 1/32, the smallest frames)
Stored per case: windows of the fp32 map (full maps for small64, with its fp64 map), the map's maximum, the reference's own fp32
error against its fp64 map, the detector's uint8 output (in full for land448 and small64), the image seeds; plus the state-dict
keys and shapes.  Run: python tests/golden/make_midas_golden.py <reference root> (several minutes on the CPU)."""
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import midas_timm_standin  # noqa: E402
from tests.midas_oracle import make_midas_state_dict, midas_image, midas_input, windows  # noqa: E402

SEED = 0
CASES = {"sq384": (384, 384, 21, True), "land448": (448, 768, 22, True), "port512": (512, 320, 23, False), "small64": (64, 96, 24, True)}


@torch.no_grad()
def main(ref_root):
    sys.modules["timm"] = midas_timm_standin
    sys.path.insert(0, ref_root)
    import condition.midas.depth as ref
    sd = make_midas_state_dict(SEED)
    out = {"seed": SEED, "keys": [(k, tuple(v.shape)) for k, v in sd.items()]}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "dpt_hybrid-midas-501f0c75.pt")
        torch.save(sd, path)
        ref.ISL_PATHS["dpt_hybrid"] = path
        det = ref.MidasDetector(device=torch.device("cpu"))
    model = det.model.model
    assert list(model.state_dict()) == list(sd), "the container's key order differs from the reference's"
    for name, (H, W, iseed, u8) in CASES.items():
        img = midas_image(H, W, iseed, uint8=u8)
        x = midas_input(img)
        y32 = model.float()(x.float())
        y64 = model.double()(x.double())
        model.float()
        out[name + "_image"] = (H, W, iseed, u8)
        out[name + "_ref_fp32_err"] = (y32.double() - y64).abs().max().item()
        out[name + "_max"] = y64.max().item()
        out[name + "_zero_frac"] = (y64 == 0).double().mean().item()
        u = torch.from_numpy(det(img.permute(2, 0, 1).permute(1, 2, 0)))           # a permuted (non-contiguous) view, as test_c2i.py passes
        if name == "small64":
            out[name] = y32[0].clone()
            out[name + "_fp64"] = y64[0].clone()
        else:
            out[name + "_windows"] = windows(y32[0])
        if name in ("land448", "small64"):
            out[name + "_u8"] = u.clone()
        else:
            out[name + "_u8_windows"] = windows(u)
        print(name, tuple(y32.shape), "max", out[name + "_max"], "zero", out[name + "_zero_frac"], "fp32 err", out[name + "_ref_fp32_err"],
              flush=True)
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "midas.pt")
    torch.save(out, dst)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
