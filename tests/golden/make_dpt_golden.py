"""Regenerate tests/golden/dpt.pt: transformers' own DPTForDepthEstimation, run on the CPU in fp32 and fp64 on the procedural
weights of tests/dpt_oracle.py (1.4 GB for DPT-Large, regenerated from the seed and never stored).  Cases:
  large_b2_384  DPT-Large, B = 2 at 384 x 384 (position grid 24 x 24, the identity resize): windows of the fp32 maps
  large_b1_512  DPT-Large, B = 1 at 512 x 512 (the sample scripts' size, position grid resized 24 -> 32): windows of the fp32 map
  small_b2_128  the small config, B = 2 at 128 x 128 (position grid 6 -> 8): full fp32 maps, the fp64 map of the first image
plus DPT-Large's state-dict keys and shapes, the seeds, the output shapes and HF's own fp32 error against its fp64 output.
Run: python tests/golden/make_dpt_golden.py (needs transformers; several minutes on the CPU)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.dpt_oracle import DPT_LARGE, DPT_SMALL, dpt_input, make_dpt_state_dict, windows  # noqa: E402

SEED = 0
CASES = {"large_b2_384": (DPT_LARGE, 2, 384, 11), "large_b1_512": (DPT_LARGE, 1, 512, 12), "small_b2_128": (DPT_SMALL, 2, 128, 13)}


@torch.no_grad()
def main():
    import transformers
    from transformers import DPTConfig, DPTForDepthEstimation
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"transformers": transformers.__version__, "seed": SEED}
    models = {}
    for name, (cfg, B, side, iseed) in CASES.items():
        key = "large" if cfg is DPT_LARGE else "small"
        if key not in models:
            m = DPTForDepthEstimation(DPTConfig(**cfg)).eval()
            sd = make_dpt_state_dict(cfg, SEED)
            m.load_state_dict(sd, strict=True)
            models[key] = m
            out[key + "_keys"] = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
            out["attn_implementation"] = m.config._attn_implementation
        m = models[key]
        x = dpt_input(B, side, iseed)
        y32 = m.float()(pixel_values=x).predicted_depth
        y64 = m.double()(pixel_values=x.double()).predicted_depth
        m.float()
        out[name + "_input_seed"] = iseed
        out[name + "_shape"] = tuple(y32.shape)
        out[name + "_ref_fp32_err"] = (y32.double() - y64).abs().max().item()
        out[name + "_max"] = y64.max().item()
        out[name + "_zero_frac"] = (y64 == 0).double().mean().item()
        if key == "large":
            out[name + "_windows"] = windows(y32)
        else:
            out[name] = y32.clone()
            out[name + "_fp64"] = y64[:1].clone()
        print(name, tuple(y32.shape), "max", out[name + "_max"], "zero", out[name + "_zero_frac"], "fp32 err", out[name + "_ref_fp32_err"],
              flush=True)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dpt.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
