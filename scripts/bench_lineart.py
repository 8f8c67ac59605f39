"""Time the LineArt detector (`car_lineart_forward`, controlar_b200/condition/lineart.py) at the batch of BASELINE config 2 (B = 8)
and 512 x 512, with CUDA events after warm-up; report ms per image and GFLOP/s of the algorithmic fp32 work (derived from the layer
shapes: 161.2 GFLOP per 512^2 image).  Prints the card name and power limit of the same run.  When the reference's unmodified
condition/lineart.py is placed at oracle/_ref/condition/lineart.py (or given with --ref), its PyTorch-eager `LineArt` is timed on the same GPU too and
the speed-up and max-abs difference are reported; that arm is fp32 with cuDNN defaults, which allow TF32 convolutions.
Weights are procedural (tests/lineart_oracle.py).  Prints one JSON line."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def lineart_gflop(H: int, W: int) -> float:
    """2 * MACs of every convolution, from the shapes of condition/lineart.py (transposed convolutions: 9 taps per input pixel)."""
    h1, w1 = (H + 1) // 2, (W + 1) // 2
    h2, w2 = (h1 + 1) // 2, (w1 + 1) // 2
    ho, wo = 4 * h2, 4 * w2
    macs = 3 * 64 * 49 * H * W + 64 * 128 * 9 * h1 * w1 + 128 * 256 * 9 * h2 * w2 + 6 * 256 * 256 * 9 * h2 * w2
    macs += 256 * 128 * 9 * h2 * w2 + 128 * 64 * 9 * (2 * h2) * (2 * w2) + 64 * 1 * 49 * ho * wo
    return 2 * macs / 1e9


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts


def load_reference(path):
    if "controlnet_aux" not in sys.modules:                 # imported at the top of the reference module, never used by LineArt
        sys.modules["controlnet_aux"] = types.SimpleNamespace(LineartDetector=None)
    spec = importlib.util.spec_from_file_location("ref_condition_lineart", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.LineArt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref", default=os.path.join(ROOT, "oracle", "_ref", "condition", "lineart.py"))
    args = ap.parse_args()
    from controlar_b200.condition.lineart import LineArt
    from tests.lineart_oracle import make_lineart_state_dict
    dev = torch.device("cuda")
    B, S = args.batch, args.size
    sd = make_lineart_state_dict(8)
    m = LineArt()
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(B, 3, S, S, generator=g) * 255).round().to(dev)
    gf = lineart_gflop(S, S)
    with torch.no_grad():
        y = m(x)
        med, ts = time_ms(lambda: m(x), args.steps, args.warmup)
    res = {"workload": "lineart", "batch": B, "size": [S, S], "gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(),
           "gflop_per_image": round(gf, 2), "ms_per_batch": round(med, 3), "ms_per_image": round(med / B, 4),
           "gflops": round(gf * B / (med / 1e3), 1), "ms_per_batch_min_max": [round(ts[0], 3), round(ts[-1], 3)],
           "steps": args.steps, "warmup": args.warmup}
    if os.path.exists(args.ref):
        Ref = load_reference(args.ref)
        r = Ref().to(dev).eval()
        r.load_state_dict(sd)
        with torch.no_grad():
            yr = r(x)
            rmed, _ = time_ms(lambda: r(x), args.steps, args.warmup)
        res["reference_eager"] = {"ms_per_batch": round(rmed, 3), "ms_per_image": round(rmed / B, 4), "speedup": round(rmed / med, 3),
                                  "max_abs_diff": (y - yr).abs().max().item(),
                                  "arithmetic": "fp32, cuDNN defaults (torch.backends.cudnn.allow_tf32=%s: TF32 convolutions allowed)"
                                                % torch.backends.cudnn.allow_tf32}
    else:
        res["reference_eager"] = "not timed: %s not present" % os.path.relpath(args.ref, ROOT)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
