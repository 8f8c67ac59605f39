"""Time the DPT depth detector (`car_dpt_forward`, controlar_b200/condition/depth.py) with DPT-Large's shapes at 512 x 512 (B = 1
and B = 8) and 384 x 384 (B = 8), with CUDA events after warm-up.  Reports ms per image, TFLOP/s of the fp32 work (dpt_gflop below:
962.7 GFLOP per 512^2 image, 516.4 per 384^2 image) and a per-stage split of the kernel time from one profiled forward (encoder
GEMMs, attention, other encoder kernels, neck, head).  When transformers is importable, HF's eager DPTForDepthEstimation runs on the
same weights with TF32 matmuls and convolutions on (as the sample script sets them) and in strict fp32; the TF32 arm's max error
against the strict map is reported.  Prints the card name and power limit, then one JSON line per workload.  Weights are procedural
(tests/dpt_oracle.py)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def dpt_gflop(side, C=1024, L=24, mlp=4096, neck=(256, 512, 1024, 1024), F=256):
    """2 * MACs of every GEMM, attention product and convolution of DPT-Large at side x side: (total, encoder incl. attention,
    attention, neck, head)."""
    h = side // 16
    T = 1 + h * h
    enc = 2 * h * h * C * 768 + L * (2 * T * C * (4 * C + 2 * mlp))
    att = L * 4 * T * T * C
    nk = 0
    for Cn, f, s in zip(neck, (4, 2, 1, 0), (4 * h, 2 * h, h, h // 2)):
        nk += 2 * h * h * 2 * C * C + 2 * h * h * C * Cn
        nk += 2 * h * h * Cn * f * f * Cn if f > 1 else (2 * s * s * 9 * Cn * Cn if f == 0 else 0)
        nk += 2 * s * s * 9 * Cn * F
    for j, s in enumerate((h // 2, h, 2 * h, 4 * h)):
        nk += (4 if j else 2) * 2 * s * s * 9 * F * F + 2 * (2 * s) ** 2 * F * F
    hd = 2 * (8 * h) ** 2 * 9 * F * F // 2 + 2 * (16 * h) ** 2 * 9 * (F // 2) * 32 + 2 * (16 * h) ** 2 * 32
    return tuple(x / 1e9 for x in (enc + att + nk + hd, enc + att, att, nk, hd))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception:
        return torch.cuda.get_device_name()


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
    return ts[len(ts) // 2]


def stage_split(fn):
    """Kernel time (ms) per stage from one profiled call, by launch order: the encoder ends at the first readout kernel, the head is
    the last five launches."""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = sorted([e for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name and "Memset" not in e.name],
                key=lambda e: e.time_range.start)
    names = [e.name for e in ev]
    first_neck = next(i for i, n in enumerate(names) if "dpt_readout_split" in n)
    out = {"encoder_gemms": 0.0, "attention": 0.0, "encoder_other": 0.0, "neck": 0.0, "head": 0.0}
    for i, e in enumerate(ev):
        t = e.time_range.elapsed_us() / 1e3
        if i >= len(ev) - 5:
            out["head"] += t
        elif i >= first_neck:
            out["neck"] += t
        elif "dpt_attention" in e.name:
            out["attention"] += t
        elif "gemm_wgmma_f32" in e.name:
            out["encoder_gemms"] += t
        else:
            out["encoder_other"] += t
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-eager", action="store_true")
    args = ap.parse_args()
    from controlar_b200.condition.depth import DPTForDepthEstimation
    from tests.dpt_oracle import DPT_LARGE, make_dpt_state_dict
    dev = torch.device("cuda")
    sd = make_dpt_state_dict(DPT_LARGE, 0)
    m = DPTForDepthEstimation(DPT_LARGE)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    hf = None
    if not args.no_eager:
        try:
            from transformers import DPTConfig, DPTForDepthEstimation as HF
            hf = HF(DPTConfig(**DPT_LARGE)).eval()
            hf.load_state_dict(sd)
            hf = hf.to(dev)
        except ImportError:
            hf = None
    print("card:", card(), flush=True)
    for B, S in ((1, 512), (8, 512), (8, 384)):
        g = torch.Generator().manual_seed(B * 1000 + S)
        x = (torch.rand(B, 3, S, S, generator=g) * 2 - 1).to(dev)
        tot, enc, att, nk, hd = dpt_gflop(S)
        with torch.no_grad():
            y = m(pixel_values=x).predicted_depth
            med = time_ms(lambda: m(pixel_values=x), args.steps, args.warmup)
            split = stage_split(lambda: m(pixel_values=x))
        res = {"workload": "dpt_large_depth", "batch": B, "size": S, "gpu": card(), "gflop_per_image": round(tot, 1),
               "gflop_split": {"encoder": round(enc - att, 1), "attention": round(att, 1), "neck": round(nk, 1), "head": round(hd, 1)},
               "ms_per_image": round(med / B, 3), "tflops_fp32_work": round(tot * B / med, 1), "stage_ms_per_batch": split,
               "steps": args.steps, "warmup": args.warmup}
        if hf is not None:
            with torch.no_grad():
                arms = {}
                for name, tf32 in (("tf32", True), ("fp32", False)):
                    torch.backends.cuda.matmul.allow_tf32 = tf32
                    torch.backends.cudnn.allow_tf32 = tf32
                    arms[name] = (hf(pixel_values=x).predicted_depth, time_ms(lambda: hf(pixel_values=x), args.steps, args.warmup))
                torch.backends.cuda.matmul.allow_tf32 = False
                torch.backends.cudnn.allow_tf32 = True
            ref = arms["fp32"][0]
            res["hf_eager"] = {"tf32_ms_per_image": round(arms["tf32"][1] / B, 3), "fp32_ms_per_image": round(arms["fp32"][1] / B, 3),
                               "tf32_max_abs_vs_fp32": (arms["tf32"][0] - ref).abs().max().item(),
                               "ours_max_abs_vs_fp32": (y - ref).abs().max().item(), "ref_max": ref.max().item(),
                               "speedup_vs_tf32": round(arms["tf32"][1] / med, 3)}
        else:
            res["hf_eager"] = "not timed: transformers not importable"
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
