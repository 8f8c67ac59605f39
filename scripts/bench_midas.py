"""Time the MiDaS DPT-Hybrid depth detector (`car_midas_forward`, controlar_b200/condition/midas.py) at 384 x 384 and 448 x 768, at
B = 1 (the reference's per-image call) and B = 8, with CUDA events after warm-up.  Reports ms per image and TFLOP/s of the fp32 work
(midas_gflop below, counted from the shapes).  The eager baseline is tests/midas_oracle.py run in fp32 on the same weights with TF32
matmuls and convolutions on: the same network in plain PyTorch ops (transformers' hybrid DPT, which accepts the square size only,
is not timed here).  Prints the card name and power limit, then one JSON line per workload.  Weights are procedural."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def midas_gflop(H, W):
    """2 * MACs of every convolution, GEMM and attention product of DPT-Hybrid at H x W: (total, trunk, ViT, neck + head)."""
    conv = lambda hw, cin, cout, k: 2 * hw * cin * cout * k * k            # noqa: E731
    trunk = conv(H * W // 4, 3, 64, 7)
    hw, cin = H * W // 16, 64
    for s, (d, c) in enumerate(zip((3, 4, 9), (256, 512, 1024))):
        for b in range(d):
            ho = hw // 4 if (s and b == 0) else hw
            mid = c // 4
            trunk += conv(hw, cin, mid, 1) + conv(ho, mid, mid, 3) + conv(ho, mid, c, 1) + (conv(ho, cin, c, 1) if b == 0 else 0)
            hw, cin = ho, c
    P = (H // 16) * (W // 16)
    T = 1 + P
    vit = 2 * P * 1024 * 768 + 12 * (2 * T * 768 * (4 * 768 + 2 * 3072) + 4 * T * T * 768)
    nk = 2 * (2 * P * 1536 * 768 + 2 * P * 768 * 768) + conv(P // 4, 768, 768, 3)
    F = 256
    sizes = [H * W // 16, H * W // 64, P, P // 4]
    for cin, s in zip((256, 512, 768, 768), sizes):
        nk += conv(s, cin, F, 3)
    for j, s in enumerate(reversed(sizes)):
        nk += (4 if j else 2) * conv(s, F, F, 3) + conv(4 * s, F, F, 1)
    nk += conv(H * W // 4, F, F // 2, 3) + conv(H * W, F // 2, 32, 3) + conv(H * W, 32, 1, 1)
    return tuple(x / 1e9 for x in (trunk + vit + nk, trunk, vit, nk))


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-eager", action="store_true")
    args = ap.parse_args()
    from controlar_b200.condition.midas import DPTDepthModel
    from tests.midas_oracle import make_midas_state_dict, midas_oracle
    dev = torch.device("cuda")
    sd = make_midas_state_dict(0)
    m = DPTDepthModel()
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    print("card:", card(), flush=True)
    for B, H, W in ((1, 384, 384), (8, 384, 384), (1, 448, 768), (8, 448, 768)):
        g = torch.Generator().manual_seed(B * 1000 + H + W)
        x = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dev)
        tot, trunk, vit, nk = midas_gflop(H, W)
        with torch.no_grad():
            y = m(x)
            med = time_ms(lambda: m(x), args.steps, args.warmup)
        res = {"workload": "midas_dpt_hybrid_depth", "batch": B, "size": [H, W], "gpu": card(), "gflop_per_image": round(tot, 1),
               "gflop_split": {"trunk": round(trunk, 1), "vit": round(vit, 1), "neck_head": round(nk, 1)},
               "ms_per_image": round(med / B, 3), "tflops_fp32_work": round(tot * B / med, 1), "steps": args.steps, "warmup": args.warmup}
        if not args.no_eager and H == W:
            torch.backends.cuda.matmul.allow_tf32 = True
            torch.backends.cudnn.allow_tf32 = True
            sdd = {k: v.to(dev) for k, v in sd.items()}              # resident weights: the timed window holds no copies
            with torch.no_grad():
                ye = midas_oracle(sdd, x, dtype=torch.float32)
                te = time_ms(lambda: midas_oracle(sdd, x, dtype=torch.float32), args.steps, args.warmup)
            torch.backends.cuda.matmul.allow_tf32 = False
            res["eager_tf32"] = {"ms_per_image": round(te / B, 3), "max_abs_vs_ours": (ye - y).abs().max().item(), "map_max": y.max().item(),
                                 "speedup_vs_eager": round(te / med, 3)}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
