"""Run the tokenizer's encoder and the four network detectors (HED, LineArt, DPT, MiDaS DPT-Hybrid) once each at two shapes, on
seeded procedural weights and inputs, and write every output to OUT/<name>.npy.  Two builds of the library run on the same card can
then be compared output for output: a change that touches only how the forwards lay out their workspace, and leaves every buffer at
the offset it had, must give bit-identical files.  `--compare A B` does that comparison and exits non-zero on any difference.
The second shape of each forward is at or near the smallest it accepts, where a scratch buffer is most likely to be short."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def outputs(dev):
    from controlar_b200.condition.depth import DPTForDepthEstimation
    from controlar_b200.condition.hed import ControlNetHED_Apache2
    from controlar_b200.condition.lineart import LineArt
    from controlar_b200.condition.midas import DPTDepthModel
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    from oracle.weights import make_hed_state_dict
    from tests.dpt_oracle import DPT_SMALL, dpt_input, make_dpt_state_dict
    from tests.lineart_oracle import make_lineart_state_dict
    from tests.midas_oracle import make_midas_state_dict

    def image(B, H, W, seed, scale):
        return (torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(seed)) * scale).to(dev)

    out = {}

    def run(name, fn):                                   # a shape one build refuses shows up as a file the other build has
        try:
            r = fn()
        except RuntimeError as e:
            print("%s: FAILED: %s" % (name, e), flush=True)
            return
        for suffix, v in (r.items() if isinstance(r, dict) else (("", r),)):
            out[name + suffix] = v

    with torch.no_grad():
        torch.manual_seed(0)
        vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(dev).eval()
        for B, H, W in ((2, 256, 256), (1, 64, 32)):
            def enc(B=B, H=H, W=W):
                quant, _, (_, _, idx) = vq.encode(image(B, H, W, 1, 2.0) - 1.0)
                return {"_quant": quant, "_idx": idx}
            run("vq_encode_%dx%dx%d" % (B, H, W), enc)
        hed = ControlNetHED_Apache2()
        hed.load_state_dict(make_hed_state_dict(seed=0), strict=True)
        hed = hed.to(dev).eval()
        for B, H, W in ((2, 256, 320), (1, 16, 16)):
            def edges(B=B, H=H, W=W):
                edge, proj = hed.run(image(B, H, W, 2, 255.0).round(), want_projections=True)
                return dict({"_edge": edge}, **{"_proj%d" % k: p for k, p in enumerate(proj)})
            run("hed_%dx%dx%d" % (B, H, W), edges)
        la = LineArt()
        la.load_state_dict(make_lineart_state_dict(8))
        la = la.to(dev).eval()
        for B, H, W in ((2, 256, 320), (1, 5, 7)):
            run("lineart_%dx%dx%d" % (B, H, W), lambda B=B, H=H, W=W: la(image(B, H, W, 3, 255.0).round()))
        dpt = DPTForDepthEstimation(DPT_SMALL)
        dpt.load_state_dict(make_dpt_state_dict(DPT_SMALL, 0))
        dpt = dpt.to(dev).eval()
        for B, S in ((2, 256), (1, 64)):
            run("dpt_%dx%d" % (B, S), lambda B=B, S=S: dpt(pixel_values=dpt_input(B, S, 4).to(dev)).predicted_depth)
        md = DPTDepthModel()
        md.load_state_dict(make_midas_state_dict(0))
        md = md.to(dev).eval()
        for B, H, W in ((2, 192, 256), (1, 64, 64)):
            run("midas_%dx%dx%d" % (B, H, W), lambda B=B, H=H, W=W: md(image(B, H, W, 5, 2.0) - 1.0))
    torch.cuda.synchronize()
    return {k: v.detach().cpu().numpy() for k, v in out.items()}


def compare(a, b):
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    missing = sorted(set(f for f in os.listdir(b) if f.endswith(".npy")) ^ set(names))
    bad = list(missing)
    for f in names:
        if f in missing:
            continue
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        same = x.shape == y.shape and x.dtype == y.dtype and x.tobytes() == y.tobytes()
        print("%-40s %-18s %s" % (f, x.shape, "identical" if same else "DIFFERENT"))
        if not same:
            bad.append(f)
    print("%d files, %d different or missing" % (len(names), len(bad)))
    return 1 if bad or not names else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="directory the outputs are written to")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="compare two output directories bit for bit")
    a = ap.parse_args()
    if a.compare:
        sys.exit(compare(*a.compare))
    os.makedirs(a.out, exist_ok=True)
    for k, v in outputs(torch.device("cuda")).items():
        np.save(os.path.join(a.out, k + ".npy"), v)
        print("%-40s %-18s mean %.6g" % (k, v.shape, float(v.astype(np.float64).mean())))


if __name__ == "__main__":
    main()
