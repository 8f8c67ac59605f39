"""Wide-batch decode at the config-2 shape (GPT-XL t2i + DINOv2-small canny, 512 x 512, CFG 4, top-k 2000): images/s end to end
(control encoder + prefill + decode + VQ decode) and decode ms/step per batch size, with the decode loop's algorithmic bytes
(car_decode_step_bytes) over its time as a share of the H100 SXM's 3.35 TB/s.

    python scripts/bench_wide.py [--batches 8,16,25,32] [--steps 1] [--compare OTHER_TREE] [--runs 2] [--out FILE]

Each measurement runs in a child process that imports the package from a source tree (built there beforehand).  With --compare,
the other tree (e.g. a checkout of an earlier commit) and this one run alternately, `--runs` times each, in one call, so both see
the same card and session; batch sizes <= 8 run on this tree only.  The card's name, power limit and SM clock are read in the same
call and printed with the results."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HBM_TBS = 3.35


def worker(args):
    import torch
    from controlar_b200 import _lib
    from controlar_b200.autoregressive.models.gpt_t2i import GPT_models
    from controlar_b200.autoregressive.models.generate import generate
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    from controlar_b200.synthetic import text_inputs, control_map
    from controlar_b200.engine import make_sampling
    assert torch.cuda.is_available(), "bench_wide.py needs a CUDA device"
    _lib.lib()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    N, T, gs = 1024, 120, 32
    gpt = GPT_models["GPT-XL"](block_size=gs * gs, cls_token_num=T, model_type="t2i", condition_type="canny", adapter_size="small").eval()
    gpt.output.weight.data.normal_(0, 0.02)
    for blk in gpt.adapter.model.encoder.layer:
        blk.layer_scale1.lambda1.data.fill_(1.0); blk.layer_scale2.lambda1.data.fill_(1.0)
    gpt = gpt.to(dev, torch.bfloat16)
    vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(dev).eval()
    kw = dict(cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True)
    for B in [int(b) for b in args.batches.split(",")]:
        cond, masks = text_inputs(T, 2048, B, 1000, torch.bfloat16)
        cmap = control_map(B, 512, 512, 2000, "canny", torch.bfloat16)
        cond, masks, cmap = cond.to(dev), masks.to(dev), cmap.to(dev)

        def one(seed):
            toks = generate(gpt, cond, N, emb_masks=masks, condition=cmap, seed=seed, **kw)
            return toks, vq.decode_code(toks, [B, 8, gs, gs])

        one(0)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            toks, img = one(1 + i)
        e1.record()
        torch.cuda.synchronize()
        e2e_ms = e0.elapsed_time(e1) / args.steps
        # the decode loop alone (prefill excluded), on the state generate() left
        st = gpt._car_state
        cc = torch.cat([cond, torch.zeros_like(cond) + gpt.cls_embedding.uncond_embedding])
        ctrl = gpt._car_encoder.forward(cmap, apply_mlp=True)
        cic = torch.cat([ctrl, torch.zeros_like(ctrl)])
        sp = make_sampling(1.0, 2000, 1.0, True, 4.0, -1, 7)
        st.prefill(cc, cic, 1.0, all_rows=False)
        e0.record(); st.generate(sp, N, None, dev); e1.record()
        torch.cuda.synchronize()
        dec_ms = e0.elapsed_time(e1)
        step_bytes = sum(st.step_bytes(T + 1 + k) for k in range(N - 1))
        print("WIDE " + json.dumps({"tree": args.worker, "B": B, "B_eff": 2 * B, "images_per_s": B / (e2e_ms * 1e-3),
                                    "e2e_ms": e2e_ms, "decode_ms": dec_ms, "decode_ms_per_step": dec_ms / (N - 1),
                                    "decode_hbm_fraction": step_bytes / (dec_ms * 1e-3) / (HBM_TBS * 1e12),
                                    "finite": bool(torch.isfinite(img).all())}), flush=True)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")]))
    except Exception as e:       # the numbers are still printed, without the card's state
        return {"error": str(e)}


def run_tree(tree, batches, steps):
    env = dict(os.environ, PYTHONPATH=tree)
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", tree, "--batches", batches, "--steps", str(steps)]
    out = subprocess.run(cmd, cwd=tree, env=env, capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError(f"{tree}: exit {out.returncode}\n{out.stderr[-4000:]}")
    return [json.loads(l[5:]) for l in out.stdout.splitlines() if l.startswith("WIDE ")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,16,25,32")
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--compare", default=None, metavar="OTHER_TREE")
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    rows = []
    info = card()
    print("CARD " + json.dumps(info), flush=True)
    wide = ",".join(b for b in args.batches.split(",") if int(b) > 8)
    for r in range(args.runs if args.compare else 1):
        if args.compare and wide:
            rows += [dict(x, run=r, which="compare") for x in run_tree(os.path.abspath(args.compare), wide, args.steps)]
        rows += [dict(x, run=r, which="this") for x in run_tree(ROOT, args.batches if r == 0 else (wide or args.batches), args.steps)]
    print("CARD_AFTER " + json.dumps(card()), flush=True)
    for x in rows:
        print(json.dumps(x), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
