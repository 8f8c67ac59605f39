"""Timing of one training step of BASELINE.json config 5 (LlamaGen-L c2i 256 x 256, canny control through DINOv2-small, bf16
autocast numerics, 32 images per GPU = global batch 256 on 8 GPUs) through the public module API, the way
autoregressive/train/train_c2i_canny.py:190-211 drives it:

    logits, loss = model(cond_idx=labels, idx=z[:, :-1], targets=z, condition=canny)   # car_dino_forward + car_train_forward
    loss.backward()                                                                    # car_train_backward
    optimizer.step()                                                                   # car_adamw_step

Prints one JSON line with CUDA-event times of the three stages (median of --steps after --warmup).  Synthetic inputs, random-init
weights.  The training step is a SURVEY.md §8 "next" row and a first correct path (unfused backward, explicit transposes): this
script exists so the number can be taken; it is not part of bench.py's contract."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="GPT-L")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--image-size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-backward", action="store_true", help="forward + loss only (what config 5 names)")
    ap.add_argument("--dropout-p", type=float, default=0.0, help="resid / ffn dropout (the train scripts' --dropout-p)")
    ap.add_argument("--token-dropout-p", type=float, default=0.0, help="token dropout (the train scripts' --token-dropout-p)")
    ap.add_argument("--drop-path-rate", type=float, default=0.0, help="stochastic depth (the c2i scripts' --drop-path-rate)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    from controlar_b200.autoregressive.models.gpt_t2i import GPT_models
    from controlar_b200.engine import ARTrainHandle
    from controlar_b200.optim import AdamW
    dev = torch.device("cuda", 0)
    n = (args.image_size // 16) ** 2
    torch.manual_seed(0)
    model = GPT_models[args.model](vocab_size=16384, block_size=n, num_classes=1000, cls_token_num=1, model_type="c2i",
                                   condition_type="canny", adapter_size="small", token_dropout_p=args.token_dropout_p,
                                   resid_dropout_p=args.dropout_p, ffn_dropout_p=args.dropout_p,
                                   drop_path_rate=args.drop_path_rate).to(dev).train()
    torch.nn.init.normal_(model.output.weight, std=0.02)         # the reference zero-inits it; zeros would make a degenerate step
    trained = {id(p) for _, p in ARTrainHandle.grad_params(model)}
    for p in model.parameters():                                  # the control encoder stays frozen under this library
        p.requires_grad_(id(p) in trained)
    opt = AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, betas=(0.9, 0.95), weight_decay=0.05)
    g = torch.Generator(device=dev).manual_seed(1)
    B = args.batch
    z = torch.randint(0, 16384, (B, n), device=dev, generator=g)
    labels = torch.randint(0, 1000, (B,), device=dev, generator=g)
    canny = (torch.rand(B, 1, args.image_size, args.image_size, device=dev, generator=g) > 0.9).float().repeat(1, 3, 1, 1) * 2 - 1
    ev = lambda: torch.cuda.Event(enable_timing=True)
    rows = []
    for it in range(args.warmup + args.steps):
        e = [ev() for _ in range(4)]
        torch.cuda.synchronize()
        with torch.enable_grad():
            e[0].record()
            _, loss = model(cond_idx=labels, idx=z[:, :-1], targets=z, condition=canny)
            e[1].record()
            if not args.no_backward:
                loss.backward()
            e[2].record()
            if not args.no_backward:
                opt.step()
                opt.zero_grad(set_to_none=True)
            e[3].record()
        torch.cuda.synchronize()
        if it >= args.warmup:
            rows.append((e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3]), float(loss)))
    med = lambda i: sorted(r[i] for r in rows)[len(rows) // 2]
    total = med(0) + med(1) + med(2)
    print(json.dumps({"workload": f"{args.model} c2i {args.image_size}^2 training step, batch {B} per GPU, bf16 autocast numerics",
                      "forward_loss_ms": med(0), "backward_ms": med(1), "adamw_ms": med(2), "images_per_s": 1000.0 * B / total,
                      "loss_first": rows[0][3], "loss_last": rows[-1][3], "steps": args.steps, "warmup": args.warmup}))


if __name__ == "__main__":
    main()
