"""Timing of one training step of BASELINE.json config 5 (LlamaGen-L c2i 256 x 256, canny control through DINOv2-small, bf16
autocast numerics, 32 images per GPU = global batch 256 on 8 GPUs) through the public module API, the way
autoregressive/train/train_c2i_canny.py:190-211 drives it:

    logits, loss = model(cond_idx=labels, idx=z[:, :-1], targets=z, condition=canny)   # car_dino_forward + car_train_forward
    loss.backward()                                                                    # car_train_backward (+ car_dino_train_backward)
    optimizer.step()                                                                   # car_adamw_step

--train-encoder makes the control encoder trainable as the reference's loop does (its forward is then car_dino_train_forward).
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
    ap.add_argument("--model-type", choices=["c2i", "t2i"], default="c2i", help="t2i: 120 caption tokens of a flan-t5-xl width")
    ap.add_argument("--train-encoder", action="store_true",
                    help="train the control encoder too, as the reference loop does (default: frozen, the transformer only)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    from controlar_b200.autoregressive.models.gpt_t2i import GPT_models
    from controlar_b200.engine import ARTrainHandle
    from controlar_b200.optim import AdamW
    dev = torch.device("cuda", 0)
    n = (args.image_size // 16) ** 2
    torch.manual_seed(0)
    t2i = args.model_type == "t2i"
    T = 120 if t2i else 1
    model = GPT_models[args.model](vocab_size=16384, block_size=n, num_classes=1000, cls_token_num=T, model_type=args.model_type,
                                   condition_type="canny", adapter_size="small", token_dropout_p=args.token_dropout_p,
                                   resid_dropout_p=args.dropout_p, ffn_dropout_p=args.dropout_p,
                                   drop_path_rate=args.drop_path_rate).to(dev).train()
    torch.nn.init.normal_(model.output.weight, std=0.02)         # the reference zero-inits it; zeros would make a degenerate step
    trained = {id(p) for _, p in ARTrainHandle.grad_params(model)}
    if args.train_encoder:
        from controlar_b200.vision import encoder_train_params
        trained |= {id(p) for _, _, p in encoder_train_params(model.adapter.model)}
    for p in model.parameters():                                  # frozen: whatever the step does not train
        p.requires_grad_(id(p) in trained)
    opt = AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, betas=(0.9, 0.95), weight_decay=0.05)
    g = torch.Generator(device=dev).manual_seed(1)
    B = args.batch
    z = torch.randint(0, 16384, (B, n), device=dev, generator=g)
    if t2i:
        labels = torch.randn(B, T, model.config.caption_dim, device=dev, generator=g) * 0.1
    else:
        labels = torch.randint(0, 1000, (B,), device=dev, generator=g)
    canny = (torch.rand(B, 1, args.image_size, args.image_size, device=dev, generator=g) > 0.9).float().repeat(1, 3, 1, 1) * 2 - 1
    canny = canny.to(torch.bfloat16)                              # condition_img.to(ptdtype), train_t2i_canny.py:167
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
    import subprocess
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True).stdout.strip()
    enc = "control encoder trained" if args.train_encoder else "control encoder frozen"
    print(json.dumps({"workload": f"{args.model} {args.model_type} {args.image_size}^2 training step, batch {B} per GPU, bf16 autocast "
                                  f"numerics, {enc}", "gpu": torch.cuda.get_device_name(dev), "power_limit": power,
                      "forward_loss_ms": med(0), "backward_ms": med(1), "adamw_ms": med(2), "images_per_s": 1000.0 * B / total,
                      "loss_first": rows[0][3], "loss_last": rows[-1][3], "steps": args.steps, "warmup": args.warmup}))


if __name__ == "__main__":
    main()
