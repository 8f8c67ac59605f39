"""Serving a queue of requests with mixed sampling configurations, at the config-2 shape (GPT-XL t2i + DINOv2-small canny,
512 x 512 = 1024 tokens, CFG 4, 8 images per launch): the serving engine with `mixed_sampling` off (one launch per group of
identical SamplingParams and control strength) and on (any 8 requests of one grid share a launch).

  python scripts/bench_mixed_serve.py [--requests 64] [--configs 8] [--out DIR]

The queue cycles through `--configs` sampling configurations (temperature, top-k, top-p, greedy) and two control strengths,
each request with its own seed, so that with the engine's default grouping the launches are small; that is the case mixed mode is
for.  Prints one JSON line: per mode the launches, wall time and images/s of the whole queue (VQ decode included), and the decode
loop's ms/step (CUDA events around car_generate, prefill excluded) of one mixed B = 8 launch against a uniform B = 8 launch,
median of alternating runs.  Needs a CUDA device; writes nothing unless --out is given."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (temperature, top_k, top_p, greedy)
SAMPLING = [(1.0, 2000, 1.0, False), (0.7, 2000, 1.0, False), (1.3, 1000, 0.95, False), (1.0, 0, 0.9, False),
            (1.0, 100, 1.0, False), (0.9, 4000, 1.0, False), (1.0, 2000, 0.8, False), (1.0, 2000, 1.0, True)]
STRENGTHS = (1.0, 0.6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--configs", type=int, default=8, help="sampling configurations in the queue (<= 8)")
    ap.add_argument("--repeats", type=int, default=3, help="alternating decode timings per kind")
    ap.add_argument("--out", default=None, help="also write the JSON line to OUT/bench_mixed_serve.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mixed_serve.py needs a CUDA device"
    from controlar_b200.autoregressive.models.gpt_t2i import GPT_models
    from controlar_b200.autoregressive.serve.llm import LLM, SamplingParams
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    from controlar_b200.synthetic import text_inputs, control_map
    from controlar_b200 import engine
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    N, T, B = 1024, 120, 8
    gpt = GPT_models["GPT-XL"](block_size=N, cls_token_num=T, model_type="t2i", condition_type="canny", adapter_size="small").eval()
    gpt.output.weight.data.normal_(0, 0.02)
    for blk in gpt.adapter.model.encoder.layer:
        blk.layer_scale1.lambda1.data.fill_(1.0); blk.layer_scale2.lambda1.data.fill_(1.0)
    gpt = gpt.to(dev, torch.bfloat16)
    vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(dev).eval()
    R = a.requests
    cond, masks = text_inputs(T, 2048, R, 1000, torch.bfloat16)
    cmap = control_map(R, 512, 512, 2000, "canny", torch.bfloat16)
    cond, masks, cmap = cond.to(dev), masks.to(dev), cmap.to(dev)
    cfgs = SAMPLING[:a.configs]

    def request(i):
        t, k, p, greedy = cfgs[i % len(cfgs)]
        sp = SamplingParams(temperature=0 if greedy else t, top_k=k, top_p=p, max_tokens=N, seed=10_000 + i)
        return dict(cond=cond[i], emb_mask=masks[i], control=cmap[i], control_strength=STRENGTHS[(i // len(cfgs)) % 2], sampling_params=sp)

    def serve(mixed, n):
        llm = LLM(model=gpt, vq=vq, cfg_scale=4.0, max_images_per_batch=B, seed=1, mixed_sampling=mixed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs = llm.generate(prompts=[request(i) for i in range(n)])
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        assert len(outs) == n and all(o.image is not None for o in outs)
        return {"launches": llm._launches, "seconds": round(s, 3), "images_per_s": round(n / s, 3)}

    # warm-up: one launch loads every module; a new batch size only adds a state's allocations (milliseconds)
    serve(True, B)
    res = {"default": serve(False, R), "mixed": serve(True, R)}

    # decode ms/step of one B = 8 launch: uniform (scalar CarSampling) against mixed (one CarRowSampling per image)
    gpt.setup_caches(2 * B, T + N, torch.bfloat16, n_img_tokens=N)
    st = gpt._car_state
    st.set_emb_mask(torch.cat([masks[:B], masks[:B]]))
    cc = torch.cat([cond[:B], torch.zeros_like(cond[:B]) + gpt.cls_embedding.uncond_embedding])
    ctrl = gpt._car_encoder.forward(cmap[:B], apply_mlp=True)
    cic = torch.cat([ctrl, torch.zeros_like(ctrl)])
    sp = engine.make_sampling(1.0, 2000, 1.0, True, 4.0, -1, 7)
    rows = []
    for b in range(B):
        t, k, p, greedy = cfgs[b % len(cfgs)]
        rows.append(engine.make_row_sampling(t, k, p, not greedy, 10_000 + b, 0, STRENGTHS[b % 2]))
    times = {"uniform": [], "mixed": []}
    for _ in range(a.repeats):
        for kind in ("uniform", "mixed"):
            st.set_row_sampling(rows if kind == "mixed" else None)
            st.prefill(cc, cic, 1.0, all_rows=False)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); st.generate(sp, N, None, dev); e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1) / (N - 1))
    st.set_row_sampling(None)
    res["decode_ms_per_step_b8"] = {k: round(statistics.median(v), 4) for k, v in times.items()}
    res["decode_ms_per_step_b8_runs"] = {k: [round(x, 4) for x in v] for k, v in times.items()}
    res["queue"] = {"requests": R, "sampling_configs": len(cfgs), "strengths": list(STRENGTHS), "images_per_launch": B,
                    "shape": "GPT-XL t2i + DINOv2-small canny 512x512, cfg 4.0"}
    res["gpu"] = torch.cuda.get_device_name(0)
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_mixed_serve.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
