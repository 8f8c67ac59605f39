"""CPU: the oracle pinned at the BENCHMARKED shape.  tests/golden/xl_b1_long.pt holds the reference's own bf16 logits for GPT-XL
(dim 1280, 36 layers, V 16384; CFG 4, left-padded masks, control_strength 0.6) along a forced token grid; the CPU restatement
(oracle/ar_oracle.py) replays prefill + 2 decode steps.  Two independent bf16 implementations of the same fp32-exact arithmetic
differ by ~2.5e-2 worst-row rel-L2 at this depth (measured here: 2.48e-2 / 2.42e-2 / 2.43e-2 at steps 0 / 1 / 2, and the same
level — 2.2e-2 ... 2.7e-2 — for the CUDA path, tests/test_zz_xl_parity_gpu.py): this is the noise floor the GPU tolerance is set against."""
import torch

from oracle.weights import GPTSpec, make_gpt_state_dict
from oracle.ar_oracle import AROracle, cfg_combine
from oracle.inputs import text_inputs, xl_ctrl_in
from tests.helpers import load_golden, rel_l2, near_tie_bound


def test_xl_oracle_vs_reference_bf16_three_steps():
    g = load_golden("xl_b1_long")
    spec = GPTSpec(**g["spec"])
    B, T, N_img = g["B"], spec.cls_token_num, g["N_img"]
    orc = AROracle(spec, make_gpt_state_dict(spec, g["seed"], with_adapter=False), torch.bfloat16)
    cond, masks = text_inputs(T, spec.caption_dim, B, g["seed"] + 1, torch.bfloat16)
    assert torch.equal(masks, g["emb_masks"])
    ctrl = xl_ctrl_in(B, N_img, spec.dim, g["seed"] + 7, torch.bfloat16).float()
    cc = torch.cat([cond.float(), torch.zeros_like(cond.float()) + orc.w["cls_embedding.uncond_embedding"]])
    cic = torch.cat([ctrl, torch.zeros_like(ctrl)])
    orc.setup_caches(2 * B, T + N_img)
    orc.apply_emb_masks(torch.cat([masks, masks]))
    lg = orc.prefill(cc, cic, g["control_strength"])[:, -1]
    forced = g["forced_tokens"].long()
    worst = 0.0
    for i in range(3):
        assert i in g["full_steps"]
        ref = g["full_logits"][:, g["full_steps"].index(i)].float()
        worst = max(worst, max(rel_l2(lg[r], ref[r]) for r in range(ref.shape[0])))
        # the oracle's greedy choice vs the reference's: equal, or a near-tie in the reference's own logits
        mine = cfg_combine(lg[None].transpose(0, 1), g["cfg_scale"])[:, 0].argmax(-1)
        for b in range(B):
            if int(mine[b]) != int(g["argmax_cfg"][b, i]):
                assert float(g["margin_cfg"][b, i]) <= 2.0 * near_tie_bound(float(g["raw_absmax"][i]), g["cfg_scale"])
        if i < 2:
            t = forced[:, i]
            lg = orc.decode(torch.cat([t, t]), T + i)
    assert worst < 3.0e-2, f"oracle vs reference at XL shape: worst-row rel-L2 {worst:.3e}"
