"""CPU: the trainable control encoder's oracle (oracle/train_encoder_oracle.py) against the reference's own training step with
the encoder trainable (tests/golden/train_enc_*.pt, tests/golden/make_train_encoder_golden.py), the parameter set the library
trains, the C entry points' argument checks, and the encoder's gradients under a world-size-2 gloo DDP step.

Measured oracle-to-reference gaps over the five cases (torch 2.11 CPU, bf16 autocast, math SDPA): feat probe 3.4e-3 .. 7.8e-3,
loss 7e-7 .. 9e-5 relative, gradient probes per tensor <= 3.1e-2 (rel-L2 of the probed values or relative norm difference; the
largest are the attention query / key weights, whose gradients are small differences of bf16-rounded terms).  The key bias is left
out of that figure: softmax is invariant to it, its gradient is zero up to rounding (norm ~1e-8) on both sides.  The bars below
sit above those figures."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.weights import GPTSpec, make_gpt_state_dict, vit_shapes, _fill
from oracle.inputs import text_inputs, class_inputs, control_map, code_inputs, train_attn_mask
from oracle.train_oracle import TrainOracle, grad_probe
from oracle.train_encoder_oracle import encoder_forward, encoder_params
from tests.helpers import load_golden, log_measurement, rel_l2

CASES = ["train_enc_dinov2s_canny_c2i_128", "train_enc_dinov2s_canny_c2i_256", "train_enc_dinov2b_depth_t2i_128",
         "train_enc_dinov2s_mr_t2i_128x192", "train_enc_vit_gptpy_c2i_64"]
FEAT_BAR, LOSS_BAR, PROBE_BAR = 1e-2, 2e-4, 5e-2


def case_setup(g):
    """(spec, full state dict, is_vit, inputs) of a golden case, as make_train_encoder_golden.py built them"""
    spec = GPTSpec(**g["spec"])
    seed, B, H, W = g["seed"], g["B"], g["H"], g["W"]
    vit = "vit_layers" in g
    if vit:
        sd = dict(make_gpt_state_dict(spec, seed, with_adapter=False))
        sd.update(_fill(vit_shapes(384, layers=g["vit_layers"], prefix="adapter.model."), seed, 0.02))
        sd["condition_norm.weight"] = torch.ones(spec.dim)
    else:
        sd = make_gpt_state_dict(spec, seed)
    N = (H // 16) * (W // 16)
    if spec.model_type == "t2i":
        cond, masks = text_inputs(spec.cls_token_num, spec.caption_dim, B, seed + 1, torch.float32)
    else:
        cond, masks = class_inputs(spec.num_classes, B, seed + 1), None
    cmap = control_map(B, H, W, seed + 2, g["kind"], torch.float32).to(torch.bfloat16)
    z = code_inputs(spec.vocab_size, B, N, seed + 4)
    mask = train_attn_mask(masks, N) if g["use_mask"] else None
    valid = None if g["valid"] is None else torch.tensor(g["valid"])
    return spec, sd, vit, (cond, cmap, z, mask, valid)


def oracle_step(g):
    """autograd over the encoder oracle followed by the transformer oracle -> (feat, loss, {encoder key: grad})"""
    spec, sd, vit, (cond, cmap, z, mask, valid) = case_setup(g)
    p = encoder_params(sd)
    if vit:         # gpt.py's token_drop gives dropped samples zeros (tests/test_train_oracle_golden.py::test_legacy_gptpy_*)
        sd = dict(sd, **{"condition_mlp.uncond_embedding": torch.zeros_like(sd["condition_mlp.uncond_embedding"])})
    heads = p["layernorm.weight"].shape[0] // 64
    with torch.enable_grad():
        feat = encoder_forward(p, cmap, vit, spec.condition_type, heads, 1e-12 if vit else 1e-6)
        _, loss = TrainOracle(spec, sd, torch.bfloat16).forward(z[:, :-1], cond, feat, g["drop_ids"], mask, z, valid)
        loss.backward()
    return feat.detach(), float(loss.detach()), {k: t.grad for k, t in p.items()}


def probe_gap(key, t, ref, n):
    """max of the rel-L2 of t's probed values against the stored ones and the relative difference of the norms"""
    pr = grad_probe(key, t, n)
    m = pr["val"].numel()
    return max(rel_l2(pr["val"], ref["val"][:m]), abs(float(pr["norm"]) - float(ref["norm"])) / float(ref["norm"]))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_training_step(name):
    g = load_golden(name)
    feat, loss, grads = oracle_step(g)
    e_feat = probe_gap("feat", feat, g["feat"], g["probe_sizes"]["feat"])
    e_loss = abs(loss - float(g["loss"])) / float(g["loss"])
    eg = g["enc_grads"]
    keys = [k[len("adapter.model."):] for k in eg["keys"]]
    assert sorted(keys) == sorted(grads), "the oracle's trainable set differs from the reference's"
    worst, worst_k = 0.0, None
    for i, k in enumerate(keys):
        if k.endswith("key.bias"):
            kw = float(grads[k.replace("key.bias", "key.weight")].norm())
            assert float(grads[k].norm()) < 1e-2 * kw and float(eg["norm"][i]) < 1e-2 * kw
            continue
        e = probe_gap(eg["keys"][i], grads[k], {"val": eg["val"][i], "norm": eg["norm"][i]}, g["probe_sizes"]["grad"])
        if e > worst:
            worst, worst_k = e, k
    log_measurement("train_encoder_oracle.txt", f"{name}: feat {e_feat:.2e} loss {e_loss:.2e} worst probe {worst:.2e} ({worst_k})\n")
    assert e_feat < FEAT_BAR and e_loss < LOSS_BAR and worst < PROBE_BAR, (e_feat, e_loss, worst, worst_k)


@pytest.mark.parametrize("name", ["train_enc_dinov2s_canny_c2i_128", "train_enc_vit_gptpy_c2i_64"])
def test_library_trains_the_reference_parameter_set(name):
    """The parameters the library hands gradients to are exactly the ones the reference's backward reaches: the encoder
    parameters on the forward path (all but embeddings.mask_token and ViT's pooler.dense.*) plus the transformer's."""
    from controlar_b200.vision import encoder_train_params
    from controlar_b200.engine import ARTrainHandle
    g = load_golden(name)
    if "vit_layers" in g:
        from controlar_b200.autoregressive.models.vit_adapter import ViT_Adapter
        ad = ViT_Adapter(layers=g["vit_layers"])
    else:
        from controlar_b200.autoregressive.models.dinov2_adapter import Dinov2_Adapter
        spec = GPTSpec(**g["spec"])
        ad = Dinov2_Adapter(adapter_size=spec.adapter_size, condition_type=spec.condition_type)
    names = {id(p): "adapter." + n for n, p in ad.named_parameters()}
    enc = sorted(names[id(p)] for _, _, p in encoder_train_params(ad.model))
    want = sorted(k for k in g["params_with_grad"] if k.startswith("adapter.model."))
    assert enc == want
    assert len(set(enc)) == len(enc)
    # the transformer side: the parameters car_train_backward produces (plus the condition norm only the legacy class has and never
    # uses in training) are the reference's non-encoder parameters with a gradient
    other = {k for k in g["params_with_grad"] if not k.startswith("adapter.")}
    assert "adapter_mlp.fc1.weight" in other and "adapter_mlp.fc2.weight" in other


def _weights_struct(vision, layers, fill=1, ls=True):
    w = vision.CarDinoWeights()
    for f in ("cls_token", "pos_emb", "patch_w", "patch_b", "ln_w", "ln_b"):
        setattr(w, f, fill)
    keep = []
    import ctypes as C
    for f in vision._DINO_ARRAYS:
        if f in ("ls1", "ls2") and not ls:
            continue
        arr = (C.c_void_p * layers)(*([fill] * layers))
        keep.append(arr)
        setattr(w, f, C.cast(arr, C.POINTER(C.c_void_p)))
    return w, keep


def test_entry_points_reject_bad_arguments_before_any_cuda_call():
    """Each call differs from a valid one in one argument; the library refuses it before it allocates or launches (the pointers
    are never dereferenced)."""
    import ctypes as C
    from controlar_b200 import _lib, vision
    lib = _lib.lib()
    good = dict(dtype=_lib.CAR_F32, hidden=384, heads=6, layers=2, patch=14, pos_grid=37, resize_mode=0, adapter_out_dim=0, eps=1e-6)
    w, keep = _weights_struct(vision, 2)
    h = C.c_void_p()

    def create(desc=None, weights=w, **kw):
        d = vision.CarDinoDesc(**dict(good, **kw)) if desc is None else desc
        return lib.car_dino_train_create(C.byref(d), C.byref(weights), None, C.byref(h))
    assert lib.car_dino_train_create(None, C.byref(w), None, C.byref(h)) < 0 and b"null" in lib.car_last_error()
    assert create(dtype=_lib.CAR_BF16) < 0 and b"fp32" in lib.car_last_error()
    assert create(heads=4) < 0 and b"head_dim" in lib.car_last_error()
    assert create(patch=8) < 0 and b"patch" in lib.car_last_error()
    assert create(layers=0) < 0 and create(resize_mode=2) < 0
    w_null, k2 = _weights_struct(vision, 2)
    w_null.ln_b = None
    assert create(weights=w_null) < 0 and b"null weight" in lib.car_last_error()
    w_hole, k3 = _weights_struct(vision, 2)
    w_hole.fc1_w[1] = None
    assert create(weights=w_hole) < 0 and b"null weight" in lib.car_last_error()
    w_ls, k4 = _weights_struct(vision, 2)
    w_ls.ls2 = None
    assert create(weights=w_ls) < 0 and b"ls1 and ls2" in lib.car_last_error()
    assert not h
    # forward / backward on no handle, bad shapes
    assert lib.car_dino_train_forward(None, 1, 1, 16, 16, 1, None) < 0 and b"null" in lib.car_last_error()
    assert lib.car_dino_train_backward(None, 1, C.byref(w), None) < 0 and b"null" in lib.car_last_error()
    assert lib.car_dino_train_destroy(None) == 0


# ---- DDP (the reference wraps the model in DistributedDataParallel with find_unused_parameters=True, train_c2i_canny.py:173) ----
# The encoder's backward reaches its parameters through a torch.autograd.Function, so DDP's hooks fire and torch all-reduces.
# Library calls are stubbed (no GPU here): each rank's encoder "backward" returns gradients equal to rank + 1, so every encoder
# .grad must end at the mean 1.5 on both ranks, and mask_token (off the path) must stay without one.
def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker_ddp(rank: int, world: int, port: int, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from torch.nn.parallel import DistributedDataParallel as DDP
        from controlar_b200 import engine, vision
        from controlar_b200.autoregressive.models import gpt_t2i

        class TrainStub:
            grad_params = staticmethod(engine.ARTrainHandle.grad_params)

            def __init__(self, module, B, n):
                self.key = tuple(p.data_ptr() for p in module.parameters())
                self.max_batch, self.max_img_tokens, self.generation = B, n, 0

            def forward(self, idx, cond, feat, drop, mask, targets, valid):
                self.generation += 1
                self.feat_shape = feat.shape
                return torch.zeros(idx.shape[0], idx.shape[1] + 1, 64), torch.tensor(float(rank))

            def backward(self, module, loss_grad=None, want_feat_grad=True):
                return ({k: torch.full_like(p, float(rank + 1)) for k, p in self.grad_params(module)},
                        torch.ones(self.feat_shape, dtype=torch.bfloat16) if want_feat_grad else None)

            def close(self):
                pass

        class EncoderStub:
            key_of = staticmethod(vision.DinoTrainHandle.key_of)

            def __init__(self, adapter):
                self.params = vision.encoder_train_params(adapter.model)
                self.key = self.key_of(adapter)
                self.generation = 0
                self.hidden = adapter.model.hidden

            def forward(self, x):
                self.generation += 1
                return torch.zeros(x.shape[0], (x.shape[2] // 16) * (x.shape[3] // 16), self.hidden)

            def backward(self, dfeat, want):
                assert dfeat.dtype == torch.float32 and float(dfeat.min()) == float(dfeat.max()) == 1.0
                return [torch.full_like(p, float(rank + 1)) if wnt else None for (_, _, p), wnt in zip(self.params, want)]

            def close(self):
                pass
        engine.ARTrainHandle = TrainStub
        vision.DinoTrainHandle = EncoderStub
        torch.manual_seed(0)
        m = gpt_t2i.Transformer(gpt_t2i.ModelArgs(dim=128, n_layer=3, n_head=2, vocab_size=64, cls_token_num=1, block_size=16, num_classes=10,
                                                  model_type="c2i", adapter_size="small", condition_type="canny", token_dropout_p=0.0,
                                                  resid_dropout_p=0.0, ffn_dropout_p=0.0, class_dropout_prob=0.1)).train()
        ddp = DDP(m, find_unused_parameters=True)
        with torch.enable_grad():
            for _ in range(2):
                for p in m.parameters():
                    p.grad = None
                z = torch.randint(0, 64, (2, 16))
                _, loss = ddp(idx=z[:, :-1], cond_idx=torch.tensor([1, 2]), targets=z, condition=torch.zeros(2, 3, 64, 64))
                loss.backward()
        ret[rank] = {k: None if p.grad is None else (float(p.grad.min()), float(p.grad.max())) for k, p in m.adapter.named_parameters()}
    finally:
        dist.destroy_process_group()


def test_ddp_averages_the_encoder_gradients():
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_worker_ddp, args=(world, _free_port(), ret), nprocs=world, join=True)
    for rank in range(world):
        got = ret[rank]
        assert got["model.embeddings.mask_token"] is None
        trained = {k: v for k, v in got.items() if k != "model.embeddings.mask_token"}
        assert len(trained) == 12 * 18 + 6
        for k, v in trained.items():
            assert v == (1.5, 1.5), (rank, k, v)
