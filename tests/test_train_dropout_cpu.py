"""CPU: the training path's dropout (token / residual / feed-forward dropout and drop path).  The oracle with the generator's masks
against the reference run with the same masks (tests/golden/make_train_dropout_golden.py -> train_*_dropout.pt), properties of the
CPU restatement of the generator (oracle/dropout_masks.py), and the C ABI's argument checks, which run before any CUDA call."""
import ctypes as C
import math

import pytest
import torch

from oracle import dropout_masks as DM
from oracle.weights import GPTSpec, make_gpt_state_dict
from oracle.train_oracle import TrainOracle
from oracle.train_dropout_oracle import DropoutTrainOracle
from oracle.inputs import class_inputs, code_inputs
from tests import dropout_fixture as DF
from tests.helpers import load_golden


def _run(g, dropout, feat=None, inputs=None):
    spec, cond, z, mask, valid, feat0 = inputs or DF.inputs(g)
    orc = DropoutTrainOracle(spec, make_gpt_state_dict(spec, g["seed"]), torch.bfloat16)
    feat = (feat0 if feat is None else feat).clone().requires_grad_(True)
    with torch.enable_grad():
        logits, loss = orc.forward(z[:, :-1], cond, feat, g["drop_ids"], mask, z, valid, dropout=dropout)
        loss.backward()
    return orc, feat, logits.detach(), loss.detach()


@pytest.mark.parametrize("name", DF.CASES)
def test_dropout_oracle_matches_reference(name):
    """Loss, logits, every parameter gradient and d loss / d control tokens of the reference run with the same masks, to the bars
    of test_train_oracle_golden.py"""
    g = load_golden(name)
    orc, feat, logits, loss = _run(g, g["dropout"])
    n = g["probe_sizes"]
    ev, _, pm = DF.probe_err("logits", logits, g["logits"], n["logits"])
    assert ev < 4e-3
    assert float((pm["val"] - g["logits"]["val"]).abs().max()) <= 2.0 ** -7 * float(g["logits"]["val"].abs().max())
    assert abs(float(loss) - float(g["loss"])) < 2e-5 * float(g["loss"])
    _, bad = DF.grad_rows(g, {k: p.grad for k, p in orc.p.items() if p.grad is not None}, 5e-3, 3e-2)
    assert not bad, "\n".join(bad)
    ef, efn, _ = DF.probe_err("feat", feat.grad, g["feat_grad"], n["feat"])
    assert ef < 3e-2 and efn < 5e-3


def test_dropout_moves_the_result_and_droppath_fixture_drops_a_branch():
    """The masks matter (the fixture is not a p = 0 run in disguise), and the drop-path case drops at least one branch."""
    g = load_golden("train_c2i_small_ac_dropout")
    _, _, lg0, _ = _run(g, None)
    ev, _, _ = DF.probe_err("logits", lg0, g["logits"], g["probe_sizes"]["logits"])
    assert ev > 1e-2
    gp = load_golden("train_c2i_small_ac_droppath_dropout")
    d = gp["dropout"]
    assert gp["dropped_paths"] > 0
    n = sum(int((~DM.path_keep(d["seed"], s, l, gp["B"], r)).sum()) for l, r in enumerate(d["drop_path"]) if r > 0
            for s in (DM.PATH_ATTN, DM.PATH_FFN))
    assert n == gp["dropped_paths"]


def test_all_keep_dropout_equals_no_dropout():
    """All-keep settings through the masked restatement equal the dropout-free TrainOracle, bit for bit"""
    g = load_golden("train_c2i_small_ac")
    spec = GPTSpec(**g["spec"])
    cond, z = class_inputs(spec.num_classes, g["B"], g["seed"] + 1), code_inputs(spec.vocab_size, g["B"], 64, g["seed"] + 4)
    ins = (spec, cond, z, None, None, g["feat"])
    orc0 = TrainOracle(spec, make_gpt_state_dict(spec, g["seed"]), torch.bfloat16)
    f0 = g["feat"].clone().requires_grad_(True)
    with torch.enable_grad():
        lg0, l0 = orc0.forward(z[:, :-1], cond, f0, g["drop_ids"], None, z, None)
        l0.backward()
    orc1, f1, lg1, l1 = _run(g, {"seed": 7, "token_p": 0.0, "resid_p": 0.0, "ffn_p": 0.0, "drop_path": [0.0] * spec.n_layer}, inputs=ins)
    assert torch.equal(lg0.detach(), lg1) and torch.equal(l0.detach(), l1) and torch.equal(f0.grad, f1.grad)
    for k, p in orc0.p.items():
        if p.grad is not None:
            assert torch.equal(p.grad, orc1.p[k].grad), k


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_fraction_within_binomial_bounds(p):
    n_rows, cols = 300, 256
    m = DM.keep_mask(0xC0FFEE, DM.RESID, 3, 2, n_rows // 2, cols, p)
    n = m.numel()
    kept = int(m.sum())
    mean, sd = n * (1 - p), math.sqrt(n * p * (1 - p))
    assert abs(kept - mean) < 5 * sd, (kept, mean, sd)
    per_col = m.float().mean(dim=(0, 1))                     # no column lane of the 4-word Philox output is biased
    for lane in range(4):
        f = float(per_col[lane::4].mean())
        assert abs(f - (1 - p)) < 5 * math.sqrt(p * (1 - p) / (n / 4)), (lane, f)


def test_sites_layers_samples_are_independent():
    seed, B, R, Cc, p = 1234567890123, 3, 40, 64, 0.5
    base = DM.keep_mask(seed, DM.FFN, 2, B, R, Cc, p)
    others = [DM.keep_mask(seed, DM.RESID, 2, B, R, Cc, p), DM.keep_mask(seed, DM.TOKEN, 2, B, R, Cc, p),
              DM.keep_mask(seed, DM.FFN, 3, B, R, Cc, p), DM.keep_mask(seed + 1, DM.FFN, 2, B, R, Cc, p),
              DM.keep_mask(seed ^ (1 << 40), DM.FFN, 2, B, R, Cc, p)]
    n = base.numel()
    for o in others:                                          # agreement of two independent fair coins: n/2 +- 5 sd
        agree = int((o == base).sum())
        assert abs(agree - n / 2) < 5 * math.sqrt(n / 4), agree
    for a, b in [(0, 1), (0, 2), (1, 2)]:
        agree = int((base[a] == base[b]).sum())
        assert abs(agree - R * Cc / 2) < 5 * math.sqrt(R * Cc / 4), (a, b, agree)
    # a sample's mask does not depend on the batch it sits in
    assert torch.equal(DM.keep_mask(seed, DM.FFN, 2, B + 2, R, Cc, p)[:B], base)


def test_drop_path_is_constant_within_a_sample():
    seed, B = 99, 64
    m = DM.keep_mask(seed, DM.PATH_ATTN, 5, B, 7, 9, 0.5)
    assert torch.equal(m, m[:, :1, :1].expand_as(m))
    k_attn, k_ffn = DM.path_keep(seed, DM.PATH_ATTN, 5, B, 0.5), DM.path_keep(seed, DM.PATH_FFN, 5, B, 0.5)
    assert torch.equal(k_attn, m[:, 0, 0])
    assert 0 < int(k_attn.sum()) < B and not torch.equal(k_attn, k_ffn)


def test_philox_known_answer():
    """Philox4x32-10 against the known-answer vectors of the Random123 distribution (kat_vectors: philox4x32_10)"""
    w = DM.philox4x32_10(0, 0, 0, 0, 0)
    assert [int(x) for x in w] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    w = DM.philox4x32_10(0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFFFFFFFFFF)
    assert [int(x) for x in w] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


@pytest.mark.parametrize("rate,n_layer", [(0.1, 24), (0.5, 6), (0.2, 36), (0.0, 12)])
def test_drop_path_rates_are_the_references_linspace(rate, n_layer):
    got = DM.drop_path_rates(rate, n_layer)
    want = [float(torch.tensor(i * rate / (n_layer - 1), dtype=torch.float32)) for i in range(n_layer)]
    assert got[0] == 0.0 and len(got) == n_layer
    assert got == [x.item() for x in torch.linspace(0, rate, n_layer)]
    assert max(abs(a - b) for a, b in zip(got, want)) < 1e-7
    assert all(float(torch.tensor(x, dtype=torch.float32)) == x for x in got)      # fp32 values, exact in the ABI's float[]


def test_scale_rules():
    assert DM.path_mult(0.1) == 1.109375                       # bf16(1 / 0.9)
    assert DM.elem_scale(0.1) == float(torch.tensor(1 / 0.9, dtype=torch.float32))
    x = torch.tensor([1.0, 3.0, -2.5], dtype=torch.bfloat16)
    y = DM.apply_dropout(x, torch.tensor([True, False, True]), 0.1)
    assert y.dtype == torch.bfloat16 and float(y[1]) == 0.0
    assert float(y[0]) == float(torch.tensor(DM.elem_scale(0.1)).to(torch.bfloat16))


# ---- C ABI: refusals happen before the handle or the device is touched (the stand-in pointers are never dereferenced) ----------
def _lib():
    from controlar_b200 import _lib
    return _lib


def test_set_dropout_rejects_bad_probabilities_and_rates():
    L = _lib()
    lib = L.lib()
    fake = C.c_void_p(1 << 20)
    seed = C.c_void_p(1 << 21)
    rates_ok = (C.c_float * 4)(0.0, 0.1, 0.2, 0.3)

    def cfg(tok=0.1, resid=0.1, ffn=0.1, rates=None, n=None, sd=seed):
        c = L.CarTrainDropout(tok, resid, ffn, 0, None, sd)
        if rates is not None:
            c.n_layer = len(rates) if n is None else n
            c.drop_path = C.cast(rates, C.c_void_p)
        return c
    bad = [cfg(tok=1.0), cfg(resid=-0.1), cfg(ffn=1.5), cfg(tok=float("nan")), cfg(sd=None),
           cfg(rates=(C.c_float * 4)(0.0, 0.1, 1.0, 0.3)), cfg(rates=(C.c_float * 2)(0.0, -0.5)),
           cfg(rates=(C.c_float * 2)(0.0, float("nan"))), cfg(rates=rates_ok, n=-1), cfg(tok=0.0, resid=0.0, ffn=0.0, rates=rates_ok, sd=None)]
    for c in bad:
        assert lib.car_train_set_dropout(fake, C.byref(c)) < 0
        assert lib.car_last_error()
    assert lib.car_train_set_dropout(None, C.byref(cfg())) < 0
    no_path = L.CarTrainDropout(0.1, 0.1, 0.1, 3, None, seed)          # n_layer without rates
    assert lib.car_train_set_dropout(fake, C.byref(no_path)) < 0


def test_keep_mask_rejects_bad_arguments():
    lib = _lib().lib()
    P = 1 << 20
    ok = dict(seed=P, site=1, layer=0, B=2, rows=3, cols=4, p=0.1, out=P)
    for change in [dict(seed=None), dict(out=None), dict(site=-1), dict(site=5), dict(layer=-1), dict(layer=70000), dict(B=0),
                   dict(rows=0), dict(cols=-3), dict(p=1.0), dict(p=-0.01), dict(p=float("nan"))]:
        a = {**ok, **change}
        rc = lib.car_dropout_keep_mask(a["seed"], a["site"], a["layer"], a["B"], a["rows"], a["cols"], a["p"], a["out"], None)
        assert rc < 0, change
        assert lib.car_last_error(), change
