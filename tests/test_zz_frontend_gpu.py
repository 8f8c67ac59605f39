"""GPU: the control-map / prompt front-end (SURVEY.md §8 row f3) through the C ABI.  Canny (reference condition/canny.py:14,
cv2.Canny) is integer work: the CUDA path must reproduce OpenCV's maps BIT-EXACTLY (fixture made by cv2 4.13.0 + the CPU oracle);
the caption left-padding (sample_t2i.py:146-156) against the reference's own lines."""
import numpy as np
import pytest
import torch

from oracle.canny_oracle import canny as canny_oracle, left_pad_captions as left_pad_oracle
from tests.golden.make_golden import canny_inputs
from tests.helpers import GOLDEN

pytestmark = pytest.mark.gpu
PAIRS = ((100, 200), (50, 150), (30.5, 90.7))


def test_canny_bit_exact_vs_opencv_fixture():
    from controlar_b200.condition.canny import CannyDetector, canny_cuda
    g = np.load(f"{GOLDEN}/canny.npz")
    det = CannyDetector()
    for name, img in canny_inputs().items():
        for lo, hi in PAIRS:
            want = g[f"{name}_{lo}_{hi}"]
            x = img if img.shape[2] == 3 else img[:, :, 0]
            got = det(x, lo, hi)                                  # numpy in, numpy out — the reference's call
            assert isinstance(got, np.ndarray) and got.dtype == np.uint8 and got.shape == want.shape
            assert np.array_equal(got, want), (name, lo, hi, int((got != want).sum()))
            got_t = canny_cuda(torch.from_numpy(np.ascontiguousarray(x)).cuda().float(), lo, hi, sweeps_per_call=1)   # device in, device out
            assert np.array_equal(got_t.cpu().numpy(), want)


def test_canny_large_and_non_square_vs_oracle():
    from controlar_b200.condition.canny import canny_cuda
    rng = np.random.default_rng(5)
    for H, W in ((768, 512), (97, 1030)):
        base = rng.integers(0, 256, (H // 8 + 2, W // 8 + 2, 3)).astype(np.float64)
        img = np.kron(base, np.ones((8, 8, 1)))[:H, :W]           # blocky image: long straight edge chains across many tiles
        img = np.clip(img + rng.normal(0, 3, img.shape), 0, 255).astype(np.uint8)
        want = canny_oracle(img, 100, 200)
        got = canny_cuda(torch.from_numpy(img).cuda(), 100, 200).cpu().numpy()
        assert np.array_equal(got, want), int((got != want).sum())
        assert 0 < int((want > 0).sum()) < H * W


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_left_pad_captions_vs_reference_lines(dt):
    from controlar_b200.frontend import left_pad_captions
    g = torch.Generator().manual_seed(3)
    B, L, D = 5, 120, 2048
    emb = torch.randn(B, L, D, generator=g).to(dt)
    lens = [120, 1, 37, 64, 119]
    mask = torch.zeros(B, L, dtype=torch.int64)
    for b, n in enumerate(lens):
        mask[b, :n] = 1
    want_e, want_m = left_pad_oracle(emb, mask)
    got_e, got_m = left_pad_captions(emb.cuda(), mask.cuda())
    assert got_e.dtype == dt and got_m.dtype == torch.int64
    assert torch.equal(got_e.cpu(), want_e) and torch.equal(got_m.cpu(), want_m)


def test_hed_detector_vs_reference_golden():
    """HED (reference condition/hed.py:17-84, fp32) on procedural weights: edge maps and the five projections against the fixture the
    reference produced (tests/golden/make_golden.py:hed_case).  fp32-grade arithmetic (split-bf16 x3 convolutions): measured values are
    logged to hed.jsonl (tests/helpers.py: log_measurement); bars 2e-2 of the 0..255 range for the edge map, 1e-3 relative for the projections."""
    import json
    from controlar_b200.condition.hed import HEDdetector
    from oracle.weights import make_hed_state_dict
    from tests.golden.make_golden import hed_inputs
    from tests.helpers import load_golden, log_measurement, rel_l2
    g = load_golden("hed")
    det = HEDdetector()
    det.netNetwork.load_state_dict(make_hed_state_dict(seed=g["seed"]), strict=True)
    det = det.cuda()
    for name, x in hed_inputs().items():
        edge = det(x.cuda())
        want = g[name + "_edge"]
        assert edge.shape == want.shape and edge.dtype == torch.float32
        err = float((edge.cpu() - want).abs().max())
        projs = det.netNetwork(x.cuda())
        perr = max(rel_l2(p.cpu(), q) for p, q in zip(projs, g[name + "_proj"]))
        for p, q in zip(projs, g[name + "_proj"]):
            assert p.shape == q.shape
        log_measurement("hed.jsonl", json.dumps({"case": name, "edge_max_abs": err, "proj_worst_rel_l2": perr,
                                                 "edge_range": [float(want.min()), float(want.max())]}) + "\n")
        assert err < 2e-2, (name, err)
        assert perr < 1e-3, (name, perr)


def _hed(seed):
    from controlar_b200.condition.hed import ControlNetHED_Apache2
    from oracle.weights import make_hed_state_dict
    m = ControlNetHED_Apache2()
    m.load_state_dict(make_hed_state_dict(seed=seed), strict=True)
    return m.cuda()


def test_hed_weight_update_rebuilds_handle():
    from oracle.weights import make_hed_state_dict
    from tests.golden.make_golden import hed_inputs
    x = next(iter(hed_inputs().values())).cuda()
    m = _hed(0)
    with torch.no_grad():
        y0 = m.run(x)[0]
        m.load_state_dict(make_hed_state_dict(seed=5))
        y5 = m.run(x)[0]
    assert torch.equal(y5, _hed(5).run(x)[0]) and not torch.equal(y0, y5)


def test_hed_failed_recreate_leaves_no_stale_handle(monkeypatch):
    """A weight update whose re-create fails leaves no handle behind: the next call builds a new one, and every handle the library
    created is destroyed exactly once.  The library's own create and destroy run; only the refusal of one create is injected."""
    import gc
    from controlar_b200 import _lib
    from tests.golden.make_golden import hed_inputs
    from tests.helpers import ObservedLib
    gc.collect()                                       # earlier tests' handles are destroyed by the library itself, not observed
    lib = ObservedLib(_lib.lib(), ["hed"])
    monkeypatch.setattr(_lib, "_lib", lib)
    x = next(iter(hed_inputs().values())).cuda()
    m = _hed(0)
    with torch.no_grad():
        m.run(x)
        m.norm.add_(1.0)                                   # an in-place update: the next call rebuilds
        lib.refuse = True
        with pytest.raises(RuntimeError, match="car_hed_create"):
            m.run(x)
        lib.refuse = False
        m.run(x)
    del m
    gc.collect()
    assert len(lib.created) == 2 and sorted(lib.destroyed) == sorted(lib.created), (lib.created, lib.destroyed)


def _t5_encoder(max_rows=64):
    from controlar_b200.language.t5 import T5EncoderB200
    from oracle.weights import make_t5_state_dict
    from tests.helpers import load_golden
    g = load_golden("t5")
    c = g["config"]
    sd = {k: v.to(torch.bfloat16) for k, v in make_t5_state_dict(**c, seed=g["seed"]).items()}
    return T5EncoderB200(sd, d_model=c["d_model"], d_kv=c["d_kv"], num_heads=c["num_heads"], d_ff=c["d_ff"], num_layers=c["num_layers"],
                         vocab_size=c["vocab"], max_rows=max_rows)


def test_t5_encoder_deep_copies():
    """A used encoder deep-copies: the copy keeps its weights, drops the library handle and builds its own on first call."""
    import copy
    from tests.golden.make_golden import t5_inputs
    ids, mask = t5_inputs()["b2_L120"]
    enc = _t5_encoder()
    want = enc(input_ids=ids.cuda(), attention_mask=mask.cuda())["last_hidden_state"]
    clone = copy.deepcopy(enc)
    assert clone._h is None and enc._h.handle
    got = clone(input_ids=ids.cuda(), attention_mask=mask.cuda())["last_hidden_state"]
    assert torch.equal(got, want)


def test_t5_failed_recreate_leaves_no_stale_handle(monkeypatch):
    """Growing `max_rows` re-creates the encoder; when that create is refused, no handle is left behind, the next call builds a new
    one, and every handle the library created is destroyed exactly once."""
    import gc
    from controlar_b200 import _lib
    from tests.golden.make_golden import t5_inputs
    from tests.helpers import ObservedLib
    gc.collect()                                       # earlier tests' handles are destroyed by the library itself, not observed
    lib = ObservedLib(_lib.lib(), ["t5"])
    monkeypatch.setattr(_lib, "_lib", lib)
    small, big = t5_inputs()["b3_L24"], t5_inputs()["b2_L120"]          # 72 rows, then 240
    enc = _t5_encoder(max_rows=72)
    want = enc(input_ids=small[0].cuda(), attention_mask=small[1].cuda())["last_hidden_state"]
    lib.refuse = True
    with pytest.raises(RuntimeError, match="car_t5_create"):
        enc(input_ids=big[0].cuda(), attention_mask=big[1].cuda())
    assert not enc._h.handle
    lib.refuse = False
    enc(input_ids=big[0].cuda(), attention_mask=big[1].cuda())
    assert enc.max_rows == 240
    assert torch.equal(enc(input_ids=small[0].cuda(), attention_mask=small[1].cuda())["last_hidden_state"], want)
    del enc
    gc.collect()
    assert len(lib.created) == 2 and sorted(lib.destroyed) == sorted(lib.created), (lib.created, lib.destroyed)


def test_t5_encoder_vs_hf_golden():
    """T5 encoder forward (reference language/t5.py:69-75 -> HF T5EncoderModel, bf16) against the fixture HF itself produced on
    procedural weights (tests/golden/make_golden.py:t5_case): right-padded prompts, a one-token prompt, distances beyond the
    relative-position clamp.  Two bf16 evaluations of the same network differ by rounding order: HF's own bf16 output sits
    1.3e-2 ... 2.2e-2 (rel-L2) from the fp32 evaluation of the same weights (stored in the fixture), so the bars are (a) at most
    2.5e-2 from HF's bf16 output and (b) at least as close to the fp32 result as HF's bf16 output is (x 1.25).  Values are logged
    to t5.jsonl (tests/helpers.py: log_measurement)."""
    import json
    from controlar_b200.language.t5 import T5EncoderB200
    from oracle.weights import make_t5_state_dict
    from tests.golden.make_golden import t5_inputs
    from tests.helpers import load_golden, log_measurement, rel_l2
    g = load_golden("t5")
    c = g["config"]
    sd = {k: v.to(torch.bfloat16) for k, v in make_t5_state_dict(**c, seed=g["seed"]).items()}
    enc = T5EncoderB200(sd, d_model=c["d_model"], d_kv=c["d_kv"], num_heads=c["num_heads"], d_ff=c["d_ff"], num_layers=c["num_layers"],
                        vocab_size=c["vocab"], max_rows=64)
    for name, (ids, mask) in t5_inputs().items():
        out = enc(input_ids=ids.cuda(), attention_mask=mask.cuda())["last_hidden_state"]
        want = g[name]
        assert out.shape == want.shape and out.dtype == torch.bfloat16
        err = rel_l2(out.float().cpu(), want.float())
        exact = g[name + "_fp32"].float()
        err_exact, hf_exact = rel_l2(out.float().cpu(), exact), rel_l2(want.float(), exact)
        log_measurement("t5.jsonl", json.dumps({"case": name, "rel_l2_vs_hf_bf16": err, "rel_l2_vs_fp32": err_exact,
                                                "hf_bf16_vs_fp32": hf_exact}) + "\n")
        assert err < 2.5e-2, (name, err)
        assert err_exact < 1.25 * hf_exact, (name, err_exact, hf_exact)
    out2 = enc(input_ids=ids.cuda(), attention_mask=mask.cuda())["last_hidden_state"]
    assert torch.equal(out, out2)
