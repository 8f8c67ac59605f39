"""CPU: the C-ABI library loads and exports every symbol include/controlar_b200.h declares (no compute)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    txt = open(os.path.join(ROOT, "include", "controlar_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(car_[a-z0-9_]+)\s*\(", txt)))


def test_library_builds_and_exports_all_symbols():
    from controlar_b200.build import build
    path = build()
    lib = ctypes.CDLL(path)
    names = _declared()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f"missing export {n}"


def test_ctypes_prototypes_cover_header():
    from controlar_b200 import _lib
    assert sorted(_lib.PROTOTYPES) == _declared()
    l = _lib.lib()
    assert l.car_version() >= 100
    # argument validation happens before any CUDA call
    assert l.car_model_create(None, None, None, None) < 0
    assert b"null" in l.car_last_error()


def test_fill_struct_places_each_entry_by_field_type(monkeypatch):
    """A pointer field, a dotted field of a nested struct, an inline-array slot and a per-layer array entry each land where the field's
    ctypes type says.  What no entry names, or names with None, stays NULL, and the struct keeps its per-layer arrays alive."""
    import gc
    import torch
    from controlar_b200 import _lib
    monkeypatch.setattr(_lib, "_ptr", lambda t: None if t is None else t.data_ptr())      # CPU tensors stand in for device ones
    a, b, c, d = (torch.zeros(4) for _ in range(4))
    s, ts = _lib.fill_struct(_lib.CarTrainWeights, [("adapter_fc1", None, a), ("w.norm", None, b), ("w.ctl_fc2", 2, c),
                                                    ("w.wqkv", 1, d), ("w.wqkv", 0, None), ("cap_uncond", None, None)], 3)
    gc.collect()
    assert s.adapter_fc1 == a.data_ptr() and s.w.norm == b.data_ptr() and list(s.w.ctl_fc2) == [None, None, c.data_ptr()]
    assert [s.w.wqkv[i] for i in range(3)] == [None, d.data_ptr(), None]
    assert not s.w.wo and s.cap_uncond is None and s.w.output is None and list(s.w.ctl_fc1) == [None] * 3
    assert [id(t) for t in ts] == [id(a), id(b), id(c), id(d)]


def test_attention_ops_reject_bad_arguments_before_any_launch():
    """Each call differs from a valid one in one argument, which the op must refuse before it touches the device (the pointers are
    never dereferenced)."""
    from controlar_b200 import _lib
    l = _lib.lib()
    P = 1 << 20                                        # a 16-byte-aligned stand-in pointer
    dec = dict(dtype=0, q=P, k=P, v=P, m=P, ld=120, pos=P, B=2, H=3, S=200, Tpre=120, nsplit=0, part=P, tickets=P, out=P)
    bad_dec = [dict(dtype=2), dict(q=None), dict(k=None), dict(pos=None), dict(part=None), dict(tickets=None), dict(out=None),
               dict(B=0), dict(H=-1), dict(S=0), dict(Tpre=-1), dict(ld=119), dict(nsplit=-1), dict(nsplit=17), dict(k=P + 8)]
    for change in bad_dec:
        a = {**dec, **change}
        rc = l.car_op_attn_decode(a["dtype"], a["q"], a["k"], a["v"], a["m"], a["ld"], a["pos"], a["B"], a["H"], a["S"], a["Tpre"],
                                  a["nsplit"], a["part"], a["tickets"], a["out"], None)
        assert rc < 0, change
        assert l.car_last_error(), change
    pre = dict(dtype=0, q=P, k=P, v=P, m=P, ld=120, B=2, H=3, S=200, Tq=150, Tpre=120, impl=1, out=P)
    bad_pre = [dict(dtype=5), dict(q=None), dict(v=None), dict(out=None), dict(Tq=0), dict(Tq=257, S=300), dict(Tq=201),
               dict(Tpre=151), dict(ld=100), dict(impl=2), dict(impl=-1), dict(dtype=1), dict(q=P + 2), dict(out=P + 2),
               dict(v=P + 4), dict(B=70000)]
    for change in bad_pre:
        a = {**pre, **change}
        rc = l.car_op_attn_prefill(a["dtype"], a["q"], a["k"], a["v"], a["m"], a["ld"], a["B"], a["H"], a["S"], a["Tq"], a["Tpre"],
                                   a["impl"], a["out"], None)
        assert rc < 0, change
        assert l.car_last_error(), change


def test_tensor_list_creates_reject_bad_lists_before_any_cuda_call():
    """The detector and tokenizer creates take a flat list of device pointers from the caller.  A null list, a null `out`, a wrong
    length, and the right length of null entries must each be refused with a message that names the entry point, before any
    allocation or launch (no entry is ever a valid pointer, so nothing is dereferenced)."""
    import ctypes as C
    import torch
    from controlar_b200 import _lib, vision
    from controlar_b200.tokenizer.tokenizer_image.vq_model import VQ_models
    l = _lib.lib()
    dpt = _lib.CarDptDesc(hidden=64, n_layers=4, n_heads=1, mlp=64, fusion=128, pos_grid=2, ln_eps=1e-12)
    for i in range(4):
        dpt.out_indices[i], dpt.neck[i] = i, 64
    with torch.device("meta"):
        vq_model = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8)
    cfg = vq_model.config
    vq = vision.CarVQDesc(codebook_size=cfg.codebook_size, embed_dim=cfg.codebook_embed_dim, ch=128, z_channels=cfg.z_channels,
                          n_levels=len(cfg.decoder_ch_mult), num_res_blocks=2)
    for i, v in enumerate(cfg.decoder_ch_mult):
        vq.ch_mult[i] = v
    creates = {
        "car_hed_create": (37, lambda ts, n, out: l.car_hed_create(ts, n, None, out)),
        "car_lineart_create": (24, lambda ts, n, out: l.car_lineart_create(ts, n, None, out)),
        "car_dpt_create": (4 + 16 * 4 + 74, lambda ts, n, out: l.car_dpt_create(C.byref(dpt), ts, n, None, out)),
        "car_midas_create": (368, lambda ts, n, out: l.car_midas_create(ts, n, None, out)),
        "car_vq_create": (len(vision.vq_tensor_order(vq_model)), lambda ts, n, out: l.car_vq_create(C.byref(vq), ts, n, None, out)),
    }

    def nulls(n):
        return C.cast((C.c_void_p * n)(), C.POINTER(C.c_void_p))
    for name, (n, create) in creates.items():
        h = C.c_void_p()
        for ts, count, out in [(None, n, C.byref(h)), (nulls(n), n, None), (nulls(n - 1), n - 1, C.byref(h)), (nulls(n), n, C.byref(h))]:
            assert create(ts, count, out) < 0, (name, count)
            assert name.encode() in l.car_last_error(), (name, count)
        assert not h, name



def test_ar_creates_reject_bad_arguments_before_any_cuda_call():
    """The model, state, training and T5 creates each refuse a null `out`, a null descriptor / model / weight table, and an unsupported
    shape, before any CUDA call: `out` stays null and the message names the entry point.  No pointer handed over is dereferenced
    (the stand-in model pointer only reaches a create whose shape check fails first)."""
    import ctypes as C
    from controlar_b200 import _lib
    from controlar_b200.language.t5 import CarT5Desc, CarT5Weights
    l = _lib.lib()
    P = 1 << 20

    def desc(dtype, **change):
        kw = dict(dtype=dtype, dim=128, n_layer=3, n_head=2, ffn_dim=384, vocab_size=64, cls_token_num=1, block_size=16, norm_eps=1e-5,
                  rope_base=1e4)
        return C.byref(_lib.CarModelDesc(**{**kw, **change}))
    bf16, f32 = _lib.CAR_BF16, _lib.CAR_F32
    w, tw = C.byref(_lib.CarWeights()), C.byref(_lib.CarTrainWeights(adapter_dim=64))
    t5 = lambda **change: C.byref(CarT5Desc(**{**dict(dtype=bf16, d_model=128, d_kv=64, n_heads=2, d_ff=256, n_layers=2, vocab=64,
                                                     num_buckets=32, max_distance=128, eps=1e-6), **change}))
    t5w = C.byref(CarT5Weights())
    kv = C.byref(C.c_void_p(P))
    calls = {
        "car_model_create": lambda out: [lambda: l.car_model_create(desc(bf16), w, None, None), lambda: l.car_model_create(None, w, None, out),
                                         lambda: l.car_model_create(desc(bf16), None, None, out),
                                         lambda: l.car_model_create(desc(bf16, n_layer=4), w, None, out)],
        "car_state_create": lambda out: [lambda: l.car_state_create(P, 2, 32, 16, kv, kv, P, None),
                                         lambda: l.car_state_create(None, 2, 32, 16, kv, kv, P, out),
                                         lambda: l.car_state_create(P, 2, 32, 16, None, kv, P, out),
                                         lambda: l.car_state_create(P, 0, 32, 16, kv, kv, P, out)],
        "car_train_create": lambda out: [lambda: l.car_train_create(desc(f32), tw, 2, 16, P, None, None),
                                         lambda: l.car_train_create(None, tw, 2, 16, P, None, out),
                                         lambda: l.car_train_create(desc(f32), None, 2, 16, P, None, out),
                                         lambda: l.car_train_create(desc(f32, n_layer=4), tw, 2, 16, P, None, out),
                                         lambda: l.car_train_create(desc(f32, n_head=0), tw, 2, 16, P, None, out)],
        "car_t5_create": lambda out: [lambda: l.car_t5_create(t5(), t5w, 64, None, None), lambda: l.car_t5_create(None, t5w, 64, None, out),
                                      lambda: l.car_t5_create(t5(), None, 64, None, out),
                                      lambda: l.car_t5_create(t5(d_kv=32), t5w, 64, None, out)],
    }
    for name, cases in calls.items():
        h = C.c_void_p()
        for i, call in enumerate(cases(C.byref(h))):
            assert call() < 0, (name, i)
            assert name.encode() in l.car_last_error(), (name, i, l.car_last_error())
        assert not h, name

def test_product_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from controlar_b200.autoregressive.models.gpt_t2i import GPT_models
    m = GPT_models["GPT-B"](block_size=64, cls_token_num=120, model_type="t2i", vocab_size=2048).eval()
    with pytest.raises(RuntimeError):
        m.setup_caches(2, 184, torch.float32)
