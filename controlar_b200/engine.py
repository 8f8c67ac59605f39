"""Host-side handles over the C ABI (include/controlar_b200.h): packed model + per-generate() state.

PyTorch is plumbing here (device memory, streams); all arithmetic happens in libcontrolar_b200.so.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional

import torch

from . import _lib
from ._lib import (CarGemmDesc, CarModelDesc, CarRowSampling, CarSampling, CarTrainWeights, CarWeights, check, cur_stream, dtype_code,
                   on_own_device, param_signature, _ptr, _ptr_array)


def _desc(m) -> CarModelDesc:
    cfg = m.config
    t2i = m.model_type == "t2i"
    return CarModelDesc(dtype=dtype_code(m.tok_embeddings.weight.dtype), dim=cfg.dim, n_layer=cfg.n_layer, n_head=cfg.n_head,
                        ffn_dim=m.layers[0].feed_forward.w1.weight.shape[0], vocab_size=cfg.vocab_size,
                        cls_token_num=cfg.cls_token_num, block_size=cfg.block_size, caption_dim=cfg.caption_dim if t2i else 0,
                        model_type=1 if t2i else 0, norm_eps=cfg.norm_eps, rope_base=cfg.rope_base)


_LAYER = [("attention_norm", "attention_norm"), ("wqkv", "attention.wqkv"), ("wo", "attention.wo"), ("ffn_norm", "ffn_norm"),
          ("w1", "feed_forward.w1"), ("w3", "feed_forward.w3"), ("w2", "feed_forward.w2")]


def _table(m):
    """(state-dict name, CarTrainWeights field, index) of every transformer parameter the library reads, in the order of
    `ARTrainHandle.grad_params`.  The "w." fields are the CarWeights of inference."""
    t = [("tok_embeddings.weight", "w.tok_embeddings", None), ("norm.weight", "w.norm", None), ("output.weight", "w.output", None)]
    for i in range(len(m.layers)):
        t += [(f"layers.{i}.{k}.weight", "w." + f, i) for f, k in _LAYER]
    if m.model_type == "t2i":
        t += [("cls_embedding.cap_proj.fc1.weight", "w.cap_fc1", None), ("cls_embedding.cap_proj.fc2.weight", "w.cap_fc2", None)]
    else:
        t += [("cls_embedding.embedding_table.weight", "w.label_table", None)]
    t += [("condition_mlp.cap_proj.fc1.weight", "w.cond_fc1", None), ("condition_mlp.cap_proj.fc2.weight", "w.cond_fc2", None)]
    for j in range(3):
        t += [(f"condition_layers.{j}.fc1.weight", "w.ctl_fc1", j), (f"condition_layers.{j}.fc2.weight", "w.ctl_fc2", j)]
    return t + [("adapter_mlp.fc1.weight", "adapter_fc1", None), ("adapter_mlp.fc2.weight", "adapter_fc2", None)]


def _param(m, name):
    """`m.get_parameter(name)` without its per-level checks, which make it several times slower; every training step looks up
    the whole table."""
    *mods, p = name.split(".")
    for k in mods:
        m = m._modules[k]
    return m._parameters[p]


def _weights(m):
    """CarWeights over the transformer's weights, and the tensors whose storage the library borrows through it."""
    return _lib.fill_struct(CarWeights, [(f[2:], i, _param(m, k).detach()) for k, f, i in _table(m) if f.startswith("w.")],
                            len(m.layers))


def train_key(m) -> tuple:
    """What an ARTrainHandle is created for: the storage of every parameter of the module."""
    return tuple(p.data_ptr() for p in m.parameters())


def _layout(m):
    """What the packed buffers were sized for: a change here needs a new CarModel, anything else a repack in place."""
    w = m.tok_embeddings.weight
    return (w.dtype, str(w.device), tuple(w.shape), len(m.layers), tuple(m.layers[0].feed_forward.w1.weight.shape))


class ARModelHandle(_lib.NativeHandle):
    """CarModel: GEMM-ready copies of the transformer weights (re-packed when the module's weights change)."""

    def __init__(self, module):
        super().__init__("car_model_destroy")
        self.lib = _lib.lib()
        self.module = module
        self._dirty = 0
        self.generation = 0          # bumped whenever the CarModel handle is re-created: states compare THIS, not the raw pointer
        self._build()

    @property
    def device(self):
        return self.module.tok_embeddings.weight.device

    def _signature(self, ts):
        """Changes when a borrowed tensor is replaced (data_ptr / dtype / device; also through `p.data = t`) or updated through
        autograd-visible in-place ops (`_version`).  Writes into `p.data` in place do NOT bump `_version`: call `invalidate()`."""
        return param_signature(ts), self._dirty

    def invalidate(self):
        """Force a repack at the next use (after in-place writes into `param.data`, which PyTorch's version counters do not see)."""
        self._dirty += 1

    @on_own_device
    def _build(self):
        m = self.module
        w, ts = _weights(m)
        d = _desc(m)
        self.close()
        check(self.lib.car_model_create(C.byref(d), C.byref(w), cur_stream(), C.byref(self.handle)), "car_model_create")
        self._keep, self.sig = ts, self._signature(ts)
        self.layout, self.dtype, self.desc = _layout(m), m.tok_embeddings.weight.dtype, d
        self.generation += 1

    @on_own_device
    def refresh(self):
        """Bring the packed copies up to date if a borrowed tensor was replaced / updated since the last pack.  Same layout:
        `car_model_repack` rewrites the library-owned buffers IN PLACE (the CarModel and every device pointer a live CarState holds
        stay valid — ADVICE r1: re-creating the model under a live state was a use-after-free).  Different dtype / device / shapes,
        or no CarModel after a failed create: a new CarModel (generation bumps; `setup_caches` then rebuilds the state)."""
        if not self.handle or _layout(self.module) != self.layout:
            self._build()
            return
        w, ts = _weights(self.module)
        sig = self._signature(ts)
        if sig == self.sig:
            return
        check(self.lib.car_model_repack(self.handle, C.byref(w), cur_stream()), "car_model_repack")
        self._keep, self.sig = ts, sig


class ARTrainHandle(_lib.NativeHandle):
    """CarTrain: the teacher-forced training forward (reference gpt_t2i.py:420-431,451-484) on the module's fp32 parameters
    under bf16-autocast numerics.  Weights are borrowed (re-cast to bf16 inside every forward, like autocast does)."""

    def __init__(self, module, max_batch: int, max_img_tokens: int):
        super().__init__("car_train_destroy")
        self.lib = _lib.lib()
        m = module
        cfg = m.config
        if m.tok_embeddings.weight.dtype != torch.float32:
            raise NotImplementedError("controlar_b200 training forward: fp32 parameters (bf16 autocast is applied inside), as the train scripts keep them")
        self.device = m.tok_embeddings.weight.device
        self.max_batch, self.max_img_tokens = max_batch, max_img_tokens
        self.V, self.T = cfg.vocab_size, cfg.cls_token_num
        self.key = train_key(m)
        self.generation = 0          # a backward belongs to the forward that produced its loss
        self._create(m)

    @on_own_device
    def _create(self, m):
        entries = [(f, i, _param(m, k).detach()) for k, f, i in _table(m)]
        if m.model_type == "t2i":
            entries.append(("cap_uncond", None, m.cls_embedding.uncond_embedding.detach().to(torch.float32).contiguous()))
        if not getattr(m, "zero_uncond_on_drop", False):       # a buffer, zeros unless a state dict says otherwise
            entries.append(("cond_uncond", None, m.condition_mlp.uncond_embedding.detach().to(torch.float32).contiguous()))
        # else: the legacy gpt.py class gives dropped samples literal zeros (gpt.py:118-119): NULL = zeros in the library
        tw, keep = _lib.fill_struct(CarTrainWeights, entries, len(m.layers))
        tw.adapter_dim = m.adapter_mlp.fc1.weight.shape[1]
        tw.num_classes = m.config.num_classes
        self.rope = m.freqs_cis.to(device=self.device, dtype=torch.float32).contiguous()
        check(self.lib.car_train_create(C.byref(_desc(m)), C.byref(tw), self.max_batch, self.max_img_tokens, _ptr(self.rope), cur_stream(),
                                        C.byref(self.handle)), "car_train_create")
        self._keep = (keep, tw)

    @on_own_device
    def forward(self, idx, cond, feat, drop_ids, mask, targets, valid, dropout=None):
        """dropout: None (every site off) or (token_p, resid_p, ffn_p, per-layer drop-path rates or None, int64 [1] device seed)."""
        B, n = idx.shape
        n_img = n + 1
        dev = idx.device
        idx = idx.to(torch.int32).contiguous()
        cond = cond.to(torch.int32).contiguous() if cond.dtype in (torch.int64, torch.int32) else cond.to(torch.float32).contiguous()
        feat = None if feat is None else feat.to(torch.bfloat16).contiguous()
        drop = drop_ids.to(torch.uint8).contiguous()
        S = self.T + n
        m8 = None
        if mask is not None:
            m8 = mask.reshape(B, S, S).to(torch.uint8).contiguous()
        tg = None if targets is None else targets.to(torch.int32).contiguous()
        vf = None if valid is None else valid.to(torch.float32).contiguous()
        logits = torch.empty(B, n_img, self.V, device=dev, dtype=torch.float32)
        loss = torch.empty(1, device=dev, dtype=torch.float32) if tg is not None else None
        seed = self._set_dropout(dropout, dev)
        check(self.lib.car_train_forward(self.handle, B, n_img, _ptr(idx), _ptr(cond), None if feat is None else _ptr(feat), _ptr(drop),
                                         None if m8 is None else _ptr(m8), None if tg is None else _ptr(tg),
                                         None if vf is None else _ptr(vf), _ptr(logits), None if loss is None else _ptr(loss), cur_stream()),
              "car_train_forward")
        self._last = (idx, cond, feat, drop, m8, tg, vf, seed)      # car_train_backward reads them again
        self.generation += 1
        return logits, (None if loss is None else loss[0])

    def _set_dropout(self, dropout, dev):
        """car_train_set_dropout for the next forward; returns the device seed the forward and its backward read (kept alive)."""
        cfg = None
        seed = None
        if dropout is not None:
            tok, resid, ffn, rates, seed = dropout
            seed = seed.to(device=dev, dtype=torch.int64).reshape(1).contiguous()
            cfg = _lib.CarTrainDropout(float(tok), float(resid), float(ffn), 0, None, _ptr(seed))
            if rates is not None:
                arr = (C.c_float * len(rates))(*rates)
                cfg.n_layer, cfg.drop_path = len(rates), C.cast(arr, C.c_void_p)
        check(self.lib.car_train_set_dropout(self.handle, None if cfg is None else C.byref(cfg)), "car_train_set_dropout")
        return seed

    # ---- backward ---------------------------------------------------------------------------------------------------
    @staticmethod
    def grad_params(m):
        """The parameters `car_train_backward` produces gradients for, in a fixed order (name, parameter)."""
        return [(k, _param(m, k)) for k, _, _ in _table(m)]

    @on_own_device
    def backward(self, module, loss_grad=None, want_feat_grad=True):
        """Gradients of the last forward(targets=...) on this handle -> ({name: fp32 grad}, d_feat bf16 or None).
        loss_grad: 0-dim / [1] fp32 CUDA tensor (d / d loss) or None = 1."""
        if getattr(self, "_last", None) is None:
            raise RuntimeError("controlar_b200: backward() needs a preceding training forward with targets")
        idx, cond, feat, drop, m8, tg, vf, _seed = self._last
        if tg is None:
            raise RuntimeError("controlar_b200: the last training forward had no targets / loss")
        table = _table(module)
        has_feat = feat is not None
        skip_wo_feat = ("condition_mlp.", "condition_layers.", "adapter_mlp.")
        G = {k: torch.empty_like(_param(module, k), dtype=torch.float32) for k, _, _ in table if has_feat or not k.startswith(skip_wo_feat)}
        gw, _ = _lib.fill_struct(CarTrainWeights, [(f, i, G.get(k)) for k, f, i in table], len(module.layers))
        dfeat = torch.empty_like(feat) if (has_feat and want_feat_grad) else None
        lg = None
        if loss_grad is not None:
            lg = loss_grad.detach().to(device=idx.device, dtype=torch.float32).reshape(1).contiguous()
        check(self.lib.car_train_backward(self.handle, C.byref(gw), None if dfeat is None else _ptr(dfeat), None if lg is None else _ptr(lg),
                                          cur_stream()), "car_train_backward")
        self._last = None
        return G, dfeat


class ARStateHandle(_lib.NativeHandle):
    """CarState: KV caches (PyTorch-owned, reference layout), control tokens, scratch, the persistent decode kernel's packet
    buffers (and the CUDA graph of the per-kernel fallback chain)."""

    def __init__(self, model: ARModelHandle, b_eff: int, S: int, N: int, k_caches, v_caches, rope: torch.Tensor):
        super().__init__("car_state_destroy")
        self.lib = model.lib
        self.model = model
        self.device = rope.device
        self.b_eff, self.S, self.N = b_eff, S, N
        self._keep = (list(k_caches), list(v_caches), rope)
        ka, va = _ptr_array(self._keep[0]), _ptr_array(self._keep[1])
        with torch.cuda.device(self.device):
            check(self.lib.car_state_create(model.handle, b_eff, S, N, C.cast(ka, C.POINTER(C.c_void_p)),
                                            C.cast(va, C.POINTER(C.c_void_p)), _ptr(rope), C.byref(self.handle)),
                  "car_state_create")
        self.V = model.desc.vocab_size
        self.T = model.desc.cls_token_num

    @on_own_device
    def set_emb_mask(self, emb_mask: Optional[torch.Tensor]):
        if emb_mask is None:
            check(self.lib.car_state_set_emb_mask(self.handle, None, cur_stream()), "car_state_set_emb_mask")
            return
        em = (emb_mask != 0).to(torch.int32).contiguous()
        assert em.shape == (self.b_eff, self.T), (em.shape, self.b_eff, self.T)
        check(self.lib.car_state_set_emb_mask(self.handle, _ptr(em), cur_stream()), "car_state_set_emb_mask")
        self._mask_keep = em

    def set_row_sampling(self, rows: Optional[List[CarRowSampling]]):
        """Per-image sampling parameters and control strengths (car_state_set_row_sampling): one CarRowSampling per image (b_eff
        or b_eff / 2 with CFG entries).  The next prefill takes the strengths, the next generate / generate_forced the sampling
        parameters; their own scalar strength and CarSampling then only supply cfg_scale and cfg_interval.  None: scalar again."""
        if rows is None:
            check(self.lib.car_state_set_row_sampling(self.handle, None, 0), "car_state_set_row_sampling")
            return
        arr = (CarRowSampling * len(rows))(*rows)
        check(self.lib.car_state_set_row_sampling(self.handle, arr, len(rows)), "car_state_set_row_sampling")

    @on_own_device
    def prefill(self, cond: torch.Tensor, condition: Optional[torch.Tensor], control_strength: float,
                all_rows: bool) -> torch.Tensor:
        dev = cond.device
        if cond.dtype in (torch.int64, torch.int32):
            cond = cond.to(torch.int32).contiguous()
        else:
            cond = cond.to(self.model.dtype).contiguous()
        if condition is not None:
            condition = condition.to(self.model.dtype).contiguous()
            assert condition.shape[0] == self.b_eff and condition.shape[1] == self.N, condition.shape
        shape = (self.b_eff, self.T, self.V) if all_rows else (self.b_eff, self.V)
        out = torch.empty(shape, dtype=torch.float32, device=dev)
        check(self.lib.car_prefill(self.handle, _ptr(cond), _ptr(condition), float(control_strength), _ptr(out),
                                   1 if all_rows else 0, cur_stream()), "car_prefill")
        self._io_keep = (cond, condition)
        return out

    @on_own_device
    def decode_step(self, tok: torch.Tensor, pos: int) -> torch.Tensor:
        tok = tok.reshape(-1).to(torch.int32).contiguous()
        assert tok.numel() == self.b_eff
        out = torch.empty((self.b_eff, self.V), dtype=torch.float32, device=tok.device)
        check(self.lib.car_decode_step(self.handle, _ptr(tok), int(pos), _ptr(out), cur_stream()), "car_decode_step")
        self._tok_keep = tok
        return out

    @on_own_device
    def generate(self, sp: CarSampling, n_tokens: int, noise: Optional[torch.Tensor], device) -> torch.Tensor:
        B = self.b_eff // 2 if sp.cfg_scale > 1.0 else self.b_eff
        out = torch.empty((B, n_tokens), dtype=torch.int32, device=device)
        if noise is not None:
            noise = noise.to(torch.float32).contiguous()
            assert noise.shape == (n_tokens, B, self.V), noise.shape
        check(self.lib.car_generate(self.handle, C.byref(sp), int(n_tokens), _ptr(noise), _ptr(out), cur_stream()),
              "car_generate")
        self._noise_keep = noise
        return out

    @on_own_device
    def generate_forced(self, sp: CarSampling, forced: torch.Tensor, trace: bool = True, noise: Optional[torch.Tensor] = None):
        """Teacher-forced device-side loop (car_generate_forced): returns (sampler choices int32 [B, n], logits fp32 [n, b_eff, V])."""
        B = self.b_eff // 2 if sp.cfg_scale > 1.0 else self.b_eff
        forced = forced.to(torch.int32).contiguous()
        assert forced.shape[0] == B, forced.shape
        n = forced.shape[1]
        out = torch.empty((B, n), dtype=torch.int32, device=forced.device)
        tr = torch.empty((n, self.b_eff, self.V), dtype=torch.float32, device=forced.device) if trace else None
        if noise is not None:
            noise = noise.to(torch.float32).contiguous()
            assert noise.shape == (n, B, self.V), noise.shape
        check(self.lib.car_generate_forced(self.handle, C.byref(sp), int(n), _ptr(noise), _ptr(forced), _ptr(tr), _ptr(out),
                                           cur_stream()), "car_generate_forced")
        self._noise_keep = (noise, forced)
        return out, tr

    def set_step_timer(self, buf: Optional[torch.Tensor]):
        """int64 [N] device tensor that receives the GPU globaltimer (ns) at the start of every decode iteration (None = off)."""
        if buf is not None:
            assert buf.dtype == torch.int64 and buf.numel() >= self.N and buf.is_cuda
        check(self.lib.car_state_set_step_timer(self.handle, _ptr(buf)), "car_state_set_step_timer")
        self._timer_keep = buf

    def step_bytes(self, n_context: int) -> int:
        return int(self.lib.car_decode_step_bytes(self.handle, int(n_context)))


def make_sampling(temperature=1.0, top_k=0, top_p=1.0, sample_logits=True, cfg_scale=1.0, cfg_interval=-1,
                  seed=0) -> CarSampling:
    # generate.py:121 turns CFG off at decode step i when `cfg_interval > -1 and i > cfg_interval`, and the sample scripts parse
    # --cfg-interval as a float.  For cfg_interval > -1, int(floor(cfg_interval)) gives the same decisions on integer steps, except
    # in (-1, 0), where the reference turns CFG off from decode step 0 and no integer can say so.
    if -1 < cfg_interval < 0:
        raise ValueError(f"cfg_interval={cfg_interval}: values in (-1, 0) are not supported (CFG off from the first decode "
                         "step cannot be expressed); use -1 to keep CFG on, or an integer >= 0")
    cfg_interval = math.floor(cfg_interval) if cfg_interval > -1 else -1
    return CarSampling(temperature=float(temperature), top_k=int(top_k or 0), top_p=float(top_p),
                       sample_logits=1 if sample_logits else 0, cfg_scale=float(cfg_scale),
                       cfg_interval=int(cfg_interval), seed=int(seed) & 0xFFFFFFFFFFFFFFFF)


def make_row_sampling(temperature=1.0, top_k=0, top_p=1.0, sample_logits=True, seed=0, noise_row=0,
                      control_strength=1.0) -> CarRowSampling:
    """One image's CarRowSampling.  noise_row is the Philox counter word: 0 (the default) makes the image's draws depend on its
    seed alone; the image index b reproduces what one CarSampling seed gives image b."""
    return CarRowSampling(temperature=float(temperature), top_k=int(top_k or 0), top_p=float(top_p),
                          sample_logits=1 if sample_logits else 0, seed=int(seed) & 0xFFFFFFFFFFFFFFFF,
                          noise_row=int(noise_row) & 0xFFFFFFFF, control_strength=float(control_strength))


def sample_rows(logits: torch.Tensor, rows: List[CarRowSampling], cfg_scale: float = 1.0, cfg_on: bool = True, step: int = 0,
                noise: Optional[torch.Tensor] = None, return_probs: bool = False, return_kept: bool = False):
    """`sample` with image b's parameters from rows[b] (car_sample_rows); B = len(rows) images, b_eff = 2B when cfg_scale > 1."""
    lib = _lib.lib()
    logits = logits.to(torch.float32).contiguous()
    b_eff, V = logits.shape
    B = len(rows)
    idx = torch.empty((B,), dtype=torch.int32, device=logits.device)
    probs = torch.empty((B, V), dtype=torch.float32, device=logits.device) if return_probs else None
    kept = torch.empty((B, V), dtype=torch.uint8, device=logits.device) if return_kept else None
    if noise is not None:
        noise = noise.to(torch.float32).contiguous()
    arr = (CarRowSampling * B)(*rows)
    with torch.cuda.device(logits.device):
        check(lib.car_sample_rows(_ptr(logits), b_eff, V, arr, B, float(cfg_scale), 1 if cfg_on else 0, int(step), _ptr(noise), _ptr(idx),
                                  _ptr(probs), _ptr(kept), cur_stream()), "car_sample_rows")
    out = (idx,) + ((probs,) if return_probs else ()) + ((kept.bool(),) if return_kept else ())
    return out if len(out) > 1 else idx


def sample(logits: torch.Tensor, sp: CarSampling, cfg_on: bool = True, step: int = 0,
           noise: Optional[torch.Tensor] = None, return_probs: bool = False, return_kept: bool = False):
    """generate.sample() + CFG combine on [b_eff, V] fp32 logits (car_sample).  Returns idx, then probs [B, V] if return_probs,
    then the kept set (bool [B, V]: survives top-k and top-p, also where its probability underflows to 0) if return_kept."""
    lib = _lib.lib()
    logits = logits.to(torch.float32).contiguous()
    b_eff, V = logits.shape
    B = b_eff // 2 if sp.cfg_scale > 1.0 else b_eff
    idx = torch.empty((B,), dtype=torch.int32, device=logits.device)
    probs = torch.empty((B, V), dtype=torch.float32, device=logits.device) if return_probs else None
    kept = torch.empty((B, V), dtype=torch.uint8, device=logits.device) if return_kept else None
    if noise is not None:
        noise = noise.to(torch.float32).contiguous()
    with torch.cuda.device(logits.device):
        check(lib.car_sample(_ptr(logits), b_eff, V, C.byref(sp), 1 if cfg_on else 0, int(step), _ptr(noise), _ptr(idx),
                             _ptr(probs), _ptr(kept), cur_stream()), "car_sample")
    out = (idx,) + ((probs,) if return_probs else ()) + ((kept.bool(),) if return_kept else ())
    return out if len(out) > 1 else idx


def op_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = 0) -> torch.Tensor:
    """y = act(x @ w.T + bias) through the library's GEMM (car_op_linear)."""
    lib = _lib.lib()
    K = x.shape[-1]
    x2 = x.reshape(-1, K).contiguous()
    N = w.shape[0]
    y = torch.empty((x2.shape[0], N), dtype=x.dtype, device=x.device)
    check(lib.car_op_linear(dtype_code(x.dtype), _ptr(x2), _ptr(w.detach().contiguous()),
                            _ptr(bias.detach().contiguous()) if bias is not None else None, _ptr(y), x2.shape[0], N, K,
                            int(act), cur_stream()), "car_op_linear")
    return y.reshape(*x.shape[:-1], N)


def op_dense_linear(x: torch.Tensor, w: torch.Tensor, resid: Optional[torch.Tensor] = None, act: int = 0) -> torch.Tensor:
    """y = act(x @ w.T) (+ resid) on the dense wgmma path (car_op_dense_linear); bf16."""
    lib = _lib.lib()
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty((M, N), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.car_op_dense_linear(_ptr(x.contiguous()), _ptr(w.detach().contiguous()), _ptr(resid.contiguous()) if resid is not None else None,
                                      _ptr(y), M, N, K, int(act), cur_stream()), "car_op_dense_linear")
    return y


def gemm_desc(**fields) -> CarGemmDesc:
    """A CarGemmDesc (gemm.h's DenseP) from keyword fields; tensors are replaced by their data pointers, alpha defaults to 1."""
    d = CarGemmDesc(alpha=1.0)
    for k, v in fields.items():
        setattr(d, k, v.data_ptr() if torch.is_tensor(v) else v)
    return d


def op_gemm_route(desc: CarGemmDesc, batch: int = 1) -> int:
    """The route gemm() takes for (desc, batch) (car_op_gemm_route): 0 wgmma plain, 1 wgmma 3x3 convolution, 2 mma.sync, 3 mma.sync
    window, or a negative error code when gemm() would refuse it (message in car_last_error).  Host only."""
    return _lib.lib().car_op_gemm_route(C.byref(desc), int(batch))


def op_gemm(desc: CarGemmDesc, batch: int = 1) -> None:
    """gemm() on the current device's current stream (car_op_gemm); raises when the descriptor is refused."""
    check(_lib.lib().car_op_gemm(C.byref(desc), int(batch), cur_stream()), "car_op_gemm")


def op_gemm_f32(A, B, M: int, N: int, K: int, bias, resid, out, ldc: int) -> None:
    """gemm_f32 (car_op_gemm_f32): out fp32 [M][ldc] = A [M][K] . B [N][K]^T + bias (+ resid).  Tensors or raw device pointers."""
    p = lambda t: t.data_ptr() if torch.is_tensor(t) else t
    check(_lib.lib().car_op_gemm_f32(p(A), p(B), M, N, K, p(bias), p(resid), p(out), ldc, cur_stream()), "car_op_gemm_f32")


def op_gemm_f32_conv3(src, fh: int, fw: int, B, nimg: int, H: int, W: int, cin: int, N: int, bias, resid, out) -> None:
    """gemm_f32_conv3 (car_op_gemm_f32_conv3): 3x3 / pad 1 convolution of the NHWC frame src [nimg][fh][fw][cin] -> out fp32
    [nimg][H][W][N] (+ bias, + resid).  Tensors or raw device pointers."""
    p = lambda t: t.data_ptr() if torch.is_tensor(t) else t
    check(_lib.lib().car_op_gemm_f32_conv3(p(src), fh, fw, p(B), nimg, H, W, cin, N, p(bias), p(resid), p(out), cur_stream()),
          "car_op_gemm_f32_conv3")


def op_rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    lib = _lib.lib()
    K = x.shape[-1]
    x2 = x.reshape(-1, K).contiguous()
    y = torch.empty_like(x2)
    check(lib.car_op_rmsnorm(dtype_code(x.dtype), _ptr(x2), _ptr(w.detach().contiguous()), _ptr(y), x2.shape[0], K,
                             float(eps), cur_stream()), "car_op_rmsnorm")
    return y.reshape(x.shape)


def _attn_mask(emb_mask: Optional[torch.Tensor]):
    """int32 [B, mask_ld] on the device, or (None, 0)."""
    if emb_mask is None:
        return None, 0
    m = emb_mask.to(torch.int32).contiguous()
    return m, m.shape[-1]


def op_attn_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, pos, Tpre: int,
                   emb_mask: Optional[torch.Tensor] = None, nsplit: int = 0, part: Optional[torch.Tensor] = None,
                   tickets: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The decode step's KV-cache attention (car_op_attn_decode): q [B, H*64] at position `pos` (int, or a device int32 scalar) against
    caches [B, H, S, 64] -> [B, H*64].  nsplit 0 = the product's choice.  part (fp32, >= B*H*16*68) and tickets (int32 [B*H], zero)
    are allocated when not given; pass them to reuse the split bookkeeping across calls.  out: optional [B, H*64] destination."""
    lib = _lib.lib()
    B, H, S, _ = k_cache.shape
    dev = q.device
    if not torch.is_tensor(pos):
        pos = torch.tensor([int(pos)], dtype=torch.int32, device=dev)
    part = torch.empty(B * H * 16 * 68, dtype=torch.float32, device=dev) if part is None else part
    tickets = torch.zeros(B * H, dtype=torch.int32, device=dev) if tickets is None else tickets
    out = torch.empty((B, H * 64), dtype=q.dtype, device=dev) if out is None else out
    m, ld = _attn_mask(emb_mask)
    with torch.cuda.device(dev):
        check(lib.car_op_attn_decode(dtype_code(q.dtype), _ptr(q.contiguous()), _ptr(k_cache), _ptr(v_cache), _ptr(m), ld, _ptr(pos),
                                     B, H, S, int(Tpre), int(nsplit), _ptr(part), _ptr(tickets), _ptr(out), cur_stream()),
              "car_op_attn_decode")
    return out


def op_attn_prefill(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, Tq: int, Tpre: int,
                    emb_mask: Optional[torch.Tensor] = None, impl: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The prefix rows' KV-cache attention (car_op_attn_prefill): q [B*Tq, H*64] at positions 0..Tq-1 against caches [B, H, S, 64]
    -> [B*Tq, H*64].  impl 0 = the scalar kernel (bf16 / fp32), 1 = the bf16 tensor-core kernel.  out: optional destination."""
    lib = _lib.lib()
    B, H, S, _ = k_cache.shape
    out = torch.empty((B * Tq, H * 64), dtype=q.dtype, device=q.device) if out is None else out
    m, ld = _attn_mask(emb_mask)
    with torch.cuda.device(q.device):
        check(lib.car_op_attn_prefill(dtype_code(q.dtype), _ptr(q.contiguous()), _ptr(k_cache), _ptr(v_cache), _ptr(m), ld, B, H, S,
                                      int(Tq), int(Tpre), int(impl), _ptr(out), cur_stream()), "car_op_attn_prefill")
    return out
