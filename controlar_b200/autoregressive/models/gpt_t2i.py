"""Drop-in for the reference module ``autoregressive/models/gpt_t2i.py`` (LlamaGen transformer with ControlAR
conditional decoding) whose inference arithmetic runs in hand-written sm_90a kernels behind the C ABI.

What is preserved (SURVEY.md §8b): ``ModelArgs`` fields, ``GPT_models`` factory names, module/parameter names
(identical state-dict keys: reference gpt_t2i.py:310-389), ``setup_caches`` / ``forward`` / ``get_fsdp_wrap_module_list``
signatures, and the attributes callers read (``adapter``, ``adapter_mlp``, ``model_type``, ``num_classes``,
``cls_embedding.uncond_embedding``, ``tok_embeddings.weight.dtype``, ``causal_mask``, ``layers[i].attention.kv_cache``).

The ``nn.Module`` objects below only *own parameters*; none of their eager ``forward``s compute anything on the
hot path.  ``Transformer.forward`` routes the two inference branches (reference gpt_t2i.py:433-470) to
``car_prefill`` / ``car_decode_step``; there is no PyTorch fallback — without the CUDA library calls raise.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch
import torch.nn as nn

from ... import engine as _engine
from .dinov2_adapter import Dinov2_Adapter


def find_multiple(n: int, k: int) -> int:
    return n if n % k == 0 else n + k - (n % k)


@dataclass
class ModelArgs:                      # field-for-field the constructor surface of reference gpt_t2i.py:31-61
    dim: int = 4096
    n_layer: int = 32
    n_head: int = 32
    n_kv_head: Optional[int] = None
    multiple_of: int = 256
    ffn_dim_multiplier: Optional[float] = None
    rope_base: float = 10000
    norm_eps: float = 1e-5
    initializer_range: float = 0.02
    token_dropout_p: float = 0.1
    attn_dropout_p: float = 0.0
    resid_dropout_p: float = 0.1
    ffn_dropout_p: float = 0.1
    drop_path_rate: float = 0.0
    num_classes: int = 1000
    caption_dim: int = 2048
    class_dropout_prob: float = 0.1
    model_type: str = "c2i"
    vocab_size: int = 16384
    cls_token_num: int = 1
    block_size: int = 256
    max_batch_size: int = 32
    max_seq_len: int = 2048
    adapter_size: str = "small"
    condition_type: str = "canny"


def precompute_freqs_cis_2d(grid_size: int, n_elem: int, base: float = 10000, cls_token_num: int = 120) -> torch.Tensor:
    """2-D RoPE table [cls_token_num + grid², n_elem/2, 2] (cos, sin), zero rows for the prefix positions.
    Same torch ops, in the same order, as reference gpt_t2i.py:506-519 so the table is bit-identical."""
    half = n_elem // 2
    inv = 1.0 / (base ** (torch.arange(0, half, 2)[: half // 2].float() / half))
    ang = torch.outer(torch.arange(grid_size), inv)
    grid = torch.concat([ang[:, None, :].expand(-1, grid_size, -1), ang[None, :, :].expand(grid_size, -1, -1)], dim=-1)
    table = torch.stack([torch.cos(grid), torch.sin(grid)], dim=-1).flatten(0, 1)
    return torch.cat([torch.zeros(cls_token_num, half, 2), table])


class MLP(nn.Module):
    """fc2(gelu_tanh(fc1(x))), bias-free (reference gpt_t2i.py:165-181); runs through the library GEMM."""

    def __init__(self, in_features: int, hidden_features: int, out_features: int):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features or in_features, bias=False)
        self.act = nn.GELU(approximate="tanh")
        self.fc2 = nn.Linear(hidden_features or in_features, out_features or in_features, bias=False)
        nn.init.zeros_(self.fc1.weight)
        nn.init.zeros_(self.fc2.weight)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = _engine.op_linear(x.to(self.fc1.weight.dtype), self.fc1.weight, act=1)
        return _engine.op_linear(h, self.fc2.weight, act=0)


class RMSNorm(nn.Module):
    def __init__(self, dim: int, eps: float = 1e-5):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return _engine.op_rmsnorm(x, self.weight, self.eps)


class LabelEmbedder(nn.Module):       # parameters only (reference gpt_t2i.py:67-97)
    def __init__(self, num_classes: int, hidden_size: int, dropout_prob: float):
        super().__init__()
        self.embedding_table = nn.Embedding(num_classes + int(dropout_prob > 0), hidden_size)
        self.num_classes = num_classes
        self.dropout_prob = dropout_prob


class CaptionEmbedder(nn.Module):     # parameters only (reference gpt_t2i.py:133-162)
    def __init__(self, in_channels: int, hidden_size: int, uncond_prob: float, token_num: int = 120):
        super().__init__()
        self.cap_proj = MLP(in_channels, hidden_size, hidden_size)
        self.register_buffer("uncond_embedding", torch.randn(token_num, in_channels) / in_channels ** 0.5)
        self.uncond_prob = uncond_prob


class ConditionEmbedder(nn.Module):   # parameters only (reference gpt_t2i.py:100-128)
    def __init__(self, in_channels: int, hidden_size: int, uncond_prob: float, token_num: int = 120, vocab_size: int = 16384):
        super().__init__()
        self.cap_proj = MLP(hidden_size, hidden_size, hidden_size)
        self.register_buffer("uncond_embedding", torch.zeros(token_num, hidden_size))
        self.uncond_prob = uncond_prob


class KVCache(nn.Module):
    """Reference layout [B, H, S, 64] (gpt_t2i.py:220-235); the kernels write/read these buffers in place."""

    def __init__(self, max_batch_size, max_seq_length, n_head, head_dim, dtype, device=None):
        super().__init__()
        shape = (max_batch_size, n_head, max_seq_length, head_dim)
        self.register_buffer("k_cache", torch.zeros(shape, dtype=dtype, device=device))
        self.register_buffer("v_cache", torch.zeros(shape, dtype=dtype, device=device))


class Attention(nn.Module):
    def __init__(self, config: ModelArgs):
        super().__init__()
        assert config.dim % config.n_head == 0
        n_kv = config.n_kv_head if config.n_kv_head is not None else config.n_head
        if n_kv != config.n_head:
            raise NotImplementedError("controlar_b200: grouped-query attention is not used by any ControlAR config")
        self.dim, self.n_head, self.head_dim, self.n_kv_head = config.dim, config.n_head, config.dim // config.n_head, n_kv
        self.wqkv = nn.Linear(config.dim, 3 * config.dim, bias=False)
        self.wo = nn.Linear(config.dim, config.dim, bias=False)
        self.kv_cache: Optional[KVCache] = None


class FeedForward(nn.Module):
    def __init__(self, config: ModelArgs):
        super().__init__()
        hidden = int(2 * (4 * config.dim) / 3)
        if config.ffn_dim_multiplier is not None:
            hidden = int(config.ffn_dim_multiplier * hidden)
        hidden = find_multiple(hidden, config.multiple_of)
        self.w1 = nn.Linear(config.dim, hidden, bias=False)
        self.w3 = nn.Linear(config.dim, hidden, bias=False)
        self.w2 = nn.Linear(hidden, config.dim, bias=False)


class TransformerBlock(nn.Module):
    def __init__(self, config: ModelArgs, drop_path: float = 0.0):
        super().__init__()
        self.attention = Attention(config)
        self.feed_forward = FeedForward(config)
        self.attention_norm = RMSNorm(config.dim, eps=config.norm_eps)
        self.ffn_norm = RMSNorm(config.dim, eps=config.norm_eps)


def _dropout_fields(cfg):
    return (cfg.token_dropout_p, cfg.attn_dropout_p, cfg.resid_dropout_p, cfg.ffn_dropout_p, cfg.drop_path_rate)


class Transformer(nn.Module):
    def __init__(self, config: ModelArgs):
        super().__init__()
        self.config = config
        self._dropout_built = _dropout_fields(config)      # the reference builds its nn.Dropout / DropPath layers here, once
        self.vocab_size, self.n_layer, self.block_size = config.vocab_size, config.n_layer, config.block_size
        self.num_classes, self.model_type, self.cls_token_num = config.num_classes, config.model_type, config.cls_token_num
        self.layer_internal = config.n_layer // 3
        self.adapter = self._make_adapter(config)
        self.adapter_mlp = MLP(384 if config.adapter_size == "small" else 768, config.dim, config.dim)
        if self.model_type == "c2i":
            self.cls_embedding = LabelEmbedder(config.num_classes, config.dim, config.class_dropout_prob)
        elif self.model_type == "t2i":
            self.cls_embedding = CaptionEmbedder(config.caption_dim, config.dim, config.class_dropout_prob)
        else:
            raise Exception("please check model type")
        self.tok_embeddings = nn.Embedding(config.vocab_size, config.dim)
        self.condition_embeddings = nn.Embedding(config.vocab_size, config.dim)   # unused in forward; must load
        self.condition_mlp = ConditionEmbedder(self.block_size, config.dim, config.class_dropout_prob, self.block_size,
                                               config.vocab_size)
        self.condition_layers = nn.ModuleList([MLP(config.dim, config.dim, config.dim) for _ in range(3)])
        self.layers = nn.ModuleList([TransformerBlock(config) for _ in range(config.n_layer)])
        self.norm = RMSNorm(config.dim, eps=config.norm_eps)
        self.output = nn.Linear(config.dim, config.vocab_size, bias=False)
        grid = int(self.block_size ** 0.5)
        assert grid * grid == self.block_size
        self.freqs_cis = precompute_freqs_cis_2d(grid, config.dim // config.n_head, config.rope_base, self.cls_token_num)
        self.max_batch_size = self.max_seq_length = -1
        self.initialize_weights()
        self.condition_token = None
        self.control_strength = 1
        self.causal_mask = None
        self._car_model: Optional[_engine.ARModelHandle] = None
        self._car_state: Optional[_engine.ARStateHandle] = None
        self._n_img = self.block_size

    def _make_adapter(self, config: ModelArgs) -> nn.Module:
        """Control encoder (gpt_t2i.py:326-333): DINOv2; the legacy c2i class (gpt.py) overrides this with ViT-S/16."""
        return Dinov2_Adapter(adapter_size=config.adapter_size, condition_type=config.condition_type)

    # same init distribution as the reference (gpt_t2i.py:366-388): N(0, 0.02) Linear/Embedding, zero head
    def initialize_weights(self):
        std = self.config.initializer_range
        for mod in self.modules():
            if isinstance(mod, nn.Linear):
                mod.weight.data.normal_(mean=0.0, std=std)
                if mod.bias is not None:
                    mod.bias.data.zero_()
            elif isinstance(mod, nn.Embedding):
                mod.weight.data.normal_(mean=0.0, std=std)
        nn.init.constant_(self.output.weight, 0)

    # ------------------------------------------------------------------------------------------------------
    def _model_handle(self) -> _engine.ARModelHandle:
        if self._car_model is None:
            self._car_model = _engine.ARModelHandle(self)
        else:
            self._car_model.refresh()
        return self._car_model

    def setup_caches(self, max_batch_size, max_seq_length, dtype, n_img_tokens: Optional[int] = None):
        """KV caches [B,H,S,64] per layer + causal mask + RoPE table (reference gpt_t2i.py:391-405), and the
        library state that borrows them.  ``n_img_tokens`` defaults to max_seq_length - cls_token_num."""
        cfg = self.config
        dev = self.tok_embeddings.weight.device
        head_dim = cfg.dim // cfg.n_head
        S = find_multiple(max_seq_length, 8)
        n_img = n_img_tokens if n_img_tokens is not None else max(1, min(cfg.block_size, max_seq_length - self.cls_token_num))
        key = (max_batch_size, S, n_img, dtype, str(dev))
        mh = self._model_handle()
        if self._car_state is not None and getattr(self, "_state_key", None) == key and self._car_state.model is mh \
                and mh.generation == self._state_model_id:
            # same shapes: reuse caches, scratch and the captured decode graph.  (The reference re-allocates zeroed
            # caches on every call; slots beyond the current position are never read, so stale contents are inert.)
            self.causal_mask = torch.tril(torch.ones(S, S, dtype=torch.bool, device=dev)).unsqueeze(0).repeat(max_batch_size, 1, 1)
            self._mask_synced = False
            return
        self.max_seq_length, self.max_batch_size = S, max_batch_size
        for b in self.layers:
            b.attention.kv_cache = KVCache(max_batch_size, S, cfg.n_head, head_dim, dtype, device=dev)
        self.causal_mask = torch.tril(torch.ones(S, S, dtype=torch.bool, device=dev)).unsqueeze(0).repeat(max_batch_size, 1, 1)
        grid = int(cfg.block_size ** 0.5)
        self.freqs_cis = precompute_freqs_cis_2d(grid, head_dim, cfg.rope_base, self.cls_token_num).to(dev)
        self._n_img = n_img
        if self._car_state is not None:
            self._car_state.close()
        self._car_state = _engine.ARStateHandle(
            mh, max_batch_size, S, self._n_img,
            [b.attention.kv_cache.k_cache for b in self.layers], [b.attention.kv_cache.v_cache for b in self.layers],
            self.freqs_cis.contiguous())
        self._state_key = key
        self._state_model_id = mh.generation
        self._mask_synced = False

    def _sync_mask(self):
        """generate() edits ``causal_mask`` in place (reference generate.py:184-193): text columns gated by
        emb_masks, diagonal forced.  A DECODE row (position T) holds exactly the per-sequence column gate: in row T-1 the forced
        diagonal makes column T-1 True even when emb_masks[:, T-1] == 0, while the reference's decode rows do gate it (ADVICE r1)."""
        T = self.cls_token_num
        row = T if self.causal_mask.shape[1] > T else T - 1
        em = self.causal_mask[:, row, :T].to(torch.int32).contiguous()
        self._car_state.set_emb_mask(em)
        self._mask_synced = True

    def forward(self, idx, cond_idx, input_pos=None, targets=None, mask=None, valid=None, condition=None,
                control_strength=1):
        """Reference gpt_t2i.py:409-484.  Inference branches -> (logits fp32, None); with both ``idx`` and ``cond_idx`` the
        teacher-forced training branch -> (logits fp32 [B, n+1, V], loss); `loss.backward()` runs the library's backward."""
        if idx is not None and cond_idx is not None:
            return self._train_forward(idx, cond_idx, targets, mask, valid, condition)
        if self._car_state is None:
            raise RuntimeError("call setup_caches() before forward(), as generate() does")
        st = self._car_state
        if cond_idx is not None:          # prefill
            self.control_strength = control_strength
            self._sync_mask()
            if condition is not None:
                self._n_img_check(condition)
            logits = st.prefill(cond_idx, condition, float(control_strength), all_rows=True)
            self.condition_token = "resident in CarState" if condition is not None else None
            return logits, None
        pos = int(input_pos.reshape(-1)[0].item()) if torch.is_tensor(input_pos) else int(input_pos)
        if not self._mask_synced:
            self._sync_mask()
        logits = st.decode_step(idx, pos)
        return logits.unsqueeze(1), None

    def _train_forward(self, idx, cond_idx, targets, mask, valid, condition):
        """Training branch, reference gpt_t2i.py:420-431,451-484 (module in train mode, fp32 parameters, bf16 autocast numerics
        inside the library).  Like the reference it only works in train mode (in eval mode the reference tuple-unpacks a bare
        tensor, SURVEY.md §8c gotcha 4)."""
        if not self.training:
            raise ValueError("forward(idx, cond_idx) is the training branch: call model.train() first (the reference fails here in eval mode too)")
        cfg = self.config
        if _dropout_fields(cfg) != getattr(self, "_dropout_built", _dropout_fields(cfg)):
            raise NotImplementedError("controlar_b200 training forward: the dropout probabilities of model.config changed after the "
                                      "model was built; like the reference, whose dropout layers are built from ModelArgs once, they "
                                      "are fixed at construction: build the model with the ModelArgs to train with")
        if cfg.attn_dropout_p > 0:
            raise NotImplementedError("controlar_b200 training forward: attention-probability dropout (attn_dropout_p > 0) is not "
                                      "supported; token, residual and feed-forward dropout and drop_path_rate are")
        B, n = idx.shape
        th = getattr(self, "_car_train", None)
        if th is None or th.key != _engine.train_key(self) or th.max_batch < B or th.max_img_tokens < n + 1:
            if th is not None:
                th.close()
            th = self._car_train = _engine.ARTrainHandle(self, B, max(n + 1, self.block_size))
        # CFG drop decision, drawn like the reference (gpt_t2i.py:83,148: torch.rand on the labels' device)
        forced = getattr(self, "_force_drop_ids", None)
        if forced is not None:
            drop = forced.to(device=idx.device).bool()
        elif cfg.class_dropout_prob > 0:
            drop = torch.rand(B, device=idx.device) < cfg.class_dropout_prob
        else:
            drop = torch.zeros(B, dtype=torch.bool, device=idx.device)
        dropout = self._train_dropout(idx.device)
        feat = self.adapter(condition) if condition is not None else None      # control encoder (CUDA path of vision.py)
        if targets is not None and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # loss.backward() works like in the reference's train loop (train_c2i_canny.py:200-211): the library's own backward
            # (car_train_backward) behind a torch.autograd.Function; gradients land in .grad of this module's parameters and, when
            # `feat` is part of an autograd graph, flow on into the control encoder
            names = _engine.ARTrainHandle.grad_params(self)
            return _TrainStep.apply(self, th, idx, cond_idx, feat, drop, mask, targets, valid, dropout, *[p for _, p in names])
        return _handle_forward(th, (idx, cond_idx, feat, drop, mask, targets, valid), dropout)

    def _train_dropout(self, device):
        """The dropout of this training forward: None when every site is off (no random draw: the dropout-free path is unchanged),
        else (token_p, resid_p, ffn_p, per-layer drop-path rates or None, seed).  The seed is one 64-bit draw from torch's default
        generator of the device, kept on the device (no host sync): torch.manual_seed reproduces a step, consecutive steps and
        differently seeded DDP ranks get different masks.  The rates are the reference's (gpt_t2i.py:347)."""
        cfg = self.config
        rates = None
        if cfg.drop_path_rate > 0:
            rates = [x.item() for x in torch.linspace(0, cfg.drop_path_rate, cfg.n_layer)]
        if max(cfg.token_dropout_p, cfg.resid_dropout_p, cfg.ffn_dropout_p) <= 0 and rates is None:
            return None
        forced = getattr(self, "_force_dropout_seed", None)
        if forced is not None:
            seed = torch.tensor([int(forced) & 0xFFFFFFFFFFFFFFFF], dtype=torch.uint64).view(torch.int64).to(device)
        else:
            seed = torch.empty(1, dtype=torch.int64, device=device).random_(-2 ** 63, None)
        return (float(cfg.token_dropout_p), float(cfg.resid_dropout_p), float(cfg.ffn_dropout_p), rates, seed)

    def _n_img_check(self, condition):
        if condition.shape[1] != self._n_img:
            raise RuntimeError(f"condition has {condition.shape[1]} tokens but the state was set up for {self._n_img}; "
                               "pass n_img_tokens to setup_caches")

    def get_fsdp_wrap_module_list(self) -> List[nn.Module]:
        return list(self.layers)


def _handle_forward(handle, args, dropout):
    """ARTrainHandle.forward; the dropout settings are passed only when a site is on"""
    return handle.forward(*args) if dropout is None else handle.forward(*args, dropout=dropout)


class _TrainStep(torch.autograd.Function):
    """(logits, loss) = car_train_forward; backward = car_train_backward.  Only `loss` is differentiable (the logits come back
    detached: the train scripts never differentiate through them)."""

    @staticmethod
    def forward(ctx, module, handle, idx, cond_idx, feat, drop, mask, targets, valid, dropout, *params):
        logits, loss = _handle_forward(handle, (idx, cond_idx, feat, drop, mask, targets, valid), dropout)
        ctx.module, ctx.handle, ctx.generation = module, handle, handle.generation
        ctx.want_feat = feat is not None and feat.requires_grad
        ctx.n_params = len(params)
        ctx.mark_non_differentiable(logits)
        return logits, loss.clone()

    @staticmethod
    def backward(ctx, _g_logits, g_loss):
        if ctx.handle.generation != ctx.generation:
            raise RuntimeError("controlar_b200: another training forward ran on this module since this loss was computed; the backward "
                               "recomputes from the state of the LAST forward (call loss.backward() before the next forward)")
        grads, dfeat = ctx.handle.backward(ctx.module, loss_grad=g_loss, want_feat_grad=ctx.want_feat)
        names = _engine.ARTrainHandle.grad_params(ctx.module)
        out = [grads.get(k) if p.requires_grad else None for k, p in names]
        return (None, None, None, None, dfeat if ctx.want_feat else None, None, None, None, None, None, *out)


def _factory(n_layer, n_head, dim):
    def make(**kwargs):
        return Transformer(ModelArgs(n_layer=n_layer, n_head=n_head, dim=dim, **kwargs))
    return make


GPT_7B, GPT_3B, GPT_1B = _factory(32, 32, 4096), _factory(24, 32, 3200), _factory(22, 32, 2048)
GPT_XXXL, GPT_XXL, GPT_XL = _factory(48, 40, 2560), _factory(48, 24, 1536), _factory(36, 20, 1280)
GPT_L, GPT_B = _factory(24, 16, 1024), _factory(12, 12, 768)

GPT_models = {"GPT-B": GPT_B, "GPT-L": GPT_L, "GPT-XL": GPT_XL, "GPT-XXL": GPT_XXL, "GPT-XXXL": GPT_XXXL,
              "GPT-1B": GPT_1B, "GPT-3B": GPT_3B, "GPT-7B": GPT_7B}
