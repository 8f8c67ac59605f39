"""Batched generation engine — the role `autoregressive/serve` plays in the reference (a vLLM 0.4.1 fork: `LLM.generate(prompt_token_ids,
sampling_params)` over a request queue, CFG-aware sampler `serve/sampler.py:38-57`, paged KV `serve/gpt_model.py:244-331`), rebuilt on
the persistent decode kernel and extended to the control path the reference's serve lacks (SURVEY.md §8 row f4).

What is different from a text LLM server, and why the design is simpler than vLLM's:
  * every request produces EXACTLY `max_tokens` image tokens from a prefix of identical length (1 class token, or 120 left-padded T5
    tokens), so iteration-level ("continuous") batching degenerates to batch-level admission: a finished batch frees all its slots at
    once, the next requests of the queue are admitted then.  No sequence ever waits on a longer neighbour.
  * the KV cache of a batch is one contiguous `[B_eff, H, S, 64]` block per layer that is fully used — paging would only add an
    indirection to the decode kernel's K/V stream.
  * CFG pairs (conditional row b, unconditional row b + B) live in the same launch and are combined inside the sampler
    (`csrc/sampler.cuh`), like the reference's `Sampler.forward` does on the split logits.
  * with `mixed_sampling=True` the images of one launch each keep their own sampling parameters, seed and control strength, as
    the reference's vLLM sampler lets every sequence group of a batch have its own; only cfg_scale is per engine.
The scheduler below is plain host logic (CPU-tested); the GPU work is `generate()` + `decode_code()` of this package."""
from __future__ import annotations

import collections
import dataclasses
from typing import Any, Callable, Deque, Dict, List, Optional, Sequence, Tuple

import torch


@dataclasses.dataclass
class SamplingParams:
    """The subset of vllm.SamplingParams the reference's serve scripts set (serve/sample_c2i.py:49-51).  top_k = -1 / 0 disables
    top-k, temperature = 0 means greedy."""
    temperature: float = 1.0
    top_p: float = 1.0
    top_k: int = -1
    max_tokens: int = 16
    seed: Optional[int] = None

    def key(self) -> Tuple:
        return (float(self.temperature), float(self.top_p), int(self.top_k), int(self.max_tokens))


@dataclasses.dataclass
class CompletionOutput:
    index: int
    token_ids: List[int]


@dataclasses.dataclass
class RequestOutput:
    request_id: int
    prompt_token_ids: Optional[List[int]]
    outputs: List[CompletionOutput]
    finished: bool = True
    image: Optional[torch.Tensor] = None       # [3, H, W] in [-1, 1] when the engine was given a VQ model


@dataclasses.dataclass
class Request:
    request_id: int
    cond: Any                                  # c2i: int class id; t2i: tensor [T, caption_dim]
    emb_mask: Optional[torch.Tensor]           # t2i: [T]
    control: Optional[torch.Tensor]            # [3, H, W] control map or None
    sampling: SamplingParams
    control_strength: float = 1.0

    def group_key(self, mixed: bool = False) -> Tuple:
        """What the requests of one launch share: the grid (token count, control-map shape, whether there are caption masks) and,
        unless the engine mixes sampling configurations, the sampling parameters and the control strength."""
        ctl = None if self.control is None else tuple(self.control.shape)
        if mixed:
            return (int(self.sampling.max_tokens), ctl, self.emb_mask is None)
        return (self.sampling.key(), ctl, float(self.control_strength), self.emb_mask is None)


def derived_seed(base_seed: int, request_id: int) -> int:
    """The seed of a request that set none, in mixed mode: a function of the engine seed and the request id only (splitmix64), so
    a request's image does not depend on when it was launched, on its row or on its neighbours."""
    z = (int(base_seed) * 0x9E3779B97F4A7C15 + (int(request_id) + 1) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return (z ^ (z >> 31)) & 0x3FFFFFFFFFFFFFFF


def _check_mixed(sp: SamplingParams, control_strength) -> None:
    """The per-image values generate() would refuse (models/generate.py:row_sampling), raised when the request is queued."""
    t, p, c = float(sp.temperature), float(sp.top_p), float(control_strength)
    if not (0.0 <= t < float("inf")):
        raise ValueError(f"temperature must be >= 0 (0 = greedy), got {sp.temperature}")
    if not (0.0 < p <= 1.0):
        raise ValueError(f"top_p must be in (0, 1], got {sp.top_p}")
    if not (abs(c) < float("inf")):
        raise ValueError(f"control_strength must be finite, got {control_strength}")


class Scheduler:
    """FIFO admission with compatibility grouping: a batch is the oldest waiting request plus the next waiting requests that share
    its group key, up to `max_images`.  One launch runs one grid size; it runs one sampling configuration unless `mixed`."""

    def __init__(self, max_images: int = 8, mixed: bool = False):
        assert max_images >= 1
        self.max_images = max_images
        self.mixed = mixed
        self.waiting: Deque[Request] = collections.deque()

    def add(self, req: Request) -> None:
        self.waiting.append(req)

    def has_unfinished(self) -> bool:
        return len(self.waiting) > 0

    def next_batch(self) -> List[Request]:
        if not self.waiting:
            return []
        key = self.waiting[0].group_key(self.mixed)
        batch, rest = [], collections.deque()
        while self.waiting:
            r = self.waiting.popleft()
            if len(batch) < self.max_images and r.group_key(self.mixed) == key:
                batch.append(r)
            else:
                rest.append(r)
        self.waiting = rest
        return batch


class LLM:
    """`LLM(model=<controlar_b200 GPT module>, vq=<VQ module or None>, cfg_scale=...)`; `generate(...)` as in the reference's
    serve/sample_c2i.py:55-58, plus `add_request` / `step` for a queue that is fed while batches run.

    `max_images_per_batch` (default 8) caps the images of one launch.  With CFG, up to 8 images (16 sequences) run on the
    persistent decode kernel; 17 to 32 images (34 to 64 sequences) of a bf16 model run on the wide decode route, one tensor-core
    pass over the weights per step (DESIGN.md §4.2); other sizes and fp32 models run on the per-kernel chain.

    `mixed_sampling` (default False) chooses how requests share a launch:
      * False: a launch holds only requests with the same SamplingParams.key() (temperature, top-p, top-k, max_tokens) and control
        strength, so a queue of 8 different configurations runs as 8 launches of one image.  The launch is seeded with the first
        request's `seed`, or, when it has none, with `seed + <number of launches so far>`; the other requests' seeds are not used,
        and an image depends on its row in the launch.  This stays the default because existing callers rely on exactly these
        groups and seeds (tests/test_serve_cpu.py pins them).
      * True: requests that differ only in sampling parameters or control strength share a launch (FIFO, up to
        `max_images_per_batch`); each image is sampled with its own parameters and strength, and its noise is keyed by its own seed:
        `SamplingParams.seed`, or `derived_seed(seed, request_id)` when unset, never the launch count or the row.  The runner then
        receives the list of per-request seeds in place of one seed."""

    def __init__(self, args=None, model=None, vq=None, cfg_scale: Optional[float] = None, max_images_per_batch: int = 8, seed: int = 0,
                 runner: Optional[Callable[[List[Request], Any], torch.Tensor]] = None, mixed_sampling: bool = False, **unused):
        if model is None and runner is None:
            raise ValueError("LLM needs the GPT module (model=...): there are no checkpoints to locate by name without a network")
        self.model, self.vq = model, vq
        self.cfg_scale = float(cfg_scale if cfg_scale is not None else getattr(args, "cfg_scale", 1.0))
        self.num_classes = getattr(model, "num_classes", getattr(args, "num_classes", 1000))
        self.mixed_sampling = bool(mixed_sampling)
        self.scheduler = Scheduler(max_images_per_batch, self.mixed_sampling)
        self.base_seed = int(seed)
        self._next_id = 0
        self._launches = 0
        self._runner = runner or self._run_batch

    # ---- queue interface
    def add_request(self, cond, sampling_params: SamplingParams, emb_mask=None, control=None, control_strength: float = 1.0) -> int:
        if self.mixed_sampling:       # checked here: a bad request raised at launch time would take its batch-mates with it
            _check_mixed(sampling_params, control_strength)
        rid = self._next_id
        self._next_id += 1
        self.scheduler.add(Request(rid, cond, emb_mask, control, sampling_params, control_strength))
        return rid

    def has_unfinished_requests(self) -> bool:
        return self.scheduler.has_unfinished()

    def step(self) -> List[RequestOutput]:
        """Admit the next batch, run it to completion (all its sequences finish together), return its outputs."""
        batch = self.scheduler.next_batch()
        if not batch:
            return []
        if self.mixed_sampling:
            seed = [r.sampling.seed if r.sampling.seed is not None else derived_seed(self.base_seed, r.request_id) for r in batch]
        else:
            seed = batch[0].sampling.seed if batch[0].sampling.seed is not None else self.base_seed + self._launches
        self._launches += 1
        tokens = self._runner(batch, seed)                   # int32 [len(batch), max_tokens]
        images = None
        if self.vq is not None and batch[0].control is not None:
            H, W = batch[0].control.shape[-2:]
            images = self.vq.decode_code(tokens, [len(batch), 8, H // 16, W // 16])
        rows = tokens.cpu().tolist()
        return [RequestOutput(r.request_id, [int(r.cond)] if isinstance(r.cond, int) else None, [CompletionOutput(0, rows[i])],
                              True, None if images is None else images[i]) for i, r in enumerate(batch)]

    # ---- the reference's offline interface
    def generate(self, prompts=None, sampling_params: Optional[SamplingParams] = None, prompt_token_ids: Optional[Sequence[Sequence[int]]] = None,
                 use_tqdm: bool = False, **unused) -> List[RequestOutput]:
        """c2i, the reference's convention (serve/sample_c2i.py:36-58): `prompt_token_ids` = one `[class]` per image, followed — when
        cfg_scale > 1 — by as many `[num_classes]` unconditional prompts; the returned list has one entry per prompt, the unconditional
        entries carrying the tokens of their conditional partner (the reference's sampler feeds both halves the same token).
        t2i / control: `prompts` = list of dicts {cond, emb_mask, control, control_strength}."""
        sp = sampling_params or SamplingParams()
        n_uncond = 0
        if prompt_token_ids is not None:
            ids = [list(p) for p in prompt_token_ids]
            if self.cfg_scale > 1.0:
                if len(ids) % 2 or any(p != [self.num_classes] for p in ids[len(ids) // 2:]):
                    raise ValueError("with cfg_scale > 1 the second half of prompt_token_ids must be [num_classes] prompts (serve/sample_c2i.py:38-39)")
                n_uncond = len(ids) // 2
                ids = ids[:n_uncond]
            order = [self.add_request(int(p[0]), sp) for p in ids]
        else:
            order = [self.add_request(p["cond"], p.get("sampling_params", sp), p.get("emb_mask"), p.get("control"), p.get("control_strength", 1.0))
                     for p in (prompts or [])]
        done: Dict[int, RequestOutput] = {}
        while self.has_unfinished_requests():
            for o in self.step():
                done[o.request_id] = o
        outs = [done[i] for i in order]
        if n_uncond:
            outs = outs + [RequestOutput(o.request_id, [self.num_classes], [CompletionOutput(0, list(o.outputs[0].token_ids))], True, None) for o in outs]
        return outs

    # ---- one batch on the GPU: generate() of this package (prefill + persistent decode kernel, CFG pairs inside)
    def _run_batch(self, batch: List[Request], seed) -> torch.Tensor:
        """seed: one int for the launch, or (mixed sampling) one per request."""
        from ..models.generate import generate
        m = self.model
        dev = m.tok_embeddings.weight.device
        sp = batch[0].sampling
        if isinstance(batch[0].cond, int):
            cond = torch.tensor([r.cond for r in batch], dtype=torch.long, device=dev)
            masks = None
        else:
            cond = torch.stack([r.cond for r in batch]).to(device=dev, dtype=m.tok_embeddings.weight.dtype)
            masks = None if batch[0].emb_mask is None else torch.stack([r.emb_mask for r in batch]).to(dev)
        control = None if batch[0].control is None else torch.stack([r.control for r in batch]).to(device=dev, dtype=m.tok_embeddings.weight.dtype)
        # per request in mixed mode, else the values the batch shares (its first request's); temperature 0 is greedy
        per = (lambda f: [f(r) for r in batch]) if self.mixed_sampling else (lambda f: f(batch[0]))
        return generate(m, cond, sp.max_tokens, emb_masks=masks, cfg_scale=self.cfg_scale, condition=control,
                        control_strength=per(lambda r: r.control_strength),
                        temperature=per(lambda r: 1.0 if r.sampling.temperature == 0 else r.sampling.temperature),
                        top_k=per(lambda r: max(int(r.sampling.top_k), 0)), top_p=per(lambda r: r.sampling.top_p),
                        sample_logits=per(lambda r: r.sampling.temperature != 0), seed=list(seed) if self.mixed_sampling else seed)
