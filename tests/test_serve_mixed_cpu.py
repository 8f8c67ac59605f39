"""CPU: the serving engine's mixed-sampling mode (controlar_b200/autoregressive/serve/llm.py, LLM(mixed_sampling=True)) and the
host checks of generate()'s per-image sampling parameters (autoregressive/models/generate.py:row_sampling).  The GPU runner is
replaced by a recording fake, as in test_serve_cpu.py."""
import pytest
import torch

from controlar_b200.autoregressive.models import generate as gen
from controlar_b200.autoregressive.serve.llm import LLM, Request, SamplingParams, Scheduler, derived_seed


def _fake_runner(log):
    def run(batch, seeds):
        log.append(([r.request_id for r in batch], seeds))
        n = batch[0].sampling.max_tokens
        return torch.tensor([[1000 * r.request_id + t for t in range(n)] for r in batch], dtype=torch.int32)
    return run


CONFIGS = [SamplingParams(max_tokens=4), SamplingParams(temperature=0.7, max_tokens=4), SamplingParams(top_k=100, max_tokens=4),
           SamplingParams(top_p=0.9, max_tokens=4), SamplingParams(temperature=0, max_tokens=4)]


def test_mixed_scheduler_batches_differing_sampling_and_strength_fifo():
    s = Scheduler(max_images=3, mixed=True)
    for i in range(7):
        s.add(Request(i, i, None, None, CONFIGS[i % len(CONFIGS)], control_strength=(0.5, 1.0)[i % 2]))
    s.add(Request(7, 7, None, None, SamplingParams(max_tokens=6)))                  # another grid: a launch of its own
    assert [r.request_id for r in s.next_batch()] == [0, 1, 2]
    assert [r.request_id for r in s.next_batch()] == [3, 4, 5]
    assert [r.request_id for r in s.next_batch()] == [6]
    assert [r.request_id for r in s.next_batch()] == [7]
    assert not s.has_unfinished()


def test_mixed_grid_key_still_separates_control_shapes_and_masks():
    ctl_a, ctl_b = torch.zeros(3, 256, 256), torch.zeros(3, 256, 512)
    sp = SamplingParams(max_tokens=4)
    reqs = [Request(0, 0, None, ctl_a, sp), Request(1, 1, None, ctl_b, sp), Request(2, 2, torch.ones(4), ctl_a, sp),
            Request(3, 3, None, ctl_a, SamplingParams(temperature=0.5, max_tokens=4), control_strength=0.3)]
    s = Scheduler(max_images=8, mixed=True)
    for r in reqs:
        s.add(r)
    assert [[r.request_id for r in s.next_batch()] for _ in range(3)] == [[0, 3], [1], [2]]


def test_mixed_engine_one_launch_per_batch_with_own_seeds():
    log = []
    llm = LLM(cfg_scale=4.0, runner=_fake_runner(log), max_images_per_batch=8, seed=11, mixed_sampling=True)
    sps = [SamplingParams(temperature=0.5 + 0.1 * i, top_k=100 * i, max_tokens=4, seed=(1234 + i if i % 3 == 0 else None))
           for i in range(10)]
    ids = [llm.add_request(i, sp, control_strength=0.25 * (1 + i % 4)) for i, sp in enumerate(sps)]
    got = {}
    while llm.has_unfinished_requests():
        for o in llm.step():
            got[o.request_id] = o
    assert sorted(got) == ids
    assert [b for b, _ in log] == [list(range(8)), [8, 9]]                                 # 10 requests, 2 launches (FIFO, cap 8)
    seeds = [s for _, ss in log for s in ss]
    for i, s in enumerate(seeds):
        assert s == (1234 + i if i % 3 == 0 else derived_seed(11, i)), i
    assert len(set(seeds)) == len(seeds)
    for i in ids:
        assert got[i].outputs[0].token_ids == [1000 * i + t for t in range(4)]


def test_derived_seed_ignores_launch_order_and_row():
    """The same request gets the same seed whether it is launched first or last, alone or among others, in any row."""
    def seeds_of(order, cap):
        log = []
        llm = LLM(cfg_scale=1.0, runner=_fake_runner(log), max_images_per_batch=cap, seed=3, mixed_sampling=True)
        for rid in order:
            llm._next_id = rid                                                             # request ids fixed by the test
            llm.add_request(rid, SamplingParams(max_tokens=2, temperature=0.5 + 0.1 * rid))
        while llm.has_unfinished_requests():
            llm.step()
        return {rid: s for batch, ss in log for rid, s in zip(batch, ss)}
    a, b, c = seeds_of([0, 1, 2, 3], 4), seeds_of([3, 2, 1, 0], 1), seeds_of([2, 0, 3, 1], 2)
    assert a == b == c
    assert a == {rid: derived_seed(3, rid) for rid in range(4)}
    assert derived_seed(3, 0) != derived_seed(4, 0) and 0 <= derived_seed(2 ** 40, 7) < 2 ** 62


def test_default_mode_is_unchanged_by_the_flag():
    log = []
    llm = LLM(cfg_scale=1.0, runner=_fake_runner(log), max_images_per_batch=4, seed=5)
    assert not llm.mixed_sampling
    for i in range(4):
        llm.add_request(i, CONFIGS[i % 2])
    while llm.has_unfinished_requests():
        llm.step()
    assert log == [([0, 2], 5), ([1, 3], 6)]                                                # grouped by key, launch-count seeds


class _Model:
    """Stands in for the GPT module: row_sampling reads nothing but the class's has_control_strength."""


def test_row_sampling_scalars_take_the_scalar_path():
    assert gen.row_sampling(_Model(), 3, True, 0.5, 7, temperature=0.9, top_k=100, top_p=0.8, sample_logits=True) is None
    assert gen.row_sampling(_Model(), 3, True, torch.tensor(0.5), None) is None           # a 0-dim tensor is a scalar


def test_row_sampling_per_image_values():
    rows = gen.row_sampling(_Model(), 3, True, [0.3, 0.6, 1.0], [5, 6, 7], temperature=[0.5, 1.0, 1.5], top_k=torch.tensor([0, 10, 2000]),
                            top_p=0.9, sample_logits=[True, False, True])
    assert [r.temperature for r in rows] == [0.5, 1.0, 1.5] and [r.top_k for r in rows] == [0, 10, 2000]
    assert [round(r.top_p, 6) for r in rows] == [0.9] * 3 and [r.sample_logits for r in rows] == [1, 0, 1]
    assert [r.seed for r in rows] == [5, 6, 7] and [r.noise_row for r in rows] == [0, 0, 0]        # per-image seeds: counter 0
    assert [round(r.control_strength, 6) for r in rows] == [0.3, 0.6, 1.0]
    rows = gen.row_sampling(_Model(), 3, True, 1.0, 42, temperature=[0.5, 1.0, 1.5])
    assert [r.seed for r in rows] == [42] * 3 and [r.noise_row for r in rows] == [0, 1, 2]        # one seed: today's rule


def test_row_sampling_forces_strength_one_without_cfg():
    rows = gen.row_sampling(_Model(), 2, False, [0.3, 0.6], 1)
    assert [r.control_strength for r in rows] == [1.0, 1.0]


@pytest.mark.parametrize("kw", [dict(temperature=[1.0, 1.0]), dict(top_k=[1, 2, 3, 4]), dict(seed=[1, 2]), dict(control_strength=[1.0]),
                                dict(sample_logits=torch.tensor([True, False]))])
def test_generate_rejects_sequences_of_the_wrong_length(kw):
    with pytest.raises(ValueError, match="values for 3 images"):
        gen.generate(_Model(), torch.zeros(3, dtype=torch.long), 4, cfg_scale=4.0, **kw)


@pytest.mark.parametrize("kw", [dict(temperature=[1.0, 0.0, 1.0]), dict(temperature=[1.0, -1.0, 1.0]), dict(top_k=[0, -1, 5]),
                                dict(top_p=[1.0, 0.0, 0.5]), dict(top_p=[1.0, 1.5, 0.5]), dict(control_strength=[1.0, float("nan"), 1.0])])
def test_generate_rejects_out_of_range_values(kw):
    with pytest.raises(ValueError):
        gen.generate(_Model(), torch.zeros(3, dtype=torch.long), 4, cfg_scale=4.0, **kw)


def test_legacy_class_refuses_strengths_other_than_one():
    from controlar_b200.autoregressive.models import gpt
    legacy = object.__new__(gpt.Transformer)                    # the class decides; no weights needed
    with pytest.raises(TypeError, match="no control_strength"):
        gen.generate(legacy, torch.zeros(2, dtype=torch.long), 4, cfg_scale=4.0, control_strength=[1.0, 0.5])
    assert gen.row_sampling(legacy, 2, True, [1.0, 1.0], [1, 2]) is not None
    assert [r.control_strength for r in gen.row_sampling(legacy, 2, False, [0.5, 0.5], [1, 2])] == [1.0, 1.0]


@pytest.mark.parametrize("bad", [dict(sp=SamplingParams(top_p=0.0)), dict(sp=SamplingParams(temperature=-1.0)),
                                 dict(sp=SamplingParams(top_p=1.5)), dict(cs=float("inf"))])
def test_mixed_mode_refuses_bad_requests_when_queued(bad):
    """A request generate() would refuse is refused by add_request, so it never reaches a launch and its batch-mates run."""
    log = []
    llm = LLM(cfg_scale=4.0, runner=_fake_runner(log), max_images_per_batch=8, mixed_sampling=True)
    llm.add_request(0, SamplingParams(max_tokens=2))
    with pytest.raises(ValueError):
        llm.add_request(1, bad.get("sp", SamplingParams(max_tokens=2)), control_strength=bad.get("cs", 1.0))
    llm.add_request(2, SamplingParams(temperature=0, max_tokens=2))
    while llm.has_unfinished_requests():
        llm.step()
    assert [b for b, _ in log] == [[0, 1]]                       # request ids 0 and 1: the refused one took no id
