"""CPU: the sampler oracle (oracle/sampler_oracle.py) against the reference's own sample() / top_k_top_p_filtering() outputs on the
edge-row catalogue (tests/golden/sampler_edges.npz, made by tests/golden/make_golden.py sampler_edges)."""
import os

import numpy as np
import pytest
import torch

from oracle.sampler_oracle import (cfg_temperature, choice_ok, div_recip_pair, fixture_configs, fixture_rows, oracle_sample,
                                   probe_cols, resolve_k)
from tests.helpers import GOLDEN


@pytest.fixture(scope="module")
def fx():
    return np.load(os.path.join(GOLDEN, "sampler_edges.npz"))


ROWS = fixture_rows()


@pytest.mark.parametrize("name", list(ROWS))
def test_oracle_matches_reference_fixture(fx, name):
    rows = ROWS[name]
    R, V = rows.shape
    cols = torch.stack([probe_cols(rows[r]) for r in range(R)])
    kept_ref = np.unpackbits(fx[f"{name}_kept"], axis=-1)[..., :V].astype(bool)
    for ci, (T, k, p) in enumerate(fixture_configs()):
        kk = resolve_k(k, V)
        z = cfg_temperature(rows, R, 1.0, True, T)
        o = oracle_sample(z, kk, p, sample_logits=False)
        what = f"{name} T={T} top_k={k} top_p={p}"
        ref = torch.from_numpy(kept_ref[ci])
        outside = ~o.band_ref
        assert torch.equal(o.kept[outside], ref[outside]), f"{what}: kept sets differ outside the nucleus band"
        # probabilities: the oracle's soft-max over the set the reference kept (its band decisions move the normaliser)
        p0 = oracle_sample(z, kk, 1.0, sample_logits=False).probs * ref
        p0 = p0 / p0.sum(-1, keepdim=True)
        pr = torch.from_numpy(fx[f"{name}_probs"][ci]).double()
        assert torch.allclose(torch.gather(p0, 1, cols), pr, atol=1e-7, rtol=2e-5), f"{what}: probabilities"
        if not bool((o.band_ref & (o.kept != ref)).any()):
            assert torch.allclose(torch.gather(o.probs, 1, cols), pr, atol=1e-7, rtol=2e-5), f"{what}: probabilities"
        idx = fx[f"{name}_idx"][ci]
        for r in range(R):
            # torch.topk's order among exact ties is unspecified: any maximal token is the reference's greedy choice then
            tie = float(o.gap[r]) == 0.0 and float(o.probs[r, int(idx[r])]) == float(o.probs[r, int(o.choice[r])])
            ok = choice_ok(int(idx[r]), o, r) or tie
            assert ok, f"{what} row {r}: reference greedy {int(idx[r])}, oracle {int(o.choice[r])} (gap {float(o.gap[r]):.2e})"


def test_fixture_covers_the_edges(fx):
    """The catalogue reaches what it is there for: ties across the top-k rank, kept -0 entries, kept -inf entries."""
    cfgs = fixture_configs()
    V = 16384
    ci = cfgs.index((1.0, 2000, 1.0))
    kept = np.unpackbits(fx["tie3000_kept"], axis=-1)[ci, 0, :V]
    assert kept.sum() > 2300                         # 2000 plus the ties at the threshold
    rows = ROWS["pm0"][0]
    kept = np.unpackbits(fx["pm0_kept"], axis=-1)[ci, 0, :V].astype(bool)
    assert kept[(rows == 0).numpy()].all(), "the reference keeps every +-0 entry tied at the threshold"
    o = oracle_sample(rows[None], 1000, 1.0, sample_logits=False)
    assert bool(o.kept[0, rows == 0].all()) and int(o.kept.sum()) == 3100
    kept = np.unpackbits(fx["tie200_kept"], axis=-1)[ci, 0, :V]
    assert kept.sum() == 2000                        # the threshold lies above the 200-way tie at top_k = 2000
    kept = np.unpackbits(fx["pm0_small_kept"], axis=-1)[ci, 0, :V].astype(bool)
    assert kept.sum() == 2100 and kept[(ROWS["pm0_small"][0] == 0).numpy()].all()
    rows = ROWS["ninf"]
    ci = cfgs.index((1.0, 2000, 1.0))
    kept = np.unpackbits(fx["ninf_kept"], axis=-1)[ci, 1, :V].astype(bool)
    assert kept.all(), "fewer finite entries than top_k: the threshold is -inf and every entry is kept"


def test_division_and_reciprocal_differ_on_the_planted_pair():
    x, y, tie_under_recip = div_recip_pair()
    t = np.float32(0.7)
    d = np.array([x, y], np.float32) / t
    m = np.array([x, y], np.float32) * (np.float32(1) / t)
    assert (d[0] == d[1]) != (m[0] == m[1])
    assert (m[0] == m[1]) == tie_under_recip


def test_cfg_temperature_is_fp32_sub_mul_add_then_reciprocal():
    g = torch.Generator().manual_seed(3)
    lg = torch.randn(4, 64, generator=g)
    z = cfg_temperature(lg, 2, 4.0, True, 0.7)
    c, u = lg[:2].numpy(), lg[2:].numpy()
    want = (u + (c - u) * np.float32(4.0)) * (np.float32(1) / np.float32(0.7))
    assert np.array_equal(z.numpy(), want.astype(np.float32))
    assert torch.equal(cfg_temperature(lg, 2, 4.0, False, 1.0), lg[:2])


def test_cfg_interval_encoding():
    """generate.py:121: CFG is off at decode step i iff `cfg_interval > -1 and i > cfg_interval`, with --cfg-interval parsed as a
    float.  Values above -1 are floored (the same decisions on integer steps); (-1, 0) cannot be expressed and is refused."""
    from controlar_b200.engine import make_sampling
    for ci, want in ((-1, -1), (-1.0, -1), (-3, -1), (-1.5, -1), (0, 0), (0.0, 0), (2.5, 2), (5, 5)):
        got = make_sampling(cfg_interval=ci).cfg_interval
        assert got == want, (ci, got)
        for i in range(8):
            assert (ci > -1 and i > ci) == (got > -1 and i > got), (ci, i)
    for ci in (-0.5, -0.999, -1e-9):
        with pytest.raises(ValueError, match="cfg_interval"):
            make_sampling(cfg_interval=ci)
