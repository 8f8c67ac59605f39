"""GPU parity of the building-block ops and the fused sampler, through the C ABI."""
import pytest
import torch

from oracle.ar_oracle import sample_from_logits, cfg_combine
from tests.helpers import load_golden, rel_l2

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(1, 256, 256), (16, 1280, 3840), (5, 3584, 1280), (33, 384, 1280), (120, 2048, 256)])
@pytest.mark.parametrize("act", [0, 1])
def test_linear_vs_torch(dt, shape, act):
    from controlar_b200 import engine
    M, K, N = shape
    g = torch.Generator().manual_seed(M * 7 + K)
    x = (torch.randn(M, K, generator=g)).to(dt)
    w = (torch.randn(N, K, generator=g) * 0.05).to(dt)
    y = engine.op_linear(x.cuda(), w.cuda(), act=act).cpu()
    want = (x.float() @ w.float().t()).to(dt).float()
    if act == 1:
        want = torch.nn.functional.gelu(want, approximate="tanh").to(dt).float()
    tol = 2e-6 if dt == torch.float32 else 3e-3
    assert rel_l2(y.float(), want) < tol
    if dt == torch.bfloat16:   # at most 1-ulp rounding flips
        assert (y.float() - want).abs().max() <= want.abs().max() * 2 ** -7


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
def test_rmsnorm_vs_reference_formula(dt):
    from controlar_b200 import engine
    g = torch.Generator().manual_seed(1)
    x = torch.randn(37, 1280, generator=g).to(dt)
    w = (1 + 0.1 * torch.randn(1280, generator=g)).to(dt)
    y = engine.op_rmsnorm(x.cuda(), w.cuda(), 1e-5).cpu()
    xf = x.float()
    want = ((xf * torch.rsqrt((xf * xf).mean(-1, keepdim=True) + 1e-5)).to(dt) * w).float()   # gpt_t2i.py:193-198
    assert rel_l2(y.float(), want) < (1e-6 if dt == torch.float32 else 2e-3)


def test_sampler_matches_reference_fixture():
    """top-k / top-p / temperature soft-max rows vs the reference's own sample() outputs (tests/golden/sampler.pt)."""
    from controlar_b200 import engine
    g = load_golden("sampler")
    logits = g["logits"][:, 0].cuda()
    for c in g["cases"]:
        sp = engine.make_sampling(c["temperature"], c["top_k"], c["top_p"], sample_logits=False, cfg_scale=1.0)
        idx, probs = engine.sample(logits, sp, return_probs=True)
        want = c["probs"]
        got = probs.cpu()
        assert torch.equal(got > 0, want > 0), (c["temperature"], c["top_k"], c["top_p"], int((got > 0).sum()), int((want > 0).sum()))
        assert torch.allclose(got, want, atol=1e-7, rtol=2e-5)
        assert torch.equal(idx.cpu().long(), torch.argmax(want, -1)), "greedy: lowest index among ties"
    # exact tie at the top (fixture plants one at indices 5 and 9 of row 0): lowest index wins
    sp = engine.make_sampling(1.0, 0, 1.0, sample_logits=False)
    assert int(engine.sample(logits, sp)[0]) == 5


def test_sampler_cfg_and_noise_race():
    """CFG combine + exponential race on caller-provided noise == oracle argmax(p / q)."""
    from controlar_b200 import engine
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(8, 16384, generator=g) * 1.5
    noise = torch.empty(4, 16384).exponential_(1.0, generator=g)
    for cfg_on in (True, False):
        sp = engine.make_sampling(0.9, 2000, 1.0, sample_logits=True, cfg_scale=4.0)
        idx = engine.sample(logits.cuda(), sp, cfg_on=cfg_on, noise=noise.cuda()).cpu()
        z = cfg_combine(logits, 4.0, cfg_on)
        want, _ = sample_from_logits(z, 0.9, 2000, 1.0, True, noise=noise)
        assert torch.equal(idx.long(), want[:, 0])


def test_sampler_philox_is_seeded_and_distributional():
    from controlar_b200 import engine
    V = 2048
    p = torch.softmax(torch.linspace(0, 4, V), 0)
    logits = torch.log(p).repeat(64, 1).cuda()
    sp = engine.make_sampling(1.0, 0, 1.0, sample_logits=True, seed=42)
    a = engine.sample(logits, sp, step=3).cpu()
    b = engine.sample(logits, sp, step=3).cpu()
    c = engine.sample(logits, sp, step=4).cpu()
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert len(set(a.tolist())) > 32          # rows use distinct sub-streams
    # many draws: empirical mean index close to the distribution's mean
    draws = torch.cat([engine.sample(logits, sp, step=s).cpu() for s in range(200)]).float()
    mean_want = float((p * torch.arange(V)).sum())
    assert abs(float(draws.mean()) - mean_want) < 25.0, (float(draws.mean()), mean_want)


@pytest.mark.parametrize("M,N,K,act,res", [(1920, 3584, 1280, 0, False), (1920, 1280, 3584, 0, True), (480, 768, 256, 1, False),
                                            (1000, 1288, 1096, 0, True), (130, 136, 72, 1, True), (16384, 1280, 1280, 1, False),
                                            (200, 100, 72, 1, True)])
def test_dense_linear_vs_torch(M, N, K, act, res):
    """gemm() (gemm.cu): y = act(x w^T) (+ resid) against an fp32 torch reference of the same rounding points (bf16 product rounding,
    GELU-tanh in bf16, residual add in bf16); includes M / N / K tails (K % 64 != 0, partial tiles).  N % 8 != 0 takes the mma.sync
    kernel, every other row the wgmma kernel (TMA + wgmma, accumulators in registers)."""
    from controlar_b200 import engine
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    x = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * (K ** -0.5)).to(torch.bfloat16)
    r = (torch.randn(M, N, device="cuda", generator=g)).to(torch.bfloat16) if res else None
    y = engine.op_dense_linear(x, w, r, act)
    ref = (x.float() @ w.float().t()).to(torch.bfloat16).float()
    if act:
        ref = torch.nn.functional.gelu(ref, approximate="tanh").to(torch.bfloat16).float()
    if res:
        ref = (ref + r.float()).to(torch.bfloat16).float()
    err = float((y.float() - ref).abs().max())
    rel = float((y.float() - ref).norm() / ref.norm())
    assert rel < 4e-3 and err < 0.1, (rel, err)        # one bf16 ulp flips where the fp32 sums differ in the last bit
