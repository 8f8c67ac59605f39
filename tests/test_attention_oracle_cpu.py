"""CPU: the fp64 attention oracle (oracle/attn_oracle.py) against F.scaled_dot_product_attention with the bool mask built the way
the reference builds it — Transformer.setup_caches (gpt_t2i.py:401-402), the emb_masks edit of generate() (generate.py:184-193) and
the row selection of the forward pass (gpt_t2i.py:447-448) — so that the oracle's mask semantics are the reference's, not a
reading of them."""
import pytest
import torch
import torch.nn.functional as F

from oracle.attn_oracle import attention_mask, masked_sdpa


def _reference_mask(B, S, emb_masks):
    causal_mask = torch.tril(torch.ones(S, S, dtype=torch.bool)).unsqueeze(0).repeat(B, 1, 1)
    if emb_masks is not None:
        T = emb_masks.shape[-1]
        causal_mask[:, :, :T] = causal_mask[:, :, :T] * emb_masks.unsqueeze(1)       # bool * int: stored back as != 0
        eye_matrix = torch.eye(causal_mask.size(1), causal_mask.size(2))
        causal_mask[:] = causal_mask * (1 - eye_matrix) + eye_matrix                   # float blend: stored back as != 0
    return causal_mask


def _masks(B, T, g):
    left = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        left[b, T - 1 - (3 * b) % T:] = 1                                             # left-padded captions, valid tokens at the end
    rnd = (torch.rand(B, T, generator=g) < 0.5).long()
    rnd[:, 0] = 0                                                                     # row 0 of the text block sees only itself
    vals = rnd * torch.tensor([2, -3, 7, 1])[torch.randint(0, 4, (B, T), generator=g)]
    return {"none": None, "ones": torch.ones(B, T, dtype=torch.int64), "zeros": torch.zeros(B, T, dtype=torch.int64),
            "leftpad": left, "random": rnd, "values": vals}


@pytest.mark.parametrize("mask", ["none", "ones", "zeros", "leftpad", "random", "values"])
@pytest.mark.parametrize("T", [1, 7, 20])
def test_oracle_matches_sdpa_with_reference_mask(mask, T):
    g = torch.Generator().manual_seed(T * 31 + len(mask))
    B, H, S = 3, 2, 40
    em = _masks(B, T, g)[mask]
    q = torch.randn(B, H, S, 64, generator=g, dtype=torch.float64)
    k = torch.randn(B, H, S, 64, generator=g, dtype=torch.float64)
    v = torch.randn(B, H, S, 64, generator=g, dtype=torch.float64)
    ref_mask = _reference_mask(B, S, em)
    assert torch.equal(attention_mask(B, S, em), ref_mask)
    # prefill: rows 0 .. Tq-1 against the cache rows the oracle is given (0 .. Tq-1); the reference soft-maxes over all S
    Tq = max(T, 13)
    want = F.scaled_dot_product_attention(q[:, :, :Tq], k, v, attn_mask=ref_mask[:, None, torch.arange(Tq)])
    got = masked_sdpa(q[:, :, :Tq], k[:, :, :Tq], v[:, :, :Tq], range(Tq), em)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    # decode: one query at pos >= T against rows 0 .. pos
    for pos in (T, T + 1, S - 1):
        want = F.scaled_dot_product_attention(q[:, :, pos:pos + 1], k, v, attn_mask=ref_mask[:, None, [pos]])
        got = masked_sdpa(q[:, :, pos:pos + 1], k[:, :, :pos + 1], v[:, :, :pos + 1], [pos], em)
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def test_oracle_edges():
    """All-zero emb_mask: a text row attends only itself, so its output is its own value row; rows past the live range never
    matter (NaN there changes nothing)."""
    B, H, T, n = 2, 1, 6, 10
    g = torch.Generator().manual_seed(5)
    q = torch.randn(B, H, n, 64, generator=g, dtype=torch.float64)
    k = torch.randn(B, H, n + 4, 64, generator=g, dtype=torch.float64)
    v = torch.randn(B, H, n + 4, 64, generator=g, dtype=torch.float64)
    k[:, :, n:] = float("nan")
    v[:, :, n:] = float("nan")
    o = masked_sdpa(q, k[:, :, :n], v[:, :, :n], range(n), torch.zeros(B, T, dtype=torch.int32))
    assert torch.isfinite(o).all()
    torch.testing.assert_close(o[:, :, :T], v[:, :, :T], rtol=0, atol=0)


def test_oracle_rounding_points():
    """out_dtype is the rounding of the fp64 result; p_dtype = bf16 moves the result by at most 2^-8 of each column's value range
    (every probability carries a relative error <= 2^-8, the same one in numerator and denominator)."""
    B, H, n = 2, 3, 50
    g = torch.Generator().manual_seed(9)
    q = torch.randn(B, H, 1, 64, generator=g, dtype=torch.float64) * 2
    k = torch.randn(B, H, n, 64, generator=g, dtype=torch.float64)
    v = torch.randn(B, H, n, 64, generator=g, dtype=torch.float64)
    exact = masked_sdpa(q, k, v, [n - 1])
    assert torch.equal(masked_sdpa(q, k, v, [n - 1], out_dtype=torch.bfloat16), exact.to(torch.bfloat16).double())
    pr = masked_sdpa(q, k, v, [n - 1], p_dtype=torch.bfloat16)
    rng = (v.amax(2) - v.amin(2))[:, :, None]
    assert bool(((pr - exact).abs() <= 2 ** -8 * rng * (1 + 2 ** -7)).all())
    assert not torch.equal(pr, exact)
