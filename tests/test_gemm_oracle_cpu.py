"""CPU: the fp64 GEMM oracle (oracle/gemm_oracle.py) against PyTorch in float64.  The oracle is written from gemm.h's index
arithmetic; these tests tie each A addressing mode, the bf16 rounding emulation, the epilogue order, the batch strides and the
window pixel map to independent PyTorch formulations, so a GPU mismatch against the oracle is the kernel's."""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm_oracle as go

F64 = torch.float64


def _gen(seed):
    g = torch.Generator().manual_seed(seed)
    return g


def _nhwc(B, H, W, C, g):
    return torch.randn(B, H, W, C, generator=g, dtype=F64)


def _conv_weight(N, C, kh, kw, g):
    w = torch.randn(N, C, kh, kw, generator=g, dtype=F64)
    return w, w.permute(0, 2, 3, 1).reshape(N, kh * kw * C).contiguous()      # B [N][(ky kw + kx) C + c]


def _run(d, batch, A, B, **bufs):
    r = go.gemm(d, batch, A.reshape(-1), B.reshape(-1), **bufs)
    return r


def test_round_bf16_matches_torch_on_fp32_values():
    """Round to nearest even, including exact ties, subnormals and values that round up into the next binade."""
    g = _gen(0)
    x = torch.randn(200000, generator=g, dtype=torch.float32) * torch.exp2(torch.randint(-140, 60, (200000,), generator=g).float())
    ties = (torch.randint(-1000, 1000, (4096,), generator=g).float() * 2 + 1) * 2.0 ** -8          # odd multiples of half an ulp
    ups = torch.tensor([255.5, 511.0, 1.99609375, -0.0078125 * 255.5, 2.0 ** -133, 3 * 2.0 ** -134])
    for v in (x, ties, ups.float()):
        assert torch.equal(go.round_bf16(v.to(F64)), v.to(torch.bfloat16).to(F64))
    m = go.bf16_midpoint_distance(torch.tensor([1.0 + 2.0 ** -8, 1.0, 1.0 + 2.0 ** -9], dtype=F64))
    assert m.tolist() == [0.0, 2.0 ** -8, 2.0 ** -9]
    lo, hi = go.bf16_cell(torch.tensor([1.0, -1.0, 1.5], dtype=F64))
    assert lo.tolist() == [1.0 - 2.0 ** -9, -1.0 - 2.0 ** -8, 1.5 - 2.0 ** -8]
    assert hi.tolist() == [1.0 + 2.0 ** -8, -1.0 + 2.0 ** -9, 1.5 + 2.0 ** -8]
    for v in (x, ties):                      # every value rounds into the cell of its rounding
        lo, hi = go.bf16_cell(go.round_bf16(v.to(F64)))
        assert ((lo <= v.to(F64)) & (v.to(F64) <= hi)).all()


@pytest.mark.parametrize("H,W", [(4, 4), (5, 7), (8, 16), (9, 17)])
@pytest.mark.parametrize("ups", [0, 1])
def test_conv3x3_matches_conv2d(H, W, ups):
    g = _gen(H * 100 + W + ups)
    B, Cin, N = 2, 8, 5
    x = _nhwc(B, H, W, Cin, g)
    w, Bm = _conv_weight(N, Cin, 3, 3, g)
    Ho, Wo = H << ups, W << ups
    d = go.Desc(M=B * Ho * Wo, N=N, K=9 * Cin, ldb=9 * Cin, amode=go.A_CONV3x3, Hs=H, Ws=W, Cin=Cin, Ho=Ho, Wo=Wo, ups=ups, ldc=N,
                out_mode=1)
    r = _run(d, 1, x, Bm)
    src = x.permute(0, 3, 1, 2)
    if ups:
        src = F.interpolate(src, scale_factor=2, mode="nearest")
    ref = F.conv2d(src, w, padding=1).permute(0, 2, 3, 1).reshape(-1)
    out = torch.full((B * Ho * Wo * N,), float("nan"), dtype=F64)
    out[r.idx.reshape(-1)] = r.val.reshape(-1)
    torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("H,W", [(4, 4), (5, 7), (8, 9), (9, 16)])
def test_conv3x3_stride2_matches_padded_conv2d(H, W):
    g = _gen(7 * H + W)
    B, Cin, N = 2, 16, 3
    x = _nhwc(B, H, W, Cin, g)
    w, Bm = _conv_weight(N, Cin, 3, 3, g)
    ref = F.conv2d(F.pad(x.permute(0, 3, 1, 2), (0, 1, 0, 1)), w, stride=2)               # Downsample: pad right / bottom by one
    Ho, Wo = ref.shape[2], ref.shape[3]
    d = go.Desc(M=B * Ho * Wo, N=N, K=9 * Cin, ldb=9 * Cin, amode=go.A_CONV3x3S2, Hs=H, Ws=W, Cin=Cin, Ho=Ho, Wo=Wo, ldc=N, out_mode=1)
    r = _run(d, 1, x, Bm)
    torch.testing.assert_close(r.val.reshape(B, Ho, Wo, N), ref.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    assert torch.equal(r.idx.reshape(-1), torch.arange(B * Ho * Wo * N))


@pytest.mark.parametrize("k,s", [(1, 1), (3, 1), (3, 2), (7, 1), (7, 2), (2, 1)])
def test_window_matches_conv2d_on_padded_source(k, s):
    g = _gen(k * 10 + s)
    B, Cin, N, Hs, Ws = 2, 8, 4, 13, 18
    x = _nhwc(B, Hs, Ws, Cin, g)
    w, Bm = _conv_weight(N, Cin, k, k, g)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, stride=s).permute(0, 2, 3, 1)
    Ho, Wo = ref.shape[1], ref.shape[2]
    ldc = N + 3
    d = go.Desc(M=B * Ho * Wo, N=N, K=k * k * Cin, ldb=k * k * Cin, amode=go.A_WIN, Hs=Hs, Ws=Ws, Cin=Cin, Ho=Ho, Wo=Wo, kh=k, kw=k, ws=s,
                ldc=ldc, out_mode=1, oH=Ho, oW=Wo)
    bias_f = torch.randn(N, generator=g, dtype=F64)
    r = _run(d, 1, x, Bm, bias_f=bias_f)
    out = torch.full((B * Ho * Wo, ldc), float("nan"), dtype=F64).reshape(-1)
    out[r.idx.reshape(-1)] = r.val.reshape(-1)
    out = out.reshape(B, Ho, Wo, ldc)
    torch.testing.assert_close(out[..., :N], ref + bias_f, rtol=1e-12, atol=1e-12)
    assert out[..., N:].isnan().all()


def test_window_parity_classes_tile_the_image():
    """The transposed-convolution split of LineArt's up-sampling: four window GEMMs, one per output parity class (ay, ax), each
    writing pixels (2 oy + ay, 2 ox + ax) of one [B][2h][2w][N] image.  Reassembled, they equal an explicit scatter and cover every
    pixel exactly once."""
    g = _gen(3)
    B, Cin, N, h, w = 2, 8, 5, 5, 6
    out = torch.full((B * 2 * h * 2 * w * N,), float("nan"), dtype=F64)
    ref = torch.full((B, 2 * h, 2 * w, N), float("nan"), dtype=F64)
    hits = torch.zeros_like(out)
    for cls in range(4):
        ay, ax = cls >> 1, cls & 1
        kh, kw = 1 + ay, 1 + ax
        x = _nhwc(B, h + 1, w + 1, Cin, g)
        wt, Bm = _conv_weight(N, Cin, kh, kw, g)
        d = go.Desc(M=B * h * w, N=N, K=kh * kw * Cin, ldb=kh * kw * Cin, amode=go.A_WIN, Hs=h + 1, Ws=w + 1, Cin=Cin, Ho=h, Wo=w, kh=kh,
                    kw=kw, ws=1, ldc=N, out_mode=1, osy=2, osx=2, oay=ay, oax=ax, oH=2 * h, oW=2 * w)
        bias_f = torch.randn(N, generator=g, dtype=F64)
        r = _run(d, 1, x, Bm, bias_f=bias_f)
        out[r.idx.reshape(-1)] = r.val.reshape(-1)
        hits[r.idx.reshape(-1)] += 1
        conv = F.conv2d(x.permute(0, 3, 1, 2), wt)[:, :, :h, :w].permute(0, 2, 3, 1) + bias_f
        ref[:, ay::2, ax::2, :] = conv
    assert (hits == 1).all()
    torch.testing.assert_close(out.reshape(B, 2 * h, 2 * w, N), ref, rtol=1e-12, atol=1e-12)


def test_nchw_output_layout():
    g = _gen(5)
    B, H, W, Cin, N = 2, 3, 5, 8, 4
    x = _nhwc(B, H, W, Cin, g)
    w, Bm = _conv_weight(N, Cin, 3, 3, g)
    d = go.Desc(M=B * H * W, N=N, K=9 * Cin, ldb=9 * Cin, amode=go.A_CONV3x3, Hs=H, Ws=W, Cin=Cin, Ho=H, Wo=W, out_mode=2)
    r = _run(d, 1, x, Bm)
    out = torch.full((B * N * H * W,), float("nan"), dtype=F64)
    out[r.idx.reshape(-1)] = r.val.reshape(-1)
    torch.testing.assert_close(out.reshape(B, N, H, W), F.conv2d(x.permute(0, 3, 1, 2), w, padding=1), rtol=1e-12, atol=1e-12)


def test_batch_strides_and_broadcasts():
    """sA = 0 or sB = 0 reuses one operand for every batch entry; C and the residual advance by sC and sR."""
    g = _gen(11)
    batch, M, N, K, lda, ldb, ldc = 3, 5, 6, 8, 10, 12, 9
    for sA, sB in [(M * lda, N * ldb), (0, N * ldb), (M * lda, 0)]:
        A = torch.randn(max(1, batch * (sA > 0)) * M * lda, generator=g, dtype=F64)
        Bb = torch.randn(max(1, batch * (sB > 0)) * N * ldb, generator=g, dtype=F64)
        rf = torch.randn(batch * M * ldc, generator=g, dtype=F64)
        d = go.Desc(M=M, N=N, K=K, lda=lda, ldb=ldb, sA=sA, sB=sB, sC=M * ldc + 1, sR=M * ldc, ldr=ldc, ldc=ldc, out_mode=1, alpha=0.5)
        r = go.gemm(d, batch, A, Bb, resid_f=rf)
        a3 = A.reshape(-1, M, lda)[:, :, :K].expand(batch, M, K)
        b3 = Bb.reshape(-1, N, ldb)[:, :, :K].expand(batch, N, K)
        ref = 0.5 * a3 @ b3.transpose(1, 2) + rf.reshape(batch, M, ldc)[:, :, :N]
        torch.testing.assert_close(r.val, ref, rtol=1e-12, atol=1e-12)
        z = torch.arange(batch).view(-1, 1, 1)
        assert torch.equal(r.idx, z * (M * ldc + 1) + torch.arange(M).view(1, -1, 1) * ldc + torch.arange(N).view(1, 1, -1))


@pytest.mark.parametrize("act", [go.ACT_NONE, go.ACT_GELU_TANH, go.ACT_GELU_ERF, go.ACT_RELU])
def test_epilogue_rounding_points_match_stepwise_torch(act):
    """The documented order, evaluated step by step with torch's own fp32 -> bf16 casts: v = acc (+ bias[n]); r(v); act (GELU
    rounds); r(v scale); r(v + resid).  Inputs are exact (small integers x 2^-3), so fp32 and fp64 agree on every value before a
    rounding point; GELU is compared on its fp64 value."""
    g = _gen(act)
    M, N, K = 7, 16, 24
    A = torch.randint(-8, 9, (M, K), generator=g).to(F64) / 8
    Bm = torch.randint(-8, 9, (N, K), generator=g).to(F64) / 8
    bias = torch.randint(-128, 129, (N,), generator=g).to(F64) / 64
    scale = torch.randint(1, 200, (N,), generator=g).to(F64) / 128
    resid = torch.randint(-128, 129, (M, N), generator=g).to(F64) / 64
    d = go.Desc(M=M, N=N, K=K, lda=K, ldb=K, act=act, ldr=N, ldc=N)
    r = go.gemm(d, 1, A.reshape(-1), Bm.reshape(-1), bias=bias, scale=scale, resid=resid.reshape(-1))
    bf = lambda t: t.to(torch.float32).to(torch.bfloat16).to(F64)
    v = bf(A @ Bm.T + bias)
    if act == go.ACT_GELU_TANH:
        v = bf(0.5 * v * (1 + torch.tanh((2 / torch.pi) ** 0.5 * (v + 0.044715 * v ** 3))))
    elif act == go.ACT_GELU_ERF:
        v = bf(F.gelu(v))
    elif act == go.ACT_RELU:
        v = v.clamp(min=0)
    v = bf(bf(v * scale) + resid)
    assert torch.equal(r.val[0], v)


def test_split3_operands_reproduce_the_fp32_product():
    """S3 . W3 (the split-bf16 triple product, split3.cuh) differs from the fp64 product of the fp32 values by at most the dropped
    lo . lo term and the rounding of lo: 2^-15 |x w| per term (see tests/test_gemm_gpu.py for the derivation)."""
    g = _gen(17)
    M, N, C = 9, 8, 40
    x = torch.randn(M, C, generator=g).float()
    w = torch.randn(N, C, generator=g).float()
    s3, w3 = go.s3_rows(x), go.w3_rows(w.view(N, 1, C)).view(N, 3 * C)
    exact = x.to(F64) @ w.to(F64).T
    err = (s3 @ w3.T - exact).abs()
    assert (err <= 2.0 ** -15 * (x.to(F64).abs() @ w.to(F64).abs().T)).all()
    hi, lo = go.x3_split(x)
    assert torch.equal(hi, x.to(torch.bfloat16).to(F64))
    assert torch.equal(lo, (x - x.to(torch.bfloat16).float()).to(torch.bfloat16).to(F64))
