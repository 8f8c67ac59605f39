"""GPU: conformance of the dense GEMM front end (csrc/gemm.h) against the fp64 oracle (oracle/gemm_oracle.py): every route of
gemm() (wgmma plain, wgmma 3x3 convolution, mma.sync, mma.sync window) and the two fp32-output functions gemm_f32 and
gemm_f32_conv3, each epilogue field, output layout and batch stride.  Every case asserts the route car_op_gemm_route reports.

Two input families:
  * exact: A and B small integers x 2^-3 (|a|, |b| <= 1), bf16 bias and residual on a 2^-6 grid, LayerScale on a 2^-7 grid, fp32
    bias / residual on a 2^-6 grid, alpha a power of two.  Every product is a multiple of 2^-6 and every partial sum stays below
    2^12 for K <= 3584, so it needs at most 18 significant bits and is exact in fp32 in any order.  This rests on one assumption
    that is not measured anywhere else: that Hopper's bf16 tensor-core accumulation into fp32 is exact when every partial sum fits
    in 24 bits.  Under it the accumulator equals the oracle's, every epilogue step before a GELU is exact or a bf16 rounding of an
    exact value, and every output must be BIT-EQUAL to the oracle.
    GELU is evaluated with tanhf / erff, 2 ulp each (CUDA C Programming Guide, single-precision mathematical functions), inside
    0.5 x (1 + t): for the tanh form the argument k0 (x + k1 x^3) carries <= 7 roundings (two constants, four products, one sum,
    no cancellation), which moves tanh by <= max(z sech^2 z) 7u = 3.2u; tanhf adds 2 ulp <= 2u (|t| < 1); 1 + t adds <= 2u; the
    final product adds u |g|.  So |gelu_f32(x) - gelu(x)| <= 0.5 |x| 7.2u + u |g| <= DELTA(x) = 4u |x| + 2u |g| (u = 2^-24); the
    erf form (two roundings in x k, erf' z <= 0.49, erff 2 ulp) is within the same bound.  A GELU output may therefore be any bf16
    value that a real within DELTA of the exact fp64 GELU rounds to: mostly the oracle's rounding or its neighbour across a nearby
    midpoint, but in the negative tail, where 1 + t cancels, DELTA spans many bf16 ulps of the tiny result.  The rest of the
    epilogue (LayerScale > 0, residual) is monotone, so the final value must lie between the oracle's epilogue applied to the two
    ends of that range.
  * gaussian: N(0, 1) operands.  The kernel's fp32 accumulator differs from the exact sum by at most 2 K u sum_k |a_k b_k| (2u per
    addition also covers adders that truncate); each epilogue addition adds u of its operands.  A bf16 output must be the rounding
    of a real within that bound of the oracle's pre-rounding value (err = the distance from the oracle's value to the set of reals
    that round to the output; near a midpoint that allows the other neighbour, near zero, where the bound is wider than an ulp, a
    few more); an fp32 output must be within the bound.  The worst err / bound and the number of outputs that differ from the
    oracle's rounding are printed.

Guards in every call: lda, ldb (and ldc where the layout has one) are larger than needed and the pad columns of A and B are NaN; C
sits inside a NaN margin.  Every element the oracle does not write must still hold its NaN bit pattern, every element it writes
must be finite.  (The source frame of gemm_f32_conv3 is zero outside the map by contract, not NaN.)  No descriptor outside gemm()'s
contract is launched here: those are tested on the CPU only (tests/test_gemm_route_cpu.py).
"""
import math

import numpy as np
import pytest
import torch

from oracle import gemm_oracle as go

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
MARGIN = 64                                  # elements of NaN before and after C (keeps C 16-byte aligned)
WGMMA, WGMMA_CONV3, MMA, MMA_WIN = 0, 1, 2, 3
REACHED = set()
DEV = "cuda"
F64 = torch.float64


def _engine():
    from controlar_b200 import engine
    return engine


def gelu_delta(x, g):
    return 4 * U * x.abs() + 2 * U * g.abs()


class Gen:
    def __init__(self, seed, fam):
        self.g = torch.Generator().manual_seed(seed)
        self.fam = fam

    def op(self, *shape):                   # A and B values
        if self.fam == "exact":
            return torch.randint(-8, 9, shape, generator=self.g).float() / 8
        return torch.randn(*shape, generator=self.g)

    def grid(self, *shape, lim=128):       # biases and residuals: 2^-6 grid (exact) or N(0, 1)
        if self.fam == "exact":
            return torch.randint(-lim, lim + 1, shape, generator=self.g).float() / 64
        return torch.randn(*shape, generator=self.g)

    def scale(self, n):
        return torch.randint(1, 256, (n,), generator=self.g).float() / 128


def nan_rows(rows, cols, ld, vals, dtype=torch.bfloat16):
    """[rows][ld] with vals in the first cols columns and NaN in the pad columns, flattened, on the device."""
    t = torch.full((rows, ld), float("nan"), dtype=dtype)
    t[:, :cols] = vals.reshape(rows, cols).to(dtype)
    return t.reshape(-1).to(DEV)


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def check_output(name, cbuf, init, base, r, fam, K, c_bf16, extra=0.0, relu=False, gelu_range=None):
    """cbuf after the call, init its contents before; the oracle's result r at offset base.  gelu_range: (lo, hi), the final values
    the exact family allows when the GELU output is any bf16 value within DELTA of the exact GELU.  Returns (worst ratio, flips)."""
    idx = r.idx.reshape(-1) + base
    written = torch.zeros(cbuf.numel(), dtype=torch.bool, device=DEV)
    written[idx] = True
    assert int(written.sum()) == idx.numel(), f"{name}: the oracle writes an element twice"
    assert torch.equal(bits(cbuf)[~written], bits(init)[~written]), f"{name}: an element outside the output changed"
    got = cbuf[idx].to(F64)
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    val = r.val.reshape(-1)
    if fam == "exact":
        if gelu_range is None:
            bad = got != val
            assert not bad.any(), f"{name}: {int(bad.sum())} of {got.numel()} differ from the exact oracle, first at " \
                                  f"{int(bad.nonzero()[0])}: {got[bad][0].item()} vs {val[bad][0].item()}"
            return 0.0, 0
        lo, hi = (t.reshape(-1) for t in gelu_range)
        ok = (got >= lo) & (got <= hi)
        assert ok.all(), f"{name}: {int((~ok).sum())} GELU outputs outside the derived tanhf / erff bound"
        flips = int((got != val).sum())
        print(f"\n{name}: exact family, {flips} of {got.numel()} outputs differ from the oracle's rounding, all within the GELU bound",
              end="")
        return 0.0, flips
    pre, absdot = r.pre.reshape(-1), r.absdot.reshape(-1)
    bound = 2 * (K + 4) * U * (absdot + pre.abs() + extra)
    t = pre.clamp(min=0) if relu else pre
    if c_bf16:
        # distance from the fp64 value to the set of reals that round to the output (the kernel's fp32 value lies in that set)
        lo, hi = go.bf16_cell(got)
        if relu:
            lo = torch.where(got == 0, torch.full_like(lo, -math.inf), lo)
        dist = torch.clamp(torch.maximum(lo - t, t - hi), min=0)
        flips = int((got != (go.round_bf16(pre).clamp(min=0) if relu else go.round_bf16(pre))).sum())
    else:
        dist = (got - t).abs()
        flips = 0
    ratio = (dist / bound).max().item()
    print(f"\n{name}: gaussian family, worst err/bound {ratio:.3g}, {flips} of {got.numel()} bf16 outputs differ from the oracle's "
          f"rounding", end="")
    assert ratio <= 1.0, f"{name}: err/bound {ratio}"
    return ratio, flips


def run(name, d, batch, route, fam, seed, *, bias=False, bias_f=False, resid_f=False, scale=False, resid=False, alias=False, c_off=0,
        alpha=None, conv_src=None):
    """Build the operands of descriptor d (oracle Desc) in family fam, launch gemm() on them, compare with the oracle."""
    e = _engine()
    g = Gen(seed, fam)
    if alpha is not None:
        d.alpha = float(np.float32(alpha))
    nA = batch if d.sA else 1
    nB = batch if d.sB else 1
    if d.amode == go.A_PLAIN:
        if d.sA:
            d.sA = d.M * d.lda
        A = nan_rows(nA * d.M, d.K, d.lda, g.op(nA * d.M, d.K))
    else:
        A = g.op(*conv_src).to(torch.bfloat16).reshape(-1).to(DEV)
    if d.sB:
        d.sB = d.N * d.ldb
    B = nan_rows(nB * d.N, d.K, d.ldb, g.op(nB * d.N, d.K))
    bufs = {}
    if bias:
        bias_n = d.M if d.bias_along_m else d.N
        bufs["bias"] = g.grid(bias_n).to(torch.bfloat16).to(DEV)
    if bias_f:
        bufs["bias_f"] = g.grid(d.N, lim=4096).to(DEV)
    if scale:
        bufs["scale"] = g.scale(d.N).to(torch.bfloat16).to(DEV)
    c_bf16 = d.out_mode == 0 and d.amode != go.A_WIN
    cdt = torch.bfloat16 if c_bf16 else torch.float32
    extent = int(go.c_index(d, batch).max()) + 1
    cbuf = torch.full((extent + 2 * MARGIN + c_off,), float("nan"), dtype=cdt, device=DEV)
    base = MARGIN + c_off
    if resid_f:
        d.sR = d.M * d.ldr if batch > 1 else 0
        bufs["resid_f"] = g.grid(batch * d.M * d.ldr, lim=4096).to(DEV)
    if resid:
        if alias:                          # the residual is C itself (x = x + f(x) in place): same rows, same pitch
            d.ldr, d.sR = d.ldc, d.sC
            live = go.c_index(d, batch).reshape(-1) + base
            cbuf[live.to(DEV)] = g.grid(live.numel()).to(cdt).to(DEV)
            rbuf = cbuf[base:]
        else:
            d.sR = d.M * d.ldr if batch > 1 else 0
            rbuf = g.grid(batch * d.M * d.ldr).to(torch.bfloat16).to(DEV)
        bufs["resid"] = rbuf
    init = cbuf.clone()
    esz = cbuf.element_size()
    ptr = lambda k: bufs[k].data_ptr() if k in bufs else None
    desc = e.gemm_desc(A=A.data_ptr(), B=B.data_ptr(), M=d.M, N=d.N, K=d.K, lda=d.lda, ldb=d.ldb, sA=d.sA, sB=d.sB, sC=d.sC, sR=d.sR,
                       amode=d.amode, Hs=d.Hs, Ws=d.Ws, Cin=d.Cin, Ho=d.Ho, Wo=d.Wo, ups=d.ups, alpha=d.alpha, bias=ptr("bias"),
                       bias_along_m=d.bias_along_m, bias_f=ptr("bias_f"), resid_f=ptr("resid_f"), act=d.act, scale=ptr("scale"),
                       resid=ptr("resid"), ldr=d.ldr, C=cbuf.data_ptr() + base * esz, ldc=d.ldc, out_mode=d.out_mode, kh=d.kh,
                       kw=d.kw, ws=d.ws, osy=d.osy, osx=d.osx, oay=d.oay, oax=d.oax, oH=d.oH, oW=d.oW)
    got_route = e.op_gemm_route(desc, batch)
    assert got_route == route, f"{name}: route {got_route}, expected {route}"
    ob = {k: (init[base:] if (k == "resid" and alias) else v) for k, v in bufs.items()}
    r = go.gemm(d, batch, A, B, **ob)
    e.op_gemm(desc, batch)
    torch.cuda.synchronize()
    REACHED.add(route)
    gelu_range = None
    if r.gelu_out is not None:             # the rest of the epilogue is monotone in the GELU output (positive LayerScale)
        delta = gelu_delta(r.gelu_in, r.gelu_out)
        tail = {k: ob.get(k) for k in ("scale", "resid")}
        gelu_range = tuple(go.epilogue_tail(d, batch, go.round_bf16(r.gelu_out + s * delta), tail) for s in (-1, 1))
    extra = sum(float(v.abs().max()) for k, v in bufs.items() if k in ("bias", "bias_f", "resid_f"))
    return check_output(name, cbuf, init, base, r, fam, d.K, c_bf16, extra, relu=d.act == go.ACT_RELU, gelu_range=gelu_range)


def plain(M, N, K, **kw):
    return go.Desc(M=M, N=N, K=K, lda=K + 8, ldb=K + 16, ldc=N + 8, ldr=N + 24, **kw)


# ---------------------------------------------------------------- wgmma plain
MS, NS, KS = [1, 127, 128, 129, 1000], [8, 120, 128, 136, 1288], [8, 56, 64, 72, 1096, 3584]
SHAPES = [(m, n, KS[(i * 5 + j) % 6]) for i, m in enumerate(MS) for j, n in enumerate(NS)] + [(129, 136, k) for k in KS]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_wgmma_plain_shapes_exact(M, N, K):
    run(f"wgmma {M}x{N}x{K}", plain(M, N, K), 1, WGMMA, "exact", M * 7 + N * 3 + K, bias=True)


@pytest.mark.parametrize("M,N,K", [(1000, 1288, 3584), (129, 136, 1096), (127, 120, 72)])
def test_wgmma_plain_gaussian(M, N, K):
    run(f"wgmma gaussian {M}x{N}x{K}", plain(M, N, K), 1, WGMMA, "gaussian", M + N + K, bias=True)


EPI = {"bias": dict(bias=True), "gelu_tanh": dict(act=1), "gelu_erf": dict(act=2), "scale": dict(scale=True), "resid": dict(resid=True),
       "all_tanh": dict(bias=True, act=1, scale=True, resid=True), "all_erf": dict(bias=True, act=2, scale=True, resid=True)}


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("route", [WGMMA, MMA])
def test_epilogue_fields_exact(epi, route):
    """Each field of the bf16 epilogue alone and all together, on the wgmma kernel and (forced there by alpha = 2^-3, which is exact)
    on the mma.sync kernel."""
    kw = dict(EPI[epi])
    act = kw.pop("act", 0)
    d = plain(257, 136, 200, act=act)
    run(f"epilogue {epi} route {route}", d, 1, route, "exact", 5 + len(epi), alpha=1.0 if route == WGMMA else 0.125, **kw)


@pytest.mark.parametrize("M", [129, 1000])
def test_wgmma_resid_aliased_to_c(M):
    """x = x + ls * f(x) in place, as DINOv2's attention output and MLP and the prefill's residual GEMMs run it."""
    d = plain(M, 384, 128)
    run(f"wgmma resid aliased M={M}", d, 1, WGMMA, "exact", M, bias=True, scale=True, resid=True, alias=True)
    d = plain(M, 384, 128, act=2)
    run(f"wgmma resid aliased gelu M={M}", d, 1, WGMMA, "exact", M + 1, bias=True, resid=True, alias=True)


# ---------------------------------------------------------------- mma.sync plain
MMA_CASES = {
    "n100": (plain(300, 100, 64), dict(bias=True)),
    "n257": (plain(300, 257, 64), dict(bias=True)),
    "relu": (plain(300, 136, 96, act=3), dict(bias=True)),
    "alpha": (plain(300, 136, 96), dict(bias=True, alpha=0.125)),
    "bias_along_m": (plain(200, 136, 64), dict(bias=True)),
    "out_mode1": (plain(300, 136, 96, out_mode=1), dict(bias=True)),
    "bias_f_resid_f": (plain(300, 136, 96, out_mode=1), dict(bias_f=True, resid_f=True)),
    "bias_f_bf16": (plain(300, 136, 96), dict(bias_f=True, resid_f=True)),
    "relu_fp32": (plain(130, 72, 64, out_mode=1, act=3), dict(bias_f=True)),
    "c_offset_one": (plain(300, 136, 96), dict(bias=True, c_off=1)),
}


@pytest.mark.parametrize("fam", ["exact", "gaussian"])
@pytest.mark.parametrize("case", list(MMA_CASES))
def test_mma_plain(case, fam):
    d0, kw = MMA_CASES[case]
    d = go.Desc(**{k: getattr(d0, k) for k in d0.__dataclass_fields__})
    if case == "bias_along_m":
        d.bias_along_m = 1
    kw = dict(kw)
    if "alpha" in kw:
        kw["alpha"] = 0.125 if fam == "exact" else 1 / math.sqrt(512)
    run(f"mma {case} {fam}", d, 1, MMA, fam, len(case) * 13 + len(fam), **kw)


@pytest.mark.parametrize("fam", ["exact", "gaussian"])
@pytest.mark.parametrize("strides", ["distinct", "a_broadcast", "b_broadcast"])
def test_mma_batched(strides, fam):
    """batch 3 through blockIdx.z: V^T with a shared weight (sA = 0, bias along m), the scores (alpha, fp32 out) and the context."""
    M, N, K = 160, 100, 96
    sA = 0 if strides == "a_broadcast" else 1
    sB = 0 if strides == "b_broadcast" else 1
    d = go.Desc(M=M, N=N, K=K, lda=K + 8, ldb=K + 8, sA=sA, sB=sB, sC=M * (N + 4) + 8, ldc=N + 4)
    run(f"mma batch {strides} {fam}", d, 3, MMA, fam, 99 + len(strides), bias=True)
    d = go.Desc(M=M, N=N, K=K, lda=K + 8, ldb=K + 8, sA=sA, sB=sB, sC=M * (N + 4), ldc=N + 4, out_mode=1)
    run(f"mma batch scores {strides} {fam}", d, 3, MMA, fam, 7 + len(strides), alpha=0.125 if fam == "exact" else 1 / math.sqrt(512))
    d = go.Desc(M=M, N=N, K=K, lda=K + 8, ldb=K + 8, sA=sA, sB=sB, sC=M * N, ldc=N, bias_along_m=1)
    run(f"mma batch bias_along_m {strides} {fam}", d, 3, MMA, fam, 3 + len(strides), bias=True)


# ---------------------------------------------------------------- 3x3 convolutions
def conv_desc(nimg, H, W, Cin, N, amode=go.A_CONV3x3, ups=0, **kw):
    Hv, Wv = H << ups, W << ups
    Ho, Wo = (Hv, Wv) if amode == go.A_CONV3x3 else ((Hv - 2) // 2 + 1, (Wv - 2) // 2 + 1)
    f = dict(M=nimg * Ho * Wo, N=N, K=9 * Cin, ldb=9 * Cin + 8, amode=amode, Hs=H, Ws=W, Cin=Cin, Ho=Ho, Wo=Wo, ups=ups, ldc=N + 8,
             ldr=N + 8)
    f.update(kw)
    return go.Desc(**f), (nimg, H, W, Cin)


CONV_WG = [(n, h, w, c, o) for n in (1, 3) for (h, w) in ((8, 16), (9, 17), (24, 40)) for c in (64, 192) for o in (64, 136)]


@pytest.mark.parametrize("nimg,H,W,Cin,N", CONV_WG)
def test_conv3x3_wgmma_exact(nimg, H, W, Cin, N):
    i = CONV_WG.index((nimg, H, W, Cin, N))
    d, src = conv_desc(nimg, H, W, Cin, N, act=i % 3)
    run(f"conv wgmma {nimg}x{H}x{W}x{Cin}->{N}", d, 1, WGMMA_CONV3, "exact", i, bias=True, resid=i % 2 == 1, conv_src=src)


CONV_MMA = {
    "cin8_4x4": dict(nimg=2, H=4, W=4, Cin=8, N=40),
    "cin24_4x4_relu": dict(nimg=2, H=4, W=4, Cin=24, N=64, act=3),
    "cin8_ups_5x7": dict(nimg=2, H=5, W=7, Cin=8, N=24, ups=1),
    "cin24_ups_9x5_gelu": dict(nimg=1, H=9, W=5, Cin=24, N=64, ups=1, act=1),
    "cin64_ups_8x16": dict(nimg=1, H=8, W=16, Cin=64, N=64, ups=1),
    "nchw_bias_f_4x4": dict(nimg=2, H=4, W=4, Cin=24, N=40, out_mode=2, ldc=0),
    "nchw_bias_f_9x17": dict(nimg=1, H=9, W=17, Cin=64, N=64, out_mode=2, ldc=0),
}


@pytest.mark.parametrize("fam", ["exact", "gaussian"])
@pytest.mark.parametrize("case", list(CONV_MMA))
def test_conv3x3_mma(case, fam):
    kw = dict(CONV_MMA[case])
    if fam == "gaussian" and kw.get("act") in (1, 2):
        pytest.skip("GELU is checked in the exact family")
    d, src = conv_desc(**kw)
    run(f"conv mma {case} {fam}", d, 1, MMA, fam, len(case), bias=d.out_mode != 2, bias_f=d.out_mode == 2, conv_src=src)


@pytest.mark.parametrize("fam", ["exact", "gaussian"])
@pytest.mark.parametrize("H,W", [(8, 8), (9, 9), (8, 9), (9, 16), (24, 40)])
def test_conv3x3_stride2(H, W, fam):
    d, src = conv_desc(2, H, W, 16, 72, amode=go.A_CONV3x3S2)
    run(f"conv s2 {H}x{W} {fam}", d, 1, MMA, fam, H * W, bias=True, conv_src=src)


# ---------------------------------------------------------------- window
@pytest.mark.parametrize("fam", ["exact", "gaussian"])
@pytest.mark.parametrize("k,s", [(1, 1), (1, 2), (3, 1), (3, 2), (7, 1), (7, 2)])
def test_window(k, s, fam):
    B, Hs, Ws, Cin, N = 2, 21, 26, 24, 40
    Ho, Wo = (Hs - k) // s + 1, (Ws - k) // s + 1
    d = go.Desc(M=B * Ho * Wo, N=N, K=k * k * Cin, ldb=k * k * Cin + 8, amode=go.A_WIN, Hs=Hs, Ws=Ws, Cin=Cin, Ho=Ho, Wo=Wo, kh=k, kw=k,
                ws=s, ldc=N + 8, out_mode=1, oH=Ho, oW=Wo)
    run(f"window {k}x{k}/{s} {fam}", d, 1, MMA_WIN, fam, k * 10 + s, bias_f=True, conv_src=(B, Hs, Ws, Cin))


def test_window_parity_classes_tile_the_image():
    """Four window GEMMs, one per parity class (ay, ax) with a (1 + ay) x (1 + ax) window, write pixels (2 oy + ay, 2 ox + ax) of one
    [B][2h][2w][ldc] image: between them every pixel exactly once, the ldc pad columns never."""
    e = _engine()
    B, h, w, Cin, N, ldc = 2, 9, 13, 24, 40, 48
    out = torch.full((B * 2 * h * 2 * w * ldc,), float("nan"), dtype=torch.float32, device=DEV)
    want = torch.full_like(out, float("nan"), dtype=F64)
    hits = torch.zeros(out.numel(), dtype=torch.int32, device=DEV)
    for cls in range(4):
        g = Gen(40 + cls, "exact")
        ay, ax = cls >> 1, cls & 1
        kh, kw = 1 + ay, 1 + ax
        d = go.Desc(M=B * h * w, N=N, K=kh * kw * Cin, ldb=kh * kw * Cin + 8, amode=go.A_WIN, Hs=h + 1, Ws=w + 1, Cin=Cin, Ho=h, Wo=w,
                    kh=kh, kw=kw, ws=1, ldc=ldc, out_mode=1, osy=2, osx=2, oay=ay, oax=ax, oH=2 * h, oW=2 * w)
        A = g.op(B, h + 1, w + 1, Cin).to(torch.bfloat16).reshape(-1).to(DEV)
        Bm = nan_rows(N, d.K, d.ldb, g.op(N, d.K))
        bias_f = g.grid(N, lim=4096).to(DEV)
        desc = e.gemm_desc(A=A, B=Bm, M=d.M, N=N, K=d.K, ldb=d.ldb, amode=go.A_WIN, Hs=d.Hs, Ws=d.Ws, Cin=Cin, Ho=h, Wo=w, kh=kh, kw=kw,
                           ws=1, bias_f=bias_f, C=out, ldc=ldc, out_mode=1, osy=2, osx=2, oay=ay, oax=ax, oH=2 * h, oW=2 * w)
        assert e.op_gemm_route(desc) == MMA_WIN
        e.op_gemm(desc)
        r = go.gemm(d, 1, A, Bm, bias_f=bias_f)
        want[r.idx.reshape(-1)] = r.val.reshape(-1)
        hits[r.idx.reshape(-1)] += 1
    torch.cuda.synchronize()
    REACHED.add(MMA_WIN)
    img = hits.reshape(B, 2 * h, 2 * w, ldc)
    assert (img[..., :N] == 1).all() and (img[..., N:] == 0).all()
    assert torch.equal(out.to(F64)[hits == 1], want[hits == 1])
    assert out[hits == 0].isnan().all()


# ---------------------------------------------------------------- gemm_f32 / gemm_f32_conv3 over split-bf16 operands
def split_bound(absdot, K3, extra):
    """Error of S3 . W3 against the fp64 product of the fp32 values.  With x = hi + lo + ex, w = hw + lw + ew (|lo| <= 2^-8 |x|
    (1 + 2^-8), |ex| <= 2^-17 |x|, split3.cuh), the three bf16 products hi hw + lo hw + hi lw miss lo lw + hi ew + lo ew + ex w:
    <= (2^-16 + 2^-17 + 2^-17) (1 + 2^-7) |x w| = 2^-15 (1 + 2^-7) |x w| per term.  The 3K products are exact in fp32 and their sum
    carries <= 2 (3K) u (1 + 2^-7) sum |x w|; the bias and residual additions add u of their operands each."""
    return (2.0 ** -15 + 2 * K3 * U) * (1 + 2.0 ** -6) * absdot + 4 * U * (absdot + extra)


@pytest.mark.parametrize("M", [1, 100, 129, 300])
@pytest.mark.parametrize("N", [8, 24, 136])
@pytest.mark.parametrize("with_resid", [False, True])
def test_gemm_f32_split3_is_fp32_grade(M, N, with_resid):
    e = _engine()
    g = torch.Generator().manual_seed(M * 3 + N + with_resid)
    C = 48 if N != 136 else 256
    ldc = N + 8
    x = torch.randn(M, C, generator=g)
    w = torch.randn(N, C, generator=g)
    A = go.s3_rows(x).to(torch.bfloat16).reshape(-1).to(DEV)
    Bm = go.w3_rows(w.view(N, 1, C)).reshape(N, 3 * C).to(torch.bfloat16).reshape(-1).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    resid = torch.randn(M * ldc, generator=g).to(DEV) if with_resid else None
    out = torch.full((M * ldc + 2 * MARGIN,), float("nan"), device=DEV)
    init = out.clone()
    e.op_gemm_f32(A, Bm, M, N, 3 * C, bias, resid, out.data_ptr() + MARGIN * 4, ldc)
    torch.cuda.synchronize()
    REACHED.add("f32")
    xd, wd = x.to(F64).to(DEV), w.to(F64).to(DEV)
    exact = xd @ wd.T + bias.to(F64)
    if with_resid:
        exact = exact + resid.to(F64).view(M, ldc)[:, :N]
    absdot = xd.abs() @ wd.abs().T
    extra = bias.abs().to(F64) + (resid.to(F64).view(M, ldc)[:, :N].abs() if with_resid else 0)
    body = out[MARGIN:MARGIN + M * ldc].view(M, ldc)
    got = body[:, :N].to(F64)
    assert torch.isfinite(got).all()
    assert torch.equal(bits(body[:, N:].contiguous()), bits(init[MARGIN:MARGIN + M * ldc].view(M, ldc)[:, N:].contiguous()))
    assert torch.equal(bits(out[:MARGIN]), bits(init[:MARGIN])) and torch.equal(bits(out[MARGIN + M * ldc:]), bits(init[MARGIN + M * ldc:]))
    ratio = ((got - exact).abs() / split_bound(absdot, 3 * C, extra)).max().item()
    print(f"\ngemm_f32 x3 {M}x{N}x3*{C} resid={with_resid}: worst err/bound {ratio:.3g}", end="")
    assert ratio <= 1.0


def conv3_f32_case(nimg, H, W, cin, N, fh, fw, fam, seed, with_resid):
    """src frame [nimg][fh][fw][cin] (zero outside the H x W map) -> fp32 NHWC; returns (got, oracle result)."""
    e = _engine()
    g = Gen(seed, fam)
    frame = torch.zeros(nimg, fh, fw, cin)
    frame[:, :H, :W, :] = g.op(nimg, H, W, cin)
    src = frame.to(torch.bfloat16).reshape(-1).to(DEV)
    Bm = g.op(N, 9 * cin).to(torch.bfloat16).reshape(-1).to(DEV)
    bias = g.grid(N, lim=4096).to(DEV)
    M = nimg * H * W
    resid = g.grid(M * N, lim=4096).to(DEV) if with_resid else None
    out = torch.full((M * N + 2 * MARGIN,), float("nan"), device=DEV)
    init = out.clone()
    e.op_gemm_f32_conv3(src, fh, fw, Bm, nimg, H, W, cin, N, bias, resid, out.data_ptr() + MARGIN * 4)
    torch.cuda.synchronize()
    REACHED.add("f32_conv3")
    d = go.Desc(M=M, N=N, K=9 * cin, ldb=9 * cin, amode=go.A_CONV3x3, Hs=H, Ws=W, Cin=cin, Ho=H, Wo=W, ldc=N, ldr=N, out_mode=1)
    img = frame[:, :H, :W, :].to(torch.bfloat16).reshape(-1).to(DEV)       # the map itself: the oracle pads with zeros
    r = go.gemm(d, 1, img, Bm, bias_f=bias, resid_f=resid)
    return out, init, r


@pytest.mark.parametrize("nimg", [1, 2])
@pytest.mark.parametrize("H,W", [(12, 20), (24, 24), (5, 9)])
@pytest.mark.parametrize("cin", [64, 256])
def test_gemm_f32_conv3_exact(nimg, H, W, cin):
    """Exact family: the fp32 output is bit-equal.  The frame is larger than the map (fh > H, fw > W; at least one 16 x 8 box)."""
    fh, fw = max(H + 3, 8), max(W + 5, 16)
    out, init, r = conv3_f32_case(nimg, H, W, cin, 136 if cin == 64 else 64, fh, fw, "exact", nimg * H + W + cin, (H + cin) % 2 == 0)
    check_output(f"gemm_f32_conv3 {nimg}x{H}x{W}x{cin}", out, init, MARGIN, r, "exact", 9 * cin, False)


def test_gemm_f32_conv3_split3_is_fp32_grade():
    """The DPT / MiDaS use: an S3 frame of 64 fp32 channels (cin = 192) against W3 weights, compared with the fp64 convolution of the
    original fp32 values under the split3 bound."""
    import torch.nn.functional as F
    e = _engine()
    g = torch.Generator().manual_seed(1)
    nimg, H, W, C, N = 2, 12, 20, 64, 72
    fh, fw = H + 2, W + 4
    x = torch.randn(nimg, H, W, C, generator=g)
    w = torch.randn(N, 3, 3, C, generator=g)
    frame = torch.zeros(nimg, fh, fw, 3 * C, dtype=F64)
    frame[:, :H, :W, :] = go.s3_rows(x)
    src = frame.to(torch.bfloat16).reshape(-1).to(DEV)
    Bm = go.w3_rows(w.view(N, 9, C)).reshape(N, 27 * C).to(torch.bfloat16).reshape(-1).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    out = torch.full((nimg * H * W * N,), float("nan"), device=DEV)
    e.op_gemm_f32_conv3(src, fh, fw, Bm, nimg, H, W, 3 * C, N, bias, None, out)
    torch.cuda.synchronize()
    REACHED.add("f32_conv3")
    xd = x.to(F64).permute(0, 3, 1, 2).to(DEV)
    wd = w.to(F64).permute(0, 3, 1, 2).to(DEV)
    exact = (F.conv2d(xd, wd, padding=1) + bias.to(F64).view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    absdot = F.conv2d(xd.abs(), wd.abs(), padding=1).permute(0, 2, 3, 1)
    got = out.view(nimg, H, W, N).to(F64)
    ratio = ((got - exact).abs() / split_bound(absdot, 27 * C, bias.abs().to(F64))).max().item()
    print(f"\ngemm_f32_conv3 x3 {nimg}x{H}x{W}x3*{C}: worst err/bound {ratio:.3g}", end="")
    assert ratio <= 1.0


def test_zz_every_route_was_reached():
    """The suite above reached all four gemm() routes and both fp32 functions: a predicate change that silently empties a route
    fails here (run the whole file)."""
    assert REACHED == {WGMMA, WGMMA_CONV3, MMA, MMA_WIN, "f32", "f32_conv3"}, REACHED
