"""fp64 reference of the dense GEMM front end (csrc/gemm.h): gemm() over a DenseP descriptor, and the split-bf16 ("x3") operand
format of csrc/split3.cuh that gemm_f32 / gemm_f32_conv3 consume.

Written from gemm.h's index arithmetic, not from the kernels:
  * A addressing: A_PLAIN row-major [M][lda]; A_CONV3x3 (3x3 / pad 1 / stride 1, optionally over the nearest-2x up-sampled view of
    the source); A_CONV3x3S2 (3x3 / stride 2 over the source padded (0, 1, 0, 1)); A_WIN (kh x kw window, stride ws, over an already
    padded source).  Row m = (b Ho + y) Wo + x, K index = tap Cin + c with tap = ky kw + kx (kw = 3 for the 3x3 modes).
  * the epilogue in DenseP's documented order, with every bf16 rounding point emulated exactly (round to nearest even from fp64):
      v = acc alpha (+ bias[n] | bias[m]) (+ bias_f[n]) (+ resid_f); v = r(v) (out_mode 0); act (GELU: r(gelu(v)), ReLU: max(v, 0));
      (v = r(v scale[n])); (v = r(v + resid)); store.
  * the output layouts: bf16 / fp32 [M][ldc] (+ z sC), fp32 NCHW C[(b N + n) Ho Wo + pix], and the window pixel map.
  * batch strides sA, sB, sC, sR in elements, 0 broadcasting.

Buffers are flat 1-D tensors holding the exact values of the device buffers (bf16 values widened to fp64); the functions return
the flat indices of C that the GEMM writes and the values it writes there, so a caller can check every other element untouched.
Everything runs in float64 on whatever device the buffers are on.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

A_PLAIN, A_CONV3x3, A_CONV3x3S2, A_WIN = 0, 1, 2, 3
ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF, ACT_RELU = 0, 1, 2, 3
F64 = torch.float64


@dataclass
class Desc:
    """gemm.h's DenseP without the pointers (the buffers are passed separately)."""
    M: int
    N: int
    K: int
    lda: int = 0
    ldb: int = 0
    sA: int = 0
    sB: int = 0
    sC: int = 0
    sR: int = 0
    amode: int = A_PLAIN
    Hs: int = 0
    Ws: int = 0
    Cin: int = 0
    Ho: int = 0
    Wo: int = 0
    ups: int = 0
    alpha: float = 1.0
    bias_along_m: int = 0
    act: int = ACT_NONE
    ldr: int = 0
    ldc: int = 0
    out_mode: int = 0
    kh: int = 0
    kw: int = 0
    ws: int = 0
    osy: int = 1
    osx: int = 1
    oay: int = 0
    oax: int = 0
    oH: int = 0
    oW: int = 0


def round_bf16(x: torch.Tensor) -> torch.Tensor:
    """Round fp64 values to the nearest bf16 (8 significant bits, ties to even, fp32's exponent range with subnormals), once."""
    x = x.to(F64)
    _, e = torch.frexp(x)                                   # |x| in [2^(e-1), 2^e)
    ulp = torch.ldexp(torch.ones_like(x), torch.clamp(e - 1, min=-126) - 7)
    return torch.round(x / ulp) * ulp                       # torch.round: half to even


def bf16_midpoint_distance(x: torch.Tensor) -> torch.Tensor:
    """Distance of fp64 x from the nearest point halfway between two adjacent bf16 values."""
    x = x.to(F64)
    _, e = torch.frexp(x)
    ulp = torch.ldexp(torch.ones_like(x), torch.clamp(e - 1, min=-126) - 7)
    q = x / ulp
    return (q - (torch.floor(q) + 0.5)).abs() * ulp


def bf16_cell(y: torch.Tensor):
    """(lo, hi): the interval of reals that round to the bf16 value y (ties ignored); at a power of two the half toward zero is
    half as wide."""
    y = y.to(F64)
    m, e = torch.frexp(y)
    ulp = torch.ldexp(torch.ones_like(y), torch.clamp(e - 1, min=-126) - 7)
    pow2 = (m.abs() == 0.5) & (e - 1 > -126)
    below = torch.where(pow2 & (y > 0), ulp / 4, ulp / 2)
    above = torch.where(pow2 & (y < 0), ulp / 4, ulp / 2)
    return y - below, y + above


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x * x * x)))


def gelu_erf(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def a_index(d: Desc, batch: int, device=None):
    """Flat index into the A buffer of element (z, m, k) of the implicit A operand, [batch][M][K] long, and a validity mask (False
    where the convolution reads padding, which contributes zero)."""
    z = torch.arange(batch, device=device).view(-1, 1, 1)
    m = torch.arange(d.M, device=device).view(1, -1, 1)
    k = torch.arange(d.K, device=device).view(1, 1, -1)
    if d.amode == A_PLAIN:
        idx = z * d.sA + m * d.lda + k
        return idx, torch.ones_like(idx, dtype=torch.bool)
    hw = d.Ho * d.Wo
    b, r = m // hw, m % hw
    y, x = r // d.Wo, r % d.Wo
    tap, c = k // d.Cin, k % d.Cin
    kw = d.kw if d.amode == A_WIN else 3
    ky, kx = tap // kw, tap % kw
    if d.amode == A_WIN:
        yy, xx = d.ws * y + ky, d.ws * x + kx
        ok = torch.ones_like(yy + xx + z, dtype=torch.bool)
        sy, sx = yy, xx
    else:
        if d.amode == A_CONV3x3:
            yy, xx = y + ky - 1, x + kx - 1
        else:
            yy, xx = 2 * y + ky, 2 * x + kx
        Hv, Wv = d.Hs << d.ups, d.Ws << d.ups
        ok = (yy >= 0) & (yy < Hv) & (xx >= 0) & (xx < Wv)
        sy, sx = torch.clamp(yy, min=0) >> d.ups, torch.clamp(xx, min=0) >> d.ups
        sy, sx = torch.clamp(sy, max=d.Hs - 1), torch.clamp(sx, max=d.Ws - 1)
    idx = z * d.sA + ((b * d.Hs + sy) * d.Ws + sx) * d.Cin + c
    idx, ok = torch.broadcast_tensors(idx, ok)
    return idx, ok


def operand_a(d: Desc, batch: int, abuf: torch.Tensor) -> torch.Tensor:
    """The implicit A operand [batch][M][K] in fp64."""
    idx, ok = a_index(d, batch, abuf.device)
    return torch.where(ok, abuf.to(F64)[idx], torch.zeros((), dtype=F64, device=abuf.device))


def operand_b(d: Desc, batch: int, bbuf: torch.Tensor) -> torch.Tensor:
    """B [batch][N][K] in fp64 (row-major [N][ldb] + z sB)."""
    dev = bbuf.device
    z = torch.arange(batch, device=dev).view(-1, 1, 1)
    n = torch.arange(d.N, device=dev).view(1, -1, 1)
    k = torch.arange(d.K, device=dev).view(1, 1, -1)
    return bbuf.to(F64)[z * d.sB + n * d.ldb + k]


def c_index(d: Desc, batch: int, device=None) -> torch.Tensor:
    """Flat index into C of output (z, m, n), [batch][M][N] long."""
    z = torch.arange(batch, device=device).view(-1, 1, 1)
    m = torch.arange(d.M, device=device).view(1, -1, 1)
    n = torch.arange(d.N, device=device).view(1, 1, -1)
    if d.amode == A_WIN:
        hw = d.Ho * d.Wo
        b, r = m // hw, m % hw
        oy, ox = r // d.Wo, r % d.Wo
        pix = (b * d.oH + d.osy * oy + d.oay) * d.oW + d.osx * ox + d.oax
        return (pix * d.ldc + n + 0 * z).expand(batch, d.M, d.N)
    if d.out_mode == 2:
        hw = d.Ho * d.Wo
        b, pix = m // hw, m % hw
        return ((b * d.N + n) * hw + pix + 0 * z).expand(batch, d.M, d.N)
    return (z * d.sC + m * d.ldc + n).expand(batch, d.M, d.N)


@dataclass
class Result:
    idx: torch.Tensor         # flat C indices written, [batch][M][N]
    val: torch.Tensor         # the values written there (fp64; bf16 values when out_mode 0)
    pre: torch.Tensor         # the epilogue value before its first rounding: acc alpha + biases (+ resid_f)
    absdot: torch.Tensor      # |alpha| sum_k |a_k b_k|, for accumulation-error bounds
    gelu_in: Optional[torch.Tensor] = None     # the GELU input (after the first rounding), when act is a GELU
    gelu_out: Optional[torch.Tensor] = None    # the exact GELU of gelu_in, before its rounding


def epilogue_tail(d: Desc, batch: int, g: torch.Tensor, bufs: dict) -> torch.Tensor:
    """LayerScale and bf16 residual after the activation (bufs: "scale", "resid" or None); monotone non-decreasing in g when the
    scale is positive."""
    dev = g.device
    n = torch.arange(d.N, device=dev)
    v = g
    if bufs.get("scale") is not None:
        v = round_bf16(v * bufs["scale"].to(F64)[n].view(1, 1, -1))
    if bufs.get("resid") is not None:
        z = torch.arange(batch, device=dev).view(-1, 1, 1)
        m = torch.arange(d.M, device=dev).view(1, -1, 1)
        v = round_bf16(v + bufs["resid"].to(F64)[z * d.sR + m * d.ldr + n.view(1, 1, -1)])
    return v


def gemm(d: Desc, batch: int, A: torch.Tensor, B: torch.Tensor, bias=None, bias_f=None, resid_f=None, scale=None,
         resid=None) -> Result:
    """gemm() of gemm.h over flat buffers (fp64 values of the device buffers).  alpha == 0 means 1."""
    a = operand_a(d, batch, A)
    b = operand_b(d, batch, B)
    dev = a.device
    alpha = 1.0 if d.alpha == 0 else float(d.alpha)
    acc = torch.matmul(a, b.transpose(1, 2))
    absdot = abs(alpha) * torch.matmul(a.abs(), b.abs().transpose(1, 2))
    z = torch.arange(batch, device=dev).view(-1, 1, 1)
    m = torch.arange(d.M, device=dev).view(1, -1, 1)
    n = torch.arange(d.N, device=dev).view(1, 1, -1)
    v = acc * alpha
    if bias is not None:
        v = v + bias.to(F64)[m if d.bias_along_m else n]
    if bias_f is not None:
        v = v + bias_f.to(F64)[n]
    if resid_f is not None:
        v = v + resid_f.to(F64)[z * d.sR + m * d.ldr + n]
    pre = v
    if d.out_mode == 0:
        v = round_bf16(v)
    res = Result(idx=c_index(d, batch, dev), val=v, pre=pre, absdot=absdot)
    bufs = dict(scale=scale, resid=resid)
    if d.act in (ACT_GELU_TANH, ACT_GELU_ERF):
        gx = (gelu_tanh if d.act == ACT_GELU_TANH else gelu_erf)(v)
        res.gelu_in = v
        res.val = epilogue_tail(d, batch, round_bf16(gx), bufs)
        res.gelu_out = gx
        return res
    if d.act == ACT_RELU:
        v = torch.clamp(v, min=0.0)
    res.val = epilogue_tail(d, batch, v, bufs)
    return res


# ---- split-bf16 ("x3") operands, csrc/split3.cuh ----
def x3_split(x: torch.Tensor):
    """fp32 values -> (hi, lo) as fp64: hi = bf16(x), lo = bf16(x - hi), x - hi exact in fp32."""
    x = x.to(torch.float32).to(F64)
    hi = round_bf16(x)
    lo = round_bf16(x - hi)
    return hi, lo


def s3_rows(x: torch.Tensor) -> torch.Tensor:
    """fp32 [..., C] -> S3 [..., 3C] = [hi | lo | hi] (the A side)."""
    hi, lo = x3_split(x)
    return torch.cat([hi, lo, hi], dim=-1)


def w3_rows(w: torch.Tensor) -> torch.Tensor:
    """fp32 [N, taps, C] -> W3 [N, taps, 3C] = [hi | hi | lo] per tap (the B side)."""
    hi, lo = x3_split(w)
    return torch.cat([hi, hi, lo], dim=-1)
