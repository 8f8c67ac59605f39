"""GPU conformance of the KV-cache attention kernels (csrc/attention.cuh) against the fp64 masked SDPA of oracle/attn_oracle.py,
through car_op_attn_decode / car_op_attn_prefill, which make the same launches as the model chains:
  * attn_decode_kernel<T> (decode step, keys split over nsplit CTAs, last CTA combines): fp32 and bf16;
  * attn_prefill_kernel<T> (scalar prefill, one warp per query row): fp32 and bf16;
  * attn_prefill_mma_kernel (bf16 tensor-core prefill, 64-row query tiles, probabilities rounded to bf16).

Every call also checks that nothing outside the live data is read or written: cache rows past the live range (> pos for decode,
>= Tq for prefill) are NaN in every (b, h) slab, and the output sits inside a NaN guard margin that must stay untouched, while every
output must be finite.

Tolerances are derived in `fp32_bound` and `mma_bound`, not fitted to a run.  Each test prints the largest error it saw in units of
its bound (`err/bound`) and, for the fp32 kernels, relative to max|V| (run pytest with -s to see them).
"""
import math

import pytest
import torch

from oracle.attn_oracle import masked_sdpa

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24          # fp32 unit roundoff
UB = 2.0 ** -8          # bf16 unit roundoff (8-bit significand)
LAM = 8.0               # probabilistic rounding-error bound parameter (see fp32_bound)
NAN = float("nan")
MARGIN = 4096           # guard elements on each side of an output


def fp32_bound(vmax, amax, n, rescales=None):
    """Bound on |y - y*| for one output of the fp32 arithmetic of the kernels (the decode kernel, the scalar prefill, and the fp32
    part of the tensor-core prefill) against the fp64 oracle y* on the same inputs (bf16 inputs are exact in fp32).

    The kernels compute y = sum_j p~_j v_j / sum_j p~_j over the visible keys, with p~_j = p_j (1 + e_j).  With the weights
    w_j = p_j / sum p, y - y* = sum_j w_j (e_j - e_bar) (v_j - c) / (1 + e_bar) for any c, so |y - y*| <= 2 vmax mean_w|e| (1 + 2 max|e|)
    where vmax = max |v|.  The relative error e_j of a probability collects:
      * its score: the fp32 dot product of 64 terms is within gamma_64 sum_e |q_e k_e| (64 u of it, u = 2^-24) of the exact one, and
        the scale 1/8 is exact, so s_j is off by at most 64 u amax with amax = max_j sum_e |q_e k_je| / 8; p_j moves by that much
        relatively (the error of the running maximum is common to all keys and cancels);
      * its exponentials: p~_j is the product of __expf(s_j - m) and of every rescale factor __expf(m_old - m_new) applied after it
        (running-maximum increases within a warp slot, the merge of the CTA's slots, the combine of the splits).  __expf is within
        2 + 1.173 |x| ulp (CUDA C Programming Guide, intrinsic functions; 1 ulp <= 2u relative), and every product adds u.  The
        |x| parts telescope to |s_j - max|, whose p-weighted mean is at most the entropy of p, <= ln n.  The number of factors is
        `rescales` + 3; with scores in random order the running maximum increases about ln n times (harmonic number), and
        2 ln n + 3 is taken.  Inputs that raise the maximum at every key (a score ramp) pass rescales = n.
    Then the two fp32 sums (per column, and the normaliser) of at most n terms add at most lambda sqrt(n) u of sum p~ |v| <= vmax sum p~
    each — the probabilistic bound of Higham and Mary (SIAM J. Sci. Comput. 41(5), 2019), which fails with probability below
    2 exp(-lambda^2 / 2) ~ 1e-14 at lambda = 8, where the worst-case n u would say nothing at n = 4216 — and the division adds u |y|.
    """
    ln_n = math.log(max(n, 2))
    f = (2 * ln_n + 3 if rescales is None else rescales) + 3
    mean_e = 64 * U * amax + U * (5 * f + 2.35 * ln_n)
    return vmax * (2 * mean_e * (1 + 4 * mean_e) + 2 * LAM * math.sqrt(n) * U + U)


def mma_bound(vmax, vrange, amax, n, ref):
    """Bound on |y - y*| for attn_prefill_mma_kernel.  Each probability is rounded to bf16 (relative error <= 2^-8) before both the
    value product and the normaliser, so with c the mid-range of the column the rounding moves y by at most
    sum_j w_j |d_j - d_bar| |v_j - c| / (1 - 2^-8) <= 2^-8 vrange / (1 - 2^-8), vrange the column's value range.  The tile-wise rounding
    (each 64-key tile is rounded against the running maximum of its time, then rescaled in fp32) keeps |d_j| <= 2^-8 + O(u).  Added:
    the fp32 errors of the scores and exponentials as in fp32_bound (on the range rather than 2 vmax), the tensor-core fp32
    accumulation of n products taken at its worst case (2u per addition, which covers truncating adders), and the final rounding to
    bf16 (2^-8 |y|)."""
    ln_n = math.log(max(n, 2))
    e32 = 64 * U * amax + U * (5 * (2 * ln_n + 6) + 2.35 * ln_n)
    y32 = vrange * (UB + e32) / (1 - UB) + 2 * n * 2 * U * vmax
    return y32 + UB * (ref.abs() + y32)


def _stats(q, k, v, n):
    """Per (b, h) [B, H, 1, 1]: vmax = max |v|, amax = max_j sum_e |q_e k_je| / 8 over the live rows; vrange per column [B, H, 1, 64]."""
    kl, vl = k[:, :, :n].double(), v[:, :, :n].double()
    vmax = vl.abs().amax(dim=(2, 3), keepdim=True)
    amax = ((q.double().abs() @ kl.abs().transpose(-1, -2)) / 8).amax(dim=(2, 3), keepdim=True)
    vrange = (vl.amax(dim=2, keepdim=True) - vl.amin(dim=2, keepdim=True))
    return vmax, amax, vrange


def _guarded(shape, dt):
    numel = math.prod(shape)
    buf = torch.full((2 * MARGIN + numel,), NAN, dtype=dt, device=DEV)
    return buf[MARGIN:MARGIN + numel].view(shape), buf


def _guard_intact(buf, what):
    assert bool(torch.isnan(buf[:MARGIN]).all()) and bool(torch.isnan(buf[-MARGIN:]).all()), f"{what}: write outside the output"


def _check(what, dt, got, ref, bound, stats_out):
    """got, ref fp64 of the same shape.  fp32: |got - ref| <= bound.  bf16 outputs of fp32 arithmetic (bound is the fp32 bound): got is
    the bf16 rounding of a value within `bound` of ref, i.e. lies in [bf16(ref - bound), bf16(ref + bound)] (rounding is monotone) —
    equal to bf16(ref) except within fp32 slack of a rounding boundary."""
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    err = (got - ref).abs()
    if dt == torch.float32:
        ok = err <= bound
    else:
        lo = (ref - bound).float().to(torch.bfloat16).double()
        hi = (ref + bound).float().to(torch.bfloat16).double()
        ok = (got >= lo) & (got <= hi)
    if not bool(ok.all()):
        i = (~ok).nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} outputs out of bounds, first at {i}: got {float(got[tuple(i)])!r}, "
                             f"fp64 {float(ref[tuple(i)])!r}, bound {float(bound.expand_as(ref)[tuple(i)]):.3e}")
    if dt != torch.float32:           # the bracket's reach: bound plus half a bf16 ulp
        bound = bound + UB * (ref.abs() + bound)
    stats_out.append(float((err / bound.expand_as(err)).max()))


# ---------------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------------
MASKS = ("none", "ones", "zeros", "leftpad", "random", "values", "selfzero", "wide")


def _mask(kind, B, Tpre, seed):
    """int32 [B, >= Tpre] on the device, or None.  The oracle uses its first Tpre columns."""
    if kind == "none" or Tpre == 0:
        return None
    g = torch.Generator().manual_seed(seed)
    if kind == "ones":
        m = torch.ones(B, Tpre, dtype=torch.int32)
    elif kind == "zeros":
        m = torch.zeros(B, Tpre, dtype=torch.int32)
    elif kind == "leftpad":                               # valid caption tokens at the end, as oracle/inputs.text_inputs makes them
        from oracle.inputs import text_inputs
        m = text_inputs(Tpre, 8, B, seed, min_valid=1)[1].to(torch.int32)
    elif kind == "random":                                # different per batch row
        m = (torch.rand(B, Tpre, generator=g) < torch.rand(B, 1, generator=g)).to(torch.int32)
    elif kind == "values":                                # any non-zero value attends
        m = (torch.rand(B, Tpre, generator=g) < 0.6).to(torch.int32) * \
            torch.tensor([1, 2, -1, 7, 1 << 30], dtype=torch.int32)[torch.randint(0, 5, (B, Tpre), generator=g)]
    elif kind == "selfzero":                              # zero at every even column: those text rows see only earlier odd columns and themselves
        m = (torch.arange(Tpre) % 2).to(torch.int32).repeat(B, 1)
        m[B - 1] = 0
    elif kind == "wide":                                  # mask_ld > Tpre: the columns >= Tpre must be ignored
        m = torch.cat([(torch.rand(B, Tpre, generator=g) < 0.5).to(torch.int32), torch.zeros(B, 5, dtype=torch.int32)], 1)
    else:
        raise ValueError(kind)
    return m.to(DEV)


def _oracle_mask(m, Tpre):
    return None if m is None else m[:, :Tpre]


def _qkv(pattern, B, H, R, S, n, dt, seed):
    """q [B, H, R, 64], k, v [B, H, S, 64] in dt; cache rows >= n are NaN.  Score patterns (s = q.k / 8):
    random ~ N(0, 1); uniform ~ N(0, 0.02^2); peaked ~ N(0, 23^2), |s| up to ~80 (large jumps of the running maximum);
    ramp: s_j ~ 80 j / (n - 1), increasing with the key index, so the maximum rises at every key (the rescale at every step)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)      # noqa: E731
    v = rn(B, H, S, 64)
    if pattern == "ramp":
        d = rn(B, H, 1, 64)
        d = d / d.norm(dim=-1, keepdim=True)
        q = d * 8 + 0.05 * rn(B, H, R, 64)
        t = torch.arange(S, device=DEV, dtype=torch.float32) / max(n - 1, 1) * 80
        k = d * t[:, None] + 0.05 * rn(B, H, S, 64)
    else:
        sc = {"random": 1.0, "uniform": 0.02 ** 0.5, "peaked": 23 ** 0.5}[pattern]
        q, k = rn(B, H, R, 64) * sc, rn(B, H, S, 64) * sc
    k[:, :, n:] = NAN
    v[:, :, n:] = NAN
    return q.to(dt), k.to(dt).contiguous(), v.to(dt).contiguous()


def _prod_nsplit(bh):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min(16, (4 * sms + bh - 1) // bh))


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------------------
def _decode(dt, B, H, S, n, Tpre, nsplit, mask_kind, pattern, seed, part, tickets, stats, rescales=None, qkv=None):
    from controlar_b200 import engine
    q, k, v = qkv if qkv is not None else _qkv(pattern, B, H, 1, S, n, dt, seed)
    m = _mask(mask_kind, B, Tpre, seed)
    out, buf = _guarded((B, H * 64), dt)
    what = f"decode {dt} B={B} H={H} S={S} n={n} Tpre={Tpre} nsplit={nsplit} mask={mask_kind} {pattern}"
    engine.op_attn_decode(q.reshape(B, H * 64), k, v, n - 1, Tpre, emb_mask=m, nsplit=nsplit, part=part, tickets=tickets, out=out)
    _guard_intact(buf, what)
    assert not bool(tickets.any()), f"{what}: tickets not reset by the combining CTA"
    ref = masked_sdpa(q, k[:, :, :n], v[:, :, :n], [n - 1], _oracle_mask(m, Tpre))[:, :, 0]
    vmax, amax, _ = _stats(q, k, v, n)
    bound = fp32_bound(vmax[:, :, 0], amax[:, :, 0], n, rescales)
    got = out.view(B, H, 64).double()
    _check(what, dt, got, ref, bound, stats)
    return out, float(((got - ref).abs() / vmax[:, :, 0]).max())


def _report(name, stats, rel=None):
    line = f"[attn] {name}: max err/bound {max(stats):.3g} over {len(stats)} calls"
    if rel:
        line += f", max err/max|V| {max(rel):.3g}"
    print(line)


def _split_edges(n_split, Tpre, S):
    """n = pos + 1 at and around the chunk boundaries of n_split splits (chunk = ceil(n / nsplit) rounded up to 8)."""
    out = set()
    for c in (8, 16, 40):
        for e in (c * n_split - 1, c * n_split, c * n_split + 1, c * (n_split - 1) + 1, c + 1):
            if Tpre < e <= S:
                out.add(e)
    return out


@pytest.mark.parametrize("Tpre", [1, 120, 256])
@pytest.mark.parametrize("nsplit", [1, 2, 3, 7, 16, 0])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_decode_vs_oracle(dt, nsplit, Tpre):
    """n = pos + 1 at 2, 7, 8, 9 (Tpre = 1), Tpre + 1, the chunk boundaries of this nsplit (trailing splits empty for small n) and S
    (full cache), under every mask kind; one part / tickets pair serves every call (the combining CTA must leave tickets zero)."""
    B, H = 2, 3
    S = Tpre + 330
    ns_eff = nsplit or _prod_nsplit(B * H)
    ns = {Tpre + 1, S} | _split_edges(ns_eff, Tpre, S)
    if Tpre == 1:
        ns |= {2, 7, 8, 9}
    part = torch.full((B * H * 16 * 68,), NAN, dtype=torch.float32, device=DEV)
    tickets = torch.zeros(B * H, dtype=torch.int32, device=DEV)
    stats, rel = [], []
    for i, n in enumerate(sorted(ns)):
        for j, mk in enumerate(MASKS):
            rel.append(_decode(dt, B, H, S, n, Tpre, nsplit, mk, "random", 1000 * i + j, part, tickets, stats)[1])
    _report(f"decode {dt} nsplit={nsplit} Tpre={Tpre}", stats, rel)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("nsplit", [1, 3, 16, 0])
def test_decode_long_context(dt, nsplit):
    """S = 120 + 4096 (a 64 x 64 token grid after a 120-token caption), pos up to the last slot."""
    B, H, Tpre, S = 2, 2, 120, 120 + 4096
    part = torch.empty(B * H * 16 * 68, dtype=torch.float32, device=DEV)
    tickets = torch.zeros(B * H, dtype=torch.int32, device=DEV)
    stats, rel = [], []
    for n in (121, 2049, 4000, S):
        for mk, pat in (("leftpad", "random"), ("random", "peaked"), ("none", "uniform")):
            rel.append(_decode(dt, B, H, S, n, Tpre, nsplit, mk, pat, n + len(mk), part, tickets, stats)[1])
    _report(f"decode long {dt} nsplit={nsplit}", stats, rel)


@pytest.mark.parametrize("BH", [(1, 1), (4, 5), (9, 16), (32, 20)], ids=lambda x: f"{x[0]}x{x[1]}")
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_decode_batch_heads(dt, BH):
    """B*H from one row to 640 (32 images x 20 heads); 9 x 16 = a CFG batch above 8, which the persistent kernel declines."""
    B, H = BH
    Tpre, S = 120, 264
    part = torch.empty(B * H * 16 * 68, dtype=torch.float32, device=DEV)
    tickets = torch.zeros(B * H, dtype=torch.int32, device=DEV)
    stats = []
    for nsplit in (0, 3):
        for n in (121, 200, S):
            _decode(dt, B, H, S, n, Tpre, nsplit, "random", "random", B * 7 + n, part, tickets, stats)
    _report(f"decode {dt} B={B} H={H}", stats)


@pytest.mark.parametrize("pattern", ["uniform", "peaked", "ramp"])
@pytest.mark.parametrize("nsplit", [1, 3, 16])
@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_decode_score_shapes(dt, nsplit, pattern):
    """Near-uniform scores; peaked scores with |s| up to ~80 (the online maximum jumps, most probabilities underflow); a ramp that
    raises the maximum at every key (a rescale on every step of every slot)."""
    B, H, Tpre, S = 2, 2, 120, 1000
    part = torch.empty(B * H * 16 * 68, dtype=torch.float32, device=DEV)
    tickets = torch.zeros(B * H, dtype=torch.int32, device=DEV)
    stats, rel = [], []
    for n in (130, 300, 1000):
        rel.append(_decode(dt, B, H, S, n, Tpre, nsplit, "leftpad", pattern, n, part, tickets, stats,
                           rescales=n if pattern == "ramp" else None)[1])
    _report(f"decode {dt} nsplit={nsplit} {pattern}", stats, rel)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_decode_equal_maxima_in_different_splits(dt):
    """Two keys with the same, dominant score (identical k rows, different v rows) in different splits, in the same split but different
    warp slots, and in the same slot: the combine must weigh them equally (the output is then close to the mean of their v rows)."""
    B, H, Tpre, S, n = 1, 2, 8, 256, 256
    part = torch.empty(B * H * 16 * 68, dtype=torch.float32, device=DEV)
    tickets = torch.zeros(B * H, dtype=torch.int32, device=DEV)
    stats = []
    for nsplit, (j1, j2) in ((4, (10, 200)), (4, (10, 75)), (2, (10, 11)), (1, (10, 26)), (16, (20, 250))):
        q, k, v = _qkv("random", B, H, 1, S, n, torch.float32, j1 * 31 + j2)
        d = q[:, :, 0] / q[:, :, 0].norm(dim=-1, keepdim=True)
        k[:, :, j1] = k[:, :, j2] = d * (12 * 8 / q[:, :, 0].norm(dim=-1, keepdim=True))       # s = 12 against ~N(0, 1) elsewhere
        out, _ = _decode(dt, B, H, S, n, Tpre, nsplit, "ones", "random", 0, part, tickets, stats,
                         qkv=(q.to(dt), k.to(dt), v.to(dt)))
        mean = (v[:, :, j1] + v[:, :, j2]).to(dt).double() / 2
        assert float((out.view(B, H, 64).double() - mean).abs().max()) < 0.05 * float(v[:, :, :n].abs().max())
    _report(f"decode {dt} equal maxima", stats)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_decode_split_bookkeeping_is_deterministic(dt):
    """The last CTA combines the partials in index order: repeated calls on the same part / tickets are bit-identical, tickets end
    zero, and nsplit = 0 is the production choice (car_state_create's formula) bit for bit."""
    from controlar_b200 import engine
    B, H, Tpre, S, n = 3, 4, 120, 700, 650
    q, k, v = _qkv("random", B, H, 1, S, n, dt, 77)
    q = q.reshape(B, H * 64)
    m = _mask("leftpad", B, Tpre, 77)
    part = torch.empty(B * H * 16 * 68, dtype=torch.float32, device=DEV)
    tickets = torch.zeros(B * H, dtype=torch.int32, device=DEV)
    for nsplit in (2, 7, 16):
        outs = [engine.op_attn_decode(q, k, v, n - 1, Tpre, m, nsplit, part, tickets).clone() for _ in range(3)]
        assert not bool(tickets.any())
        assert all(torch.equal(o, outs[0]) for o in outs[1:]), f"nsplit={nsplit}: repeated calls differ"
    prod = engine.op_attn_decode(q, k, v, n - 1, Tpre, m, 0, part, tickets)
    assert torch.equal(prod, engine.op_attn_decode(q, k, v, n - 1, Tpre, m, _prod_nsplit(B * H), part, tickets))


def test_decode_rejects_pos_outside_cache():
    """pos must be an image position inside the cache: the decode kernel relies on the key at pos being visible."""
    from controlar_b200 import engine
    B, H, Tpre, S = 1, 1, 120, 200
    q, k, v = _qkv("random", B, H, 1, S, S, torch.float32, 0)
    for pos in (Tpre - 1, S, -1):
        with pytest.raises(RuntimeError, match="pos"):
            engine.op_attn_decode(q.reshape(B, 64), k, v, pos, Tpre)


# ---------------------------------------------------------------------------------------------------------------------------------
# prefill
# ---------------------------------------------------------------------------------------------------------------------------------
IMPLS = {"scalar-fp32": (0, torch.float32), "scalar-bf16": (0, torch.bfloat16), "mma-bf16": (1, torch.bfloat16)}
TQS = [1, 15, 16, 17, 63, 64, 65, 120, 127, 128, 129, 200, 255, 256]


def _prefill(impl_name, B, H, S, Tq, Tpre, mask_kind, pattern, seed, stats, rel=None, rescales=None, qkv=None):
    from controlar_b200 import engine
    impl, dt = IMPLS[impl_name]
    q, k, v = qkv if qkv is not None else _qkv(pattern, B, H, Tq, S, Tq, dt, seed)
    m = _mask(mask_kind, B, Tpre, seed)
    out, buf = _guarded((B * Tq, H * 64), dt)
    what = f"prefill {impl_name} B={B} H={H} S={S} Tq={Tq} Tpre={Tpre} mask={mask_kind} {pattern}"
    q_rows = q.permute(0, 2, 1, 3).reshape(B * Tq, H * 64).contiguous()
    engine.op_attn_prefill(q_rows, k, v, Tq, Tpre, emb_mask=m, impl=impl, out=out)
    _guard_intact(buf, what)
    ref = masked_sdpa(q, k[:, :, :Tq], v[:, :, :Tq], range(Tq), _oracle_mask(m, Tpre))
    got = out.view(B, Tq, H, 64).permute(0, 2, 1, 3).double()
    vmax, amax, vrange = _stats(q, k, v, Tq)
    if impl == 1:
        assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
        bound = mma_bound(vmax, vrange, amax, Tq, ref)
        err = (got - ref).abs()
        bad = err > bound
        assert not bool(bad.any()), f"{what}: {int(bad.sum())} outputs out of bounds, worst err/bound {float((err / bound).max()):.3g}"
        stats.append(float((err / bound).max()))
    else:
        _check(what, dt, got, ref, fp32_bound(vmax, amax, Tq, rescales), stats)
        if rel is not None:
            rel.append(float(((got - ref).abs() / vmax).max()))
    return got, ref


@pytest.mark.parametrize("Tq", TQS)
@pytest.mark.parametrize("impl", list(IMPLS))
def test_prefill_vs_oracle(impl, Tq):
    """Every mask kind (including a zero at the query's own column, which only the forced diagonal keeps visible), with the text block
    the whole prefix (Tpre = Tq, as the product runs it) and a part of it; S > Tq with NaN past Tq."""
    B, H, S = 2, 3, Tq + 24
    stats, rel = [], []
    for Tpre in sorted({Tq, Tq // 2}):
        for j, mk in enumerate(MASKS):
            _prefill(impl, B, H, S, Tq, Tpre, mk, "random", Tq * 100 + Tpre * 10 + j, stats, rel)
    _report(f"prefill {impl} Tq={Tq}", stats, rel)


@pytest.mark.parametrize("impl", list(IMPLS))
def test_prefill_all_text_masked_rows_see_only_themselves(impl):
    """emb_mask all zero over the whole prefix: each row attends only its own key (the forced diagonal), so the output is that row's
    value vector, exactly."""
    B, H, Tq = 2, 2, 130
    got, ref = _prefill(impl, B, H, Tq + 8, Tq, Tq, "zeros", "random", 3, [])
    assert torch.equal(got, ref)


@pytest.mark.parametrize("BH", [(1, 1), (5, 4), (16, 2)], ids=lambda x: f"{x[0]}x{x[1]}")
@pytest.mark.parametrize("impl", list(IMPLS))
def test_prefill_batch_heads(impl, BH):
    B, H = BH
    stats = []
    for Tq in (120, 129):
        _prefill(impl, B, H, Tq + 40, Tq, Tq, "leftpad", "random", Tq + B, stats)
    _report(f"prefill {impl} B={B} H={H}", stats)


@pytest.mark.parametrize("pattern", ["uniform", "peaked", "ramp"])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_prefill_score_shapes(impl, pattern):
    stats, rel = [], []
    for Tq in (65, 200, 256):
        _prefill(impl, 2, 2, Tq + 8, Tq, Tq, "leftpad", pattern, Tq, stats, rel, rescales=Tq if pattern == "ramp" else None)
    _report(f"prefill {impl} {pattern}", stats, rel)


@pytest.mark.parametrize("pattern", ["random", "peaked"])
def test_prefill_scalar_vs_mma_gap(pattern):
    """The two bf16 prefill kernels on the same inputs: their gap is what the mma path's bf16 probabilities cost.  Printed in units of
    2^-8 of the column value range; bounded by the sum of the two kernels' own bounds."""
    from controlar_b200 import engine
    gaps = []
    for Tq in (120, 256):
        B, H, S = 2, 3, Tq + 8
        q, k, v = _qkv(pattern, B, H, Tq, S, Tq, torch.bfloat16, Tq + 5)
        m = _mask("leftpad", B, Tq, Tq)
        q_rows = q.permute(0, 2, 1, 3).reshape(B * Tq, H * 64).contiguous()
        sc = engine.op_attn_prefill(q_rows, k, v, Tq, Tq, m, impl=0).view(B, Tq, H, 64).permute(0, 2, 1, 3).double()
        mm = engine.op_attn_prefill(q_rows, k, v, Tq, Tq, m, impl=1).view(B, Tq, H, 64).permute(0, 2, 1, 3).double()
        ref = masked_sdpa(q, k[:, :, :Tq], v[:, :, :Tq], range(Tq), m)
        vmax, amax, vrange = _stats(q, k, v, Tq)
        b_sc = fp32_bound(vmax, amax, Tq) + UB * (ref.abs() + fp32_bound(vmax, amax, Tq))
        gap = (sc - mm).abs()
        assert bool((gap <= mma_bound(vmax, vrange, amax, Tq, ref) + b_sc).all())
        gaps.append(float((gap / (UB * vrange)).max()))
        print(f"[attn] scalar vs mma bf16 {pattern} Tq={Tq}: max gap {float(gap.max()):.3e} = {gaps[-1]:.3g} x 2^-8 of the column range, "
              f"mean {float(gap.mean()):.3e}")
    assert max(gaps) > 0
