"""Exact restatement of the reference's sampling semantics (autoregressive/models/generate.py:17-74 with the CFG combine and the
cfg_interval rule of :89-131), and the seeded row catalogue the sampler tests run it on.

  * CFG and temperature in fp32, as the reference computes them on the GPU: ``u + (c - u) * s`` as separate sub, mul and add, then
    ``z * fp32(1 / fp32(T))`` — ATen's CUDA true-divide by a CPU scalar multiplies by the fp32 reciprocal (the CPU divides).
  * top-k by exact comparison of fp32 values: keep ``z >= `` the k-th largest value, k = min(max(top_k, 1), V); ties are kept and
    -0.0 == +0.0.
  * nucleus and soft-max in fp64.  A token is kept iff the probability mass of the tokens strictly above it is <= fp32(top_p).  The
    reference's fp32 cumsum is not exact, so tokens whose fp64 "mass above" lies within DELTA of top_p (the ambiguity band) may go
    either way; the reference also splits exact ties at the boundary in whatever order torch.sort left them (``band_ref``).
  * the draw: argmax(p / q) for Exp(1) noise q, or argmax(p) for greedy, lowest index among exact ties; the runner-up and the
    relative gap are returned so that a caller can tell a disagreement from a rounding-level near-tie.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch

# relative gap between the best and the second-best race score below which two fp32 evaluations may legitimately pick either
NEAR_TIE = 1e-5


def cfg_temperature(logits: torch.Tensor, B: int, cfg_scale: float, cfg_on: bool, temperature: float) -> torch.Tensor:
    """[b_eff, V] fp32 raw logits -> [B, V] fp32 rows the reference hands to top_k_top_p_filtering on the GPU."""
    x = logits.detach().to(torch.float32).cpu()
    if cfg_scale > 1.0:
        c, u = x[:B], x[B:2 * B]
        z = (u + (c - u) * torch.tensor(cfg_scale, dtype=torch.float32)) if cfg_on else c.clone()
    else:
        z = x[:B].clone()
    inv = np.float32(1.0) / np.float32(max(temperature, 1e-5))
    return z * torch.tensor(float(inv), dtype=torch.float32)


def delta_for(n: int) -> float:
    """Width of the nucleus ambiguity band for a row with n candidate tokens: the reference sums n fp32 probabilities one after the
    other (torch.cumsum), each add rounding by at most 2^-24 of the running sum (<= 1), and each soft-max term carries a few ulp of
    its own; (n + 8) * 2^-24 bounds both.  The fused kernel's fixed-point mass is exact to n * 2^-40 plus expf's 2 ulp per term, far
    inside the band."""
    return (n + 8) * 2.0 ** -24


@dataclass
class OracleOut:
    kept: torch.Tensor        # bool [R, V]: kept after top-k and nucleus (ties kept together, the kernel's rule)
    topk_kept: torch.Tensor   # bool [R, V]: kept after top-k only
    band: torch.Tensor        # bool [R, V]: nucleus decision within DELTA of top_p (either way is correct)
    band_ref: torch.Tensor    # bool [R, V]: band, plus tokens whose fate the reference leaves to torch.sort's order among ties
    probs: torch.Tensor       # fp64 [R, V]: soft-max over the kept set
    choice: torch.Tensor      # int64 [R]
    second: torch.Tensor      # int64 [R]   (-1: only one candidate)
    gap: torch.Tensor         # fp64 [R]: (s1 - s2) / s1 of the race scores (0 = exact tie, decided by the lowest index)


def oracle_sample(z: torch.Tensor, top_k: int, top_p: float, noise: Optional[torch.Tensor] = None,
                  sample_logits: bool = True) -> OracleOut:
    """z: fp32 [R, V] rows after CFG and temperature (cfg_temperature).  noise: [R, V] Exp(1) draws, or None for greedy."""
    z = z.detach().to(torch.float32).cpu()
    R, V = z.shape
    zd = z.double()
    if top_k > 0:
        k = min(max(top_k, 1), V)
        thr = torch.sort(z, dim=-1, descending=True).values[:, k - 1:k]
        tk = z >= thr
    else:
        tk = torch.ones_like(z, dtype=torch.bool)
    mx = torch.where(tk, zd, torch.full_like(zd, -float("inf"))).amax(-1, keepdim=True)
    e = torch.where(tk, torch.exp(zd - mx), torch.zeros_like(zd))
    p = e / e.sum(-1, keepdim=True)
    kept = tk.clone()
    band = torch.zeros_like(tk)
    band_ref = torch.zeros_like(tk)
    tp = float(np.float32(top_p))
    if top_p < 1.0:
        for r in range(R):
            pr = p[r]
            order = torch.sort(pr, descending=True, stable=True).indices
            ps = pr[order]
            # tie groups of equal probability in sorted order: strict mass above = exclusive cumsum at the group's first member
            csum = torch.cumsum(ps, 0)
            excl = csum - ps
            new_grp = torch.ones(V, dtype=torch.bool)
            new_grp[1:] = ps[1:] != ps[:-1]
            gid = torch.cumsum(new_grp.long(), 0) - 1
            first = torch.nonzero(new_grp).view(-1)
            last = torch.cat([first[1:] - 1, torch.tensor([V - 1])])
            strict = excl[first][gid]
            hi = (csum[last][gid]) - ps                     # the most the reference's cumsum before this token can be
            d = delta_for(int(tk[r].sum()))
            ks = strict <= tp
            b = (strict - tp).abs() <= d
            br = b | ((strict <= tp + d) & (hi > tp - d))
            kept[r, order] = ks & tk[r, order]
            band[r, order] = b & tk[r, order]
            band_ref[r, order] = br & tk[r, order]
        e = torch.where(kept, e, torch.zeros_like(e))
        p = e / e.sum(-1, keepdim=True)
    probs = p
    if sample_logits and noise is not None:
        score = probs / noise.detach().double().cpu()
    else:
        score = probs.clone()
    score = torch.where(kept & (probs > 0), score, torch.full_like(score, -1.0))
    choice = torch.empty(R, dtype=torch.int64)
    second = torch.empty(R, dtype=torch.int64)
    gap = torch.empty(R, dtype=torch.float64)
    idx = torch.arange(V)
    for r in range(R):
        s = score[r].numpy()
        o = np.lexsort((idx.numpy(), -s))              # by score descending, then index ascending
        choice[r] = int(o[0])
        if V > 1 and s[o[1]] >= 0:
            second[r] = int(o[1])
            gap[r] = float((s[o[0]] - s[o[1]]) / s[o[0]])
        else:
            second[r] = -1
            gap[r] = float("inf")
    return OracleOut(kept, tk, band, band_ref, probs, choice, second, gap)


def choice_ok(got: int, o: OracleOut, r: int) -> bool:
    """The kernel's draw for row r agrees with the oracle: exact, unless the oracle reports a rounding-level near-tie (then either of
    its top two); exact ties always go to the lowest index."""
    if got == int(o.choice[r]):
        return True
    g = float(o.gap[r])
    return 0.0 < g < NEAR_TIE and got == int(o.second[r])


# ------------------------------------------------------------------------------------------------------------------------------
# seeded row catalogue
# ------------------------------------------------------------------------------------------------------------------------------
def div_recip_pair(T: float = 0.7, lo: float = 3.0):
    """Two adjacent fp32 values x < y (y = nextafter(x)) that the reciprocal multiply z * fp32(1/T) maps to the SAME value while the
    true division z / T keeps them apart (or the other way round): top-k ties and greedy choices then depend on which one a
    sampler computes."""
    t = np.float32(T)
    inv = np.float32(1.0) / t
    x = np.arange(np.float32(lo).view(np.int32), np.float32(lo).view(np.int32) + (1 << 20), dtype=np.int32).view(np.float32)
    d, m = x / t, x * inv
    same_d, same_m = d[1:] == d[:-1], m[1:] == m[:-1]
    i = int(np.nonzero(same_d != same_m)[0][0])
    return float(x[i]), float(x[i + 1]), bool(same_m[i])


def _g(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def catalogue(V: int = 16384, seed: int = 0) -> Dict[str, torch.Tensor]:
    """name -> fp32 [R, V] rows (V a multiple of 4; the edge rows need V >= 8192)."""
    out: Dict[str, torch.Tensor] = {}
    g = _g(seed)
    out["normal"] = torch.randn(2, V, generator=g) * 2.0
    out["bf16"] = (torch.randn(2, V, generator=g) * 3.0).to(torch.bfloat16).float()
    c = (torch.randn(1, V, generator=g) * 3.0).to(torch.bfloat16).float()
    u = (c + torch.randn(1, V, generator=g) * 0.5).to(torch.bfloat16).float()
    out["bf16_cfg4"] = u + (c - u) * torch.tensor(4.0)        # the production tie structure after CFG
    r = torch.randn(1, V, generator=g)
    r[0, 777] = 1e4                                            # far outlier: the histogram's bin scale collapses
    out["outlier"] = r
    out["equal"] = torch.full((1, V), 0.5)
    r = torch.randn(2, V, generator=g) * 2.0
    r[0, torch.randperm(V, generator=g)[:1000]] = -float("inf")
    r[1, torch.randperm(V, generator=g)[:V - 384]] = -float("inf")   # fewer finite entries than top_k
    out["ninf"] = r
    r = torch.randn(1, V, generator=g)
    r[0, torch.randperm(V, generator=g)[:3000]] = 1.5          # ~900 above, so the tie block spans ranks ~900 .. ~3900
    out["tie3000"] = r
    r = -1.0 - torch.rand(1, V, generator=g)                   # negative body
    perm = torch.randperm(V, generator=g)
    r[0, perm[:100]] = 1.0 + torch.rand(100, generator=g)
    r[0, perm[100:1600]] = 0.0
    r[0, perm[1600:3100]] = -0.0
    out["pm0"] = r
    x, y, _ = div_recip_pair()
    r = torch.randn(1, V, generator=g)
    r[0, 10], r[0, 20] = x, y                                  # the row's two largest values, adjacent floats
    out["divrecip"] = r
    # 2200 distinct values above a 200-way exact tie (ranks 2201 .. 2400): the tie fits the boundary bin (<= 1024 candidates, exact
    # ranks), yet at top_k 2201 .. 2240 the kept list overflows (2400 > 2304 entries) after the ranks are known
    r = torch.randn(1, V, generator=g)
    order = torch.sort(r[0], descending=True).indices
    r[0, order[2200:2400]] = float(r[0, order[2200]])
    out["tie200"] = r
    # +-0 ties few enough for the exact-rank comparison: 1900 positive values, 100 x +0, 100 x -0, negative body
    r = -1.0 - torch.rand(1, V, generator=g)
    perm = torch.randperm(V, generator=g)
    r[0, perm[:1900]] = 1.0 + torch.rand(1900, generator=g)
    r[0, perm[1900:2000]] = 0.0
    r[0, perm[2000:2100]] = -0.0
    out["pm0_small"] = r
    return out


SMALL_V = (4, 12, 1000, 4100)


def small_v_rows(seed: int = 1) -> Dict[int, torch.Tensor]:
    g = _g(seed)
    return {V: torch.randn(2, V, generator=g) * 2.0 for V in SMALL_V}


# the (top_k, top_p) pairs and temperatures the reference fixture covers (temperatures where z / T == z * (1 / T) exactly)
FIXTURE_TEMPS = (1.0, 0.5, 2.0)
FIXTURE_PAIRS = ((0, 1.0), (1, 1.0), (100, 1.0), (2000, 1.0), (2241, 1.0), ("V-1", 1.0), ("V+5", 1.0), (-1, 0.9), (0, 0.9),
                 (0, 0.5), (2000, 0.9), (100, 0.5), (2000, 1e-6), (0, 0.0), (8000, 0.999))


def resolve_k(k, V: int) -> int:
    return {"V-1": V - 1, "V": V, "V+5": V + 5}.get(k, k) if isinstance(k, str) else int(k)


def fixture_configs():
    """(temperature, top_k, top_p): every pair at T = 1; the nucleus pairs (the only ones a power-of-two temperature can change)
    also at T = 0.5 and 2."""
    out = []
    for T in FIXTURE_TEMPS:
        for k, p in FIXTURE_PAIRS:
            if T == 1.0 or p < 1.0:
                out.append((T, k, p))
    return out


def fixture_rows():
    """name -> fp32 [R, V] rows of the reference fixture: the catalogue at V = 16384 plus the small vocabularies."""
    rows = dict(catalogue())
    for V, r in small_v_rows().items():
        rows[f"v{V}"] = r
    return rows


def probe_cols(z: torch.Tensor, seed: int = 5) -> torch.Tensor:
    """Columns whose probabilities the fixture stores for row z [V]: the 64 largest values and 64 seeded random columns."""
    V = z.numel()
    top = torch.sort(z, descending=True, stable=True).indices[:64]
    rnd = torch.randperm(V, generator=_g(seed))[:64]
    return torch.cat([top, rnd])
