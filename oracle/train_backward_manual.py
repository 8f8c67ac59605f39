"""TEST INFRASTRUCTURE — the hand-derived backward of the teacher-forced training forward (SURVEY.md §8 row f1), written out
op by op in the decomposition `car_train_backward` (controlar_b200/csrc/car_train.cu, train_bwd.cuh) uses: layer-wise recompute
from the saved fp32 residual stream, bf16 gradients wherever autograd under bf16 autocast produces bf16 ones (every nn.Linear
operand / result, SDPA, GELU / SiLU), fp32 on the residual stream, RMSNorm and the loss.  Never shipped or called by the product.

It restates autograd's result for `oracle/train_oracle.py::TrainOracle.forward` (itself pinned against gradients the reference
produced, tests/test_train_oracle_golden.py); tests/test_train_backward_cpu.py checks the two against each other, which
validates the formulas before they are transcribed to CUDA, and the GPU test compares the CUDA gradients with autograd's.

Reference lines (relative to the reference checkout): autoregressive/models/gpt_t2i.py:420-431,451-484 (forward), RMSNorm :193-198,
Attention :257-291, FeedForward :216-217, MLP :177-181, loss :474-481; the backward itself is autograd's in the reference
(autoregressive/train/train_c2i_canny.py:200-211: `scaler.scale(loss).backward()` on bf16 no-op scaling)."""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

BF = torch.bfloat16


def _b(x: torch.Tensor) -> torch.Tensor:
    return x.to(BF)


def _lin(x, w):                     # bf16 operands, fp32 accumulate, bf16 result (what the tensor-core GEMM returns)
    return _b(x.float() @ w.float().t())


def _gelu_tanh(t):                  # on the bf16 tensor, result bf16
    return _b(F.gelu(t.float(), approximate="tanh"))


def _gelu_tanh_grad(t):
    x = t.float()
    k0, k1 = 0.7978845608028654, 0.044715
    u = k0 * (x + k1 * x ** 3)
    th = torch.tanh(u)
    return 0.5 * (1 + th) + 0.5 * x * (1 - th * th) * k0 * (1 + 3 * k1 * x * x)


def _rms_fwd(h, w, eps):
    rstd = torch.rsqrt((h * h).mean(-1, keepdim=True) + eps)
    n = h * rstd
    return _b(n * w), n, rstd


def _rms_bwd(dy_b, n, rstd, w):
    """dy_b: bf16 gradient of the bf16-cast norm output.  Returns (dh fp32, dw fp32)."""
    dy = dy_b.float()
    dw = (dy * n).reshape(-1, n.shape[-1]).sum(0)
    dn = dy * w
    dh = rstd * (dn - n * (dn * n).mean(-1, keepdim=True))
    return dh, dw


def _rope(x, fr, inverse=False):
    """x [..., S, H, 64] any float dtype -> fp32 rotated (inverse = transpose rotation: the backward)"""
    xs = x.float().reshape(*x.shape[:-1], -1, 2)
    c, s = fr[:, None, :, 0], fr[:, None, :, 1]
    if inverse:
        s = -s
    o = torch.stack([xs[..., 0] * c - xs[..., 1] * s, xs[..., 1] * c + xs[..., 0] * s], dim=-1)
    return o.flatten(-2)


class ManualTrainBackward:
    def __init__(self, spec, params: Dict[str, torch.Tensor], freqs: torch.Tensor):
        self.sp = spec
        self.p = {k: v.detach().float() for k, v in params.items()}
        self.fr = freqs
        self.g: Dict[str, torch.Tensor] = {}

    def wb(self, key):
        return _b(self.p[key])

    # ---- MLP (fc1 -> GELU-tanh -> fc2, no bias) -------------------------------------------------------------------
    def mlp_fwd(self, x_b, prefix):
        t = _lin(x_b, self.wb(prefix + ".fc1.weight"))
        a = _gelu_tanh(t)
        return _lin(a, self.wb(prefix + ".fc2.weight")), t, a

    def mlp_bwd(self, x_b, prefix, dy_b, need_dx=True):
        _, t, a = self.mlp_fwd(x_b, prefix)
        w1, w2 = self.wb(prefix + ".fc1.weight"), self.wb(prefix + ".fc2.weight")
        x2, dy2 = x_b.reshape(-1, x_b.shape[-1]), dy_b.reshape(-1, dy_b.shape[-1])
        t2, a2 = t.reshape(-1, t.shape[-1]), a.reshape(-1, a.shape[-1])
        self.g[prefix + ".fc2.weight"] = _b(dy2.float().t() @ a2.float()).float()
        da = _b(dy2.float() @ w2.float())
        dt = _b(da.float() * _gelu_tanh_grad(t2))
        self.g[prefix + ".fc1.weight"] = _b(dt.float().t() @ x2.float()).float()
        return _b(dt.float() @ w1.float()).reshape(x_b.shape) if need_dx else None

    # ---- one block, forward pieces needed by its backward ---------------------------------------------------------
    def block_recompute(self, l, h0, mask):
        sp, P = self.sp, self.p
        B, S, d = h0.shape
        pre = f"layers.{l}."
        x1, n1, r1 = _rms_fwd(h0, P[pre + "attention_norm.weight"], sp.norm_eps)
        qkv = _lin(x1, self.wb(pre + "attention.wqkv.weight"))
        q, k, v = qkv.split([d, d, d], dim=-1)
        fr = self.fr[:S]
        q = _b(_rope(q.view(B, S, sp.n_head, 64), fr)).transpose(1, 2)
        k = _b(_rope(k.view(B, S, sp.n_head, 64), fr)).transpose(1, 2)
        v = v.reshape(B, S, sp.n_head, 64).transpose(1, 2)
        sc = (q.float() @ k.float().transpose(-1, -2)) * 0.125
        keep = torch.tril(torch.ones(S, S, dtype=torch.bool)) if mask is None else mask
        sc = sc.masked_fill(~keep, float("-inf"))
        p = torch.softmax(sc, dim=-1)
        att = _b(p @ v.float()).transpose(1, 2).reshape(B, S, d)
        o = _lin(att, self.wb(pre + "attention.wo.weight"))
        hm = h0 + o.float()
        x2, n2, r2 = _rms_fwd(hm, P[pre + "ffn_norm.weight"], sp.norm_eps)
        g = _lin(x2, self.wb(pre + "feed_forward.w1.weight"))
        u = _lin(x2, self.wb(pre + "feed_forward.w3.weight"))
        s = _b(F.silu(g.float()))
        act = _b(s.float() * u.float())
        o2 = _lin(act, self.wb(pre + "feed_forward.w2.weight"))
        return dict(x1=x1, n1=n1, r1=r1, q=q, k=k, v=v, p=p, att=att, hm=hm, x2=x2, n2=n2, r2=r2, g=g, u=u, s=s, act=act,
                    out=hm + o2.float())

    def block_bwd(self, l, c, dh):
        """dh: fp32 gradient of the block's output stream; returns the gradient of its input stream (fp32)."""
        sp, P, G = self.sp, self.p, self.g
        pre = f"layers.{l}."
        B, S, d = dh.shape
        R = B * S
        f2 = lambda t: t.reshape(R, -1).float()
        # feed-forward
        do2 = _b(dh)
        G[pre + "feed_forward.w2.weight"] = _b(f2(do2).t() @ f2(c["act"])).float()
        dact = _b(f2(do2) @ self.wb(pre + "feed_forward.w2.weight").float())
        ds = _b(dact.float() * f2(c["u"]))
        du = _b(dact.float() * f2(c["s"]))
        gf = f2(c["g"])
        sig = torch.sigmoid(gf)
        dg = _b(ds.float() * (sig * (1 + gf * (1 - sig))))
        G[pre + "feed_forward.w1.weight"] = _b(dg.float().t() @ f2(c["x2"])).float()
        G[pre + "feed_forward.w3.weight"] = _b(du.float().t() @ f2(c["x2"])).float()
        dx2 = _b(_b(dg.float() @ self.wb(pre + "feed_forward.w1.weight").float()).float()
                 + _b(du.float() @ self.wb(pre + "feed_forward.w3.weight").float()).float()).reshape(B, S, d)
        dhn, G[pre + "ffn_norm.weight"] = _rms_bwd(dx2, c["n2"], c["r2"], P[pre + "ffn_norm.weight"])
        dh = dh + dhn
        # attention
        do = _b(dh)
        G[pre + "attention.wo.weight"] = _b(f2(do).t() @ f2(c["att"])).float()
        datt = _b(f2(do) @ self.wb(pre + "attention.wo.weight").float()).reshape(B, S, sp.n_head, 64).transpose(1, 2)   # [B,H,S,64]
        p, q, k, v = c["p"], c["q"].float(), c["k"].float(), c["v"].float()
        dO = datt.float()
        dv = _b(p.transpose(-1, -2) @ dO)
        dp = dO @ v.transpose(-1, -2)
        dsc = p * (dp - (dp * p).sum(-1, keepdim=True))
        dq = _b((dsc @ k) * 0.125)
        dk = _b((dsc.transpose(-1, -2) @ q) * 0.125)
        fr = self.fr[:S]
        dq = _b(_rope(dq.transpose(1, 2), fr, inverse=True)).reshape(B, S, d)
        dk = _b(_rope(dk.transpose(1, 2), fr, inverse=True)).reshape(B, S, d)
        dqkv = torch.cat((dq, dk, dv.transpose(1, 2).reshape(B, S, d)), dim=-1)
        G[pre + "attention.wqkv.weight"] = _b(f2(dqkv).t() @ f2(c["x1"])).float()
        dx1 = _b(f2(dqkv) @ self.wb(pre + "attention.wqkv.weight").float()).reshape(B, S, d)
        dhn, G[pre + "attention_norm.weight"] = _rms_bwd(dx1, c["n1"], c["r1"], P[pre + "attention_norm.weight"])
        return dh + dhn

    # ---- whole model ----------------------------------------------------------------------------------------------
    def run(self, idx, cond, feat, drop_ids, mask, targets, valid):
        """Forward (saving the stream at every block input) + backward.  Returns (loss, d_feat bf16); gradients in self.g."""
        sp, P, G = self.sp, self.p, self.g
        T = sp.cls_token_num
        drop = drop_ids.bool()
        B, n = idx.shape
        n_img = n + 1
        if sp.model_type == "t2i":
            cap_b = _b(torch.where(drop[:, None, None], P["cls_embedding.uncond_embedding"], cond.float()))
            ce = self.mlp_fwd(cap_b, "cls_embedding.cap_proj")[0][:, :T].float()
        else:
            lab = torch.where(drop, torch.full_like(cond, sp.num_classes), cond)
            ce = P["cls_embedding.embedding_table.weight"][lab].unsqueeze(1)
        te = P["tok_embeddings.weight"][idx]
        h = torch.cat((ce, te), dim=1)
        feat_b = cin = ctok = None
        if feat is not None:
            feat_b = _b(feat)
            cin = self.mlp_fwd(feat_b, "adapter_mlp")[0]
            unc = _b(P["condition_mlp.uncond_embedding"][:n_img])                # ConditionEmbedder.token_drop gpt_t2i.py:110-120
            cin = torch.where(drop[:, None, None], unc[None], cin)
            ctok = self.mlp_fwd(cin, "condition_mlp.cap_proj")[0]
        step = sp.n_layer // 3
        saved = []
        for l in range(sp.n_layer):
            saved.append(h)
            if l % step == 0 and ctok is not None:
                add = self.mlp_fwd(ctok, f"condition_layers.{l // step}")[0]
                h = torch.cat((h[:, : T - 1], h[:, T - 1:] + add.float()), dim=1)
            h = self.block_recompute(l, h, mask)["out"]
        S = h.shape[1]
        xf, nf, rf = _rms_fwd(h[:, T - 1:], P["norm.weight"], sp.norm_eps)
        lg = _lin(xf, self.wb("output.weight")).float()                       # [B, n_img, V]
        lse = torch.logsumexp(lg, dim=-1)
        nll = lse - lg.gather(-1, targets[..., None]).squeeze(-1)
        if valid is not None:
            wrow = valid.float()[:, None].expand(B, n_img)
            den = max(float(wrow.sum()), 1.0)
        else:
            wrow = torch.ones(B, n_img)
            den = float(B * n_img)
        loss = (nll * wrow).sum() / den
        # ---- backward ----
        prob = torch.exp(lg - lse[..., None])
        onehot = F.one_hot(targets, lg.shape[-1]).float()
        dlg = _b((prob - onehot) * (wrow / den)[..., None]).reshape(B * n_img, -1)
        G["output.weight"] = _b(dlg.float().t() @ xf.reshape(B * n_img, -1).float()).float()
        dxf = _b(dlg.float() @ self.wb("output.weight").float()).reshape(B, n_img, -1)
        dht, G["norm.weight"] = _rms_bwd(dxf, nf, rf, P["norm.weight"])
        dh = torch.zeros(B, S, h.shape[-1])
        dh[:, T - 1:] = dht
        dctok = None
        for l in reversed(range(sp.n_layer)):
            h0 = saved[l]
            if l % step == 0 and ctok is not None:
                add = self.mlp_fwd(ctok, f"condition_layers.{l // step}")[0]
                h0 = torch.cat((h0[:, : T - 1], h0[:, T - 1:] + add.float()), dim=1)
            c = self.block_recompute(l, h0, mask)
            dh = self.block_bwd(l, c, dh)
            if l % step == 0 and ctok is not None:
                dadd = _b(dh[:, T - 1:])
                dc = self.mlp_bwd(ctok, f"condition_layers.{l // step}", dadd)
                dctok = dc if dctok is None else _b(dctok.float() + dc.float())
        # embeddings
        dE = torch.zeros_like(P["tok_embeddings.weight"])
        dE.index_add_(0, idx.reshape(-1), dh[:, T:].reshape(-1, dh.shape[-1]))
        G["tok_embeddings.weight"] = dE
        if sp.model_type == "t2i":
            self.mlp_bwd(cap_b, "cls_embedding.cap_proj", _b(dh[:, :T]), need_dx=False)
        else:
            dT = torch.zeros_like(P["cls_embedding.embedding_table.weight"])
            lab = torch.where(drop, torch.full_like(cond, sp.num_classes), cond)
            dT.index_add_(0, lab, dh[:, 0])
            G["cls_embedding.embedding_table.weight"] = dT
        dfeat = None
        if feat is not None:
            dcin = self.mlp_bwd(cin, "condition_mlp.cap_proj", dctok)
            dcin = torch.where(drop[:, None, None], torch.zeros_like(dcin), dcin)
            dfeat = self.mlp_bwd(feat_b, "adapter_mlp", dcin)
        return loss, dfeat
