"""Float64 reference of the T5 attention kernel's decoder modes (rpx_debug_attention_ex) and a checker, on the
rounding model of tests/attention_ref.py: causal self-attention (keys j <= i, the decoder's unidirectional bias
table) and cross-attention (queries of one packed matrix, keys / values of another with their own offsets, no bias).

Per sequence, every term of attention_ref's tolerance is formed over the keys the kernel visits.  A masked key has
p = 0 and adds nothing to any term; its score is set to the row maximum (finite) before the tolerance is formed, so
the per-key error factors stay finite where they are multiplied by p = 0.
"""
from __future__ import annotations

import math

import torch

from tests.attention_ref import ETA_EX2, HD, KT, ROW_ELEMS, U, U_BF
from tests.gemm_ref import BF16_NAN_BITS, Findings, bf16_bracket_bad, check_sentinels, gamma_acc, gamma_n


def _ref_qk(q, k, v, bias, mask):
    """q [H, Lq, 64], k / v [H, Lk, 64] float64; bias [H, Lq, Lk] or None; mask [Lq, Lk] bool (visible)."""
    S = q @ k.transpose(-1, -2)
    SA = q.abs() @ k.abs().transpose(-1, -2)
    s = S + bias if bias is not None else S
    s = s.masked_fill(~mask, -math.inf)
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    o = (p @ v) / l
    s_fin = torch.where(mask, s, m.expand_as(s))
    return s_fin, SA * mask, m, p, l, o


def _tolerance_qk(Lk, v, s, SA, m, p, l, o):
    """attention_ref._tolerance for Lq queries over Lk keys (s finite everywhere, p = 0 on masked keys).  Tensors carry a leading
    batch dimension of 1."""
    n_kt = -(-Lk // KT)
    dS = gamma_acc(HD) * SA
    rho_s = dS + U * (s.abs() + dS)
    E = rho_s.amax(-1, keepdim=True)
    d = m - s + 2 * E
    Mabs = s.abs().amax(-1, keepdim=True) + E
    rho = torch.expm1(rho_s + U * (4 * d + Mabs) * (1 + 2 * U) + n_kt * ETA_EX2)
    den = l * (1 - rho.amax(-1, keepdim=True))
    w = p * rho
    va = v.abs()
    A = (p * (1 + rho)) @ va
    Lq = o.shape[-2]
    t1 = torch.empty_like(o)
    nb = max(1, ROW_ELEMS // max(1, v.shape[0] * v.shape[1] * Lk * HD))
    for r0 in range(0, Lq, nb):
        r1 = min(Lq, r0 + nb)
        diff = (v[:, :, None, :, :] - o[:, :, r0:r1, None, :]).abs()
        t1[:, :, r0:r1] = (w[:, :, r0:r1, :, None] * diff).sum(3)
        del diff
    t1 = t1 / den
    t2 = U_BF * A / den
    t3 = (math.ceil(Lk / 16) * 18 * 2.0 ** -23 + n_kt * U) * (1 + U_BF) * A / den
    lam = gamma_n(Lk + n_kt + 2)
    t4 = o.abs() * (lam + 2 * U) * (1 + lam)
    t5 = Lk * 2.0 ** -126 * (va.amax(2, keepdim=True) + o.abs()) / l
    return 1.01 * (t1 + t2 + t3 + t4) + t5


def hf_bias_lut_unidirectional(rel_bias: torch.Tensor, num_buckets: int, R: int) -> torch.Tensor:
    """hf_bias_lut with HF's unidirectional (decoder) buckets."""
    from transformers.models.t5.modeling_t5 import T5Attention

    delta = torch.arange(-R, R + 1, dtype=torch.long)
    b = T5Attention._relative_position_bucket(delta, bidirectional=False, num_buckets=num_buckets, max_distance=R)
    return rel_bias.detach().cpu().float()[b].t().double().contiguous().to(rel_bias.device)


def check_attention_mode(out: torch.Tensor, q_mat: torch.Tensor, kv_mat: torch.Tensor, cu_q: list, cu_k: list, H: int,
                         causal: bool, lut: torch.Tensor | None = None, R: int = 0) -> list:
    """Findings of out (bf16, >= cu_q[-1] rows; rows from cu_q[-1] on must hold the NaN sentinel) for the causal mode
    (q_mat = kv_mat = qkv [T, 3 H 64], cu_k = cu_q, lut the decoder's table) or the cross mode (q_mat [Tq, H 64],
    kv_mat [Tk, 2 H 64] k | v, no bias)."""
    inner = H * HD
    f = Findings("attn.out")
    for s_i in range(len(cu_q) - 1):
        a, b = cu_q[s_i], cu_q[s_i + 1]
        c, e = cu_k[s_i], cu_k[s_i + 1]
        Lq, Lk = b - a, e - c
        if Lq == 0:
            continue
        if causal:
            x = q_mat[a:b].double()
            q = x[:, :inner].reshape(Lq, H, HD).transpose(0, 1)
            k = x[:, inner:2 * inner].reshape(Lq, H, HD).transpose(0, 1)
            v = x[:, 2 * inner:].reshape(Lq, H, HD).transpose(0, 1)
            pos = torch.arange(Lq, device=q.device)
            rel = pos[None, :] - pos[:, None]
            bias = lut.to(q.device).double()[:, rel.clamp(-R, R) + R]
            mask = rel <= 0
        else:
            q = q_mat[a:b].double().reshape(Lq, H, HD).transpose(0, 1)
            y = kv_mat[c:e].double()
            k = y[:, :inner].reshape(Lk, H, HD).transpose(0, 1)
            v = y[:, inner:].reshape(Lk, H, HD).transpose(0, 1)
            bias = None
            mask = torch.ones(Lq, Lk, dtype=torch.bool, device=q.device)
        s, SA, m, p, l, o = _ref_qk(q, k, v, bias, mask)
        n_keys = Lq if causal else Lk
        tol = _tolerance_qk(n_keys, v[None], s[None], SA[None], m[None], p[None], l[None], o[None])[0]
        got = out[a:b].reshape(Lq, H, HD).transpose(0, 1)
        bad = bf16_bracket_bad(got, o, tol)
        if bool(bad.any()):
            for h, i, col in bad.nonzero().tolist():
                f.n_bad += 1
                if len(f.where) < f.keep:
                    f.where.append((a + i, h * HD + col))
                if len(f.samples) < 16:
                    f.samples.append({"row": a + i, "col": h * HD + col, "got": float(got[h, i, col]),
                                      "want": float(o[h, i, col]), "tol": float(tol[h, i, col])})
    return [f, check_sentinels("attn.pad", out, cu_q[-1] * inner, BF16_NAN_BITS)]
