"""Float64 reference of the encoder's T5 attention (t5_attention_kernel) and a checker whose tolerance follows
from the rounding each step of the kernel performs.

Layout as the kernel sees it: qkv [T, 3 H 64] bf16 (q | k | v, head h in columns [64 h, 64 h + 64) of each),
sequences packed back to back at token offsets cu[0] = 0 < cu[1] < ... < cu[n] <= T, out [T, H 64] bf16,
and the relative-position bias table lut [H, 2R + 1] fp32 with lut[h][delta + R] the bias of delta = key - query
(clamped to [-R, R]).  For every sequence and head, from the exact bf16 inputs in float64:
    s_ij = q_i . k_j + lut[h][clamp(j - i, -R, R) + R],   p_ij = exp(s_ij - m_i),  m_i = max_j s_ij,
    l_i = sum_j p_ij,   o_i = sum_j p_ij v_j / l_i,       j over the keys 0 <= j < len of the same sequence.
Sequences are processed in groups of equal length, chunked so that a group's score tensor stays below
SCORE_CHUNK elements: thousands of short sequences and 2048-token ones both fit.  The reference LUT comes from
HF's own T5Attention._relative_position_bucket (hf_bias_lut), not from the library's bucket function, so the
GPU suite pins the sign convention (key - query; positive delta in the upper half of the buckets) on its own.

Notation as in tests/gemm_ref.py: u = 2^-24, gamma_n = n u / (1 - n u), gamma_acc(K) = ceil(K / 16) 18 2^-23
(the truncating block-FMA model of wgmma); u_bf = 2^-8 is the unit roundoff of bf16.  L2E = fp32(log2 e).

Per-key relative error rho_j of p_j (the same factor in numerator and denominator)
    A relative error rho_j of the weight p_j, present in both sum_j p_j v_j and l, moves o_i by
        |sum_j p_j rho_j (v_j - o_i)| / sum_j p_j (1 + rho_j)  <=  sum_j p_j rho_j |v_j - o_i| / (l (1 - max rho)).
    Errors common to a whole row (the value of the running maximum m, any factor shared by every key) cancel
    between numerator and denominator and do not appear.  What differs from key to key, as a shift dx_j of the
    exponent in log2 units (p_j moves by a factor 2^dx_j, i.e. rho_j = expm1(ln 2 |dx_j|)) or directly as rho_j:
      - the score: S = Q K^T by wgmma over K = 64 (4 block FMAs), |dS| <= gamma_acc(64) sum_c |q_ic| |k_jc|, then
        fl(S + bias): u (|s| + dS).  A shift ds of s_j is a relative error ds of p_j:  rho_s = dS + u (|s| + dS).
      - the argument fmaf(s, L2E, -fl(m_t L2E)) of step t (m_t the running maximum after that step): one rounding
        of the fmaf, u |x_j| with |x_j| <= (m - s_j + 2 E) L2E (E = the largest rho_s of the row, m the final
        maximum); the rounding of mb = fl(m_t L2E), u |m_t| L2E, which differs between key steps; the error of
        L2E itself, at most u (m - s_j) L2E over the whole exponent.
      - the rescale of o and l when a later step raises the maximum, ex2((m_old - m_new) L2E): two roundings per
        step, and the (m_old - m_new) of the steps after key j's telescope to at most m - s_j + 2 E, so
        2 u (m - s_j + 2 E) L2E in all.
        Together (ln 2 L2E = 1 to within u):  rho_x = u (4 (m - s_j + 2 E) + max_j |s_j| + E) (1 + 2u).
      - ex2.approx.ftz.f32: the PTX ISA ("ex2", Floating Point Instructions) bounds its maximum relative error
        below 2^-22.  Key j's weight passes through its own ex2 and through the scale ex2 of every later step,
        at most n_kt = ceil(len / 64) of them:  rho_ex2 = n_kt 2^-22.
      - results below 2^-126 are flushed to 0: an absolute error of at most 2^-126 per key, at most
        len 2^-126 (max |v| + |o|) / l in the output (l >= 1: the maximal key has p = 1).
    rho_j = expm1(rho_s + rho_x + rho_ex2).
P rounded to bf16 (numerator only)
    The PV MMA takes P as a bf16 operand (round to nearest, relative error u_bf) while l sums the fp32 values,
    so this error is not shared with the denominator:  u_bf sum_j p_j (1 + rho_j) |v_j| / (l (1 - max rho)).
PV accumulation
    o accumulates over ceil(len / 16) wgmma k16 instructions (steps of masked keys add exact zeros), each off by
    at most 18 2^-23 of a magnitude bounded by the sum of the magnitudes added so far; the per-step rescale
    multiplications of o add one rounding each (n_kt of them).  The magnitudes are bounded by
    sum_j p~_j |v_j| <= (1 + u_bf) sum_j p_j (1 + rho_j) |v_j|:
        (ceil(len / 16) 18 2^-23 + n_kt u) (1 + u_bf) sum_j p_j (1 + rho_j) |v_j| / (l (1 - max rho)).
Row sum and final scaling
    l is the sum of len non-negative fp32 values plus n_kt rescale multiplications and the two quad additions:
    relative error lambda = gamma_(len + n_kt + 2).  The kernel then forms the IEEE quotient 1.f / l (the library
    is compiled without fast-math) and the product o * inv: 2 u.  Together |o| (lambda + 2 u) (1 + lambda).
Products of two of these relative errors (each below 2^-6) are covered by a factor 1.01 on the sum.

The output check is the bf16 bracket of gemm_ref: out must lie in [bf16_rn(ref - tol), bf16_rn(ref + tol)].

What this tolerance cannot see.  The bf16 rounding of P is the dominant term, u_bf sum_j p_j |v_j| / l, about
2^-8 mean |v| on a long flat row.  When the v_j cancel (o small against mean |v|) that is many output ulps, so
an error confined to a few keys of such a row, or a slightly wrong weight spread over many keys, can pass.
The exact cases of tests/test_attention_gpu.py (one-hot routing, the bias-bucket sweep, bit-identity across
packings) carry the discriminating power there.
"""
from __future__ import annotations

import math
from collections import Counter

import torch

from tests.gemm_ref import (BF16_NAN_BITS, U, Findings, _f32_outward, bf16_bracket_bad, check_sentinels, gamma_acc,
                            gamma_n)

HD = 64  # head dim
KT = 64  # keys per kernel step
QT = 64  # queries per CTA
U_BF = 2.0 ** -8
ETA_EX2 = 2.0 ** -22  # ex2.approx.f32 maximum relative error (PTX ISA)
L2E = float(torch.tensor(math.log2(math.e), dtype=torch.float32))
SCORE_CHUNK = 1 << 23  # score-tensor elements per reference chunk
ROW_ELEMS = 1 << 24  # elements of the [rows, keys, 64] |v_j - o_i| product per block


def hf_bias_lut(rel_bias: torch.Tensor, num_buckets: int, R: int) -> torch.Tensor:
    """lut [H, 2R + 1] (float64, fp32 values) from an HF relative_attention_bias table [buckets, H], through HF's
    own bidirectional bucket function."""
    from transformers.models.t5.modeling_t5 import T5Attention

    delta = torch.arange(-R, R + 1, dtype=torch.long)
    b = T5Attention._relative_position_bucket(delta, bidirectional=True, num_buckets=num_buckets, max_distance=R)
    return rel_bias.detach().cpu().float()[b].t().double().contiguous().to(rel_bias.device)


def random_qkv(T: int, H: int, gen: torch.Generator, device="cpu") -> torch.Tensor:
    """qkv [T, 3 H 64] bf16 whose score rows range from flat to sharp: q rows scaled by 0.06..3 (log-uniform),
    k rows by 0.5..2 / sqrt(8), so the score spread 8 |q_scale| |k_scale| runs from about 0.1 (|s| ~ 1 after
    the bias) to about 17 (|s| ~ 50 at the top of a 2048-key row); v ~ N(0, 1)."""
    inner = H * HD
    x = torch.randn(T, 3 * inner, generator=gen, device=device)
    qs = torch.exp(torch.empty(T, H, 1, device=device).uniform_(math.log(0.06), math.log(3.0), generator=gen))
    ks = torch.exp(torch.empty(T, H, 1, device=device).uniform_(math.log(0.5), math.log(2.0), generator=gen)) / math.sqrt(8)
    x[:, :inner] = (x[:, :inner].reshape(T, H, HD) * qs).reshape(T, inner)
    x[:, inner:2 * inner] = (x[:, inner:2 * inner].reshape(T, H, HD) * ks).reshape(T, inner)
    return x.to(torch.bfloat16)


def _groups(cu: list[int]):
    """(length, tensor of start offsets) for each distinct sequence length."""
    by_len: dict[int, list[int]] = {}
    for s in range(len(cu) - 1):
        by_len.setdefault(cu[s + 1] - cu[s], []).append(cu[s])
    return sorted(by_len.items())


class AttnFindings(Findings):
    """Findings that also keep, per recorded bad element, (sequence, head, query position, key step of the
    largest-weight key) for the diagnostic."""

    def __init__(self, name: str):
        super().__init__(name)
        self.meta: list[tuple[int, int, int, int]] = []


def _ref_chunk(qkv, starts, L, H, lut, R):
    """float64 reference of n sequences of length L: returns q, k, v [n, H, L, 64], s, p [n, H, L, L], o, l."""
    dev = qkv.device
    inner = H * HD
    rows = starts[:, None] + torch.arange(L, device=dev)[None, :]  # [n, L]
    x = qkv[rows].double()  # [n, L, 3 inner]
    n = rows.shape[0]
    q = x[..., :inner].reshape(n, L, H, HD).transpose(1, 2)
    k = x[..., inner:2 * inner].reshape(n, L, H, HD).transpose(1, 2)
    v = x[..., 2 * inner:].reshape(n, L, H, HD).transpose(1, 2)
    pos = torch.arange(L, device=dev)
    idx = (pos[None, :] - pos[:, None]).clamp(-R, R) + R  # [L(query), L(key)]
    bias = lut.to(dev).double()[:, idx]  # [H, L, L]
    S = q @ k.transpose(-1, -2)
    SA = q.abs() @ k.abs().transpose(-1, -2)
    s = S + bias[None]
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    o = (p @ v) / l
    return rows, v, s, SA, m, p, l, o


def reference(qkv: torch.Tensor, cu: list[int], H: int, lut: torch.Tensor, R: int) -> torch.Tensor:
    """o [T, H 64] float64 (rows outside every sequence are NaN)."""
    T = qkv.shape[0]
    out = torch.full((T, H * HD), math.nan, dtype=torch.float64, device=qkv.device)
    for L, starts, rows, _, _, _, _, _, _, o in _iter_chunks(qkv, cu, H, lut, R):
        out[rows.reshape(-1)] = o.transpose(1, 2).reshape(-1, H * HD)
    return out


def _iter_chunks(qkv, cu, H, lut, R):
    for L, starts in _groups(cu):
        st = torch.tensor(starts, dtype=torch.long, device=qkv.device)
        per = max(1, SCORE_CHUNK // (H * L * L))
        for c0 in range(0, len(starts), per):
            sc = st[c0:c0 + per]
            rows, v, s, SA, m, p, l, o = _ref_chunk(qkv, sc, L, H, lut, R)
            yield L, sc, rows, v, s, SA, m, p, l, o


def _tolerance(L, v, s, SA, m, p, l, o):
    """tol [n, H, L, 64] of every output element (docstring)."""
    n_kt = -(-L // KT)
    dS = gamma_acc(HD) * SA
    rho_s = dS + U * (s.abs() + dS)
    E = rho_s.amax(-1, keepdim=True)
    d = m - s + 2 * E
    Mabs = s.abs().amax(-1, keepdim=True) + E
    rho_x = U * (4 * d + Mabs) * (1 + 2 * U)
    rho = torch.expm1(rho_s + rho_x + n_kt * ETA_EX2)  # [n, H, L, L]
    rmax = rho.amax(-1, keepdim=True)
    den = l * (1 - rmax)
    w = p * rho  # [n, H, L, L]
    va = v.abs()
    A = (p * (1 + rho)) @ va  # [n, H, L, 64]
    # sum_j w_ij |v_j - o_i|, in blocks of query rows
    t1 = torch.empty_like(o)
    nb = max(1, ROW_ELEMS // max(1, v.shape[0] * v.shape[1] * L * HD))
    for r0 in range(0, L, nb):
        r1 = min(L, r0 + nb)
        diff = (v[:, :, None, :, :] - o[:, :, r0:r1, None, :]).abs()  # [n, H, rows, L, 64]
        t1[:, :, r0:r1] = (w[:, :, r0:r1, :, None] * diff).sum(3)
        del diff
    t1 = t1 / den
    t2 = U_BF * A / den
    t3 = (math.ceil(L / 16) * 18 * 2.0 ** -23 + n_kt * U) * (1 + U_BF) * A / den
    lam = gamma_n(L + n_kt + 2)
    t4 = o.abs() * (lam + 2 * U) * (1 + lam)
    t5 = L * 2.0 ** -126 * (va.amax(2, keepdim=True) + o.abs()) / l
    return 1.01 * (t1 + t2 + t3 + t4) + t5


def check_attention(out: torch.Tensor, qkv: torch.Tensor, cu: list[int], H: int, lut: torch.Tensor, R: int,
                    stats: dict | None = None) -> list[Findings]:
    """Findings of out [>= T rows, H 64] bf16 against the reference; rows from cu[-1] on must still hold the NaN
    sentinel.  `stats` receives the largest error over the allowed half-width of the bracket (<= 1 passes; an
    output on the bracket's edge gives 1), the largest error beyond half a bf16 ulp (the final rounding) over
    tol, the median tol in bf16 ulps, and the count of outputs that are not bf16_rn(ref)."""
    T = cu[-1]
    f = AttnFindings("attn.out")
    seq_of = {}
    for s_i in range(len(cu) - 1):
        seq_of[cu[s_i]] = s_i
    worst_bracket = 0.0
    worst_excess = 0.0
    n_not_rn = 0
    tol_ulps = []
    for L, starts, rows, v, s, SA, m, p, l, o in _iter_chunks(qkv, cu, H, lut, R):
        tol = _tolerance(L, v, s, SA, m, p, l, o)
        n = rows.shape[0]
        got = out[rows.reshape(-1)].reshape(n, L, H, HD).transpose(1, 2)  # [n, H, L, 64]
        bad = bf16_bracket_bad(got, o, tol)
        g = got.double()
        err = (g - o).abs()
        lo = _f32_outward(o - tol, down=True).to(torch.bfloat16).double()
        hi = _f32_outward(o + tol, down=False).to(torch.bfloat16).double()
        allowed = torch.where(g >= o, hi - o, o - lo)
        ratio = torch.where(allowed > 0, err / allowed.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        worst_bracket = max(worst_bracket, float(ratio.nan_to_num(math.inf).max()))
        half_ulp = _bf16_half_ulp(torch.maximum(g.abs(), o.abs()))
        beyond = (err - half_ulp).clamp_min(0)
        excess = torch.where(beyond > 0, beyond / tol, torch.zeros_like(tol)).nan_to_num(math.inf)
        worst_excess = max(worst_excess, float(excess.max()))
        n_not_rn += int((g != o.float().to(torch.bfloat16).double()).sum())
        tol_ulps.append(float((tol / (2 * half_ulp).clamp_min(1e-300)).median()))
        if bool(bad.any()):
            amax_step = p.argmax(-1) // KT  # [n, H, L]
            for si, h, i, c in bad.nonzero().tolist():
                if len(f.where) >= f.keep:
                    f.n_bad += 1
                    continue
                t0 = int(starts[si])
                f.n_bad += 1
                f.where.append((t0 + i, h * HD + c))
                f.meta.append((seq_of[t0], h, i, int(amax_step[si, h, i])))
                if len(f.samples) < 16:
                    f.samples.append({"row": t0 + i, "col": h * HD + c, "got": float(g[si, h, i, c]),
                                      "want": float(o[si, h, i, c]), "tol": float(tol[si, h, i, c])})
        del tol, bad, g, err, lo, hi, allowed, ratio, excess
    if stats is not None:
        stats.update(max_err_over_bracket=worst_bracket, max_excess_over_tol=worst_excess, n_not_rn_of_ref=n_not_rn,
                     median_tol_in_ulps=(sorted(tol_ulps)[len(tol_ulps) // 2] if tol_ulps else 0.0))
    return [f, check_sentinels("attn.pad", out, T * H * HD, BF16_NAN_BITS)]


def _bf16_half_ulp(x: torch.Tensor) -> torch.Tensor:
    """Half the bf16 spacing at |x| (normal range)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 8)


def diagnose(f: Findings) -> dict:
    """Where the bad elements sit: per sequence, head, 64-query tile, wgmma fragment row (query % 16) and the
    64-key step holding the row's largest-weight key."""
    meta = getattr(f, "meta", [])
    return {
        "output": f.name,
        "n_bad": f.n_bad,
        "first": f.where[:40],
        "samples": f.samples,
        "by_sequence": Counter(m[0] for m in meta).most_common(24),
        "by_head": sorted(Counter(m[1] for m in meta).items()),
        "by_query_tile": sorted(Counter(m[2] // QT for m in meta).items()),
        "by_fragment_row": sorted(Counter(m[2] % 16 for m in meta).items()),
        "by_max_weight_key_step": sorted(Counter(m[3] for m in meta).items()),
    }
