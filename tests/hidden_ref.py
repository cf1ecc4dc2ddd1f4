"""Float64 reference of the encoder's per-token output (`rpx_encode_ids_hidden`, `hidden_store_kernel`) and a
checker whose tolerance follows from the rounding steps of the kernel.  Notation and helpers as in
tests/gemm_ref.py (u = 2^-24, gamma_n, the 2-ulp rsqrtf, the bf16 bracket).

The kernel writes, for token t at row (b, p) of a padded [B, L, D] output (t = cu[b] + p, p < len_b),
    y = fl(fl(h[t] * rs[t]) * w),   rs[t] = rsqrtf(fl(sum_q ss[q][t]) * fl(1/D) + eps),
and zeros at p >= len_b.  The checker gets the fp32 residual stream h [T, D] the kernel read (packed tokens),
not the partial sums ss: the reference row scale is 1 / sqrt(sum_c h[t, c]^2 / D + eps) in float64.

Row scale   every part is an fp32 sum of at most 128 squares (the residual epilogue: one part per 128 columns
            on the throughput path, per 32 on the latency path), and the P parts are summed in fp32: the
            relative error of the sum of squares is at most gamma_{128 + P}.  Then fp32(1/D), the product and
            + eps take 3 roundings, rsqrtf 2 ulp, and 1/sqrt halves a relative error of its argument:
                eps_rs = ((gamma_{128 + P} + 3u) / 2 + 2^-22) (1 + 1e-3).
Output      two fp32 products: |y - ref| <= |ref| (eps_rs + 2u) (1 + 1e-3).  An fp32 output must lie within
            that; a bf16 output in [bf16_rn(ref - tol), bf16_rn(ref + tol)].
Padding     positions past a row's length must be exactly +0.0 (bit pattern 0), and nothing past B * L rows may
            be written (NaN sentinels survive).
"""
from __future__ import annotations

from typing import Sequence

import torch

from tests import gemm_ref as R


def eps_hidden(n_parts: int) -> float:
    eps_rs = ((R.gamma_n(128 + n_parts) + 3 * R.U) / 2 + R.RSQRT_REL) * (1 + 1e-3)
    return (eps_rs + 2 * R.U) * (1 + 1e-3)


def reference(h32: torch.Tensor, ln_w: torch.Tensor, eps: float) -> torch.Tensor:
    """float64 final RMSNorm of packed rows h32 [T, D]; eps is the fp32 value the kernel receives."""
    h = h32.double()
    rs = 1.0 / torch.sqrt((h * h).sum(1, keepdim=True) / h.shape[1] + eps)
    return h * rs * ln_w.double()


def check_hidden(out: torch.Tensor, h32: torch.Tensor, ln_w: torch.Tensor, lens: Sequence[int], eps: float,
                 n_parts: int) -> list:
    """All findings (empty list: clean) for a padded output out [B, L, D] (bf16 or fp32) against the packed
    residual stream h32 [T, D] of the same call, T = sum(lens)."""
    B, L, D = out.shape
    assert h32.shape == (sum(lens), D), (h32.shape, sum(lens), D)
    want = reference(h32, ln_w, eps)
    tol = want.abs() * eps_hidden(n_parts)
    vals, pads = R.Findings("hidden.values"), R.Findings("hidden.padding")
    t0 = 0
    for b, n in enumerate(lens):
        got, ref, t = out[b, :n], want[t0:t0 + n], tol[t0:t0 + n]
        if got.dtype == torch.bfloat16:
            bad = R.bf16_bracket_bad(got, ref, t)
        else:
            bad = ~((got.double() - ref).abs() <= t)
        vals.add(bad, t0, got.double(), ref, t)
        pad = out[b, n:]
        bits = pad.reshape(-1, D).view(torch.int16 if pad.element_size() == 2 else torch.int32)
        pads.add(bits != 0, b * L + n)
        t0 += n
    return [f for f in (vals, pads) if f]
