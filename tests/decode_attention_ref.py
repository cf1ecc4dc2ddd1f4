"""Float64 reference of the generator's decode self-attention (rpx_debug_decode_attention) and its checker.

Step t, row r, head h: keys / values p = 0..t come from cache row p * R + lin[r][p] of a [max_length][R][3 inner]
q | k | v cache; the query is cache row t * R + r.  Scores are q.k (unscaled) + lut[h][max(p - t, -md) + md].

Tolerance per output element, derived as tests/attention_mode_ref.py derives its own:
  - the kernel rounds its fp32 result to bf16: half an ulp, 2^-8 |ref|;
  - each fp32 score carries at most ~2^-20 * sum_i |q_i k_i| of rounding from its 64 products, plus the bias; a score
    error e moves the output by at most e * max_p |v_p - ref| (the softmax weights shift by at most e in ratio);
  - the fp32 softmax and the value sum: a few units of 2^-23 of max |v| each over t + 1 terms.
`fp32_model` restates the kernel in fp32 and must pass; each of `DEFECTS` injected into it must fail.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

DEFECTS = ("bias_plus_1", "bias_minus_1", "drop_own_key", "admit_next_key", "sibling_slot", "lin_not_gathered",
           "wrong_head")


@dataclass
class Case:
    cache: torch.Tensor  # [ML, R, 3 inner] fp32 (bf16 values)
    lin: torch.Tensor    # [R, ML] int64
    lut: torch.Tensor    # [H, 2 md + 1] fp32
    t: int
    H: int
    md: int


def random_lineage(t: int, R: int, ML: int, g: torch.Generator) -> torch.Tensor:
    """lin [R, ML] of a random beam search that reached step t: each step every row continues a random parent, whose
    lineage it copies, and takes its own slot at the new position.  Positions past t + 1 hold random slots."""
    lin = torch.randint(0, R, (R, ML), generator=g)
    cur = torch.arange(R)[:, None].clone()
    for p in range(1, t + 1):
        parent = torch.randint(0, R, (R,), generator=g)
        cur = torch.cat([cur[parent], torch.arange(R)[:, None]], 1)
    lin[:, :t + 1] = cur
    return lin


def random_case(t: int, R: int, H: int = 6, ML: int = 0, max_distance: int = 128, seed: int = 0,
                device="cpu") -> Case:
    g = torch.Generator().manual_seed(seed)
    ML = ML or t + 2
    inner = H * 64
    cache = torch.randn(ML, R, 3 * inner, generator=g)
    cache[..., :2 * inner] *= 0.35
    cache = cache.bfloat16().float()
    lut = (torch.randn(H, 2 * max_distance + 1, generator=g) * 2.0).float()
    return Case(cache.to(device), random_lineage(t, R, ML, g).to(device), lut.to(device), t, H, max_distance)


def reference(case: Case) -> torch.Tensor:
    """[R, inner] float64."""
    c = case.cache.double().cpu()
    lin = case.lin.cpu()
    lut = case.lut.double().cpu()
    ML, R, W = c.shape
    inner = W // 3
    t, md = case.t, case.md
    p = torch.arange(t + 1)
    rows = c[p[None, :], lin[:, :t + 1]]  # [R, t + 1, 3 inner]
    q = c[t, torch.arange(R)][:, :inner].view(R, case.H, 64)
    k = rows[..., inner:2 * inner].view(R, t + 1, case.H, 64)
    v = rows[..., 2 * inner:].view(R, t + 1, case.H, 64)
    s = torch.einsum("rhd,rphd->rhp", q, k) + lut[:, (p - t).clamp(min=-md) + md][None]
    w = torch.softmax(s, -1)
    return torch.einsum("rhp,rphd->rhd", w, v).reshape(R, inner)


def tolerance(case: Case, ref: torch.Tensor) -> torch.Tensor:
    c = case.cache.double().cpu()
    lin = case.lin.cpu()
    ML, R, W = c.shape
    inner = W // 3
    t = case.t
    p = torch.arange(t + 1)
    rows = c[p[None, :], lin[:, :t + 1]]
    q = c[t, torch.arange(R)][:, :inner].view(R, case.H, 64)
    k = rows[..., inner:2 * inner].view(R, t + 1, case.H, 64)
    v = rows[..., 2 * inner:].view(R, t + 1, case.H, 64)
    qk_abs = torch.einsum("rhd,rphd->rhp", q.abs(), k.abs()).amax(-1)  # [R, H]
    e_score = qk_abs * 2.0 ** -20 + case.lut.abs().max().item() * 2.0 ** -23 + 1e-7
    ref3 = ref.view(R, case.H, 64)
    spread = (v - ref3[:, None]).abs().amax(1)  # [R, H, 64]
    vmax = v.abs().amax(1)
    tol = 2.0 ** -8 * ref3.abs() + 4 * e_score[..., None] * spread + (t + 8) * 2.0 ** -22 * vmax
    return tol.reshape(R, inner)


def check(out: torch.Tensor, case: Case) -> int:
    """How many elements of `out` [R, inner] fall outside the tolerance (NaNs count)."""
    ref = reference(case)
    err = (out.double().cpu() - ref).abs()
    bad = ~(err <= tolerance(case, ref))
    return int(bad.sum())


def fp32_model(case: Case, defect: str = "") -> torch.Tensor:
    """The kernel's arithmetic in fp32 (scores, softmax, value sum), output rounded to bf16; `defect` injects one of
    DEFECTS."""
    c = case.cache.float().cpu()
    lin = case.lin.cpu().clone()
    ML, R, W = c.shape
    inner = W // 3
    H, t, md = case.H, case.t, case.md
    n = t + 2 if defect == "admit_next_key" else t + 1
    p = torch.arange(n)
    if defect == "drop_own_key":
        p = p[:t]
    slots = lin[:, p]
    if defect == "sibling_slot":
        slots = torch.where(p[None, :] < t, lin[(torch.arange(R) + 1) % R][:, p], slots)
    if defect == "lin_not_gathered":
        slots = torch.arange(R)[:, None].expand_as(slots)
    rows = c[p[None, :], slots]
    q = c[t, torch.arange(R)][:, :inner].view(R, H, 64)
    k = rows[..., inner:2 * inner].view(R, len(p), H, 64)
    if defect == "wrong_head":
        k = k.roll(1, dims=2)
    v = rows[..., 2 * inner:].view(R, len(p), H, 64)
    delta = (p - t).clamp(min=-md) + md
    if defect == "bias_plus_1":
        delta = (delta + 1).clamp(max=2 * md)
    if defect == "bias_minus_1":
        delta = (delta - 1).clamp(min=0)
    s = torch.einsum("rhd,rphd->rhp", q, k) + case.lut.float().cpu()[:, delta][None]
    w = torch.softmax(s, -1)
    out = torch.einsum("rhp,rphd->rhd", w, v).reshape(R, inner)
    return out.bfloat16()
