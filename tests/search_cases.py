"""Constructed logits for the search step, fed to the engine through `rpx_debug_search` and to tests/beam_ref.py.

A case's logits are fp32 [max_length - 1, B * nb, V]: step t reads slab t, row b * nb + j being beam j of state b.
Random engine weights give continuous log-probs that almost never tie, so each family here aims at a path those
runs leave alone:

    plateau          logits from a few integer levels: log-probs tie exactly within a row, and beams with equal
                     running scores tie across rows.  At nb = 128, V = 384 hundreds of keys tie at the 2 nb-th
                     place, spread over many of the step kernel's 48-key thread chunks.
    identical        every beam of a state reads the same row at each step, so equal running scores tie across
                     parents.
    eos_pressure     EOS close to each row's best token, with a per-state strength: hypotheses finish at many lengths,
                     the finished merge replaces kept entries, and in one batch some states end by the early-stop
                     heuristic while others run to max_length.
    mask_magnitude   logits spread over 1e7 - 1e8: running and finished scores reach the -1e9 mask, where fp32's
                     spacing (64 - 128) decides ranks.
    parent_churn     each step one random beam other than beam 0 gets a sharp peak while the others are flat, so the
                     best beam's parent moves at most steps, over up to 511 steps (the lineage table and the finished
                     set's double buffers, sequences past 32 tokens).
    exact_levels     log-probs of exactly 0 and multiples of -1e4, so scores of hypotheses that finish at different
                     steps tie exactly, kept ones against new candidates in the finished merge.
    greedy_ties      nb = 1: equal maxima across lanes, warps and the 256-thread stride (ids j, j + 32, j + 256),
                     rows with -inf, all-equal rows, EOS at chosen steps.

`host_logprobs` is what beam_ref is fed on the CPU: the fp32 rounding of a float64 log_softmax, which is what the
step kernel computes up to its fp64 rounding (test_search_step_gpu.py checks that bound).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import torch

from tests import beam_ref

EOS, START = 1, 0


def _gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def plateau(B, nb, V, ML, seed, levels=3):
    """Integer levels 0 .. levels - 1, drawn per element."""
    g = _gen(seed)
    return torch.randint(0, levels, (ML - 1, B * nb, V), generator=g).float()


def identical(B, nb, V, ML, seed, levels: Optional[int] = 4):
    """One row per (step, state), repeated over its beams: integer levels, or N(0, 2) when levels is None."""
    g = _gen(seed)
    if levels is None:
        rows = torch.randn(ML - 1, B, 1, V, generator=g) * 2.0
    else:
        rows = torch.randint(0, levels, (ML - 1, B, 1, V), generator=g).float()
    return rows.expand(ML - 1, B, nb, V).reshape(ML - 1, B * nb, V).contiguous()


def eos_pressure(B, nb, V, ML, seed, eos=EOS):
    """N(0, 1.5) logits; EOS set to the row's maximum plus an offset drawn around a per-state strength (state 0
    strong, the last state never close), so states end at different steps and by different rules."""
    g = _gen(seed)
    x = torch.randn(ML - 1, B, nb, V, generator=g) * 1.5
    strength = torch.linspace(0.5, -6.0, B) if B > 1 else torch.tensor([-0.5])
    off = strength[None, :, None] + torch.randn(ML - 1, B, nb, generator=g) * 1.5
    x[..., eos] = x.amax(-1) + off
    return x.reshape(ML - 1, B * nb, V).contiguous()


def mask_magnitude(B, nb, V, ML, seed, scale=1e8, eos=EOS):
    """N(0, scale) logits, with EOS lifted to the row's median so that hypotheses finish with scores near the mask."""
    g = _gen(seed)
    x = torch.randn(ML - 1, B * nb, V, generator=g) * scale
    x[..., eos] = x.median(-1).values + torch.randn(ML - 1, B * nb, generator=g) * scale
    return x.contiguous()


def parent_churn(B, nb, V, ML, seed, eos=EOS):
    """Flat rows (N(0, 0.3)), and per (step, state) one random beam j >= 1 whose random token is lifted by 12 (log-prob
    near 0).  EOS sits 3.5 above the flat rows, so hypotheses keep finishing."""
    g = _gen(seed)
    x = torch.randn(ML - 1, B, nb, V, generator=g) * 0.3
    x[..., eos] += 3.5
    hot_beam = torch.randint(1, nb, (ML - 1, B), generator=g)
    hot_tok = torch.randint(2, V, (ML - 1, B), generator=g)
    t_idx, b_idx = torch.meshgrid(torch.arange(ML - 1), torch.arange(B), indexing="ij")
    x[t_idx, b_idx, hot_beam, hot_tok] += 12.0
    return x.reshape(ML - 1, B * nb, V).contiguous()


def exact_levels(B, nb, V, ML, seed, eos=EOS):
    """One token per row at 0, every other at -1e4 k (k = 1, 2, 3), so the log-probs are exactly 0 and -1e4 k in fp32
    and fp64 alike (the other terms of the softmax sum underflow) and every score is a multiple of 1e4: hypotheses
    that finish at different steps tie exactly, kept ones against the step's candidates in the finished merge.  EOS
    is the row's top token with probability 1/4."""
    g = _gen(seed)
    x = -1e4 * torch.randint(1, 4, (ML - 1, B * nb, V), generator=g).float()
    top = torch.randint(2, V, (ML - 1, B * nb), generator=g)
    top = torch.where(torch.rand(ML - 1, B * nb, generator=g) < 0.25, torch.full_like(top, eos), top)
    x.scatter_(-1, top[..., None], 0.0)
    return x.contiguous()


def greedy_ties(B, V, ML, seed, eos=EOS):
    """nb = 1.  Row r of step t takes one of: equal maxima at ids j, j + 32, j + 256 (those below V; j in [2, 32)),
    an all-equal row (id 0), a row of -inf with those ids tied at a finite value, a row half -inf, a row of all -inf
    (id 0).  Row r's EOS becomes its unique maximum at step r % (ML - 1), so the rows end at different steps, row 0
    at t = 0."""
    g = _gen(seed)
    x = torch.randn(ML - 1, B, V, generator=g)
    for t in range(ML - 1):
        for r in range(B):
            kind = (t + 3 * r) % 5
            j = 2 + (7 * t + 5 * r) % 30
            ids = [i for i in (j, j + 32, j + 256) if i < V]
            row = x[t, r]
            if kind == 0:
                row[ids] = row.max() + 1.0
            elif kind == 1:
                row[:] = 0.25
            elif kind == 2:
                row[:] = -math.inf
                row[ids] = 3.0
            elif kind == 3:
                row[torch.randperm(V, generator=g)[: V // 2]] = -math.inf
            else:
                row[:] = -math.inf
            if t == r % (ML - 1):
                finite = row[row.isfinite()]
                row[eos] = (float(finite.max()) if finite.numel() else 0.0) + 1.0
    return x.contiguous()


FAMILIES = {"plateau": plateau, "identical": identical, "eos_pressure": eos_pressure,
            "mask_magnitude": mask_magnitude, "parent_churn": parent_churn, "exact_levels": exact_levels}


@dataclass
class Case:
    """One search: its shape, its settings and the family (with extra keyword arguments) that builds its logits."""

    family: str
    B: int
    nb: int
    V: int
    ML: int
    lp: float
    n_ret: int
    seed: int
    kw: dict = field(default_factory=dict)

    @property
    def name(self) -> str:
        return f"{self.family}_B{self.B}_nb{self.nb}_V{self.V}_ML{self.ML}_lp{self.lp:g}_ret{self.n_ret}"

    def logits(self) -> torch.Tensor:
        if self.family == "greedy_ties":
            return greedy_ties(self.B, self.V, self.ML, self.seed, **self.kw)
        return FAMILIES[self.family](self.B, self.nb, self.V, self.ML, self.seed, **self.kw)


# The beam cases the GPU suite runs.  nb in {2, 3, 8, 64, 128}; V in {384, 256 (2 nb = V at nb = 128), 416 (nb V 4 =
# 212 992 B, the most that fits at nb = 128)}; B in {1, 5}; max_length in {2, 3, 40, 512}; length_penalty in
# {-0.5, 0, 1, 2}; num_return in {1, nb - 1, nb}.
BEAM_CASES = [
    Case("plateau", 1, 128, 384, 40, 1.0, 128, 1),
    Case("plateau", 1, 128, 256, 12, 0.0, 1, 2, {"levels": 2}),
    Case("plateau", 1, 128, 416, 12, -0.5, 127, 3),
    Case("plateau", 5, 64, 384, 40, 1.0, 63, 4),
    Case("plateau", 5, 3, 384, 40, 2.0, 2, 5, {"levels": 4}),
    Case("identical", 5, 8, 384, 40, 1.0, 8, 6),
    Case("identical", 1, 128, 384, 12, 0.0, 128, 7),
    Case("identical", 5, 2, 384, 2, 1.0, 1, 8),
    Case("identical", 5, 3, 256, 40, -0.5, 3, 9, {"levels": None}),
    Case("eos_pressure", 5, 8, 384, 40, 1.0, 8, 10),
    Case("eos_pressure", 5, 64, 384, 40, 0.0, 64, 11),
    Case("eos_pressure", 5, 3, 256, 3, -0.5, 3, 12),
    Case("eos_pressure", 5, 2, 384, 40, -0.5, 1, 13),
    Case("eos_pressure", 1, 128, 416, 40, 1.0, 127, 14),
    Case("mask_magnitude", 5, 8, 384, 40, 1.0, 7, 15),
    Case("mask_magnitude", 5, 2, 416, 40, 0.0, 2, 16, {"scale": 3e7}),
    Case("mask_magnitude", 1, 128, 384, 12, 2.0, 128, 17),
    Case("exact_levels", 5, 8, 384, 40, 0.0, 8, 21),
    Case("exact_levels", 5, 2, 384, 40, 0.0, 2, 22),
    Case("parent_churn", 1, 8, 384, 512, 2.0, 8, 18),
    Case("parent_churn", 5, 3, 256, 512, 2.0, 3, 19),
    Case("parent_churn", 1, 64, 384, 160, 2.0, 63, 20),
]

GREEDY_CASES = [
    Case("greedy_ties", 40, 1, 384, 40, 1.0, 1, 30),
    Case("greedy_ties", 5, 1, 384, 2, 1.0, 1, 31),
    Case("greedy_ties", 7, 1, 300, 3, 1.0, 1, 32),
    Case("greedy_ties", 5, 1, 32128, 12, 1.0, 1, 33),
]


def host_logprobs(logits: torch.Tensor) -> torch.Tensor:
    """fp32 rounding of the float64 log_softmax over the last dim."""
    return torch.log_softmax(logits.double(), -1).float()


def reference(case: Case, scores: torch.Tensor, defect: Optional[str] = None,
              stats: Optional[beam_ref.SearchStats] = None):
    """beam_ref on per-step scores [ML - 1, R, V] (log-probs for beam search, logits for greedy): (sequences,
    scores or None)."""
    step = lambda t, prefixes: scores[t]  # noqa: E731
    if case.nb == 1:
        return beam_ref.greedy(step, case.B, case.ML, EOS, START, START, stats=stats), None
    return beam_ref.beam_search(step, case.B, case.nb, case.n_ret, case.ML, case.lp, EOS, START, START, stats=stats,
                                defect=defect)
