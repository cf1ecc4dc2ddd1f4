"""A restatement of HF 5.5 `GenerationMixin._beam_search` (early_stopping=False, one EOS id, no logits processor)
and greedy `_sample`, driven by a step function, with the engine's tie rule: every top-k ranks (score desc, index
asc).  `tests/test_generate_cpu.py` pins it against HF `generate`; the GPU tests feed it the engine's traced step
log-probs, so the search bookkeeping is checked apart from the arithmetic.

    step_fn(t, prefixes [R, t + 1] int64) -> fp32 [R, V]   log-probs (beam search) or logits (greedy)

`beam_search(defect=...)` plants one bookkeeping mistake a step kernel could make (default None: none), so that
tests/test_search_cases_cpu.py can show that the constructed cases of tests/search_cases.py tell it apart:

    thr_high_index       of the keys equal to the 2 nb-th largest, those of the highest flat indices are taken
    run_desc             the running choice breaks ties by descending position
    merge_cand_first     the finished merge ranks the step's candidates before the kept hypotheses on ties
    penalty_at_t         finished scores divided by t ** lp instead of (t + 1) ** lp (1 at t = 0)
    heuristic_prev       the early-stop heuristic tests the finished set of the step before
    fin_wrong_lineage    a finished hypothesis copies its tokens from the next beam's row, not its parent's
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional

import torch

MASK = -1.0e9


DEFECTS = ("thr_high_index", "run_desc", "merge_cand_first", "penalty_at_t", "heuristic_prev", "fin_wrong_lineage")


def _topk(x: torch.Tensor, k: int):
    """torch.topk along the last dim with ties by index ascending."""
    vals, idx = torch.sort(x, dim=-1, descending=True, stable=True)
    return vals[..., :k], idx[..., :k]


def _topk_desc(x: torch.Tensor, k: int):
    """torch.topk along the last dim with ties by index descending."""
    n = x.shape[-1]
    vals, idx = torch.sort(x.flip(-1), dim=-1, descending=True, stable=True)
    return vals[..., :k], (n - 1 - idx)[..., :k]


def _topk_thr_high(x: torch.Tensor, k: int):
    """The k largest with the ties at the k-th value taken from the highest indices, then ranked (value desc, index
    asc) like _topk."""
    sel = _topk_desc(x, k)[1].sort(-1).values
    vals, order = torch.sort(torch.gather(x, -1, sel), dim=-1, descending=True, stable=True)
    return vals, torch.gather(sel, -1, order)


def _gather(t: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    while idx.dim() < t.dim():
        idx = idx.unsqueeze(-1)
    return torch.gather(t, 1, idx.expand(*idx.shape[:2], *t.shape[2:]))


@dataclass
class SearchStats:
    steps: int = 0
    finish_lengths: set = field(default_factory=set)   # generated lengths of hypotheses that entered a finished set
    heuristic_done_step: List[Optional[int]] = field(default_factory=list)  # per state: step its heuristic turned
    ended_by: str = ""                                  # "heuristic", "max_length" or "eos" (greedy)
    # per state: the smallest decision margin of its search, each gap divided by the weight of the summed log-probs
    # in the scores it separates (n for a running score, n ** (1 - length_penalty) for a finished one), so it
    # compares with a per-step log-prob error.  Beam search: the gaps at the
    # nb / nb + 1 boundary of the running choice and of the finished merge, between the returned hypotheses, and the
    # early-stop test; greedy: the top-1 / top-2 logit gap of each step.
    margins: List[float] = field(default_factory=list)


def _gap(sorted_vals: torch.Tensor, i: int) -> float:
    """sorted_vals[i] - sorted_vals[i + 1], or inf where either side carries a -1e9 mask."""
    if i + 1 >= sorted_vals.shape[-1]:
        return float("inf")
    a, b = float(sorted_vals[i]), float(sorted_vals[i + 1])
    return float("inf") if b < MASK / 2 or a < MASK / 2 else a - b


def beam_search(step_fn: Callable, batch: int, num_beams: int, num_return: int, max_length: int,
                length_penalty: float, eos: int, pad: int, start: int, stats: Optional[SearchStats] = None,
                defect: Optional[str] = None):
    """(sequences [batch * num_return, L_out] int64, sequences_scores [batch * num_return] fp32)."""
    assert defect is None or defect in DEFECTS, defect
    B, nb = batch, num_beams
    fill = pad or eos
    cur_len = 1
    running = torch.full((B, nb, max_length), fill, dtype=torch.int64)
    running[:, :, 0] = start
    sequences = running.clone()
    running_scores = torch.zeros(B, nb)
    running_scores[:, 1:] = MASK
    beam_scores = torch.full((B, nb), MASK)
    is_finished = torch.zeros(B, nb, dtype=torch.bool)
    unsat = torch.ones(B, 1, dtype=torch.bool)
    gen_len = torch.zeros(B, nb, dtype=torch.int64)       # generated tokens of each finished slot
    top_mask = torch.cat([torch.ones(nb, dtype=torch.bool), torch.zeros(nb, dtype=torch.bool)])
    stats = stats if stats is not None else SearchStats()
    stats.heuristic_done_step = [None] * B
    margin = [float("inf")] * B
    t = 0
    while True:
        lp = step_fn(t, running[:, :, :cur_len].reshape(B * nb, cur_len)).float()
        V = lp.shape[-1]
        lp = lp.view(B, nb, V) + running_scores[:, :, None]
        lp = lp.reshape(B, nb * V)
        top_lp, top_idx = (_topk_thr_high if defect == "thr_high_index" else _topk)(lp, 2 * nb)
        live = unsat[:, 0].clone()
        n_terms = t + 1                                 # log-probs summed into a running score
        fin_terms = n_terms ** (1 - length_penalty)     # ... their weight in a length-penalised score
        parent = top_idx // V
        tok = top_idx % V
        top_seq = _gather(running, parent)
        top_seq[:, :, cur_len] = tok
        hits = (tok == eos) | (cur_len + 1 >= max_length)
        # running beams for the next step
        run_lp = top_lp + hits.to(torch.float32) * MASK
        nxt = (_topk_desc if defect == "run_desc" else _topk)(run_lp, nb)[1]
        for b in range(B):
            if live[b]:
                margin[b] = min(margin[b], _gap(_topk(run_lp[b], 2 * nb)[0], nb - 1) / n_terms)
        new_running = _gather(top_seq, nxt)
        new_running_scores = _gather(run_lp, nxt)
        # finished beams
        did = hits & top_mask[None, :]
        pen_len = max(cur_len - 1, 1) if defect == "penalty_at_t" else cur_len + 1 - 1
        fin = top_lp / (pen_len ** length_penalty)
        fin += (~unsat).to(torch.float32) * MASK
        fin += (~did) * MASK
        for b in range(B):
            for c in range(nb):
                if did[b, c] and unsat[b, 0]:
                    stats.finish_lengths.add(cur_len)
        fin_seq = top_seq
        if defect == "fin_wrong_lineage":
            fin_seq = _gather(running, (parent + 1) % nb)
            fin_seq[:, :, cur_len] = tok
        merged_seq = torch.cat([sequences, fin_seq], 1)
        merged_scores = torch.cat([beam_scores, fin], 1)
        merged_fin = torch.cat([is_finished, did], 1)
        merged_len = torch.cat([gen_len, torch.full((B, 2 * nb), cur_len)], 1)
        if defect == "merge_cand_first":  # the candidates first: position order [candidates, kept]
            perm = torch.cat([torch.arange(nb, 3 * nb), torch.arange(nb)])
            keep = perm[_topk(merged_scores[:, perm], nb)[1]]
        else:
            keep = _topk(merged_scores, nb)[1]
        prev_scores, prev_finished = beam_scores, is_finished
        for b in range(B):
            if live[b]:
                margin[b] = min(margin[b], _gap(_topk(merged_scores[b], 3 * nb)[0], nb - 1) / fin_terms)
        sequences = _gather(merged_seq, keep)
        beam_scores = _gather(merged_scores, keep)
        is_finished = _gather(merged_fin, keep)
        gen_len = _gather(merged_len, keep)
        running, running_scores = new_running, new_running_scores
        cur_len += 1
        t += 1
        best = running_scores[:, :1] / ((cur_len - 1) ** length_penalty)
        if defect == "heuristic_prev":
            worst = torch.where(prev_finished, torch.min(prev_scores, dim=1, keepdim=True)[0], MASK)
        else:
            worst = torch.where(is_finished, torch.min(beam_scores, dim=1, keepdim=True)[0], MASK)
        new_unsat = unsat & torch.any(best > worst, dim=-1, keepdim=True)
        for b in range(B):
            if live[b] and bool(is_finished[b].all()):
                margin[b] = min(margin[b], abs(float(best[b, 0]) - float(worst[b, 0])) / fin_terms)
        for b in range(B):
            if bool(unsat[b, 0]) and not bool(new_unsat[b, 0]):
                stats.heuristic_done_step[b] = t - 1
        unsat = new_unsat
        if bool(hits.all()):
            stats.ended_by = "max_length"
            break
        if not bool(unsat.any()):
            stats.ended_by = "heuristic"
            break
    stats.steps = t
    for b in range(B):  # the order of the returned hypotheses
        for j in range(min(num_return, nb - 1)):
            margin[b] = min(margin[b], _gap(beam_scores[b], j) / max(int(gen_len[b, j]), 1) ** (1 - length_penalty))
    stats.margins = margin
    seqs = sequences[:, :num_return].reshape(B * num_return, max_length)
    scores = beam_scores[:, :num_return].reshape(B * num_return)
    out_len = 1 + int(gen_len[:, :num_return].max())
    return seqs[:, :out_len], scores


def greedy(step_fn: Callable, batch: int, max_length: int, eos: int, pad: int, start: int,
           stats: Optional[SearchStats] = None):
    """HF `_sample` with do_sample=False: sequences [batch, L_out] int64."""
    ids = torch.full((batch, 1), start, dtype=torch.int64)
    unfinished = torch.ones(batch, dtype=torch.int64)
    stats = stats if stats is not None else SearchStats()
    margin = [float("inf")] * batch
    t = 0
    while True:
        logits = step_fn(t, ids).float()
        top2 = torch.topk(logits, 2, dim=-1).values
        for b in range(batch):
            if unfinished[b]:
                margin[b] = min(margin[b], float(top2[b, 0] - top2[b, 1]))
        nxt = torch.argmax(logits, dim=-1)  # the first maximum: the lowest id on ties
        nxt = nxt * unfinished + pad * (1 - unfinished)
        ids = torch.cat([ids, nxt[:, None]], -1)
        done = (nxt == eos) | (ids.shape[1] >= max_length)
        unfinished = unfinished & ~done
        t += 1
        if int(unfinished.max()) == 0:
            stats.ended_by = "max_length" if ids.shape[1] >= max_length else "eos"
            break
    stats.steps = t
    stats.margins = margin
    return ids
