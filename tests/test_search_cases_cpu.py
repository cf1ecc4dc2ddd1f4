"""The constructed search cases of tests/search_cases.py can fail: for every bookkeeping defect that
tests/beam_ref.py can plant, at least one case the GPU suite runs (tests/test_search_step_gpu.py) gives other sequences
or scores than the defect-free search, on the host log-probs (fp32 rounding of a float64 log_softmax).  Also that
the families reach the endings they are built for."""
import pytest
import torch

from tests import beam_ref
from tests import search_cases as SC


@pytest.fixture(scope="module")
def beam_runs():
    runs = []
    for case in SC.BEAM_CASES:
        lp = SC.host_logprobs(case.logits())
        st = beam_ref.SearchStats()
        runs.append((case, lp, SC.reference(case, lp, stats=st), st))
    return runs


def _differs(a, b):
    (sa, ca), (sb, cb) = a, b
    return sa.shape != sb.shape or not torch.equal(sa, sb) or not torch.equal(ca, cb)


@pytest.mark.parametrize("defect", beam_ref.DEFECTS)
def test_every_defect_changes_some_case(beam_runs, defect):
    caught = [case.name for case, lp, want, _ in beam_runs if _differs(SC.reference(case, lp, defect=defect), want)]
    assert caught, f"no case tells {defect} apart"


def test_cases_reach_their_endings(beam_runs):
    """In one eos_pressure batch some states end by the heuristic and others run to max_length; hypotheses finish at
    many lengths; the parent_churn search of max_length 512 runs all 511 steps."""
    by_name = {case.name: (case, st) for case, _, _, st in beam_runs}
    case, st = by_name["eos_pressure_B5_nb8_V384_ML40_lp1_ret8"]
    last = st.heuristic_done_step
    assert any(s < case.ML - 2 for s in last) and any(s == case.ML - 2 for s in last), last
    assert len(st.finish_lengths) >= 20
    case, st = by_name["parent_churn_B1_nb8_V384_ML512_lp2_ret8"]
    assert st.steps == 511 and max(st.finish_lengths) > 32


def test_exact_levels_are_exact():
    """The exact_levels log-probs are 0 and multiples of -1e4 in fp32, so sums of them tie exactly."""
    x = SC.exact_levels(2, 3, 384, 5, 0)
    lp = SC.host_logprobs(x)
    assert torch.equal(lp, x)
    assert bool(((lp == 0).sum(-1) == 1).all())


def test_greedy_cases_hit_ties_and_end_at_different_steps():
    case = SC.GREEDY_CASES[0]
    x = case.logits()
    st = beam_ref.SearchStats()
    seqs, _ = SC.reference(case, x, stats=st)
    ends = [(row[1:] == SC.EOS).nonzero() for row in seqs]
    first = sorted({int(e[0]) for e in ends if len(e)})
    assert first[:3] == [0, 1, 2] and len(first) >= 10, first
    # a row whose maximum ties at ids j, j + 32, j + 256 takes j
    t, r = 0, 0
    while not ((x[t, r] == x[t, r].max()).sum() == 3):
        r += 1
    ids = (x[t, r] == x[t, r].max()).nonzero().flatten().tolist()
    assert ids[1] - ids[0] == 32 and ids[2] - ids[0] == 256 and int(torch.argmax(x[t, r])) == ids[0]
