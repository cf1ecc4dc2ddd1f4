"""The search step on constructed logits (tests/search_cases.py), run through `rpx_debug_search`, which launches the
init, step and finish kernels with the arguments `rpx_seq2seq_generate` builds, without a decoder.

Log-softmax.  The beam step computes, per row of fp32 logits x over V entries,
    mx = max_j x_j (exact),  d_j = fl64(x_j - mx),  s = sum_j exp(d_j) in fp64 (lane-strided, then a xor tree),
    lp_j = fp32(fl64(d_j - fl64(log s))).
With u = 2^-53 and gamma_n = n u / (1 - n u):
  - d_j rounds once: |d_j - (x_j - mx)| <= u |x_j - mx|.  Through exp that moves term j by at most
    e^{d_j} u |d_j| <= u / e (x e^-x <= 1/e), so the sum by at most V u / e;
  - exp is correctly rounded to within 1 ulp (CUDA C++ Programming Guide, double-precision functions): 2u relative;
  - the fp64 sum of V non-negative terms in any order errs by gamma_{V-1} relative;
  - s >= 1 (the maximum's term is exp(0) = 1), so log s moves by at most rho (1 + rho) with
    rho = gamma_{V-1} + 2u + V u / e, and log itself adds 1 ulp, 2u log s;
  - the final subtraction rounds once more: u |lp|.
    delta_k = u |x_j - mx| + 1.001 rho + 2.002 u log s + u (|x_j - mx| + log s + 1).
The float64 reference (torch.log_softmax) is computed the same way and errs by at most as much, so the traced fp32
value must lie in [fp32(ref - 2 delta_k), fp32(ref + 2 delta_k)], both ends rounded to nearest as the kernel's last
step rounds: equality with fp32(ref) away from a rounding boundary, and no empirical floor.

Bookkeeping.  The traced log-probs fed to tests/beam_ref.py must give the engine's sequences and scores exactly
(torch.equal), its step count and its output length; the rows a step traces must be exactly those of the states
whose search had not ended."""
import ctypes as C
import math

import pytest
import torch

from reprover_b200 import _native
from tests import beam_ref
from tests import search_cases as SC

pytestmark = pytest.mark.gpu
U64 = 2.0 ** -53


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _run(lib, case, x, dev):
    """rpx_debug_search on logits x [ML - 1, R, V]: sequences [B n_ret, out_len], scores, steps, out_len, the trace
    [ML - 1, R, V] (NaN rows: not traced), all on the host; sentinels past every output checked."""
    B, nb, V, ML, n_ret = case.B, case.nb, case.V, case.ML, case.n_ret
    R = B * nb
    assert x.shape == (ML - 1, R, V)
    d_x = x.to(dev).contiguous()
    need = lib.rpx_debug_search_workspace_bytes(B, nb, ML)
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    seqs = torch.full((B * n_ret * ML + 16,), -7, dtype=torch.int64, device=dev)
    scores = torch.full((B * n_ret + 4,), float("nan"), device=dev) if nb > 1 else None
    tr_s = torch.full((ML - 1, R, V), float("nan"), device=dev)
    tr_p = torch.full((ML - 1, R), -1, dtype=torch.int32, device=dev)
    tr_t = torch.full((ML - 1, R), -1, dtype=torch.int32, device=dev)
    trace = _native.GenerateTrace(tr_s.data_ptr(), tr_p.data_ptr(), tr_t.data_ptr(), ML - 1)
    out_len, steps = C.c_int32(0), C.c_int32(0)
    _native.check(lib.rpx_debug_search(d_x.data_ptr(), B, nb, V, n_ret, ML, case.lp, SC.EOS, SC.START, seqs.data_ptr(),
                                       None if scores is None else scores.data_ptr(), C.byref(out_len),
                                       C.byref(steps), C.byref(trace), ws.data_ptr(), need, _stream()))
    torch.cuda.synchronize()
    n = B * n_ret * ML
    assert bool((seqs[n:] == -7).all()), "wrote past the sequences"
    full = seqs[:n].view(B * n_ret, ML).cpu()
    L = out_len.value
    assert 2 <= L <= ML
    fill = SC.EOS if (nb > 1 and SC.START == 0) else SC.START
    assert bool((full[:, L:] == fill).all()), "columns past out_len must hold the fill id"
    res = {"seqs": full[:, :L], "steps": steps.value, "out_len": L, "trace": tr_s.cpu(), "parents": tr_p.cpu(),
           "tokens": tr_t.cpu(), "scores": None}
    if scores is not None:
        assert bool(scores[B * n_ret:].isnan().all()), "wrote past the scores"
        res["scores"] = scores[:B * n_ret].cpu()
    return res


def _delta(x: torch.Tensor) -> torch.Tensor:
    """2 delta_k of the module docstring, per element of logits x [..., V] (float64)."""
    V = x.shape[-1]
    x = x.double()
    d = (x - x.amax(-1, keepdim=True)).abs()
    log_s = torch.logsumexp(x, -1, keepdim=True) - x.amax(-1, keepdim=True)
    gamma = (V - 1) * U64 / (1 - (V - 1) * U64)
    rho = gamma + 2 * U64 + V * U64 / math.e
    return 2 * (U64 * d + 1.001 * rho + 2.002 * U64 * log_s + U64 * (d + log_s + 1))


def _check_log_softmax(got: torch.Tensor, x: torch.Tensor):
    """Traced fp32 log-probs got [n, V] against the float64 log_softmax of logits x [n, V]: the fp32 bracket."""
    ref = torch.log_softmax(x.double(), -1)
    dl = _delta(x)
    lo, hi = (ref - dl).float(), (ref + dl).float()
    bad = ~((got >= lo) & (got <= hi))
    assert not bool(bad.any()), (int(bad.sum()), bad.nonzero()[:4].tolist(),
                                 [(float(got[tuple(i)]), float(ref[tuple(i)])) for i in bad.nonzero()[:4].tolist()])


def _live_rows(case, last_step):
    """[ML - 1, R] bool: rows of states whose search had not ended before step t (last_step[b]: its final step)."""
    live = torch.zeros(case.ML - 1, case.B * case.nb, dtype=torch.bool)
    for b, e in enumerate(last_step):
        e = case.ML - 2 if e is None else e
        live[: e + 1, b * case.nb:(b + 1) * case.nb] = True
    return live


def _bookkeeping(lib, case, x, dev):
    """Run the case, check the log-softmax of every traced row, replay the traced log-probs through beam_ref."""
    got = _run(lib, case, x, dev)
    tr = got["trace"]
    traced = ~tr.isnan().any(-1)
    _check_log_softmax(tr[traced], x[traced])
    scores = torch.where(traced[..., None], tr, SC.host_logprobs(x))
    st = beam_ref.SearchStats()
    want, want_scores = SC.reference(case, scores, stats=st)
    assert torch.equal(got["seqs"], want), case.name
    assert torch.equal(got["scores"], want_scores), case.name
    assert got["steps"] == st.steps and got["out_len"] == want.shape[1]
    assert torch.equal(traced, _live_rows(case, st.heuristic_done_step)), "a finished state's step did not return"
    return got, st


@pytest.mark.parametrize("case", SC.BEAM_CASES, ids=lambda c: c.name)
def test_bookkeeping_against_beam_ref(rpx_lib, cuda_device, case):
    _bookkeeping(rpx_lib, case, case.logits(), cuda_device)


def test_log_softmax_bound_on_extreme_rows(rpx_lib, cuda_device):
    """One step (max_length 2) over 5 states of 8 beams, every row traced: all-equal rows (exactly -log V), one
    dominant entry (the other terms underflow), spreads of +-1e4 and +-1e8, and rows of N(0, 1)."""
    case = SC.Case("extreme", 5, 8, 384, 2, 1.0, 8, 0)
    g = torch.Generator().manual_seed(50)
    x = torch.randn(1, 40, 384, generator=g)
    x[0, 0:4] = torch.tensor([0.0, 7.5, -3.25, 1e6])[:, None]              # all equal
    x[0, 4:8, 17] += torch.tensor([50.0, 200.0, 1e4, 1e8])                  # one dominant entry
    x[0, 8:16] = (torch.rand(8, 384, generator=g) * 2 - 1) * 1e4            # spread +-1e4
    x[0, 16:24] = (torch.rand(8, 384, generator=g) * 2 - 1) * 1e8           # spread +-1e8
    x[0, 24:28] = torch.randn(4, 384, generator=g) * 1e4
    got = _run(rpx_lib, case, x, cuda_device)
    tr = got["trace"][0]
    assert not bool(tr.isnan().any()), "every row of a live state is traced"
    _check_log_softmax(tr, x[0])
    want = torch.tensor(-math.log(384.0)).float()
    assert bool((tr[0:4] == want).all()), "all-equal rows must give fp32(-log V)"
    assert bool((tr[5:8, 17] == 0).all()), "the dominant entry's log-prob rounds to 0 once the others underflow"
    assert bool((tr[6:8].sort(-1, descending=True).values[:, 1] <= -1e4 + 10).all())


def test_vocab_limits_at_128_beams(rpx_lib, cuda_device):
    """nb V 4 bytes of keys must fit beside the step's static arrays: V = 416 runs at nb = 128 (a case above), V = 448
    is refused as the engine refuses it, and 2 nb > V is invalid."""
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device=cuda_device)
    p = buf.data_ptr()
    out_len, steps = C.c_int32(0), C.c_int32(0)

    def call(V, nb=128):
        return rpx_lib.rpx_debug_search(p, 1, nb, V, 1, 4, 1.0, SC.EOS, SC.START, p, p, C.byref(out_len),
                                        C.byref(steps), None, p, buf.numel(), _stream())

    assert call(448) == _native.RPX_ERR_UNSUPPORTED and "shared memory" in _native.last_error()
    assert call(255) == _native.RPX_ERR_INVALID
    torch.cuda.synchronize()
    assert int(buf.count_nonzero()) == 0, "a refused call wrote to the device"


ISOLATION_CASES = [c for c in SC.BEAM_CASES if c.name in (
    "eos_pressure_B5_nb8_V384_ML40_lp1_ret8", "eos_pressure_B5_nb64_V384_ML40_lp0_ret64",
    "identical_B5_nb3_V256_ML40_lp-0.5_ret3", "eos_pressure_B5_nb2_V384_ML40_lp-0.5_ret1")]


@pytest.mark.parametrize("case", ISOLATION_CASES, ids=lambda c: c.name)
def test_finished_state_isolation(rpx_lib, cuda_device, case):
    """After a state's search ends (its last step from beam_ref), NaN or +1e30 logits in its rows at every later step
    leave every output bit-identical; and each state alone gives what it gives inside the batch of five."""
    x = case.logits()
    base, st = _bookkeeping(rpx_lib, case, x, cuda_device)
    last = st.heuristic_done_step
    assert any(e < case.ML - 2 for e in last), last
    nb, n_ret = case.nb, case.n_ret
    for poison in (float("nan"), 1e30):
        y = x.clone()
        for b, e in enumerate(last):
            y[e + 1:, b * nb:(b + 1) * nb] = poison
        got = _run(rpx_lib, case, y, cuda_device)
        assert torch.equal(got["seqs"], base["seqs"]) and torch.equal(got["scores"], base["scores"]), poison
        assert got["steps"] == base["steps"]
    for b in range(case.B):
        one = SC.Case(case.family, 1, nb, case.V, case.ML, case.lp, n_ret, case.seed)
        got = _run(rpx_lib, one, x[:, b * nb:(b + 1) * nb].contiguous(), cuda_device)
        rows = slice(b * n_ret, (b + 1) * n_ret)
        L = got["out_len"]
        assert torch.equal(got["seqs"], base["seqs"][rows, :L]), b
        assert bool((base["seqs"][rows, L:] == SC.EOS).all()), b
        assert torch.equal(got["scores"], base["scores"][rows]), b
        assert got["steps"] == last[b] + 1, b


@pytest.mark.parametrize("case", SC.GREEDY_CASES, ids=lambda c: c.name)
def test_greedy(rpx_lib, cuda_device, case):
    """Lowest id on ties (across lanes, warps and the 256-thread stride), -inf and all-equal rows, EOS at t = 0 and
    max_length 2, rows ending at different steps; every traced row is the logits row bit for bit, and exactly the rows
    still running are traced."""
    x = case.logits()
    got = _run(rpx_lib, case, x, cuda_device)
    st = beam_ref.SearchStats()
    want, _ = SC.reference(case, x, stats=st)
    assert torch.equal(got["seqs"], want)
    assert got["steps"] == st.steps and got["out_len"] == want.shape[1]
    assert got["scores"] is None
    tr = got["trace"]
    traced = ~tr.isnan().any(-1)
    assert torch.equal(tr[traced].view(torch.int32), x[traced].view(torch.int32)), "traced logits differ"
    ends = []
    for r in range(case.B):
        e = (want[r, 1:] == SC.EOS).nonzero()
        ends.append(int(e[0]) if len(e) else case.ML - 2)
    live = torch.stack([torch.tensor([t <= e for e in ends]) for t in range(case.ML - 1)])
    assert torch.equal(traced, live), "a finished row's step did not return"
    wide = torch.full((case.B, case.ML), SC.START, dtype=torch.int64)
    wide[:, :want.shape[1]] = want
    assert torch.equal(got["tokens"][traced].long(), wide[:, 1:].t()[traced])


def test_greedy_nan_rows_follow_torch_argmax(rpx_lib, cuda_device):
    """HF's greedy step is torch.argmax: a NaN is above every number, the first NaN wins; an all-NaN row gives id 0."""
    case = SC.Case("greedy_nan", 6, 1, 384, 3, 1.0, 1, 0)
    g = torch.Generator().manual_seed(51)
    x = torch.randn(2, 6, 384, generator=g)
    nan = float("nan")
    x[:, 0, [300, 5]] = nan                 # first NaN: 5
    x[:, 1, :] = nan                        # all NaN: 0
    x[:, 2, 383] = nan                      # the last id
    x[:, 3, :] = math.inf
    x[:, 3, [40, 290]] = nan                # NaN above +inf: 40
    x[:, 4, 256 + 7] = nan                  # past the 256-thread stride
    x[:, 4, 7] = 1e30
    x[:, 5, 33] = 1e30                      # no NaN: the maximum
    got = _run(rpx_lib, case, x, cuda_device)
    first = got["seqs"][:, 1]
    assert first.tolist() == [5, 0, 383, 40, 263, 33]
    assert torch.equal(first, torch.argmax(x[0], -1))
    want = beam_ref.greedy(lambda t, prefixes: x[t], case.B, case.ML, SC.EOS, SC.START, SC.START)
    assert torch.equal(got["seqs"], want)
