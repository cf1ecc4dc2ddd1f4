"""The epilogue checker of tests/gemm_ref.py, tested on the CPU: a straightforward fp32 implementation of each
encoder GEMM epilogue passes it, and each subtle defect a kernel could have fails it.  This is how the suite
shows that the GPU epilogue tests would catch such an error, without running anything faulty on a GPU."""
import math

import pytest
import torch

from tests import gemm_ref as R

T, PAD = 150, 3  # two 128-row tiles, the second ragged; PAD sentinel rows below the output
D, INNER, F = 192, 64, 256  # d_model with a 64-column tail tile on the throughput path; 2 x 128 hidden units
EPS = float(torch.tensor(1e-6, dtype=torch.float32))

DEFECTS = {
    # defect: sites it applies to
    "swap_rows_r_r8": ("qkv", "oproj", "ffn_up", "ffn_down"),
    "drop_kblock": ("qkv", "oproj", "ffn_up", "ffn_down"),
    "neighbour_row_scale": ("qkv", "ffn_up"),
    "swap_gate_linear_8cols": ("ffn_up",),
    "ss_part_to_neighbour_slot": ("oproj", "ffn_down"),
    "bf16_truncation": ("qkv", "oproj", "ffn_up", "ffn_down"),
    "tail_column_written": ("qkv", "oproj", "ffn_up", "ffn_down"),
}


def _data(site, seed=0):
    g = torch.Generator().manual_seed(seed)
    K = {"qkv": D, "oproj": INNER, "ffn_up": D, "ffn_down": F}[site]
    N = {"qkv": 3 * INNER, "oproj": D, "ffn_up": 2 * F, "ffn_down": D}[site]
    A = torch.randn(T, K, generator=g).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(torch.bfloat16)
    # row scales that differ by up to 4x between rows
    ms = torch.exp(torch.empty(T).uniform_(math.log(1 / 4), math.log(4), generator=g))
    return A, W, ms, g


def _ss_in(ms, latency, g):
    P = R.ss_parts(D, latency)
    w = torch.rand(P, T, generator=g) + 0.1
    return (w / w.sum(0) * ms * D).float()


def _acc(A, B, defect):
    acc = A.float() @ B.float().t()
    if defect == "swap_rows_r_r8":  # rows 3 and 11 of the second fragment of tile 0, columns 0..7
        acc[[16 + 3, 16 + 11], :8] = acc[[16 + 11, 16 + 3], :8]
    if defect == "drop_kblock":  # tile (0, 0) misses k-block 1 (or 0 when K = 64)
        kb = 1 if A.shape[1] > 64 else 0
        acc[:128, :128] -= A[:128, 64 * kb:64 * kb + 64].float() @ B[:128, 64 * kb:64 * kb + 64].float().t()
    return acc


def _rs(ss, defect):
    s = ss.sum(0)
    rs = torch.rsqrt(s * torch.tensor(1.0 / D, dtype=torch.float32) + torch.tensor(EPS, dtype=torch.float32))
    if defect == "neighbour_row_scale":
        rs[5] = rs[6]
    return rs


def _to_bf16(x, defect):
    if defect == "bf16_truncation":
        return (x.contiguous().view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)
    return x.to(torch.bfloat16)


def _nan_buffer(rows, cols, dtype):
    return torch.full((rows, cols), float("nan"), dtype=dtype)


def _tail_write(buf, n, defect):
    """The last row's tile writes one column past the matrix: in a row-major [rows, n] buffer that is
    element (T, 0), the first sentinel."""
    if defect == "tail_column_written":
        buf.view(-1)[T * n] = 1.0


def sim_qkv(A, B, ss, defect):
    acc = _acc(A, B, defect)
    out = _nan_buffer(T + PAD, B.shape[0], torch.bfloat16)
    out[:T] = _to_bf16(acc * _rs(ss, defect)[:, None], defect)
    _tail_write(out, B.shape[0], defect)
    return out


def sim_ffn_up(A, Bp, ss, defect):
    acc = _acc(A, Bp, defect)
    j = torch.arange(F)
    gate_rows = 256 * (j // 128) + j % 128
    lin_rows = gate_rows + 128
    if defect == "swap_gate_linear_8cols":
        gate_rows[40:48], lin_rows[40:48] = lin_rows[40:48].clone(), gate_rows[40:48].clone()
    rs = _rs(ss, defect)[:, None]
    x, y = acc[:, gate_rows] * rs, acc[:, lin_rows] * rs
    k0, k1 = torch.tensor(R.GELU_K0, dtype=torch.float32), torch.tensor(R.GELU_K1, dtype=torch.float32)
    gel = 0.5 * x * (1.0 + torch.tanh(k0 * (x + k1 * x * x * x)))
    out = _nan_buffer(T + PAD, F, torch.bfloat16)
    out[:T] = _to_bf16(gel * y, defect)
    _tail_write(out, F, defect)
    return out


def sim_residual(A, B, h32_in, latency, defect):
    N = B.shape[0]
    acc = _acc(A, B, defect)
    h32 = _nan_buffer(T + PAD, N, torch.float32)
    h32[:T] = h32_in + acc
    h16 = _nan_buffer(T + PAD, N, torch.bfloat16)
    h16[:T] = _to_bf16(h32[:T], defect)
    pc, P = R.part_cols(latency), R.ss_parts(N, latency)
    ss = torch.full(((P + 1) * T,), float("nan"), dtype=torch.float32)
    for p in range(P):
        blk = h32[:T, p * pc:(p + 1) * pc]
        ss[p * T:(p + 1) * T] = (blk * blk).sum(1)
    if defect == "ss_part_to_neighbour_slot":  # part 0 lands in slot 1, slot 0 is never written
        ss[T:2 * T] = ss[:T].clone()
        ss[:T] = float("nan")
    _tail_write(h32, N, defect)
    return h32, h16, ss


def run_and_check(site, latency, defect):
    """All findings (empty list: clean) of the fp32 model of `site` with `defect` injected."""
    A, W, ms, g = _data(site)
    found = []
    if site == "qkv":
        ss = _ss_in(ms, latency, g)
        out = sim_qkv(A, W, ss, defect)
        found += [R.check_qkv(out[:T], A, W, ss, D, EPS), R.check_sentinels("qkv.pad", out, T * W.shape[0], R.BF16_NAN_BITS)]
    elif site == "ffn_up":
        W0, W1 = W[:F], W[F:]
        ss = _ss_in(ms, latency, g)
        out = sim_ffn_up(A, R.pack_ffn_up(W0, W1), ss, defect)
        found += [R.check_ffn_up(out[:T], A, W0, W1, ss, D, EPS), R.check_sentinels("ffn_up.pad", out, T * F, R.BF16_NAN_BITS)]
    else:
        h32_in = torch.randn(T, W.shape[0], generator=g)
        h32, h16, ss = sim_residual(A, W, h32_in, latency, defect)
        P = R.ss_parts(W.shape[0], latency)
        found += R.check_residual(h32_in, h32[:T], h16[:T], ss[:P * T].view(P, T), A, W, latency)
        n = W.shape[0]
        found += [R.check_sentinels("h32.pad", h32, T * n, R.F32_NAN_BITS),
                  R.check_sentinels("h16.pad", h16, T * n, R.BF16_NAN_BITS),
                  R.check_sentinels("ss.pad", ss, P * T, R.F32_NAN_BITS)]
    return [f for f in found if f]


@pytest.mark.parametrize("latency", [False, True], ids=["throughput", "latency"])
@pytest.mark.parametrize("site", ["qkv", "oproj", "ffn_up", "ffn_down"])
def test_fp32_model_passes(site, latency):
    bad = run_and_check(site, latency, None)
    assert not bad, [f.summary() for f in bad]


@pytest.mark.parametrize("latency", [False, True], ids=["throughput", "latency"])
@pytest.mark.parametrize("site,defect", [(s, d) for d, sites in DEFECTS.items() for s in sites])
def test_injected_defect_is_caught(site, defect, latency):
    assert run_and_check(site, latency, defect), f"{defect} in the {site} epilogue went unnoticed"


def test_pack_ffn_up_matches_the_documented_layout():
    W0 = torch.arange(384 * 2, dtype=torch.float32).reshape(384, 2)
    W1 = -W0
    P = R.pack_ffn_up(W0, W1)
    for j in (0, 127, 128, 255, 383):
        assert torch.equal(P[256 * (j // 128) + j % 128], W0[j])
        assert torch.equal(P[256 * (j // 128) + 128 + j % 128], W1[j])


def test_gelu_lipschitz_constant():
    x = torch.linspace(-30, 30, 600_001, dtype=torch.float64, requires_grad=True)
    R.gelu_new64(x).sum().backward()
    assert x.grad.abs().max().item() < R.GELU_LIP


def test_bf16_bracket_is_exact_away_from_boundaries():
    ref = torch.tensor([1.0 + 2 ** -9, 1.0 + 3 * 2 ** -9, 3.0], dtype=torch.float64)  # mid-ulp, mid-ulp, exact
    tol = torch.full_like(ref, 1e-6)
    exact = ref.float().to(torch.bfloat16)
    assert not R.bf16_bracket_bad(torch.tensor([3.0], dtype=torch.bfloat16), ref[2:], tol[2:]).any()
    # within tol of a tie: either neighbour is accepted; 1 ulp further is not
    both = R.bf16_bracket_bad(torch.tensor([1.0, 1.0 + 2 ** -8], dtype=torch.bfloat16), ref[:1].expand(2), tol[:1].expand(2))
    assert not both.any()
    assert R.bf16_bracket_bad(torch.tensor([1.0 + 2 ** -7], dtype=torch.bfloat16), ref[:1], tol[:1]).all()
    off = R.bf16_bracket_bad(exact[2:] + 2 ** -6, ref[2:], tol[2:])
    assert off.all()
