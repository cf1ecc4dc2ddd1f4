"""The per-token checker of tests/hidden_ref.py, tested on the CPU: a straightforward fp32 implementation of the
final-norm store (`hidden_store_kernel`) passes it, and each defect such a kernel could have fails it.  This is
how the suite shows that the GPU tests of `rpx_encode_ids_hidden` would catch such an error."""
import math

import pytest
import torch

from tests import gemm_ref as R
from tests import hidden_ref as H

D = 192  # a 64-column last part on the throughput path, like d_model 1472
LENS = [5, 1, 9, 3]
L = 9  # the longest row; the others are padded
PAD = 2  # sentinel rows past batch * seq_len
EPS = float(torch.tensor(1e-6, dtype=torch.float32))

DEFECTS = ("rows_shifted", "padded_row_not_zero", "weight_missing", "neighbour_row_scale", "last_ss_part_dropped")


def _data(seed=0):
    g = torch.Generator().manual_seed(seed)
    T = sum(LENS)
    # row magnitudes that differ by up to 4x, so a neighbour's row scale is visibly wrong
    scale = torch.exp(torch.empty(T, 1).uniform_(math.log(1 / 4), math.log(4), generator=g))
    h32 = (torch.randn(T, D, generator=g) * scale).float()
    ln_w = (torch.rand(D, generator=g) + 0.5).float()
    return h32, ln_w


def _ss_parts(h32, latency):
    pc, P = R.part_cols(latency), R.ss_parts(D, latency)
    return torch.stack([(h32[:, q * pc:(q + 1) * pc] ** 2).sum(1) for q in range(P)])  # fp32 [P, T]


def sim_store(h32, ln_w, latency, dtype, defect):
    """fp32 model of hidden_store_kernel writing into a NaN-filled buffer of B * L + PAD rows."""
    ss = _ss_parts(h32, latency)
    if defect == "last_ss_part_dropped":
        ss = ss[:-1]
    total = torch.zeros(ss.shape[1], dtype=torch.float32)
    for q in range(ss.shape[0]):
        total = total + ss[q]
    rs = torch.rsqrt(total * torch.tensor(1.0 / D, dtype=torch.float32) + torch.tensor(EPS, dtype=torch.float32))
    if defect == "neighbour_row_scale":
        rs[6] = rs[7]
    y = h32 * rs[:, None]
    if defect != "weight_missing":
        y = y * ln_w
    B = len(LENS)
    out = torch.full((B * L + PAD, D), float("nan"), dtype=dtype)
    t0 = 0
    for b, n in enumerate(LENS):
        for p in range(L):
            row = b * L + p
            if p < n:
                t = min(t0 + p + 1, len(y) - 1) if defect == "rows_shifted" else t0 + p
                out[row] = y[t].to(dtype)
            elif defect != "padded_row_not_zero":
                out[row] = 0
        t0 += n
    return out


def run_and_check(latency, dtype, defect):
    h32, ln_w = _data()
    buf = sim_store(h32, ln_w, latency, dtype, defect)
    B = len(LENS)
    found = H.check_hidden(buf[:B * L].view(B, L, D), h32, ln_w, LENS, EPS, R.ss_parts(D, latency))
    nan_bits = R.BF16_NAN_BITS if dtype == torch.bfloat16 else R.F32_NAN_BITS
    found.append(R.check_sentinels("hidden.past_end", buf, B * L * D, nan_bits))
    return [f for f in found if f]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("latency", [False, True], ids=["throughput", "latency"])
def test_fp32_model_passes(latency, dtype):
    bad = run_and_check(latency, dtype, None)
    assert not bad, [f.summary() for f in bad]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("latency", [False, True], ids=["throughput", "latency"])
@pytest.mark.parametrize("defect", DEFECTS)
def test_injected_defect_is_caught(defect, latency, dtype):
    assert run_and_check(latency, dtype, defect), f"{defect} in the hidden-state store went unnoticed"


def test_engine_config_reads_like_an_hf_config():
    """`encoder.config.hidden_size` (retrieval/model.py:90) on the dict the rest of the package reads."""
    from reprover_b200.engine import EncoderConfig, EncoderOutput

    cfg = EncoderConfig({"d_model": 1472, "num_layers": 12})
    assert cfg.hidden_size == 1472 and cfg.d_model == 1472 and cfg["num_layers"] == 12
    assert isinstance(cfg, dict) and dict(cfg) == {"d_model": 1472, "num_layers": 12}
    with pytest.raises(AttributeError):
        cfg.vocab_size
    out = EncoderOutput(torch.zeros(1, 2, 3))
    assert out[0] is out.last_hidden_state
