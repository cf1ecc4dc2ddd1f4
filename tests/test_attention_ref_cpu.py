"""The attention checker (tests/attention_ref.py) is neither too loose nor too tight: a plain fp32 model of
t5_attention_kernel passes it, and the same model with one injected defect fails it.

The model follows the kernel step by step: 64-key steps, an online softmax in fp32 with the exponent argument
fmaf(s, L2E, -fl(m L2E)) and the rescale exp2((m_old - m_new) L2E), P rounded to bf16 before the PV product
while l sums the fp32 values, keys past the end of the packed buffer read as zeros (TMA zero fill), and the
output o * (1 / l) rounded to bf16 into a NaN-filled buffer with two spare rows.  Each defect case is built so
that the defect moves some output far outside the tolerance by construction; the test says why."""
import math

import pytest
import torch

from tests import attention_ref as A

PAD = 2


def _trunc_bf16(x: torch.Tensor) -> torch.Tensor:
    return (x.contiguous().view(torch.int32) & ~0xFFFF).view(torch.float32)


def model(qkv, cu, H, lut, R, defect=None):
    """fp32 model of the kernel; `defect` names one injected bug."""
    T = qkv.shape[0]
    inner = H * A.HD
    out = torch.full((T + PAD, inner), math.nan, dtype=torch.bfloat16)
    xz = torch.cat([qkv.float(), torch.zeros(A.KT + 1, 3 * inner)])  # rows past T read as zeros
    lut = lut.float()
    l2e = A.L2E
    for s_i in range(len(cu) - 1):
        t0, L = cu[s_i], cu[s_i + 1] - cu[s_i]
        n_keys = L + 1 if defect == "mask_admits_len" else (L - 1 if defect == "mask_drops_last" else L)
        qpos = torch.arange(L)
        for h in range(H):
            hk = (h + 1) % H if defect == "k_neighbour_head" else h
            q = xz[t0:t0 + L, h * 64:(h + 1) * 64]
            m = torch.full((L,), -math.inf)
            l = torch.zeros(L)
            o = torch.zeros(L, 64)
            for kb in range(0, L, A.KT):
                keys = torch.arange(kb, kb + A.KT)
                k = xz[t0 + kb:t0 + kb + A.KT, inner + hk * 64:inner + (hk + 1) * 64]
                v = xz[t0 + kb:t0 + kb + A.KT, 2 * inner + h * 64:2 * inner + (h + 1) * 64]
                s = q @ k.t()
                if defect == "scaled_scores":
                    s = s / 8
                delta = keys[None, :] - qpos[:, None]
                if defect == "bias_plus1":
                    delta = delta + 1
                elif defect == "bias_minus1":
                    delta = delta - 1
                elif defect == "bias_sign":
                    delta = -delta
                hi = R - 1 if defect == "lut_clamp_r_minus_1" else R
                idx = delta.clamp(-hi, hi) + R
                s = s + lut[h][idx]
                s = torch.where(keys[None, :] < n_keys, s, torch.full_like(s, -math.inf))
                mn = torch.maximum(m, s.amax(1))
                scale = torch.exp2((m - mn) * l2e)
                mb = (mn * l2e)[:, None]
                p = (s.double() * l2e - mb.double()).float()  # fmaf: one rounding
                p = torch.exp2(p)
                l = (l if defect == "l_no_rescale" else l * scale) + p.sum(1)
                if defect != "o_no_rescale":
                    o = o * scale[:, None]
                pb = _trunc_bf16(p) if defect == "p_truncated" else p.to(torch.bfloat16).float()
                o = o + pb @ v
                m = mn
            res = (o * (1.0 / l)[:, None]).to(torch.bfloat16)
            if defect == "swap_fragment_rows":
                perm = torch.arange(L) ^ 8
                ok = perm < L
                res = torch.where(ok[:, None], res[perm.clamp(max=L - 1)], res)
            out[t0:t0 + L, h * 64:(h + 1) * 64] = res
    return out


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return cu


def _fails(out, qkv, cu, H, lut, R):
    return any(f for f in A.check_attention(out, qkv, cu, H, lut, R))


# ----------------------------------------------------------------------------------------------- cases
def case_random(seed=0, lens=(1, 63, 64, 65, 130), H=3, buckets=32, R=128):
    """Random q / k / v with flat and sharp rows, the HF bias table of a random relative_attention_bias."""
    g = torch.Generator().manual_seed(seed)
    cu = _cu(lens)
    qkv = A.random_qkv(cu[-1], H, g)
    rel = torch.randn(buckets, H, generator=g) * 2
    return qkv, cu, H, A.hf_bias_lut(rel, buckets, R), R


def _zeros_case(lens, H, R, seed):
    g = torch.Generator().manual_seed(seed)
    cu = _cu(lens)
    qkv = torch.zeros(cu[-1], 3 * H * 64)
    qkv[:, 2 * H * 64:] = torch.randn(cu[-1], H * 64, generator=g)
    return qkv, cu, g


def case_ladder():
    """q = k = 0: the scores are the bias alone.  Every head's LUT is a shuffled ladder with steps of 0.5, so
    reading any entry other than the right one (delta +- 1, -delta, delta clamped at R - 1 for |delta| >= R)
    scales some key's weight by at least e^0.5 in rows of up to 130 keys with v ~ N(0, 1)."""
    H, R = 2, 8
    qkv, cu, g = _zeros_case((1, 20, 65, 130), H, R, 1)
    lut = torch.stack([torch.randperm(2 * R + 1, generator=g).double() * 0.5 - R / 2 for _ in range(H)])
    return qkv.to(torch.bfloat16), cu, H, lut, R


def case_flat_marked():
    """q = k = 0 and a zero bias: every row averages v over its keys uniformly.  The first key of every
    sequence carries v = 32 and the last v = -32, so admitting key len (the next sequence's first key, or a
    zero row past the buffer) or dropping key len - 1 moves every output of a row of len <= 130 keys by at
    least 32 / 131 (a 1-token sequence that drops its only key gives 0 / 0)."""
    H, R = 2, 8
    qkv, cu, _ = _zeros_case((1, 20, 65, 130, 7), H, R, 2)
    for s in range(len(cu) - 1):
        qkv[cu[s], 2 * H * 64:] = 32
        if cu[s + 1] - cu[s] > 1:
            qkv[cu[s + 1] - 1, 2 * H * 64:] = -32
    return qkv.to(torch.bfloat16), cu, H, torch.zeros(H, 2 * R + 1, dtype=torch.float64), R


def case_rising_max():
    """Keys 0-63 score 0 (k = 0, v = 1), keys 64-129 score 16 (k = 4 e_0 against q = 4 e_0, v = 2): every row's
    maximum rises by 16 in the second key step, and the answer is 2 to within e^-16.  Without the rescale of o
    the first step's 64 unit values stay in the sum (~2.97); without that of l the sum is divided by ~130
    instead of 66 (~1.02); scores scaled by 1/8 give the first step a weight of e^-2 (~1.88)."""
    H, R = 2, 8
    lens = (65, 130)
    cu = _cu(lens)
    qkv = torch.zeros(cu[-1], 3 * H * 64)
    for h in range(H):
        qkv[:, h * 64] = 4
        for s in range(len(lens)):
            t0 = cu[s]
            qkv[t0 + 64:cu[s + 1], H * 64 + h * 64] = 4
            qkv[t0:t0 + 64, 2 * H * 64 + h * 64:2 * H * 64 + (h + 1) * 64] = 1
            qkv[t0 + 64:cu[s + 1], 2 * H * 64 + h * 64:2 * H * 64 + (h + 1) * 64] = 2
    return qkv.to(torch.bfloat16), cu, H, torch.zeros(H, 2 * R + 1, dtype=torch.float64), R


def case_head_routing():
    """Head h's keys are zero except key h (k = 4 e_0 against q = 4 e_0: a margin of 16), and v_j = j + 1 in
    every column: head h outputs h + 1, and K taken from head h + 1 outputs h + 2."""
    H, R = 3, 8
    cu = _cu((20,))
    qkv = torch.zeros(20, 3 * H * 64)
    for h in range(H):
        qkv[:, h * 64] = 4
        qkv[h, H * 64 + h * 64] = 4
        qkv[:, 2 * H * 64 + h * 64:2 * H * 64 + (h + 1) * 64] = torch.arange(1, 21, dtype=torch.float32)[:, None]
    return qkv.to(torch.bfloat16), cu, H, torch.zeros(H, 2 * R + 1, dtype=torch.float64), R


def case_diagonal():
    """q = k = 0 and a bias of +20 at delta = 0 only: query i attends key i (weight 1 - O(len e^-20)), and
    v_j = j + 1: row i outputs i + 1, so rows i and i ^ 8 of a fragment swapped differ by 8."""
    H, R = 2, 8
    cu = _cu((20, 70))
    qkv = torch.zeros(90, 3 * H * 64)
    for s in range(2):
        L = cu[s + 1] - cu[s]
        qkv[cu[s]:cu[s + 1], 2 * H * 64:] = torch.arange(1, L + 1, dtype=torch.float32)[:, None]
    lut = torch.zeros(H, 2 * R + 1, dtype=torch.float64)
    lut[:, R] = 20
    return qkv.to(torch.bfloat16), cu, H, lut, R


def case_truncation():
    """q = k = 0, v = 1, bias 0 at delta = 0 and b = fp32(ln(0.5 + 0.95 2^-8)) elsewhere: in every row one key
    has p = 1 and 63 have p = 0.5 + 0.95 2^-8, which rounds to bf16 0.5 + 2^-8 and truncates to 0.5.  Rounded,
    the output is 1.0004 -> 1; truncated, 32.5 / 32.73 = 0.9929 -> bf16 0.9922, below the bracket
    [bf16(1 - tol), ...] with tol ~ 2^-8 (the P-rounding term with v = 1)."""
    H, R = 1, 8
    cu = _cu((64,))
    qkv = torch.zeros(64, 3 * 64)
    qkv[:, 128:] = 1
    b = float(torch.tensor(math.log(0.5 + 0.95 * 2 ** -8), dtype=torch.float32))
    lut = torch.full((H, 2 * R + 1), b, dtype=torch.float64)
    lut[:, R] = 0
    return qkv.to(torch.bfloat16), cu, H, lut, R


CASES = {
    "random": case_random,
    "random_short_bucket_range": lambda: case_random(5, (2, 17, 64, 129), 2, 8, 4),
    "ladder": case_ladder,
    "flat_marked": case_flat_marked,
    "rising_max": case_rising_max,
    "head_routing": case_head_routing,
    "diagonal": case_diagonal,
    "truncation": case_truncation,
}

DEFECTS = {
    "bias_plus1": "ladder",
    "bias_minus1": "ladder",
    "bias_sign": "ladder",
    "lut_clamp_r_minus_1": "ladder",
    "mask_admits_len": "flat_marked",
    "mask_drops_last": "flat_marked",
    "o_no_rescale": "rising_max",
    "l_no_rescale": "rising_max",
    "scaled_scores": "rising_max",
    "k_neighbour_head": "head_routing",
    "swap_fragment_rows": "diagonal",
    "p_truncated": "truncation",
}


@pytest.mark.parametrize("name", list(CASES))
def test_fp32_model_passes(name):
    qkv, cu, H, lut, R = CASES[name]()
    out = model(qkv, cu, H, lut, R)
    stats = {}
    found = A.check_attention(out, qkv, cu, H, lut, R, stats)
    assert not any(found), [f.summary() for f in found if f]
    assert stats["max_err_over_bracket"] <= 1.0


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_injected_defect_fails(defect):
    qkv, cu, H, lut, R = CASES[DEFECTS[defect]]()
    assert not _fails(model(qkv, cu, H, lut, R), qkv, cu, H, lut, R)
    out = model(qkv, cu, H, lut, R, defect)
    found = A.check_attention(out, qkv, cu, H, lut, R)
    assert found[0], f"{defect} passed the checker"
    d = A.diagnose(found[0])
    assert d["n_bad"] > 0 and d["by_head"] and d["by_fragment_row"]


def test_write_past_the_last_sequence_is_reported():
    qkv, cu, H, lut, R = case_random(3, (5, 9))
    out = model(qkv, cu, H, lut, R)
    out[cu[-1], 3] = 0
    found = A.check_attention(out, qkv, cu, H, lut, R)
    assert found[1] and not found[0]


def test_reference_matches_plain_softmax():
    """The grouped, chunked float64 reference equals a direct per-sequence softmax."""
    qkv, cu, H, lut, R = case_random(4, (3, 70, 3, 1, 70))
    ref = A.reference(qkv, cu, H, lut, R)
    x = qkv.double()
    inner = H * 64
    for s in range(len(cu) - 1):
        t0, L = cu[s], cu[s + 1] - cu[s]
        for h in range(H):
            q = x[t0:t0 + L, h * 64:(h + 1) * 64]
            k = x[t0:t0 + L, inner + h * 64:inner + (h + 1) * 64]
            v = x[t0:t0 + L, 2 * inner + h * 64:2 * inner + (h + 1) * 64]
            i = torch.arange(L)
            b = lut[h][(i[None, :] - i[:, None]).clamp(-R, R) + R]
            want = torch.softmax(q @ k.t() + b, -1) @ v
            torch.testing.assert_close(ref[t0:t0 + L, h * 64:(h + 1) * 64], want, rtol=1e-12, atol=1e-12)


def test_hf_lut_sign_convention():
    """Positive delta = key - query maps to the upper half of the buckets; |delta| >= max_distance clamps."""
    rel = torch.arange(32, dtype=torch.float32)[:, None]
    lut = A.hf_bias_lut(rel, 32, 128)[0]
    assert lut[128] == 0 and lut[129] == 17 and lut[127] == 1
    assert lut[0] == 15 and lut[-1] == 31
