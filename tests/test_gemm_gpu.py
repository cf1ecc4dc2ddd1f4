"""Parity of the wgmma/TMA contraction core against a plain PyTorch fp32 matmul
of the same bf16 operands (C = A @ B^T, fp32 accumulate)."""
import json

import pytest
import torch

from reprover_b200 import _native

pytestmark = pytest.mark.gpu


ENTRY = "rpx_gemm_bf16_f32"


@pytest.fixture(params=["rpx_gemm_bf16_f32", "rpx_gemm1_bf16_f32", "rpx_gemm2_bf16_f32"], autouse=True)
def _entry(request):
    """Every test runs through the warp-specialised 128 x 256 throughput core, the single-CTA 128 x 128 core and
    its paired (2-CTA cluster, multicast B) form."""
    global ENTRY
    ENTRY = request.param
    yield


def _run_gemm(lib, A, B):
    M, K = A.shape
    N = B.shape[0]
    Cout = torch.full((M, N), float("nan"), device=A.device, dtype=torch.float32)
    st = torch.cuda.current_stream().cuda_stream
    _native.check(getattr(lib, ENTRY)(A.data_ptr(), B.data_ptr(), Cout.data_ptr(), M, N, K, st))
    torch.cuda.synchronize()
    return Cout


def _diagnose(C, R, tag, out_dir):
    """Summarise where a mismatch sits (rows / columns / blocks) to debug descriptor bugs."""
    bad = ~torch.isclose(C, R, rtol=2e-3, atol=2e-3) | torch.isnan(C)
    info = {
        "tag": tag,
        "shape": list(C.shape),
        "n_bad": int(bad.sum()),
        "n_nan": int(torch.isnan(C).sum()),
        "max_abs_err": float((C - R).abs().nan_to_num(1e30).max()),
        "bad_rows_first": bad.any(1).nonzero().flatten()[:40].tolist(),
        "bad_cols_first": bad.any(0).nonzero().flatten()[:40].tolist(),
        "bad_per_row_block128": bad.any(1).float().reshape(-1).unfold(0, min(128, C.shape[0]), min(128, C.shape[0])).sum(1).tolist()[:16]
        if C.shape[0] >= 128 else [],
        "sample_C": C[:4, :8].tolist(),
        "sample_R": R[:4, :8].tolist(),
    }
    (out_dir / f"gemm_diag_{tag}.json").write_text(json.dumps(info, indent=1))
    return info


@pytest.mark.parametrize(
    "M,N,K",
    [
        (128, 256, 64),      # one tile, one k-block
        (128, 256, 256),     # one tile, ring wraps once
        (128, 256, 1472),    # encoder K
        (256, 512, 384),     # 2x2 tiles
        (300, 1472, 384),    # ragged M, ragged N tail (192 cols), o-proj shape
        (1000, 1152, 1472),  # qkv shape, N tail 128
        (4096, 7168, 1472),  # ffn-up shape, many tiles per CTA (persistent loop, accumulator tile hand-off)
        (777, 1472, 3584),   # ffn-down shape
        (20000, 256, 128),   # >132 tiles along M
    ],
)
def test_gemm_matches_torch(rpx_lib, cuda_device, out_dir, M, N, K):
    g = torch.Generator(device="cpu").manual_seed(1234 + M + N + K)
    A = torch.randn(M, K, generator=g).to(torch.bfloat16).to(cuda_device)
    B = torch.randn(N, K, generator=g).to(torch.bfloat16).to(cuda_device)
    C = _run_gemm(rpx_lib, A, B)
    R = A.float() @ B.float().t()
    ok = torch.allclose(C, R, rtol=2e-3, atol=2e-3)
    if not ok:
        info = _diagnose(C, R, f"{M}x{N}x{K}", out_dir)
        pytest.fail(f"GEMM mismatch {M}x{N}x{K}: {json.dumps(info)[:1500]}")


def test_gemm_structured_operands(rpx_lib, cuda_device, out_dir):
    """Identity-like B exposes any swizzle / descriptor permutation exactly."""
    M, N, K = 128, 256, 256
    A = (torch.arange(M * K, dtype=torch.float32).reshape(M, K) % 251 - 125).to(torch.bfloat16).to(cuda_device)
    B = torch.zeros(N, K, dtype=torch.float32)
    B[torch.arange(N), torch.arange(N) % K] = 1.0
    B = B.to(torch.bfloat16).to(cuda_device)
    C = _run_gemm(rpx_lib, A, B)
    R = A.float() @ B.float().t()
    if not torch.equal(C, R):
        info = _diagnose(C, R, "structured", out_dir)
        pytest.fail(f"structured GEMM mismatch: {json.dumps(info)[:1500]}")


def test_gemm_rejects_bad_shapes(rpx_lib, cuda_device):
    A = torch.zeros(128, 100, dtype=torch.bfloat16, device=cuda_device)
    B = torch.zeros(256, 100, dtype=torch.bfloat16, device=cuda_device)
    C = torch.zeros(128, 256, device=cuda_device)
    st = torch.cuda.current_stream().cuda_stream
    rc = getattr(rpx_lib, ENTRY)(A.data_ptr(), B.data_ptr(), C.data_ptr(), 128, 256, 100, st)
    assert rc == _native.RPX_ERR_UNSUPPORTED
    assert "multiple of 64" in _native.last_error()
