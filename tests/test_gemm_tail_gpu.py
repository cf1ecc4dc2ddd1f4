"""The last n-tile of the 128 x 256 throughput core, whose MMAs are only as wide as its columns rounded up to 64.

When N is not a multiple of 256 the consumers run that tile's k-loop on wgmma.m64n64k16, m64n128k16 or
m64n192k16 instead of m64n256k16.  Checked here:
  - the encoder GEMMs on the throughput path (rpx_debug_encoder_gemm, the forward pass's own dispatch) at
    geometries whose QKV and residual sites between them have every tail width (64, 128 and 192), against the
    float64 reference of tests/gemm_ref.py, with NaN sentinels past row T and past the used RMSNorm parts;
  - the token counts around the edges of the two-CTA clusters (one tile, an odd number of m-tiles, 16384 and
    16385 tokens: with and without programmatic dependent launch);
  - rows computed at one T are bit-identical to the same rows computed at another;
  - the bare core (rpx_gemm_bf16_f32) at N % 256 in {32, 96, 160, 224}: bit for bit the columns a full-width
    MMA computes when B is padded with zero rows to a multiple of 256."""
import math

import pytest
import torch

from reprover_b200 import _native
from tests import gemm_ref as R

pytestmark = pytest.mark.gpu

# (d_model, d_ff, heads) -> tail width of QKV (N = 192 heads) / of O-proj and FFN-down (N = d_model)
GEOMS = {
    "byt5_small": (1472, 3584, 6),  # QKV 128, residual 192
    "tiny": (64, 128, 1),  # QKV 192, residual 64 (one n-tile)
    "d384_h3": (384, 768, 3),  # QKV 64, residual 128
}
SITES = ("qkv", "oproj", "ffn_down")
SITE_ID = {"qkv": _native.RPX_EGEMM_QKV, "oproj": _native.RPX_EGEMM_OPROJ, "ffn_down": _native.RPX_EGEMM_FFN_DOWN}
# one tile; 3 m-tiles (the last cluster pair half past M); 128 and 129 m-tiles, PDL on up to 16384 tokens
TOKENS = [1, 257, 16384, 16385]
PAD = 2  # sentinel rows below every output
EPS = float(torch.tensor(1e-6, dtype=torch.float32))


def _ptr(t):
    return None if t is None else t.data_ptr()


class Case:
    """Inputs and NaN-filled outputs of one throughput-path site: A [T, K], B [N, K]; QKV: ss_in [P, T] with row
    scales that differ by up to 4x between rows; O-proj / FFN-down: h32_in [T, N]."""

    def __init__(self, site, geom, T, seed, dev, A=None, B=None, ss_in=None, h32_in=None):
        D, F, H = GEOMS[geom]
        self.site, self.geom, self.T, self.D = site, geom, T, D
        self.N, self.K = {"qkv": (192 * H, D), "oproj": (D, 64 * H), "ffn_down": (D, F)}[site]
        self.P = R.ss_parts(D, False)
        g = torch.Generator(device=dev).manual_seed(seed)
        N, K = self.N, self.K
        self.A = torch.randn(T, K, generator=g, device=dev).to(torch.bfloat16) if A is None else A
        self.B = (torch.randn(N, K, generator=g, device=dev) / math.sqrt(K)).to(torch.bfloat16) if B is None else B
        if site == "qkv":
            if ss_in is None:
                ms = torch.exp(torch.empty(T, device=dev).uniform_(math.log(1 / 4), math.log(4), generator=g))
                w = torch.rand(self.P, T, generator=g, device=dev) + 0.1
                ss_in = (w / w.sum(0) * ms * D).float().contiguous()
            self.ss_in = ss_in
            self.out = torch.full((T + PAD, N), float("nan"), dtype=torch.bfloat16, device=dev)
        else:
            self.h32_in = torch.randn(T, N, generator=g, device=dev) if h32_in is None else h32_in
            self.h32 = torch.full((T + PAD, N), float("nan"), device=dev)
            self.h32[:T] = self.h32_in
            self.h16 = torch.full((T + PAD, N), float("nan"), dtype=torch.bfloat16, device=dev)
            self.ss_out = torch.full(((self.P + 1) * T,), float("nan"), device=dev)

    def run(self, lib):
        st = torch.cuda.current_stream().cuda_stream
        if self.site == "qkv":
            args = (_ptr(self.ss_in), _ptr(self.out), None, None, None)
        else:
            args = (None, None, _ptr(self.h32), _ptr(self.h16), _ptr(self.ss_out))
        _native.check(lib.rpx_debug_encoder_gemm(SITE_ID[self.site], 0, _ptr(self.A), _ptr(self.B), self.T, self.N,
                                                 self.K, EPS, *args, None, 0, st))

    def outputs(self, rows):
        """Every output's first `rows` rows (the partial sums as [P, rows])."""
        if self.site == "qkv":
            return [self.out[:rows]]
        return [self.h32[:rows], self.h16[:rows], self.ss_out[:self.P * self.T].view(self.P, self.T)[:, :rows]]

    def findings(self):
        T = self.T
        if self.site == "qkv":
            return [R.check_qkv(self.out[:T], self.A, self.B, self.ss_in, self.D, EPS),
                    R.check_sentinels("out.pad", self.out, T * self.N, R.BF16_NAN_BITS)]
        return R.check_residual(self.h32_in, self.h32[:T], self.h16[:T], self.ss_out[:self.P * T].view(self.P, T),
                                self.A, self.B, False) + [
            R.check_sentinels("h32.pad", self.h32, T * self.N, R.F32_NAN_BITS),
            R.check_sentinels("h16.pad", self.h16, T * self.N, R.BF16_NAN_BITS),
            R.check_sentinels("ss_out.pad", self.ss_out, self.P * T, R.F32_NAN_BITS)]


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("site", SITES)
@pytest.mark.parametrize("T", TOKENS)
def test_tail_tile_matches_reference(rpx_lib, cuda_device, site, geom, T):
    case = Case(site, geom, T, 13 * T + 5, cuda_device)
    case.run(rpx_lib)
    torch.cuda.synchronize()
    bad = [f for f in case.findings() if f]
    assert not bad, f"{site} {geom} T={T}: " + "; ".join(f.summary() for f in bad)[:3000]


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("site", SITES)
def test_tail_rows_do_not_depend_on_T(rpx_lib, cuda_device, site, geom):
    """16385 tokens (129 m-tiles, no PDL) against its first 1 and 257 rows (one tile; 3 m-tiles under PDL)."""
    big = Case(site, geom, 16385, 59, cuda_device)
    big.run(rpx_lib)
    for T in (1, 257):
        small = Case(site, geom, T, 0, cuda_device, A=big.A[:T].contiguous(), B=big.B,
                     ss_in=big.ss_in[:, :T].contiguous() if site == "qkv" else None,
                     h32_in=big.h32_in[:T].contiguous() if site != "qkv" else None)
        small.run(rpx_lib)
        torch.cuda.synchronize()
        for i, (x, y) in enumerate(zip(big.outputs(T), small.outputs(T))):
            diff = (_bits(x) != _bits(y)).nonzero()
            assert diff.numel() == 0, f"{site} {geom}: T=16385 vs T={T}: output {i} differs at {diff[:8].tolist()}"


@pytest.mark.parametrize("N", [288, 352, 416, 480, 1312])
@pytest.mark.parametrize("M", [1, 300, 16385])
def test_bare_core_tail_equals_full_width(rpx_lib, cuda_device, M, N):
    """rpx_gemm_bf16_f32 with N % 256 in {32, 96, 160, 224}: the tail tile runs m64n64 / n128 / n192 / n256
    MMAs.  Its columns equal bit for bit those of the same product with B padded by zero rows to a multiple of
    256 (every tile full width), and lie within the accumulation bound of the float64 product."""
    K = 1472
    g = torch.Generator(device=cuda_device).manual_seed(M * 7 + N)
    A = torch.randn(M, K, generator=g, device=cuda_device).to(torch.bfloat16)
    B = torch.randn(N, K, generator=g, device=cuda_device).to(torch.bfloat16)
    n_pad = -(-N // 256) * 256
    B_pad = torch.zeros(n_pad, K, dtype=torch.bfloat16, device=cuda_device)
    B_pad[:N] = B
    st = torch.cuda.current_stream().cuda_stream
    C = torch.full((M + PAD, N), float("nan"), device=cuda_device)
    C_pad = torch.full((M, n_pad), float("nan"), device=cuda_device)
    _native.check(rpx_lib.rpx_gemm_bf16_f32(A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, st))
    _native.check(rpx_lib.rpx_gemm_bf16_f32(A.data_ptr(), B_pad.data_ptr(), C_pad.data_ptr(), M, n_pad, K, st))
    torch.cuda.synchronize()
    diff = (_bits(C[:M]) != _bits(C_pad[:, :N].contiguous())).nonzero()
    assert diff.numel() == 0, f"tail columns differ from the full-width MMA at {diff[:8].tolist()}"
    E, S = R.accumulate(A, B)
    err = (C[:M].double() - E).abs()
    assert bool((err <= R.gamma_acc(K) * S + R.U * E.abs()).all()), f"max error {float(err.max())}"
    assert bool(torch.isnan(C[M:]).all()), "a store landed past row M"
