"""Every encoder GEMM epilogue, launched exactly as the forward pass launches it (rpx_debug_encoder_gemm runs
the same tile-shape dispatch as forward_layer()), on both paths and every tile shape,
against the float64 reference and rounding-aware checker of tests/gemm_ref.py.

Sites: QKV (RMSNorm row scale, bf16 store), O-proj and FFN-down (fp32 residual update, bf16 copy, partial
sums of h^2 for the next RMSNorm), FFN-up (gated GELU over the interleaved gate / linear rows), and the generator's
output head (row scale, fp32 store; on the throughput core with either layout of partial sums, as the teacher-forced
forward and the decode steps run it).  On top of
the per-site checks: chained launches under programmatic dependent launch, the L2-prefetch helper CTAs of
the latency QKV projection, and bit-identical rows across tile shapes.

Every output buffer carries NaN sentinels past row T (and past the used parts of ss_out) that must survive.
The observed accumulation error of every residual case is written next to its bound to
gemm_epilogue_accuracy.json; a failing case writes gemm_epilogue_diag_<case>.json (bad elements by tile and
by wgmma fragment position)."""
import json
import math

import pytest
import torch

from reprover_b200 import _native
from tests import gemm_ref as R

pytestmark = pytest.mark.gpu

# (d_model, d_ff, heads, vocab)
GEOMS = {
    "byt5_small": (1472, 3584, 6, 384),  # 64-column tail on 128-wide tiles; 46 latency parts (two RowScale batches);
                                         # the head's last n-tile is 128 columns wide
    "d768": (768, 2048, 12, 32128),  # exactly 24 latency parts; T5's vocabulary
    "byt5_base_like": (1536, 3968, 12, 416),  # d_ff an odd multiple of 128: split-B tiles start at unit 64 of a
                                              # block; the head's last n-tile is 160 columns on a 192-wide MMA
    "tiny": (64, 128, 1, 32),  # one tile narrower than the tile width; the head is one 64-wide MMA over 32 columns
}
# BM = 64 / 128 switch at 384, FFN-up 32 / 64 hidden units per tile at 128, ragged tiles
LAT_T = [1, 17, 63, 64, 65, 127, 128, 129, 383, 384, 385, 700, 1025]
# PDL on up to 16384 tokens; 40000 gives many tiles per persistent CTA on both cores
THR_T = [1, 129, 1000, 16384, 16385, 40000]
SITES = ("qkv", "oproj", "ffn_up", "ffn_down", "head")
SITE_ID = {"qkv": _native.RPX_EGEMM_QKV, "oproj": _native.RPX_EGEMM_OPROJ, "ffn_up": _native.RPX_EGEMM_FFN_UP,
           "ffn_down": _native.RPX_EGEMM_FFN_DOWN, "head": _native.RPX_EGEMM_HEAD}
PAD = 2  # sentinel rows below every output
EPS = float(torch.tensor(1e-6, dtype=torch.float32))

ACCURACY = []


@pytest.fixture(scope="module", autouse=True)
def _accuracy_artefact(out_dir):
    yield
    (out_dir / "gemm_epilogue_accuracy.json").write_text(json.dumps(ACCURACY, indent=0))


def _dims(site, geom):
    """(N, K, d_model) of one site."""
    D, F, H, V = GEOMS[geom]
    inner = 64 * H
    return {"qkv": (3 * inner, D, D), "oproj": (D, inner, D), "ffn_up": (2 * F, D, D), "ffn_down": (D, F, D),
            "head": (V, D, D)}[site]


def _ptr(t):
    return None if t is None else t.data_ptr()


def _launch(lib, site, latency, T, N, K, A, B, ss_in=None, out=None, h32=None, h16=None, ss_out=None, prefetch=None,
            stream=None):
    st = torch.cuda.current_stream().cuda_stream if stream is None else stream
    return lib.rpx_debug_encoder_gemm(SITE_ID[site], int(latency), _ptr(A), _ptr(B), T, N, K, EPS, _ptr(ss_in), _ptr(out),
                                      _ptr(h32), _ptr(h16), _ptr(ss_out), _ptr(prefetch),
                                      0 if prefetch is None else prefetch.numel() * prefetch.element_size(), st)


class Case:
    """Inputs and sentinel-filled outputs of one site: A [T, K], B [N, K] (FFN-up: packed from W0 / W1),
    ss_in [P, T] with row scales that differ by up to 4x between rows, h32_in [T, N] for the residual sites."""

    def __init__(self, site, geom, T, latency, seed, dev):
        self.site, self.geom, self.T, self.latency = site, geom, T, latency
        self.N, self.K, self.D = _dims(site, geom)
        g = torch.Generator(device=dev).manual_seed(seed)
        N, K, D = self.N, self.K, self.D
        self.A = torch.randn(T, K, generator=g, device=dev).to(torch.bfloat16)
        if site == "ffn_up":
            self.W0 = (torch.randn(N // 2, K, generator=g, device=dev) / math.sqrt(K)).to(torch.bfloat16)
            self.W1 = (torch.randn(N // 2, K, generator=g, device=dev) / math.sqrt(K)).to(torch.bfloat16)
            self.B = R.pack_ffn_up(self.W0, self.W1).contiguous()
        else:
            self.B = (torch.randn(N, K, generator=g, device=dev) / math.sqrt(K)).to(torch.bfloat16)
        self.P = R.ss_parts(D, latency)
        if site in ("qkv", "ffn_up", "head"):
            ms = torch.exp(torch.empty(T, device=dev).uniform_(math.log(1 / 4), math.log(4), generator=g))
            w = torch.rand(self.P, T, generator=g, device=dev) + 0.1
            self.ss_in = (w / w.sum(0) * ms * D).float().contiguous()
            cols = N // 2 if site == "ffn_up" else N
            dtype = torch.float32 if site == "head" else torch.bfloat16
            self.out = torch.full((T + PAD, cols), float("nan"), dtype=dtype, device=dev)
        else:
            self.h32_in = torch.randn(T, N, generator=g, device=dev)
            self.h32 = torch.full((T + PAD, N), float("nan"), device=dev)
            self.h32[:T] = self.h32_in
            self.h16 = torch.full((T + PAD, N), float("nan"), dtype=torch.bfloat16, device=dev)
            self.ss_out = torch.full(((self.P + 1) * T,), float("nan"), device=dev)

    @property
    def residual(self):
        return self.site in ("oproj", "ffn_down")

    def run(self, lib, **kw):
        if self.residual:
            return _launch(lib, self.site, self.latency, self.T, self.N, self.K, self.A, self.B, h32=self.h32, h16=self.h16,
                           ss_out=self.ss_out, **kw)
        return _launch(lib, self.site, self.latency, self.T, self.N, self.K, self.A, self.B, ss_in=self.ss_in, out=self.out, **kw)

    def outputs(self):
        return (self.h32, self.h16, self.ss_out) if self.residual else (self.out,)

    def tile(self):
        """(rows, output columns) of one tile, for the diagnostic."""
        T = self.T
        if self.site == "ffn_up":
            return (128, 128) if not self.latency else (128, 32 if T <= 128 else 64)
        if not self.latency or self.site == "head":
            return (128, 128)
        return (64 if T <= 384 else 128, 64)

    def check(self, A=None, ss_in=None, h32_in=None):
        """Findings of every output against the reference (A / ss_in / h32_in default to this case's inputs)."""
        T = self.T
        A = self.A if A is None else A
        stats = {}
        if self.site == "qkv":
            ss = self.ss_in if ss_in is None else ss_in
            found = [R.check_qkv(self.out[:T], A, self.B, ss, self.D, EPS, stats),
                     R.check_sentinels("out.pad", self.out, T * self.N, R.BF16_NAN_BITS)]
        elif self.site == "head":
            ss = self.ss_in if ss_in is None else ss_in
            found = [R.check_head(self.out[:T], A, self.B, ss, self.D, EPS, stats),
                     R.check_sentinels("out.pad", self.out, T * self.N, R.F32_NAN_BITS)]
        elif self.site == "ffn_up":
            ss = self.ss_in if ss_in is None else ss_in
            found = [R.check_ffn_up(self.out[:T], A, self.W0, self.W1, ss, self.D, EPS, stats),
                     R.check_sentinels("out.pad", self.out, T * self.N // 2, R.BF16_NAN_BITS)]
        else:
            hin = self.h32_in if h32_in is None else h32_in
            found = R.check_residual(hin, self.h32[:T], self.h16[:T], self.ss_out[:self.P * T].view(self.P, T), A, self.B,
                                     self.latency, stats)
            found += [R.check_sentinels("h32.pad", self.h32, T * self.N, R.F32_NAN_BITS),
                      R.check_sentinels("h16.pad", self.h16, T * self.N, R.BF16_NAN_BITS),
                      R.check_sentinels("ss_out.pad", self.ss_out, self.P * T, R.F32_NAN_BITS)]
        return found, stats

    def tag(self):
        return f"{self.site}_{'lat' if self.latency else 'thr'}_{self.geom}_T{self.T}"


def _fail_on(case, found, out_dir, what=""):
    bad = [f for f in found if f]
    if not bad:
        return
    tm, tn = case.tile()
    diag = {"case": case.tag(), "what": what, "tile": [tm, tn], "findings": [R.diagnose(f, tm, tn) for f in bad]}
    (out_dir / f"gemm_epilogue_diag_{case.tag()}{what}.json").write_text(json.dumps(diag, indent=1))
    pytest.fail(f"{case.tag()}{what}: " + "; ".join(f.summary() for f in bad)[:3000])


def _run_and_check(lib, case, out_dir):
    _native.check(case.run(lib))
    torch.cuda.synchronize()
    found, stats = case.check()
    ACCURACY.append({"case": case.tag(), "K": case.K, **stats})
    _fail_on(case, found, out_dir)


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("site", SITES)
@pytest.mark.parametrize("T", LAT_T)
def test_latency_epilogue(rpx_lib, cuda_device, out_dir, site, geom, T):
    _run_and_check(rpx_lib, Case(site, geom, T, True, 7 * T + 1, cuda_device), out_dir)


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("site", SITES)
@pytest.mark.parametrize("T", THR_T)
def test_throughput_epilogue(rpx_lib, cuda_device, out_dir, site, geom, T):
    _run_and_check(rpx_lib, Case(site, geom, T, False, 11 * T + 3, cuda_device), out_dir)


@pytest.mark.parametrize("latency,T", [(True, 200), (False, 300)], ids=["latency", "throughput"])
def test_ffn_up_structured_pairing(rpx_lib, cuda_device, out_dir, latency, T):
    """Gate row j reads only column 2j mod K of A and linear row j only column 2j + 1: gate and linear values are
    single exact products, so a wrong column pairing shows up exactly in the failure message."""
    case = Case("ffn_up", "byt5_small", T, latency, 5, cuda_device)
    F, K = case.N // 2, case.K
    A = (torch.arange(T * K, device=cuda_device, dtype=torch.float32).reshape(T, K) % 61 - 30) / 8
    case.A = A.to(torch.bfloat16)
    j = torch.arange(F, device=cuda_device)
    case.W0 = torch.zeros(F, K, device=cuda_device, dtype=torch.bfloat16)
    case.W1 = torch.zeros_like(case.W0)
    case.W0[j, (2 * j) % K] = 1
    case.W1[j, (2 * j + 1) % K] = 1
    case.B = R.pack_ffn_up(case.W0, case.W1).contiguous()
    _run_and_check(rpx_lib, case, out_dir)


CHAINS = [("oproj", "ffn_up"), ("ffn_up", "ffn_down"), ("ffn_down", "qkv")]


@pytest.mark.parametrize("latency,T", [(True, 200), (False, 1000)], ids=["latency", "throughput"])
@pytest.mark.parametrize("first,second", CHAINS)
def test_chained_launches_under_pdl(rpx_lib, cuda_device, out_dir, first, second, latency, T):
    """Two consecutive GEMMs enqueued back to back (programmatic dependent launch is on for both paths at these
    T); the second reads what the first writes and is checked against the reference built from the first's
    actual outputs.  The intermediate buffers start as NaN, so a read before the first GEMM's writes land fails."""
    a = Case(first, "byt5_small", T, latency, 21, cuda_device)
    b = Case(second, "byt5_small", T, latency, 22, cuda_device)
    # wire a's outputs into b's inputs (b's own inputs of that kind are replaced by NaN-filled buffers of a)
    if first == "ffn_up":  # ffn [T, d_ff] -> FFN-down A
        b_A = a.out
    else:  # h16 [T, d_model] and the partial sums -> FFN-up / QKV A and ss_in
        b_A = a.h16
        b.ss_in = a.ss_out[:a.P * T].view(a.P, T)
    b.A = b_A  # rows past T are not read (A is [T, K] to the kernel)
    _native.check(a.run(rpx_lib))
    _native.check(b.run(rpx_lib))
    torch.cuda.synchronize()
    found_a, _ = a.check()
    _fail_on(a, found_a, out_dir, "_chain_first")
    found_b, _ = b.check(A=b_A[:T])
    _fail_on(b, found_b, out_dir, f"_chain_after_{first}")


@pytest.mark.parametrize("T", [17, 385])
def test_latency_qkv_prefetch_helpers_change_nothing(rpx_lib, cuda_device, out_dir, T):
    """Latency QKV with the next layer's weights to prefetch, as forward_layer runs it: the surplus CTAs
    only read.  Outputs are bit-identical to a run without prefetch, sentinels and the prefetched buffer intact."""
    case = Case("qkv", "byt5_small", T, True, 31, cuda_device)
    _native.check(case.run(rpx_lib))
    torch.cuda.synchronize()
    plain = case.out.clone()
    case.out.fill_(float("nan"))
    nxt = torch.randint(-2 ** 31, 2 ** 31 - 1, (36 << 20 >> 2,), dtype=torch.int32, device=cuda_device)
    before = nxt.clone()
    _native.check(case.run(rpx_lib, prefetch=nxt))
    torch.cuda.synchronize()
    assert torch.equal(case.out.view(torch.int16), plain.view(torch.int16)), "prefetch helpers changed the QKV output"
    assert torch.equal(nxt, before), "prefetch helpers wrote to the prefetched buffer"
    found, _ = case.check()
    _fail_on(case, found, out_dir, "_prefetch")


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _sub_case(big, T):
    """The same inputs as `big`, cut to its first T rows, with fresh sentinel-filled outputs."""
    small = Case(big.site, big.geom, T, big.latency, 0, big.A.device)
    small.A, small.B = big.A[:T].contiguous(), big.B
    if big.site == "ffn_up":
        small.W0, small.W1 = big.W0, big.W1
    if big.residual:
        small.h32_in = big.h32_in[:T].contiguous()
        small.h32[:T] = small.h32_in
    else:
        small.ss_in = big.ss_in[:, :T].contiguous()
    return small


def _same_rows(lib, big, T):
    """Run `big` and its first-T-rows copy; the shared rows of every output must be bit-identical."""
    small = _sub_case(big, T)
    _native.check(big.run(lib))
    _native.check(small.run(lib))
    torch.cuda.synchronize()
    if big.residual:
        pairs = [(big.h32[:T], small.h32[:T]), (big.h16[:T], small.h16[:T]),
                 (big.ss_out[:big.P * big.T].view(big.P, big.T)[:, :T], small.ss_out[:small.P * T].view(small.P, T))]
    else:
        pairs = [(big.out[:T], small.out[:T])]
    for i, (x, y) in enumerate(pairs):
        diff = (_bits(x) != _bits(y)).nonzero()
        assert diff.numel() == 0, f"{big.tag()} vs T={T}: output {i} differs at {diff[:8].tolist()}"


@pytest.mark.parametrize("site", ["oproj", "ffn_down"])
def test_latency_residual_rows_identical_across_tile_heights(rpx_lib, cuda_device, site):
    """T = 385 runs 128-row tiles, T = 384 64-row tiles: h32, h16 and the 32-column partial sums agree bit for bit."""
    _same_rows(rpx_lib, Case(site, "byt5_small", 385, True, 41, cuda_device), 384)


def test_latency_ffn_up_rows_identical_across_tile_widths(rpx_lib, cuda_device):
    """T = 129 runs 64 hidden units per tile, T = 128 32 units."""
    _same_rows(rpx_lib, Case("ffn_up", "byt5_small", 129, True, 43, cuda_device), 128)


@pytest.mark.parametrize("site", SITES)
def test_throughput_rows_do_not_depend_on_T(rpx_lib, cuda_device, site):
    for T in (1, 129):
        _same_rows(rpx_lib, Case(site, "byt5_small", 1000, False, 47, cuda_device), T)


def test_entry_point_rejects_bad_site_and_input(rpx_lib, cuda_device):
    """Sites outside [RPX_EGEMM_QKV, RPX_EGEMM_HEAD] and incomplete arguments are refused, and nothing is written."""
    t = torch.zeros(4096, dtype=torch.float32, device=cuda_device)
    p = t.data_ptr()
    st = torch.cuda.current_stream().cuda_stream

    def call(site, latency=0, N=256, K=64, ss_in=p, out=p, h32=None, h16=None, ss_out=None, pf=None):
        return rpx_lib.rpx_debug_encoder_gemm(site, latency, p, p, 4, N, K, EPS, ss_in, out, h32, h16, ss_out, pf, 64, st)

    assert call(5) == _native.RPX_ERR_INVALID
    assert call(-1) == _native.RPX_ERR_INVALID
    assert call(_native.RPX_EGEMM_QKV, ss_in=None) == _native.RPX_ERR_INVALID
    assert call(_native.RPX_EGEMM_FFN_UP, out=None) == _native.RPX_ERR_INVALID
    assert call(_native.RPX_EGEMM_OPROJ, N=64, h32=p, h16=p, ss_out=None) == _native.RPX_ERR_INVALID
    assert call(_native.RPX_EGEMM_FFN_DOWN, N=64, h32=None, h16=p, ss_out=p) == _native.RPX_ERR_INVALID
    assert call(_native.RPX_EGEMM_QKV, latency=0, pf=p) == _native.RPX_ERR_INVALID  # only latency QKV prefetches
    assert call(_native.RPX_EGEMM_FFN_UP, N=384) == _native.RPX_ERR_UNSUPPORTED
    assert "multiple of 256" in _native.last_error()
    assert call(_native.RPX_EGEMM_QKV, K=96) == _native.RPX_ERR_UNSUPPORTED  # d_model = K not a multiple of 64
    for latency in (0, 1):
        assert call(_native.RPX_EGEMM_HEAD, latency, ss_in=None) == _native.RPX_ERR_INVALID
        assert call(_native.RPX_EGEMM_HEAD, latency, out=None) == _native.RPX_ERR_INVALID
        assert call(_native.RPX_EGEMM_HEAD, latency, pf=p) == _native.RPX_ERR_INVALID  # the head never prefetches
        assert call(_native.RPX_EGEMM_HEAD, latency, N=400) == _native.RPX_ERR_UNSUPPORTED
        assert "multiple of 32" in _native.last_error()
    torch.cuda.synchronize()
    assert torch.count_nonzero(t) == 0
