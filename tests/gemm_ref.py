"""Float64 references of the encoder GEMM epilogues and a checker whose tolerances follow from the rounding
each step of the kernel performs.

Every function takes torch tensors on any device (the GPU suite runs them on the H100, the CPU suite on the
host) and works on row chunks, so a 40 000-token case fits in memory.

Notation: u = 2^-24 is the unit roundoff of fp32 round-to-nearest, gamma_n = n u / (1 - n u) the classical
bound on the relative error of a sum of n non-negative fp32 terms in any order (Higham, "Accuracy and
Stability of Numerical Algorithms", 2nd ed., Lemma 3.1 and section 4.2).

Accumulation (all four sites)
    E = A B^T is formed in float64.  A product of two bf16 values has at most 16 significant bits, so every
    product is exact in float64 and in fp32; the float64 sum of K such terms is within K 2^-53 S of the exact
    sum, S = |A| |B|^T, which is below 1e-12 S for the K used here: E is exact for these purposes.
    The kernels issue wgmma with K = 16 per instruction: the fp32 accumulator receives ceil(K / 16) block
    fused multiply-adds, each adding 16 exact products to it.  Take the pessimistic model of such a block
    FMA on NVIDIA tensor cores (Fasi et al., "Numerical behavior of NVIDIA tensor cores", PeerJ CS 2021):
    the 17 addends are aligned to the largest exponent with their significands truncated to 24 bits, summed,
    and the result truncated to 24 bits.  Each truncation loses less than one unit in the 24th bit of the
    largest addend or of the result, i.e. less than 2^-23 times a magnitude that is at most the sum of the
    magnitudes of the addends, which is at most S for that element.  One block FMA therefore errs by less
    than 18 * 2^-23 * S and the whole accumulation by
        |acc - E| <= gamma_acc(K) * S,     gamma_acc(K) = ceil(K / 16) * 18 * 2^-23.
    gamma_acc(1472) = 2.0e-4, gamma_acc(3968) = 5.3e-4.  Any fp32 summation order with round-to-nearest obeys
    the same bound (gamma_K < gamma_acc(K)), so the plain CPU model in test_gemm_ref_cpu.py passes it too.
    The GPU suite records the observed max |acc - E| / S of every case (residual sites, where the
    accumulator is visible through h32_out - h32_in, so the figure includes that addition's rounding) next to
    gamma_acc in its artefact.  On an NVIDIA H100 80GB HBM3 at a 400 W power limit, the 152 residual cases of
    the suite measured at most 1.5e-7 (K = 64, gamma_acc = 8.6e-6, a margin of 56x) and 7.6e-7 at K = 3968
    (margin 700x).  The
    derived bound is kept rather than a tighter one fitted to random operands, which need not hold for other
    data.  A dropped 64-wide k-block or a swapped row is off by
    about sqrt(64) resp. sqrt(K) times a typical product, far outside gamma_acc * S.

Row scale (QKV, FFN-up)
    rs[m] = 1 / sqrt(sum_p ss_in[p][m] / D + eps) in float64 from the same fp32 partial sums the kernel reads.
    The kernel sums the P non-negative parts in fp32 (relative error gamma_{P-1}), multiplies by fp32(1/D)
    (2 roundings: the constant and the product), adds eps (1 rounding), and takes rsqrtf, whose maximum
    error is 2 ulp (CUDA C++ Programming Guide, single-precision mathematical functions), i.e. a relative
    error of at most 2 * 2^-23.  A relative error e of the argument moves 1/sqrt by at most e / 2 (+ O(e^2)):
        eps_rs(P) = (gamma_{P-1} + 3u) / 2 + 2^-22, plus a 1e-3 relative allowance for the second-order terms.

bf16 outputs
    The kernel rounds an fp32 value v to bf16 with round-to-nearest-even.  When |v - ref| <= tol, rounding is
    monotone, so the output must lie in [bf16_rn(ref - tol), bf16_rn(ref + tol)] (the bounds are moved
    outward to fp32 first, so that no double rounding can narrow the bracket).  Away from a bf16 rounding
    boundary this is exact equality; there is no global rtol.

QKV        v = fl(acc * rs_k):  tol = rs (gamma S + (|E| + gamma S)(eps_rs + u)).

FFN-up     x = fl(g * rs_k), y = fl(l * rs_k) with g, l the gate and linear accumulators: dx, dy as for QKV.
           gelu_new(x) = x/2 (1 + tanh(k0 (x + k1 x^3))), evaluated in float64 with an exact tanh for the
           reference.  The kernel:
             - the argument of tanh takes 5 roundings plus the fp32 constants k0, k1: |du| <= 7u k0 (|x| + k1 |x|^3),
               and |tanh'| <= 1, so t moves by at most that;
             - tanh.approx.f32 has a maximum relative error of 2^-10.987 (PTX ISA, "tanh"): |dt| <= ETA |t| <= ETA;
             - x/2 (1 + t): 1 + t and the product take 2 roundings, 4u x/2 with |1 + t| <= 2;
             - the perturbation dx of the argument moves gelu_new by at most GELU_LIP dx (max |gelu_new'| < 1.13).
           dg = GELU_LIP dx + (|x| + dx)/2 (dt_arith (1 + ETA) + ETA + 4u);
           out = fl(gelu * y): tol = dg (|y| + dy) + |gelu| dy + u (|gelu| + dg)(|y| + dy).

Residual   h32_out = fl(h32_in + acc): |h32_out - (h32_in + E)| <= gamma S + u (|h32_in + E| + gamma S).
(O-proj,   h16_out must equal bf16_rn(h32_out) bit for bit, from the kernel's own h32_out.
FFN-down)  ss_out[p][m] is compared with the float64 sum of h32_out[m, c]^2 over exactly the columns c of part p
           (a 128-column tile on the throughput path, a 32-column chunk on the latency path): the kernel squares
           and sums n <= 128 fp32 values in some order, relative error <= gamma_{n+1}.
"""
from __future__ import annotations

import math

import torch

U = 2.0 ** -24
ETA_TANH = 2.0 ** -10.987  # tanh.approx.f32, maximum relative error (PTX ISA)
RSQRT_REL = 2 * 2.0 ** -23  # rsqrtf: 2 ulp
GELU_LIP = 1.13  # max |d/dx gelu_new(x)| = 1.1289... (pinned by test_gemm_ref_cpu.py)
GELU_K0 = math.sqrt(2.0 / math.pi)
GELU_K1 = 0.044715
ROW_CHUNK = 4096

F32_NAN_BITS = 0x7FC00000
BF16_NAN_BITS = 0x7FC0


def gamma_n(n: int) -> float:
    return n * U / (1 - n * U)


def gamma_acc(K: int) -> float:
    return math.ceil(K / 16) * 18 * 2.0 ** -23


def eps_rowscale(n_parts: int) -> float:
    return ((gamma_n(max(n_parts - 1, 0)) + 3 * U) / 2 + RSQRT_REL) * (1 + 1e-3)


def ss_parts(d_model: int, latency: bool) -> int:
    """RMSNorm partial sums per row: one per 128-column tile (throughput) or 32-column chunk (latency)."""
    return -(-d_model // (32 if latency else 128))


def part_cols(latency: bool) -> int:
    return 32 if latency else 128


def accumulate(A: torch.Tensor, B: torch.Tensor):
    """E = A B^T and S = |A| |B|^T in float64 (A [T, K], B [N, K], any float dtype)."""
    A64, B64 = A.double(), B.double()
    return A64 @ B64.t(), A64.abs() @ B64.abs().t()


def rowscale(ss_in: torch.Tensor, d_model: int, eps: float) -> torch.Tensor:
    """float64 rs[m] from fp32 partial sums ss_in [P, T]; eps is the fp32 value the kernel receives."""
    return 1.0 / torch.sqrt(ss_in.double().sum(0) / d_model + eps)


def gelu_new64(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.tanh(GELU_K0 * (x + GELU_K1 * x ** 3)))


def _f32_outward(x: torch.Tensor, down: bool) -> torch.Tensor:
    """float64 -> fp32 rounded toward -inf (down) or +inf, so that a later bf16 rounding brackets correctly."""
    y = x.float()
    if down:
        return torch.where(y.double() > x, torch.nextafter(y, torch.full_like(y, -math.inf)), y)
    return torch.where(y.double() < x, torch.nextafter(y, torch.full_like(y, math.inf)), y)


def bf16_bracket_bad(out: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> torch.Tensor:
    """True where the bf16 output lies outside [bf16_rn(ref - tol), bf16_rn(ref + tol)] (or is NaN)."""
    lo = _f32_outward(ref - tol, down=True).to(torch.bfloat16).double()
    hi = _f32_outward(ref + tol, down=False).to(torch.bfloat16).double()
    o = out.double()
    return ~((o >= lo) & (o <= hi))


class Findings:
    """Bad elements of one output, gathered over row chunks: count, the first few (row, col), and the data to
    group them by tile and fragment position for a diagnostic."""

    def __init__(self, name: str, keep: int = 4096):
        self.name = name
        self.n_bad = 0
        self.keep = keep
        self.where: list[tuple[int, int]] = []
        self.samples: list[dict] = []

    def add(self, bad: torch.Tensor, row0: int, got=None, want=None, tol=None) -> None:
        n = int(bad.sum())
        if n == 0:
            return
        self.n_bad += n
        if len(self.where) < self.keep:
            idx = bad.nonzero()[: self.keep - len(self.where)]
            for r, c in idx.tolist():
                self.where.append((row0 + r, c))
                if len(self.samples) < 16 and got is not None:
                    self.samples.append({"row": row0 + r, "col": c, "got": float(got[r, c]), "want": float(want[r, c]),
                                         "tol": float(tol[r, c]) if tol is not None else 0.0})

    def __bool__(self) -> bool:  # truthy when something is wrong
        return self.n_bad > 0

    def summary(self) -> str:
        return f"{self.name}: {self.n_bad} bad, first {self.where[:8]}, samples {self.samples[:4]}"


def _chunks(T: int):
    for r0 in range(0, T, ROW_CHUNK):
        yield r0, min(T, r0 + ROW_CHUNK)


def check_sentinels(name: str, buf: torch.Tensor, start: int, fill_bits: int) -> Findings:
    """Every element of the flat buffer from `start` on must still hold the NaN sentinel `fill_bits`."""
    f = Findings(name)
    flat = buf.reshape(-1)
    bits = flat.view(torch.int16 if flat.element_size() == 2 else torch.int32)[start:]
    bad = bits != fill_bits
    if bool(bad.any()):
        idx = bad.nonzero().flatten()
        f.n_bad = int(idx.numel())
        row_len = buf.shape[-1] if buf.dim() > 1 else 1
        f.where = [divmod(start + i, row_len) for i in idx[:64].tolist()]
    return f


def check_qkv(out: torch.Tensor, A: torch.Tensor, B: torch.Tensor, ss_in: torch.Tensor, d_model: int, eps: float,
              stats: dict | None = None) -> Findings:
    """out [T, N] bf16 = bf16(A B^T * rs[m])."""
    T, K = A.shape
    g = gamma_acc(K)
    e_rs = eps_rowscale(ss_in.shape[0])
    f = Findings("qkv.out")
    n_boundary = 0
    for r0, r1 in _chunks(T):
        E, S = accumulate(A[r0:r1], B)
        rs = rowscale(ss_in[:, r0:r1], d_model, eps)[:, None]
        ref = E * rs
        tol = rs * (g * S + (E.abs() + g * S) * (e_rs + U))
        o = out[r0:r1]
        bad = bf16_bracket_bad(o, ref, tol)
        f.add(bad, r0, o.float(), ref, tol)
        n_boundary += int((o.double() != ref.float().to(torch.bfloat16).double()).sum())
    if stats is not None:
        stats.update(gamma=g, eps_rs=e_rs, n_not_rn_of_ref=n_boundary)
    return f


def check_ffn_up(out: torch.Tensor, A: torch.Tensor, W0: torch.Tensor, W1: torch.Tensor, ss_in: torch.Tensor,
                 d_model: int, eps: float, stats: dict | None = None) -> Findings:
    """out [T, F] bf16 = bf16(gelu_new(A W0^T rs) * (A W1^T rs)); W0 / W1 [F, K] are the gate / linear weights
    (the reference takes them unpacked, so it also pins the packed layout the kernel reads)."""
    T, K = A.shape
    g = gamma_acc(K)
    e_rs = eps_rowscale(ss_in.shape[0])
    f = Findings("ffn_up.out")
    n_boundary = 0
    for r0, r1 in _chunks(T):
        G, SG = accumulate(A[r0:r1], W0)
        L, SL = accumulate(A[r0:r1], W1)
        rs = rowscale(ss_in[:, r0:r1], d_model, eps)[:, None]
        x, y = G * rs, L * rs
        dx = rs * (g * SG + (G.abs() + g * SG) * (e_rs + U))
        dy = rs * (g * SL + (L.abs() + g * SL) * (e_rs + U))
        del G, SG, L, SL
        gel = gelu_new64(x)
        xa = x.abs() + dx
        dt_arith = 7 * U * GELU_K0 * (xa + GELU_K1 * xa ** 3)
        dg = GELU_LIP * dx + 0.5 * xa * (dt_arith * (1 + ETA_TANH) + ETA_TANH + 4 * U)
        ref = gel * y
        ya = y.abs() + dy
        tol = dg * ya + gel.abs() * dy + U * (gel.abs() + dg) * ya
        o = out[r0:r1]
        bad = bf16_bracket_bad(o, ref, tol)
        f.add(bad, r0, o.float(), ref, tol)
        n_boundary += int((o.double() != ref.float().to(torch.bfloat16).double()).sum())
    if stats is not None:
        stats.update(gamma=g, eps_rs=e_rs, n_not_rn_of_ref=n_boundary)
    return f


def check_residual(h32_in: torch.Tensor, h32_out: torch.Tensor, h16_out: torch.Tensor, ss_out: torch.Tensor,
                   A: torch.Tensor, B: torch.Tensor, latency: bool, stats: dict | None = None) -> list[Findings]:
    """h32_out [T, N] = h32_in + A B^T; h16_out = bf16(h32_out); ss_out [P, T] partial sums of h32_out^2 per
    part (ss_out is the [P, T] view of the kernel's buffer, stride T)."""
    T, K = A.shape
    N = B.shape[0]
    g = gamma_acc(K)
    pc = part_cols(latency)
    P = ss_parts(N, latency)
    fh, f16, fss = Findings("residual.h32"), Findings("residual.h16"), Findings("residual.ss")
    obs = 0.0
    for r0, r1 in _chunks(T):
        E, S = accumulate(A[r0:r1], B)
        hin = h32_in[r0:r1].double()
        hout = h32_out[r0:r1].double()
        ref = hin + E
        tol = g * S + U * (ref.abs() + g * S)
        err = (hout - ref).abs()
        fh.add(~(err <= tol), r0, hout, ref, tol)
        ratio = torch.where(S > 0, err / S.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        obs = max(obs, float(ratio.nan_to_num(math.inf).max()))
        del E, S, tol, err
        want16 = h32_out[r0:r1].to(torch.bfloat16).view(torch.int16)
        f16.add(h16_out[r0:r1].view(torch.int16) != want16, r0, h16_out[r0:r1].float(), h32_out[r0:r1].to(torch.bfloat16).float())
        sq = torch.zeros(r1 - r0, P * pc, dtype=torch.float64, device=hout.device)
        sq[:, :N] = hout * hout
        want_ss = sq.reshape(r1 - r0, P, pc).sum(2)  # [rows, P]
        n_terms = torch.full((P,), pc, dtype=torch.float64, device=hout.device)
        n_terms[-1] = N - (P - 1) * pc
        rel = torch.tensor([gamma_n(int(n) + 1) for n in n_terms.tolist()], dtype=torch.float64, device=hout.device)
        got_ss = ss_out[:, r0:r1].t().double()
        tol_ss = rel[None, :] * want_ss
        fss.add(~((got_ss - want_ss).abs() <= tol_ss), r0, got_ss, want_ss, tol_ss)
    if stats is not None:
        stats.update(gamma=g, observed_acc_err_over_S=obs, margin=(g / obs if obs > 0 else math.inf))
    return [fh, f16, fss]


def pack_ffn_up(W0: torch.Tensor, W1: torch.Tensor) -> torch.Tensor:
    """The packed FFN-up weight rpx_encoder_create writes: rows [256j, 256j + 128) are wi_0 rows
    [128j, 128j + 128), rows [256j + 128, 256j + 256) the wi_1 rows of the same hidden units."""
    F, K = W0.shape
    assert F % 128 == 0
    return torch.stack([W0.reshape(F // 128, 128, K), W1.reshape(F // 128, 128, K)], 1).reshape(2 * F, K)


def diagnose(findings: Findings, tile_m: int, tile_n: int) -> dict:
    """Where the bad elements of one output sit: per tile, per fragment row (row % 16: rows r and r + 8 of a
    wgmma fragment) and per fragment column (col % 8), per 32-column chunk."""
    from collections import Counter

    rows = [r for r, _ in findings.where]
    cols = [c for _, c in findings.where]
    return {
        "output": findings.name,
        "n_bad": findings.n_bad,
        "first": findings.where[:40],
        "samples": findings.samples,
        "by_tile": Counter(f"{r // tile_m},{c // tile_n}" for r, c in findings.where).most_common(24),
        "by_fragment_row": sorted(Counter(r % 16 for r in rows).items()),
        "by_fragment_col": sorted(Counter(c % 8 for c in cols).items()),
        "by_chunk32": Counter(c // 32 for c in cols).most_common(24),
        "rows": sorted(set(rows))[:64],
    }
