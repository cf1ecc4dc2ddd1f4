"""The encoder's T5 attention kernel, launched exactly as the forward pass launches it (rpx_debug_attention calls
the same launch_t5_attention, PDL scope as forward() sets it), against the float64 reference and the
rounding-aware checker of tests/attention_ref.py, plus exact cases that need no tolerance.

Every case writes into a NaN-filled [T + 2, H 64] output (rows past the last sequence must keep the sentinel)
and checks that qkv is unchanged afterwards.  The observed error of every tolerance case is written to
attention_accuracy.json; a failing case writes attention_diag_<case>.json (bad elements by sequence, head,
64-query tile, wgmma fragment row and the 64-key step of the row's largest-weight key)."""
import json
import math
import random

import numpy as np
import pytest
import torch

from reprover_b200 import _native, synth
from tests import attention_ref as A
from tests import gemm_ref as G
from tests.test_gemm_epilogues_gpu import Case as GemmCase

pytestmark = pytest.mark.gpu

PAD = 2
ACCURACY = []
LENGTHS = [1, 2, 63, 64, 65, 127, 128, 129, 255, 257, 1023, 1024, 2047, 2048]


@pytest.fixture(scope="module", autouse=True)
def _accuracy_artefact(out_dir):
    yield
    (out_dir / "attention_accuracy.json").write_text(json.dumps(ACCURACY, indent=0))


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cu(lens):
    return [0] + np.cumsum(lens).tolist()


def _lut(lib, rel_bias, R):
    """Device LUT from rpx_debug_attention_lut; it must equal the table built from HF's bucket function."""
    B, H = rel_bias.shape
    lut = torch.full((H, 2 * R + 1), float("nan"), device=rel_bias.device)
    _native.check(lib.rpx_debug_attention_lut(rel_bias.data_ptr(), H, B, R, lut.data_ptr(), _stream()))
    want = A.hf_bias_lut(rel_bias, B, R)
    assert torch.equal(lut.double(), want), f"LUT ({B}, {R}) differs from HF's bucket table"
    return lut


def _buffers(cu, n_tokens, H, dev):
    """Device cu_seqlens and a NaN-filled [n_tokens + 2, H 64] output.  Copying the host list to the device
    synchronises the stream, so a chained launch must make these before its first kernel."""
    out = torch.full((n_tokens + PAD, H * 64), float("nan"), dtype=torch.bfloat16, device=dev)
    return torch.tensor(cu, dtype=torch.int32, device=dev), out


def _launch(lib, qkv, cu, cu_d, out, H, lut, R, max_len=None, n_tokens=None, latency=False):
    """Enqueue the attention only: no allocation, copy or synchronisation."""
    n_tokens = qkv.shape[0] if n_tokens is None else n_tokens
    max_len = max(b - a for a, b in zip(cu, cu[1:])) if max_len is None else max_len
    _native.check(lib.rpx_debug_attention(int(latency), qkv.data_ptr(), out.data_ptr(), cu_d.data_ptr(), lut.data_ptr(),
                                          n_tokens, len(cu) - 1, max_len, H, R, _stream()))


def _attend(lib, qkv, cu, H, lut, R, max_len=None, n_tokens=None, latency=False):
    """Launch on a NaN-filled [n_tokens + 2, H 64] output and synchronise; returns it, qkv checked unchanged."""
    n_tokens = qkv.shape[0] if n_tokens is None else n_tokens
    cu_d, out = _buffers(cu, n_tokens, H, qkv.device)
    before = qkv.clone()
    _launch(lib, qkv, cu, cu_d, out, H, lut, R, max_len, n_tokens, latency)
    torch.cuda.synchronize()
    assert torch.equal(qkv.view(torch.int16), before.view(torch.int16)), "attention wrote to qkv"
    return out


def _check(tag, out, qkv, cu, H, lut, R, out_dir, record=True):
    stats = {}
    found = A.check_attention(out, qkv, cu, H, lut.double(), R, stats)
    if record:
        ACCURACY.append({"case": tag, "heads": H, "n_seqs": len(cu) - 1, "n_tokens": cu[-1], **stats})
    bad = [f for f in found if f]
    if bad:
        diag = {"case": tag, "findings": [A.diagnose(f) for f in bad]}
        (out_dir / f"attention_diag_{tag}.json").write_text(json.dumps(diag, indent=1))
        pytest.fail(f"{tag}: " + "; ".join(f.summary() for f in bad)[:3000])


def _packing(seed):
    """The lengths of LENGTHS shuffled, the longest last in the buffer."""
    rng = random.Random(seed)
    lens = LENGTHS[:-1]
    rng.shuffle(lens)
    return lens + [LENGTHS[-1]]


# ------------------------------------------------------------------------------------- random vs tolerance
@pytest.mark.parametrize("H", [1, 6, 12, 16])
@pytest.mark.parametrize("packing", ["shuffled", "max_len_over", "pdl_off"])
def test_random_against_reference(rpx_lib, cuda_device, out_dir, H, packing):
    """Lengths at every 64-boundary and up to 2048 in a shuffled packing (t0 mod 64 takes many values); q rows
    from flat (|s| ~ 1) to sharp (|s| ~ 50).
      shuffled      the sequences fill the call: the last one's TMA boxes run past n_tokens (zero fill)
      max_len_over  max_len 2100: the CTAs of query tiles past every length exit early
      pdl_off       the call has 16400 tokens, so PDL is off; the 9167 rows after the last sequence belong to
                    no sequence: its boxes read them as real data, and their output rows must not be written"""
    seed = 100 * H + len(packing)
    lens = _packing(seed)
    cu = _cu(lens)
    n_tokens = 16400 if packing == "pdl_off" else cu[-1]
    g = torch.Generator(device=cuda_device).manual_seed(seed)
    qkv = A.random_qkv(n_tokens, H, g, cuda_device)
    rel = torch.randn(32, H, generator=g, device=cuda_device) * 2
    lut = _lut(rpx_lib, rel, 128)
    max_len = 2100 if packing == "max_len_over" else None
    out = _attend(rpx_lib, qkv, cu, H, lut, 128, max_len=max_len)
    _check(f"random_H{H}_{packing}", out, qkv, cu, H, lut, 128, out_dir)


def test_many_short_sequences(rpx_lib, cuda_device, out_dir):
    """4000 sequences of 1-40 tokens (ByT5-small heads)."""
    rng = np.random.default_rng(7)
    cu = _cu(rng.integers(1, 41, size=4000).tolist())
    g = torch.Generator(device=cuda_device).manual_seed(7)
    qkv = A.random_qkv(cu[-1], 6, g, cuda_device)
    lut = _lut(rpx_lib, torch.randn(32, 6, generator=g, device=cuda_device), 128)
    out = _attend(rpx_lib, qkv, cu, 6, lut, 128)
    _check("many_short_H6", out, qkv, cu, 6, lut, 128, out_dir)


# --------------------------------------------------------------------------------------------- exact routing
ROUTING_LENS = [130, 1, 65, 2, 300, 63, 1000, 2048]
N_BITS = 11  # codes of key indices < 2048


def _code(j):
    """[..., 11] +-1 binary code of the integers j."""
    bits = (j[..., None] >> torch.arange(N_BITS, device=j.device)) & 1
    return bits.float() * 2 - 1


def _routing_case(dev):
    """Head h routes query i to key pi_h(i) of its own sequence: k_j = code(j), q_i = 64 code(pi_h(i)) in dims
    0-10, so q.k = 64 (11 - 2 hamming) and every other key sits at least 128 below the target (a weight of
    e^-126 or less after the bias, |bias| <= 1: exactly 0 in fp32 even without ftz).  Every sequence uses the
    same codes, so a key leaking in from a neighbour ties with the target when it carries the target's code:
    with head 2 (every query -> key 0) a leak of key len, the next sequence's key 0, averages the output with
    that key's v (another sequence id), and
    head 3 (every query -> key len - 1) loses its target if the mask drops that key.  In the other heads a
    leaked key scores at least 128 below the target and weighs 0, so there only the random cases can see a
    leak.  A target pi(i) >= 64
    has Hamming-1 neighbours pi(i) - 2^b (b >= 6) in earlier key steps, which hold the row maximum until the
    target's step: the rescale path runs.  v holds bf16-exact integers: key index mod 128, key index // 128,
    sequence, head."""
    H = 5
    lens = ROUTING_LENS
    cu = _cu(lens)
    T, inner = cu[-1], H * 64
    qkv = torch.zeros(T, 3 * inner, device=dev)
    g = torch.Generator().manual_seed(3)
    pis = []
    for s, L in enumerate(lens):
        t0 = cu[s]
        j = torch.arange(L, device=dev)
        per_head = [j, L - 1 - j, torch.zeros_like(j), torch.full_like(j, L - 1), torch.randperm(L, generator=g).to(dev)]
        pis.append(per_head)
        for h in range(H):
            qkv[t0:t0 + L, h * 64:h * 64 + N_BITS] = 64 * _code(per_head[h])
            qkv[t0:t0 + L, inner + h * 64:inner + h * 64 + N_BITS] = _code(j)
            vb = 2 * inner + h * 64
            qkv[t0:t0 + L, vb + 0] = (j % 128).float()
            qkv[t0:t0 + L, vb + 1] = (j // 128).float()
            qkv[t0:t0 + L, vb + 2] = s
            qkv[t0:t0 + L, vb + 3] = h
            qkv[t0:t0 + L, vb + 4:vb + 64] = ((j[:, None] * 7 + torch.arange(60, device=dev)) % 61 - 30).float()
    return qkv.to(torch.bfloat16), cu, H, pis


def test_exact_routing(rpx_lib, cuda_device, out_dir):
    qkv, cu, H, pis = _routing_case(cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(4)
    rel = torch.rand(32, H, generator=g, device=cuda_device) * 2 - 1
    lut = _lut(rpx_lib, rel, 128)
    out = _attend(rpx_lib, qkv, cu, H, lut, 128)
    inner = H * 64
    wrong = []
    for s in range(len(cu) - 1):
        t0, L = cu[s], cu[s + 1] - cu[s]
        for h in range(H):
            want = qkv[t0 + pis[s][h], 2 * inner + h * 64:2 * inner + (h + 1) * 64]
            got = out[t0:t0 + L, h * 64:(h + 1) * 64]
            rows = (got.view(torch.int16) != want.view(torch.int16)).any(1).nonzero().flatten()
            for i in rows[:4].tolist():
                key = float(got[i, 0]) + 128 * float(got[i, 1])
                wrong.append(f"seq {s} head {h} query {i}: want key {int(pis[s][h][i])}, got key {key} of seq "
                             f"{float(got[i, 2])} head {float(got[i, 3])}")
    assert not wrong, "\n".join(wrong[:40])
    pad = G.check_sentinels("attn.pad", out, cu[-1] * inner, G.BF16_NAN_BITS)
    assert not pad, pad.summary()
    _check("exact_routing", out, qkv, cu, H, lut, 128, out_dir)


# ---------------------------------------------------------------------------------------- bias-bucket sweep
BUCKET_CONFIGS = [(32, 128), (32, 16), (8, 4), (64, 2048)]


@pytest.mark.parametrize("buckets,R", BUCKET_CONFIGS)
def test_bias_bucket_sweep(rpx_lib, cuda_device, out_dir, buckets, R):
    """q = k = 0, one head per bucket, head h's table +150 on bucket h and 0 elsewhere: each query averages v
    over exactly the keys whose delta = key - query falls in bucket h (uniformly over all keys when none does);
    every other key's weight is e^-150, exactly 0 in the kernel.  All weights of a row are the same fp32 value
    p within 2^-16 of 1 (it rounds to bf16 1.0), and v holds small integers whose sums are exact, so the errors
    are |p - 1|, the fp32 sum l of up to 2048 copies of p, 1 / l and the product, all relative to the output,
    plus the rescale factor ex2(0) of each key step: the PTX ISA bounds it only to within 2^-22 of 1, which
    moves the weights of earlier steps against later ones by up to n_kt 2^-22 and the output by that times
    max_j |v_j - ref|.  That last allowance is absolute: on a row whose mean is near 0 it spans several bf16
    ulps (up to a few tens on 2048-key rows), so the check is bit-exact only on rows with |ref| well above
    n_kt 2^-22 max |v - ref|.  A key in the wrong bucket still moves its row by about |v_j - ref| / n, far
    outside that.  The lengths reach |delta| = max_distance - 1, max_distance, max_distance + 1 and 2047."""
    H = buckets
    lens = [R + 2, 5] if R >= 2048 else [R + 2, 5, 2048]
    cu = _cu(lens)
    T, inner = cu[-1], H * 64
    qkv = torch.zeros(T, 3 * inner, device=cuda_device)
    j = torch.arange(T, device=cuda_device)[:, None]
    c = torch.arange(inner, device=cuda_device)[None, :]
    qkv[:, 2 * inner:] = ((j * 5 + c * 3) % 17 - 8).float()
    qkv = qkv.to(torch.bfloat16)
    rel = torch.eye(buckets, device=cuda_device) * 150
    lut = _lut(rpx_lib, rel, R)
    out = _attend(rpx_lib, qkv, cu, H, lut, R)
    from transformers.models.t5.modeling_t5 import T5Attention

    bad = []
    for s in range(len(cu) - 1):
        t0, L = cu[s], cu[s + 1] - cu[s]
        pos = torch.arange(L)
        bucket = T5Attention._relative_position_bucket(pos[None, :] - pos[:, None], True, buckets, R).to(cuda_device)
        n_kt = -(-L // 64)
        for h in range(H):
            M = (bucket == h).double()
            n = M.sum(1, keepdim=True)
            M = torch.where(n > 0, M, torch.ones_like(M))
            n = M.sum(1, keepdim=True)
            v = qkv[t0:t0 + L, 2 * inner + h * 64:2 * inner + (h + 1) * 64].double()
            ref = (M @ v) / n
            spread = torch.maximum(v.amax(0) - ref, ref - v.amin(0))  # >= |v_j - ref_i| for every key j
            tol = 1.01 * (ref.abs() * (2.0 ** -16 + G.gamma_n(L + n_kt + 2) + 2 * G.U) + n_kt * A.ETA_EX2 * spread) + 1e-30
            got = out[t0:t0 + L, h * 64:(h + 1) * 64]
            b = G.bf16_bracket_bad(got, ref, tol)
            if bool(b.any()):
                i, col = b.nonzero()[0].tolist()
                bad.append(f"seq {s} (len {L}) head/bucket {h}: {int(b.sum())} bad, first query {i} col {col}: "
                           f"got {float(got[i, col])} want {float(ref[i, col])} over {int(n[i])} keys")
    pad = G.check_sentinels("attn.pad", out, T * inner, G.BF16_NAN_BITS)
    assert not bad and not pad, "\n".join(bad[:40]) + (pad.summary() if pad else "")


# ----------------------------------------------------------------------------------------- packing invariance
def test_packing_invariance(rpx_lib, cuda_device):
    """One 150-token sequence's output is bit-identical alone, at t0 = 1, 17, 63, 64 between other sequences,
    with a larger max_len, and in a call past 16384 tokens, with PDL off (throughput path) and on (latency
    path).  Below 16384 tokens both paths run under PDL, so the latency flag changes nothing there."""
    H, R, L = 6, 128, 150
    g = torch.Generator(device=cuda_device).manual_seed(9)
    x = A.random_qkv(L, H, g, cuda_device)
    filler = A.random_qkv(20000, H, g, cuda_device)
    lut = _lut(rpx_lib, torch.randn(32, H, generator=g, device=cuda_device), R)
    alone = _attend(rpx_lib, x, [0, L], H, lut, R)[:L]

    def embedded(t0, tail_lens, **kw):
        before = [t0] if t0 < 64 else [t0 - 40, 40]
        lens = before + [L] + tail_lens
        n = sum(lens)
        qkv = torch.cat([filler[:t0], x, filler[t0:t0 + n - t0 - L]])
        out = _attend(rpx_lib, qkv, _cu(lens), H, lut, R, **kw)
        return out[t0:t0 + L]

    runs = {f"t0={t0}": embedded(t0, [90, 33]) for t0 in (1, 17, 63, 64)}
    runs["max_len=1000"] = _attend(rpx_lib, x, [0, L], H, lut, R, max_len=1000)[:L]
    runs["pdl_off"] = embedded(17, [1000] * 17)  # 17 + 150 + 17000 tokens
    runs["pdl_on_latency"] = embedded(17, [1000] * 17, latency=True)  # the latency path keeps PDL on at any size
    for name, got in runs.items():
        diff = (got.view(torch.int16) != alone.view(torch.int16)).nonzero()
        assert diff.numel() == 0, f"{name}: differs from the sequence alone at {diff[:8].tolist()}"


# --------------------------------------------------------------------------------------------------- grid limit
def test_grid_limit_65535_sequences(rpx_lib, cuda_device, out_dir):
    rng = np.random.default_rng(11)
    cu = _cu(rng.integers(1, 4, size=65535).tolist())
    H = 2
    g = torch.Generator(device=cuda_device).manual_seed(11)
    qkv = A.random_qkv(cu[-1], H, g, cuda_device)
    lut = _lut(rpx_lib, torch.randn(32, H, generator=g, device=cuda_device), 128)
    out = _attend(rpx_lib, qkv, cu, H, lut, 128)
    _check("grid_65535_seqs", out, qkv, cu, H, lut, 128, out_dir)


def test_grid_limit_65536_sequences_rejected(rpx_lib, cuda_device):
    cu = torch.arange(65537, dtype=torch.int32, device=cuda_device)
    H = 1
    qkv = torch.zeros(65536, 3 * 64, dtype=torch.bfloat16, device=cuda_device)
    lut = torch.zeros(H, 257, device=cuda_device)
    out = torch.full((65536 + PAD, 64), float("nan"), dtype=torch.bfloat16, device=cuda_device)
    rc = rpx_lib.rpx_debug_attention(0, qkv.data_ptr(), out.data_ptr(), cu.data_ptr(), lut.data_ptr(), 65536, 65536, 1, H,
                                     128, _stream())
    assert rc == _native.RPX_ERR_UNSUPPORTED and "65535" in _native.last_error()
    torch.cuda.synchronize()
    assert bool((out.view(torch.int16) == G.BF16_NAN_BITS).all()), "a rejected call wrote output"


def test_engine_splits_calls_at_the_grid_limit(rpx_lib, cuda_device):
    """encode_bytes of 65635 short strings (one call's token budget) == the first 65535 and the last 100 encoded
    separately, bit for bit: the engine cuts calls at MAX_SEQS_PER_CALL sequences."""
    from reprover_b200.engine import T5EncoderEngine

    cfg = synth.tiny_config(num_layers=2)
    eng = T5EncoderEngine(cfg, synth.random_t5_state_dict(cfg, seed=12), cuda_device)
    n = T5EncoderEngine.MAX_SEQS_PER_CALL + 100
    data, offsets = synth.synth_byte_strings(n, seed=13, min_len=1, max_len=3)
    together = eng.encode_bytes(data, offsets, 2048, out_dtype=torch.float32)
    k = T5EncoderEngine.MAX_SEQS_PER_CALL
    first = eng.encode_bytes(data[:offsets[k]], offsets[:k + 1], 2048, out_dtype=torch.float32)
    last = eng.encode_bytes(data[offsets[k]:], offsets[k:] - offsets[k], 2048, out_dtype=torch.float32)
    torch.cuda.synchronize()
    assert torch.equal(together[:k], first) and torch.equal(together[k:], last)


# ------------------------------------------------------------------------------------------ chain under PDL
@pytest.mark.parametrize("latency,T,lens", [(True, 200, [37, 100, 63]), (False, 1000, [300, 64, 1, 635])],
                         ids=["latency", "throughput"])
def test_chain_qkv_attention_oproj_under_pdl(rpx_lib, cuda_device, out_dir, latency, T, lens):
    """QKV projection -> attention -> O-proj enqueued back to back on one stream with no synchronisation, into
    NaN-initialised intermediates (PDL is on at these T), so each kernel may start while its predecessor still
    runs.  Every buffer, cu_seqlens included, exists before the first launch, and PyTorch's sync debug mode
    raises on the synchronising tensor operations it detects between the launches (copying a Python list to
    the device is one).  Attention is checked against
    the reference built from the qkv actually written, O-proj against the attention output actually written: a
    read before the predecessor's writes land shows up as NaN or stale data."""
    H, R = 6, 128
    a = GemmCase("qkv", "byt5_small", T, latency, 51, cuda_device)
    b = GemmCase("oproj", "byt5_small", T, latency, 52, cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(53)
    lut = _lut(rpx_lib, torch.randn(32, H, generator=g, device=cuda_device), R)
    cu = _cu(lens)
    assert cu[-1] == T
    cu_d, attn = _buffers(cu, T, H, cuda_device)
    b.A = attn
    qkv = a.out[:T]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _native.check(a.run(rpx_lib))
        _launch(rpx_lib, qkv, cu, cu_d, attn, H, lut, R, latency=latency)
        _native.check(b.run(rpx_lib))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    found_a, _ = a.check()
    assert not any(found_a), [f.summary() for f in found_a if f]
    _check(f"chain_{'lat' if latency else 'thr'}_T{T}", attn, a.out[:T].contiguous(), cu, H, lut, R, out_dir)
    found_b, _ = b.check(A=attn[:T])
    assert not any(found_b), [f.summary() for f in found_b if f]


# ----------------------------------------------------------------------------------------------- entry points
def test_entry_points_reject_bad_input(rpx_lib, cuda_device):
    t = torch.zeros(1 << 16, dtype=torch.float32, device=cuda_device)
    p = t.data_ptr()
    st = _stream()

    def att(qkv=p, out=p, cu=p, lut=p, n_tokens=4, n_seqs=1, max_len=4, H=1, R=128):
        return rpx_lib.rpx_debug_attention(0, qkv, out, cu, lut, n_tokens, n_seqs, max_len, H, R, st)

    for kw in ({"qkv": None}, {"out": None}, {"cu": None}, {"lut": None}, {"n_tokens": 0}, {"max_len": 0}, {"H": 0},
               {"n_seqs": 0}, {"R": 0}):
        assert att(**kw) == _native.RPX_ERR_INVALID, kw
    assert att(n_seqs=65536) == _native.RPX_ERR_UNSUPPORTED
    lut = rpx_lib.rpx_debug_attention_lut
    assert lut(None, 6, 32, 128, p, st) == _native.RPX_ERR_INVALID
    assert lut(p, 6, 32, 128, None, st) == _native.RPX_ERR_INVALID
    assert lut(p, 0, 32, 128, p, st) == _native.RPX_ERR_INVALID
    for buckets, R in ((32, 8), (8, 2), (30, 64), (32, 2049)):
        assert lut(p, 6, buckets, R, p, st) == _native.RPX_ERR_UNSUPPORTED, (buckets, R)
        assert "relative attention config" in _native.last_error()
    torch.cuda.synchronize()
    assert torch.count_nonzero(t) == 0
