"""The tactic generator's forward on the H100: the attention kernel's causal and cross modes against the float64
reference of tests/attention_mode_ref.py (with exact cases), the whole forward (`T5GeneratorEngine`, rpx_seq2seq_forward)
against HF `T5ForConditionalGeneration` in fp32 and bf16, batch invariance, error codes and output bounds."""
import json
import math

import pytest
import torch

from reprover_b200 import _native, synth
from reprover_b200.generator import T5GeneratorEngine
from tests import attention_mode_ref as M
from tests import attention_ref as A
from tests import seq2seq_ref as S

pytestmark = pytest.mark.gpu
H = 6
INNER = H * 64


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cu(lens):
    out = [0]
    for n in lens:
        out.append(out[-1] + n)
    return out


def _dec_lut(lib, dev, seed=1, R=128, nb=32):
    g = torch.Generator().manual_seed(seed)
    rel = (torch.randn(nb, H, generator=g) * 2.0).to(dev)
    lut = torch.full((H, 2 * R + 1), float("nan"), device=dev)
    _native.check(lib.rpx_debug_attention_lut_ex(rel.data_ptr(), H, nb, R, 0, lut.data_ptr(), _stream()))
    assert torch.equal(lut.double(), M.hf_bias_lut_unidirectional(rel, nb, R)), "decoder LUT differs from HF's buckets"
    return lut


def _run(lib, mode, q, kv, cu_q, cu_k, lut, n_q, n_k, R=128):
    out = torch.full((n_q + 2, INNER), float("nan"), dtype=torch.bfloat16, device=q.device)
    cq = torch.tensor(cu_q, dtype=torch.int32, device=q.device)
    ck = torch.tensor(cu_k, dtype=torch.int32, device=q.device)
    max_len = max(b - a for a, b in zip(cu_q, cu_q[1:]))
    _native.check(lib.rpx_debug_attention_ex(mode, q.data_ptr(), None if kv is None else kv.data_ptr(), out.data_ptr(),
                                             cq.data_ptr(), ck.data_ptr(), None if lut is None else lut.data_ptr(),
                                             n_q, n_k, len(cu_q) - 1, max_len, H, R, _stream()))
    torch.cuda.synchronize()
    return out


def _assert_ok(findings):
    for f in findings:
        assert f.n_bad == 0, (f.name, f.n_bad, f.samples[:4])


@pytest.mark.parametrize("lens", [[1, 2, 63, 64, 65, 129, 300], [1024, 17, 640]])
def test_causal_attention_against_float64(rpx_lib, cuda_device, lens):
    lut = _dec_lut(rpx_lib, cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(sum(lens))
    cu = _cu(lens)
    qkv = A.random_qkv(cu[-1], H, g, device=cuda_device)
    out = _run(rpx_lib, _native.RPX_ATTN_CAUSAL, qkv, None, cu, cu, lut, cu[-1], 0)
    _assert_ok(M.check_attention_mode(out, qkv, qkv, cu, cu, H, True, lut, 128))


def test_causal_future_key_changes_nothing_before_it(rpx_lib, cuda_device):
    """A key with a huge score and value at position j0 must leave every query before it bit-identical."""
    lut = _dec_lut(rpx_lib, cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(7)
    lens = [300, 200]
    cu = _cu(lens)
    qkv = A.random_qkv(cu[-1], H, g, device=cuda_device)
    base = _run(rpx_lib, _native.RPX_ATTN_CAUSAL, qkv, None, cu, cu, lut, cu[-1], 0)
    for j0 in (0 + 100, 300 + 64):  # mid-tile in sequence 0, first key of a tile in sequence 1
        hot = qkv.clone()
        hot[j0, INNER:2 * INNER] = 30.0
        hot[j0, 2 * INNER:] = 1e4
        out = _run(rpx_lib, _native.RPX_ATTN_CAUSAL, hot, None, cu, cu, lut, cu[-1], 0)
        same = torch.arange(cu[-1], device=cuda_device)
        same = (same < j0) | (same >= (300 if j0 < 300 else cu[-1]))
        assert torch.equal(out[:cu[-1]][same].view(torch.int16), base[:cu[-1]][same].view(torch.int16))
        assert not torch.equal(out[j0], base[j0]), "the hot key is invisible to its own query"


def test_causal_bias_sweep_one_hot(rpx_lib, cuda_device):
    """q = k = 0: every visible score is the bias alone, so query i's weights are softmax over j <= i of
    lut[h][j - i]; one-hot values (v_j = e_(j mod 64) per head) read the weights back, each within bf16 rounding of the
    float64 value, across every unidirectional bucket (distances 0..700)."""
    lut = _dec_lut(rpx_lib, cuda_device, seed=3)
    L = 700
    qkv = torch.zeros(L, 3 * INNER, dtype=torch.bfloat16, device=cuda_device)
    for h in range(H):
        qkv[torch.arange(L), 2 * INNER + 64 * h + (torch.arange(L) % 64)] = 1.0
    out = _run(rpx_lib, _native.RPX_ATTN_CAUSAL, qkv, None, [0, L], [0, L], lut, L, 0)
    _assert_ok(M.check_attention_mode(out, qkv, qkv, [0, L], [0, L], H, True, lut, 128))


@pytest.mark.parametrize("case", [([1, 63, 64, 65, 7], [2300, 1, 64, 65, 63]), ([512, 3], [100, 2300])])
def test_cross_attention_against_float64(rpx_lib, cuda_device, case):
    lq, lk = case
    g = torch.Generator(device=cuda_device).manual_seed(len(lq) + sum(lk))
    cq, ck = _cu(lq), _cu(lk)
    xq = A.random_qkv(cq[-1], H, g, device=cuda_device)[:, :INNER].contiguous()
    xk = A.random_qkv(ck[-1], H, g, device=cuda_device)[:, INNER:].contiguous()  # k | v
    out = _run(rpx_lib, _native.RPX_ATTN_CROSS, xq, xk, cq, ck, None, cq[-1], ck[-1])
    _assert_ok(M.check_attention_mode(out, xq, xk, cq, ck, H, False))


# ---------------------------------------------------------------------------------------------- whole forward
def _hf(path, dtype):
    from transformers import T5ForConditionalGeneration

    m = T5ForConditionalGeneration.from_pretrained(path, torch_dtype=dtype).cuda().eval()
    return m


def _batch(cfg, in_lens, out_lens, seed, ignore_mid=True):
    g = torch.Generator().manual_seed(seed)
    rows = []
    for n in out_lens:
        r = torch.randint(3, cfg["vocab_size"], (n,), generator=g).tolist()
        if ignore_mid and n > 4:
            r[n // 2] = S.IGNORE
        rows.append(r if n else [S.IGNORE])
    return S.random_batch(cfg, in_lens, rows, seed)


def _compare(tmp_path, cfg, sd, ids, mask, labels, floor_logit, floor_lp, tag, out_dir):
    torch.set_float32_matmul_precision("highest")
    torch.backends.cuda.matmul.allow_tf32 = False
    synth.save_hf_checkpoint(str(tmp_path), cfg, sd)
    gen = T5GeneratorEngine.from_hf_dir(str(tmp_path), torch.device("cuda:0"))
    got = gen(input_ids=ids, attention_mask=mask, labels=labels)
    lens = S.decoder_lengths(labels)
    valid = (torch.arange(labels.shape[1])[None, :] < lens[:, None]).cuda()
    res = {}
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        m = _hf(str(tmp_path), dt)
        if "lm_head.weight" in sd and dt == torch.float32:
            assert S.untied_head_is_distinct(m.cpu(), sd), "HF oracle runs with a tied head"
            m.cuda()
        with torch.no_grad():
            o = m(input_ids=ids.cuda(), attention_mask=mask.cuda(), labels=labels.cuda())
        lg = o.logits.float()
        lp = torch.log_softmax(lg.double(), -1).gather(2, labels.cuda().clamp_min(0)[..., None])[..., 0]
        seq = torch.where(labels.cuda() != S.IGNORE, lp, torch.zeros_like(lp)).sum(1)
        res[name] = (lg, seq, float(o.loss))
        del m
        torch.cuda.empty_cache()
    ref_lg, ref_seq, ref_loss = res["fp32"]
    bf_lg, bf_seq, bf_loss = res["bf16"]
    e_lg = float((got.logits - ref_lg).abs()[valid].max())
    b_lg = float((bf_lg - ref_lg).abs()[valid].max())
    e_seq = float((got.sequence_log_probs - ref_seq).abs().max())
    b_seq = float((bf_seq - ref_seq).abs().max())
    e_loss, b_loss = abs(float(got.loss) - ref_loss), abs(bf_loss - ref_loss)
    stats = dict(tag=tag, engine_logit=e_lg, hf_bf16_logit=b_lg, engine_seq_lp=e_seq, hf_bf16_seq_lp=b_seq,
                 engine_loss=e_loss, hf_bf16_loss=b_loss, loss=ref_loss)
    with open(out_dir / f"generator_accuracy_{tag}.json", "w") as fh:
        json.dump(stats, fh, indent=1)
    assert torch.equal(got.num_tokens.cpu(), (labels != S.IGNORE).sum(1).int())
    assert bool((got.logits[~valid] == 0).all()), "logits past a row's decoder length must be zeros"
    # acceptance: no worse than HF bf16 against HF fp32 on the same inputs, with a floor
    assert e_lg <= max(b_lg, floor_logit), stats
    assert e_seq <= max(b_seq, floor_lp), stats
    assert e_loss <= max(b_loss, floor_lp / 100), stats
    gen.close()
    return got


def test_forward_against_hf_2_plus_2_layers(tmp_path, cuda_device, out_dir):
    cfg = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=21)
    ids, mask, labels = _batch(cfg, [2300, 1, 64, 65, 300, 17], [40, 1, 65, 0, 128, 512], seed=4)
    _compare(tmp_path, cfg, sd, ids, mask, labels, 0.05, 0.5, "2x2", out_dir)


def test_forward_against_hf_tied_head(tmp_path, cuda_device, out_dir):
    cfg = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0)
    cfg.pop("tie_word_embeddings")
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=22)
    ids, mask, labels = _batch(cfg, [200, 33, 5], [20, 64, 7], seed=5)
    _compare(tmp_path, cfg, sd, ids, mask, labels, 0.05, 0.5, "tied", out_dir)


def test_forward_against_hf_full_geometry_validation_batch(tmp_path, cuda_device, out_dir):
    cfg = dict(synth.BYT5_SMALL, decoder_start_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=23)
    g = torch.Generator().manual_seed(9)
    in_lens = torch.randint(100, 2301, (64,), generator=g).tolist()
    in_lens[0] = 2300
    out_lens = torch.randint(8, 513, (64,), generator=g).tolist()
    out_lens[1] = 512
    ids, mask, labels = _batch(cfg, in_lens, out_lens, seed=6)
    _compare(tmp_path, cfg, sd, ids, mask, labels, 0.1, 2.0, "12x4_b64", out_dir)


@pytest.fixture(scope="module")
def small_gen(tmp_path_factory):
    cfg = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=31)
    gen = T5GeneratorEngine(cfg, sd, torch.device("cuda:0"))
    yield cfg, gen
    gen.close()


def test_batch_invariance(cuda_device, small_gen):
    """Each row's sequence log-probability and logits are bit-identical scored alone and inside a 64-row batch
    padded to other lengths."""
    cfg, gen = small_gen
    g = torch.Generator().manual_seed(12)
    in_lens = torch.randint(1, 700, (64,), generator=g).tolist()
    out_lens = torch.randint(1, 200, (64,), generator=g).tolist()
    ids, mask, labels = _batch(cfg, in_lens, out_lens, seed=13)
    big = gen(input_ids=ids, attention_mask=mask, labels=labels)
    for b in (0, 17, 63):
        n_in, n_out = in_lens[b], out_lens[b]
        one = gen(input_ids=ids[b:b + 1, :n_in], attention_mask=mask[b:b + 1, :n_in], labels=labels[b:b + 1, :n_out])
        assert torch.equal(one.sequence_log_probs, big.sequence_log_probs[b:b + 1]), b
        assert torch.equal(one.logits[0], big.logits[b, :n_out]), b


def test_errors_and_bounds(cuda_device, small_gen):
    cfg, gen = small_gen
    lib = gen.lib
    ids, mask, labels = _batch(cfg, [30, 20], [10, 5], seed=14)
    bad = ids.clone()
    bad[1, 3] = cfg["vocab_size"]
    with pytest.raises(_native.RpxError) as ei:
        gen(input_ids=bad, attention_mask=mask, labels=labels)
    assert ei.value.code == _native.RPX_ERR_INVALID
    bl = labels.clone()
    bl[0, 2] = -5
    with pytest.raises(_native.RpxError) as ei:
        gen(input_ids=ids, attention_mask=mask, labels=bl)
    assert ei.value.code == _native.RPX_ERR_INVALID
    bm = mask.clone()
    bm[0, 0] = 0
    with pytest.raises(_native.RpxError) as ei:
        gen(input_ids=ids, attention_mask=bm, labels=labels)
    assert ei.value.code == _native.RPX_ERR_MASK
    with pytest.raises(NotImplementedError, match="past_key_values"):
        gen(input_ids=ids, attention_mask=mask, labels=labels, past_key_values=())
    # NaN sentinels past every output survive
    B, L_in = ids.shape
    L_out, V = labels.shape[1], cfg["vocab_size"]
    d_ids, d_mask, d_lab = ids.cuda(), mask.cuda(), labels.cuda()
    logits = torch.full((B * L_out * V + 1024,), float("nan"), device=cuda_device)
    lp = torch.full((B + 8,), float("nan"), dtype=torch.float64, device=cuda_device)
    cnt = torch.full((B + 8,), -7, dtype=torch.int32, device=cuda_device)
    ws = gen._workspace(B, L_in, L_out)
    _native.check(lib.rpx_seq2seq_forward(gen._handle, gen.encoder._handle, d_ids.data_ptr(), d_mask.data_ptr(), B, L_in,
                                          d_lab.data_ptr(), L_out, logits.data_ptr(), lp.data_ptr(), cnt.data_ptr(),
                                          ws.data_ptr(), ws.numel(), _stream()))
    torch.cuda.synchronize()
    assert bool(logits[B * L_out * V:].isnan().all()) and not bool(logits[:B * L_out * V].isnan().any())
    assert bool(lp[B:].isnan().all()) and bool((cnt[B:] == -7).all())
    ref = gen(input_ids=ids, attention_mask=mask, labels=labels)
    assert torch.equal(lp[:B], ref.sequence_log_probs)
    # a row with no counted label: loss over the others; all rows ignored: NaN as HF's empty mean
    none = torch.full_like(labels, S.IGNORE)
    out = gen(input_ids=ids, attention_mask=mask, labels=none)
    assert math.isnan(float(out.loss)) and bool((out.logits == 0).all())


# ---------------------------------------------------------------------------------------------- log-probs vs logits
U64 = 2.0 ** -53


def _logprob_bound(logits: torch.Tensor, labels: torch.Tensor):
    """Float64 sum of log_softmax(logits)[label] over each row's counted positions, and the bound on its difference
    from the engine's sum.  Per token, token_logprob_kernel computes d = fl64(x_y - mx), s = sum_j exp(fl64(x_j - mx))
    over V terms in fp64 and d - log s, whose error is delta_k = u |d| + 1.001 rho + 2.002 u log s + u (|d| + log s +
    1) with rho = gamma_{V-1} + 2u + V u / e (u = 2^-53; derived in tests/test_search_step_gpu.py, which runs the same
    arithmetic); seq_logprob_kernel adds the n counted terms in token order, gamma_n sum |lp|.  The float64 reference
    errs by at most as much again, so tol = 2 (sum delta_k + gamma_n sum |lp|)."""
    x = logits.double()
    V = x.shape[-1]
    mx = x.amax(-1, keepdim=True)
    log_s = (torch.logsumexp(x, -1, keepdim=True) - mx)[..., 0]
    lp = torch.log_softmax(x, -1).gather(-1, labels.clamp_min(0)[..., None])[..., 0]
    d = (x.gather(-1, labels.clamp_min(0)[..., None])[..., 0] - mx[..., 0]).abs()
    gamma = (V - 1) * U64 / (1 - (V - 1) * U64)
    rho = gamma + 2 * U64 + V * U64 / math.e
    delta = U64 * d + 1.001 * rho + 2.002 * U64 * log_s + U64 * (d + log_s + 1)
    counted = labels != S.IGNORE
    lp = torch.where(counted, lp, torch.zeros_like(lp))
    n = counted.sum(1)
    g_n = n.double() * U64 / (1 - n.double() * U64)
    tol = 2 * (torch.where(counted, delta, torch.zeros_like(delta)).sum(1) + g_n * lp.abs().sum(1))
    return lp.sum(1), n, tol


def _edge_labels(cfg, seed):
    """Rows with -100 at the first, a middle and the last position, single-token rows, rows whose only counted label is
    at out_len - 1, and longer rows with scattered -100."""
    g = torch.Generator().manual_seed(seed)
    V, L = cfg["vocab_size"], 40

    def rnd(n):
        return torch.randint(3, V, (n,), generator=g).tolist()

    I = S.IGNORE
    rows = [
        [I] + rnd(18) + [I] + rnd(19) + [I],         # -100 first, middle and last
        rnd(1),                                       # one token
        [I] * (L - 1) + rnd(1),                       # the only counted label at out_len - 1
        [I] * 7 + rnd(1),                             # one counted label after -100s, in a shorter row
        rnd(L),
        [I, I] + rnd(5) + [I] * 3 + rnd(9),
        rnd(1) + [I] * 20,                            # one token, then -100 to the end
    ]
    return rows


@pytest.mark.parametrize("head_scale", [1.0, 3000.0], ids=["plain", "logits_span_thousands"])
def test_sequence_log_probs_against_own_logits(tmp_path, cuda_device, head_scale):
    """sequence_log_probs is the float64 sum of log_softmax(logits)[label] over each row's counted positions of the
    engine's own returned logits, within the derived fp64 bound (about 1e-12 relative); the counts match and the loss
    is -sum(lp) / sum(n).  A dropped, duplicated or misaligned token's term is off by a whole log-probability."""
    cfg = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=33)
    sd["lm_head.weight"] = sd["lm_head.weight"] * head_scale
    gen = T5GeneratorEngine(cfg, sd, cuda_device)
    rows = _edge_labels(cfg, 7)
    ids, mask, labels = S.random_batch(cfg, [50, 3, 700, 17, 129, 64, 1], rows, seed=8)
    out = gen(input_ids=ids, attention_mask=mask, labels=labels)
    logits = out.logits.cpu()
    lens = S.decoder_lengths(labels)
    spread = logits[0, :int(lens[0])].amax(-1) - logits[0, :int(lens[0])].amin(-1)
    if head_scale > 1:
        assert float(spread.min()) > 1000, "the scaled head must give logits spanning thousands"
    want, n, tol = _logprob_bound(logits, labels)
    got = out.sequence_log_probs.cpu()
    assert torch.equal(out.num_tokens.cpu().long(), n)
    err = (got - want).abs()
    assert bool((err <= tol).all()), (err.tolist(), tol.tolist())
    assert bool((tol <= 1e-11 * want.abs().clamp_min(1.0)).all()), "the bound is of order 1e-12 relative"
    assert float(out.loss) == float(-out.sequence_log_probs.sum() / out.num_tokens.sum().double())
    assert abs(float(out.loss) - float(-want.sum() / n.sum())) <= float(tol.sum() / n.sum())
    gen.close()
