"""The encoder's per-token output (`T5EncoderEngine.__call__`, `rpx_encode_ids_hidden`) against HF
`T5EncoderModel` in fp32 and bf16, against the float64 checker of tests/hidden_ref.py, against the engine's own
pooled embedding, and as the `encoder` of the reference's own pooling code."""
import ctypes as C
import json
import math

import pytest
import torch

from reprover_b200 import _native, synth
from reprover_b200.engine import T5EncoderEngine
from tests import gemm_ref as R
from tests import hidden_ref as H
from tests.helpers import EMB_MAX_ABS, EMB_MIN_COS, compare_embeddings, ref

pytestmark = pytest.mark.gpu

EPS = float(torch.tensor(1e-6, dtype=torch.float32))
# lengths in tokens: 1-token rows, both sides of the 64 / 128 tile boundaries, a 2048-token row (tiny checkpoint only)
TINY_LENS = [1, 63, 64, 65, 127, 128, 129, 2048]
FULL_LENS = [1, 64, 65, 128, 129, 300]


@pytest.fixture(scope="module")
def tiny():
    cfg = synth.tiny_config(num_layers=2)
    return cfg, synth.random_t5_state_dict(cfg, seed=13)


@pytest.fixture(scope="module")
def full():
    cfg = dict(synth.BYT5_SMALL)
    return cfg, synth.random_t5_state_dict(cfg, seed=synth.SEED)


@pytest.fixture(scope="module")
def report(out_dir):
    rows = {}
    yield rows
    (out_dir / "encoder_hidden_accuracy.json").write_text(json.dumps(rows, indent=1))


def _padded_ids(lens, seed):
    """Right-padded int64 ids and prefix mask: random byte ids (3..258), EOS (1) last, pad id 0."""
    g = torch.Generator().manual_seed(seed)
    L = max(lens)
    ids = torch.zeros(len(lens), L, dtype=torch.int64)
    mask = torch.zeros(len(lens), L, dtype=torch.int64)
    for b, n in enumerate(lens):
        ids[b, :n - 1] = torch.randint(3, 259, (n - 1,), generator=g)
        ids[b, n - 1] = 1
        mask[b, :n] = 1
    return ids, mask


@torch.no_grad()
def _hf_rows(model, ids, lens):
    """HF last_hidden_state of each row's real tokens, each row run on its own (no padding), as fp64."""
    return [model(input_ids=ids[b:b + 1, :n]).last_hidden_state[0].double() for b, n in enumerate(lens)]


def _errors(got_rows, want_rows):
    """(max |got - want|, worst cosine of a token row) over every real position."""
    got, want = torch.cat(got_rows).double(), torch.cat(want_rows).double()
    cos = torch.nn.functional.cosine_similarity(got, want, dim=1)
    return float((got - want).abs().max()), float(cos.min())


def _hf_models(cfg, sd):
    torch.set_float32_matmul_precision("highest")
    f32 = ref.build_hf_encoder(cfg, sd)
    b16 = ref.build_hf_encoder(cfg, sd).to(torch.bfloat16)
    return f32, b16


def _vs_hf(eng, cfg, sd, lens, seed, report, tag):
    """Test (1): per token, the engine's error against HF fp32 is no worse than HF's bf16 model's."""
    ids, mask = _padded_ids(lens, seed)
    f32, b16 = _hf_models(cfg, sd)
    want = _hf_rows(f32, ids, lens)
    hf16 = _errors(_hf_rows(b16, ids, lens), want)
    rows = {"lens": lens, "hf_bf16": {"max_abs": hf16[0], "min_cos": hf16[1]}}
    for dtype in (torch.bfloat16, torch.float32):
        out = eng(ids.to(eng.device), mask.to(eng.device), out_dtype=dtype).last_hidden_state.cpu()
        assert out.shape == (len(lens), max(lens), cfg["d_model"]) and out.dtype == dtype
        got = _errors([out[b, :n] for b, n in enumerate(lens)], want)
        rows[f"engine_{str(dtype).split('.')[-1]}"] = {"max_abs": got[0], "min_cos": got[1]}
        for b, n in enumerate(lens):
            assert (out[b, n:] == 0).all() and not torch.signbit(out[b, n:]).any(), (b, n)
        assert got[0] <= hf16[0] and got[1] >= hf16[1], (tag, rows)
    report[tag] = rows


def test_tiny_matches_hf_per_token(rpx_lib, cuda_device, tiny, report):
    cfg, sd = tiny
    _vs_hf(T5EncoderEngine(cfg, sd, cuda_device), cfg, sd, TINY_LENS, 1, report, "tiny_throughput")


def test_byt5_small_matches_hf_per_token(rpx_lib, cuda_device, full, report):
    cfg, sd = full
    _vs_hf(T5EncoderEngine(cfg, sd, cuda_device), cfg, sd, FULL_LENS, 2, report, "byt5_small_throughput")


def test_latency_path_matches_hf_per_token(rpx_lib, cuda_device, tiny, report):
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    eng.set_latency_tokens(4096)
    _vs_hf(eng, cfg, sd, TINY_LENS[:-1], 3, report, "tiny_latency")


@pytest.mark.parametrize("latency", [False, True], ids=["throughput", "latency"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_store_against_float64_reference(rpx_lib, cuda_device, tiny, latency, dtype):
    """The final-norm store itself: every real row against the float64 RMSNorm of the final residual stream the
    kernel read (the engine's debug dump), zeros past each length."""
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    if latency:
        eng.set_latency_tokens(4096)
    lens = TINY_LENS[:-1] if latency else TINY_LENS
    ids, mask = _padded_ids(lens, 4)
    dump = eng.set_debug_hidden(sum(lens))
    out = eng(ids, mask, out_dtype=dtype).last_hidden_state
    torch.cuda.synchronize()
    h32 = dump[cfg["num_layers"]].clone()
    eng.set_debug_hidden(None)
    ln_w = sd["encoder.final_layer_norm.weight"].to(cuda_device)
    bad = H.check_hidden(out, h32, ln_w, lens, EPS, R.ss_parts(cfg["d_model"], latency))
    assert not bad, [f.summary() for f in bad]


def _readme_example(model, tokenizer, state, premises, k, device=None):
    """The reference README's "Premise Retriever" example (encode without an attention mask, unnormalised masked
    mean, dot-product top-k) with the model swapped in; `device`: where the tokenizer output goes."""
    def encode(s):
        squeeze = isinstance(s, str)
        tok = tokenizer([s] if squeeze else s, return_tensors="pt", padding=True)
        if device is not None:
            tok = tok.to(device)
        hidden = model(tok.input_ids).last_hidden_state
        lens = tok.attention_mask.sum(dim=1)
        features = (hidden * tok.attention_mask.unsqueeze(2)).sum(dim=1) / lens.unsqueeze(1)
        return (features.squeeze() if squeeze else features), hidden, tok

    with torch.no_grad():
        state_emb, _, _ = encode(state)
        premise_embs, hidden, tok = encode(premises)
        scores = state_emb @ premise_embs.T
    return scores.topk(k).indices.tolist(), scores.double().cpu(), hidden, tok


def test_no_mask_is_the_readme_example(rpx_lib, cuda_device, tiny, report):
    """attention_mask=None: pad tokens are encoded as ordinary tokens, as HF does; every position matches HF."""
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    f32, b16 = _hf_models(cfg, sd)
    tok = ref.build_hf_tokenizer()
    pd, po = synth.synth_premises(8, seed=21, min_len=10, max_len=300)
    premises = [s.decode() for s in synth.split_strings(pd, po)]
    state = synth.split_strings(*synth.synth_states(1, seed=22, min_len=50, max_len=200))[0].decode()
    top_ref, s_ref, h_ref, t_ref = _readme_example(f32, tok, state, premises, 4)
    _, s_b16, h_b16, _ = _readme_example(b16, tok, state, premises, 4)
    top_eng, s_eng, h_eng, t_eng = _readme_example(eng, tok, state, premises, 4, cuda_device)
    assert (t_ref.attention_mask == 0).any(), "the batch must have padded rows"
    assert torch.equal(t_eng.input_ids.cpu(), t_ref.input_ids)
    B, L = t_ref.input_ids.shape
    every = lambda h: [h[b].cpu() for b in range(B)]  # noqa: E731 - every position, pads included
    bar = _errors(every(h_b16), every(h_ref))
    got = _errors(every(h_eng), every(h_ref))
    bar_s, got_s = float((s_b16 - s_ref).abs().max()), float((s_eng - s_ref).abs().max())
    report["readme_no_mask"] = {"hf_bf16": bar, "engine": got, "score_err_hf_bf16": bar_s, "score_err_engine": got_s,
                                "top_ref": top_ref, "top_engine": top_eng}
    assert got[0] <= bar[0] and got[1] >= bar[1], report["readme_no_mask"]
    assert top_eng == top_ref and got_s <= bar_s, report["readme_no_mask"]


def test_drop_in_for_the_reference_encode_and_reindex(rpx_lib, cuda_device, tiny):
    """The engine as `self.encoder` under the reference's own `_encode` and a `reindex_corpus`-shaped loop."""
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    tokenizer = ref.build_hf_tokenizer()
    data, offsets = synth.synth_premises(20, seed=23, min_len=1, max_len=600)
    texts = [s.decode() for s in synth.split_strings(data, offsets)]
    torch.set_float32_matmul_precision("highest")
    want = ref.reindex_corpus(ref.build_hf_encoder(cfg, sd), tokenizer, texts, 8, 512)
    # retrieval/model.py:190-208 with the engine as the encoder: ids and mask moved to the device (:205)
    got = torch.zeros(len(texts), eng.config.hidden_size, dtype=eng.dtype, device=cuda_device)
    for i in range(0, len(texts), 8):
        tok = ref.tokenize(tokenizer, texts[i:i + 8], 512).to(cuda_device)
        got[i:i + 8] = ref.encode(eng, tok.input_ids, tok.attention_mask)
    max_abs, min_cos = compare_embeddings(got, want)
    assert got.dtype == torch.bfloat16
    assert max_abs <= EMB_MAX_ABS + 2e-3 and min_cos >= EMB_MIN_COS, (max_abs, min_cos)  # + bf16 pooling
    # `self.encoder(input_ids, attention_mask)[0]` (retrieval/model.py:97-99) is the same tensor
    tok = ref.tokenize(tokenizer, texts[:8], 512).to(cuda_device)
    assert torch.equal(eng(tok.input_ids, tok.attention_mask)[0],
                       eng(input_ids=tok.input_ids, attention_mask=tok.attention_mask, return_dict=True).last_hidden_state)


@pytest.mark.parametrize("latency", [False, True], ids=["throughput", "latency"])
def test_fp32_hidden_pools_to_the_engine_embedding(rpx_lib, cuda_device, tiny, latency):
    """Masked mean + L2 normalise of the fp32 hidden output, in float64, against `encode_ids(out_dtype=fp32)`.

    Both use the same fp32 row scale and differ only in rounding.  Per element e, with S_e = sum_t |y_te| / len:
    the pool kernel's fp32 sum over len tokens errs by gamma_len S_e, its scaling by w / len and the stored
    products v * rs by 4u S_e; the hidden output's two products by 2u S_e.  So |x_e - x'_e| <= E_e =
    (gamma_len + 8u) S_e before normalisation.  x / ||x|| then moves by at most E_e / n + |out_e| ||E|| / n with
    n = ||x||, plus the fp32 norm (gamma_D) and the final products: |out_e| (gamma_D + 8u)."""
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    if latency:
        eng.set_latency_tokens(4096)
    lens = TINY_LENS[:-1] if latency else TINY_LENS
    ids, mask = _padded_ids(lens, 5)
    ids, mask = ids.to(cuda_device), mask.to(cuda_device)
    hid = eng(ids, mask, out_dtype=torch.float32).last_hidden_state.double()
    emb = eng.encode_ids(ids, mask, out_dtype=torch.float32).double()
    D = cfg["d_model"]
    for b, n in enumerate(lens):
        y = hid[b, :n]
        x = y.sum(0) / n
        norm = x.norm()
        out = x / norm
        E = (R.gamma_n(n) + 8 * R.U) * y.abs().sum(0) / n
        bound = (E / norm + out.abs() * (E.norm() / norm + R.gamma_n(D) + 8 * R.U)) * 1.01
        assert ((emb[b] - out).abs() <= bound).all(), (b, n, float(((emb[b] - out).abs() / bound).max()))


@pytest.mark.parametrize("latency", [False, True], ids=["throughput", "latency"])
def test_rows_do_not_depend_on_the_batch(rpx_lib, cuda_device, full, latency):
    """On each path a sequence's rows are bit-identical alone and inside a padded batch."""
    cfg, sd = full
    cfg = dict(cfg, num_layers=3)
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    if latency:
        eng.set_latency_tokens(4096)
    lens = [1, 64, 65, 128, 129, 300]
    ids, mask = _padded_ids(lens, 6)
    ids, mask = ids.to(cuda_device), mask.to(cuda_device)
    batch = eng(ids, mask, out_dtype=torch.float32).last_hidden_state
    for b, n in enumerate(lens):
        alone = eng(ids[b:b + 1, :n], out_dtype=torch.float32).last_hidden_state
        assert torch.equal(alone[0], batch[b, :n]), (b, n)


def test_rows_past_the_output_are_untouched(rpx_lib, cuda_device, tiny):
    """rpx_encode_ids_hidden writes batch * seq_len rows and nothing after them (NaN sentinels), with and
    without a mask."""
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    lens = [3, 70, 1]
    ids, mask = _padded_ids(lens, 7)
    ids, mask = ids.to(cuda_device), mask.to(cuda_device)
    B, L = ids.shape
    D = cfg["d_model"]
    ws = eng._workspace(B * L, B)
    for dtype, nan_bits in ((torch.bfloat16, R.BF16_NAN_BITS), (torch.float32, R.F32_NAN_BITS)):
        for m in (mask, None):
            buf = torch.full((B * L + 5, D), float("nan"), dtype=dtype, device=cuda_device)
            _native.check(eng.lib.rpx_encode_ids_hidden(
                eng._handle, ids.data_ptr(), None if m is None else m.data_ptr(), B, L, buf.data_ptr(),
                eng._out_dtype(dtype), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream))
            torch.cuda.synchronize()
            f = R.check_sentinels("past_end", buf.cpu(), B * L * D, nan_bits)
            assert not f, f.summary()
            assert not buf[:B * L].isnan().any()
            want = eng(ids, m, out_dtype=dtype).last_hidden_state.reshape(B * L, D)
            assert torch.equal(buf[:B * L], want)


def test_bad_input_raises_as_encode_ids_does(rpx_lib, cuda_device, tiny):
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    ids = torch.randint(3, 259, (2, 16), device=cuda_device)
    mask = torch.ones(2, 16, dtype=torch.int64, device=cuda_device)
    mask[1, 5] = 0  # hole: not a prefix mask
    for call in (eng, eng.encode_ids):
        with pytest.raises(_native.RpxError) as ei:
            call(ids, mask)
        assert ei.value.code == _native.RPX_ERR_MASK
    bad = ids.clone()
    bad[0, 0] = 999
    for m in (torch.ones_like(mask), None):
        with pytest.raises(_native.RpxError) as ei:
            eng(bad, m)
        assert ei.value.code == _native.RPX_ERR_INVALID and "outside" in str(ei.value)
    for kw in ({"output_hidden_states": True}, {"output_attentions": True}, {"inputs_embeds": torch.zeros(2, 16, 1472)},
               {"head_mask": torch.ones(2, 6)}):
        with pytest.raises(NotImplementedError):
            eng(ids, **kw)
    assert eng.dtype == torch.bfloat16 and eng.config.hidden_size == cfg["d_model"]
    assert math.isfinite(float(eng(ids).last_hidden_state.float().abs().max()))
