"""Parity of the CUDA encoder path (rpx_encode_bytes / rpx_encode_ids through the C ABI)
against the HF-based CPU oracle on the same synthetic checkpoint and inputs."""
import json

import numpy as np
import pytest
import torch

from reprover_b200 import _native, synth
from reprover_b200.engine import T5EncoderEngine
from tests.helpers import EMB_MAX_ABS, EMB_MIN_COS, compare_embeddings, oracle_embeddings, ref

pytestmark = pytest.mark.gpu


def _hidden_report(engine, cfg, sd, data, offsets, max_len, out_dir, tag):
    """Layer-by-layer relative error of the residual stream (diagnostic artefact)."""
    texts = [s.decode() for s in synth.split_strings(data, offsets)]
    enc = ref.build_hf_encoder(cfg, sd)
    tok = ref.tokenize(ref.build_hf_tokenizer(), texts, max_len)
    with torch.no_grad():
        hs = enc(input_ids=tok.input_ids, attention_mask=tok.attention_mask, output_hidden_states=True).hidden_states
    lens = tok.attention_mask.sum(1).tolist()
    T = int(sum(lens))
    dump = engine.set_debug_hidden(T)
    engine.encode_bytes(data, offsets, max_len)
    torch.cuda.synchronize()
    dump = dump.cpu()
    engine.set_debug_hidden(None)
    rows = []
    for l in range(cfg["num_layers"]):
        want = torch.cat([hs[l][b, :lens[b]] for b in range(len(lens))], 0)
        err = (dump[l] - want).abs().max().item()
        rel = err / want.abs().max().item()
        rows.append({"layer_in": l, "max_abs": err, "rel_to_max": rel})
    (out_dir / f"encoder_hidden_{tag}.json").write_text(json.dumps(rows, indent=1))
    return rows


@pytest.fixture(scope="module")
def tiny():
    cfg = synth.tiny_config(num_layers=2)
    return cfg, synth.random_t5_state_dict(cfg, seed=11)


def test_tiny_encoder_matches_oracle(rpx_lib, cuda_device, out_dir, tiny):
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    # ragged lengths incl. 1-byte strings, tile boundaries (63/64/65, 127/128) and > 2 key tiles
    lens = [1, 5, 62, 63, 64, 127, 128, 200, 300, 511]
    rng = np.random.default_rng(5)
    strs = [bytes(rng.choice(synth._ALPHABET, size=n).tolist()) for n in lens]
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in strs])]).astype(np.int64)
    data = np.frombuffer(b"".join(strs), dtype=np.uint8)
    got = eng.encode_bytes(data, offsets, 512, out_dtype=torch.float32)
    want = oracle_embeddings(cfg, sd, data, offsets, 512)
    max_abs, min_cos = compare_embeddings(got, want)
    rows = _hidden_report(eng, cfg, sd, data, offsets, 512, out_dir, "tiny")
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos, rows)
    norms = got.float().norm(dim=1)
    assert torch.allclose(norms, torch.ones_like(norms), atol=1e-4)


def test_truncation_and_bf16_output(rpx_lib, cuda_device, tiny):
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    data, offsets = synth.synth_premises(12, seed=3, min_len=100, max_len=400)
    # max_seq_len 128 truncates most strings to 127 bytes + EOS (HF: truncation includes the EOS)
    got = eng.encode_bytes(data, offsets, 128, out_dtype=torch.bfloat16)
    want = oracle_embeddings(cfg, sd, data, offsets, 128)
    max_abs, min_cos = compare_embeddings(got, want)
    assert max_abs <= EMB_MAX_ABS + 2e-3 and min_cos >= EMB_MIN_COS, (max_abs, min_cos)  # + bf16 output rounding


def test_encode_ids_signature_parity(rpx_lib, cuda_device, tiny):
    """`_encode(input_ids, attention_mask)` on padded int64 tensors == the packed-bytes path."""
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    data, offsets = synth.synth_premises(7, seed=9, min_len=3, max_len=90)
    texts = [s.decode() for s in synth.split_strings(data, offsets)]
    tok = ref.tokenize(ref.build_hf_tokenizer(), texts, 64)
    a = eng.encode_ids(tok.input_ids.to(cuda_device), tok.attention_mask.to(cuda_device), out_dtype=torch.float32)
    b = eng.encode_bytes(data, offsets, 64, out_dtype=torch.float32)
    assert torch.equal(a, b)
    want = ref.encode(ref.build_hf_encoder(cfg, sd), tok.input_ids, tok.attention_mask)
    max_abs, min_cos = compare_embeddings(a, want)
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos)


def test_encode_ids_rejects_non_prefix_mask(rpx_lib, cuda_device, tiny):
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    ids = torch.randint(3, 259, (2, 16), device=cuda_device)
    mask = torch.ones(2, 16, dtype=torch.int64, device=cuda_device)
    mask[1, 5] = 0  # hole
    with pytest.raises(_native.RpxError) as ei:
        eng.encode_ids(ids, mask)
    assert ei.value.code == _native.RPX_ERR_MASK
    mask = torch.ones(2, 16, dtype=torch.int64, device=cuda_device)
    mask[0, :] = 0  # empty row (the reference would divide by zero)
    with pytest.raises(_native.RpxError):
        eng.encode_ids(ids, mask)
    bad = ids.clone()
    bad[0, 0] = 999
    with pytest.raises(_native.RpxError):
        eng.encode_ids(bad, torch.ones(2, 16, dtype=torch.int64, device=cuda_device))


def test_byt5_small_cfg1(rpx_lib, cuda_device, out_dir):
    """BASELINE config 1: full ByT5-small geometry, 8 premises + 1 state, cosine top-3."""
    cfg = dict(synth.BYT5_SMALL)
    sd = synth.random_t5_state_dict(cfg, seed=synth.SEED)
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    pd, po = synth.synth_premises(8, seed=synth.SEED)
    sdt, so = synth.synth_states(1, seed=synth.SEED + 1)
    data = np.concatenate([pd, sdt])
    offsets = np.concatenate([po, po[-1] + so[1:]])
    got = eng.encode_bytes(data, offsets, 512, out_dtype=torch.float32)
    want = oracle_embeddings(cfg, sd, data, offsets, 512)
    max_abs, min_cos = compare_embeddings(got, want)
    rows = _hidden_report(eng, cfg, sd, data, offsets, 512, out_dir, "byt5small")
    (out_dir / "encoder_cfg1.json").write_text(json.dumps({"max_abs": max_abs, "min_cos": min_cos}))
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos, rows)
    sims_got = (got[8:] @ got[:8].t()).cpu()
    sims_want = want[8:] @ want[:8].t()
    assert torch.allclose(sims_got, sims_want, atol=4e-3)


def test_long_sequences_and_max_len_2048(rpx_lib, cuda_device, tiny):
    """The reference indexes with max_seq_len = 2048 (retrieval/index.py:33): sequences longer than the
    relative-bias range (|delta| >= 128 saturates), multi-tile attention, truncation at 2048 incl. EOS."""
    cfg, sd = tiny
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    lens = [2047, 2500, 1025, 700, 129]
    rng = np.random.default_rng(8)
    strs = [bytes(rng.choice(synth._ALPHABET, size=n).tolist()) for n in lens]
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in strs])]).astype(np.int64)
    data = np.frombuffer(b"".join(strs), dtype=np.uint8)
    got = eng.encode_bytes(data, offsets, 2048, out_dtype=torch.float32)
    want = oracle_embeddings(cfg, sd, data, offsets, 2048, batch_size=2)
    max_abs, min_cos = compare_embeddings(got, want)
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos)


def test_byt5_small_full_depth_at_max_seq_len_2048(rpx_lib, cuda_device, out_dir):
    """The production indexing shape at FULL depth: 12-layer ByT5-small, max_seq_len = 2048
    (retrieval/index.py:33, prover/evaluate.py:106), lengths around every tiling boundary of the long
    path — 1023 / 1024 tokens (8 query tiles, 16 key steps), 2047 / 2048 tokens, and a 2500-byte
    string truncated to 2047 bytes + EOS — against the HF fp32 oracle (tolerance of SURVEY 8c)."""
    cfg = dict(synth.BYT5_SMALL)
    sd = synth.random_t5_state_dict(cfg, seed=synth.SEED)
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    lens = [1022, 1023, 2046, 2500, 2047]          # bytes; + EOS -> 1023, 1024, 2047, 2048 (truncated), 2048 tokens
    rng = np.random.default_rng(21)
    strs = [bytes(rng.choice(synth._ALPHABET, size=n).tolist()) for n in lens]
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in strs])]).astype(np.int64)
    data = np.frombuffer(b"".join(strs), dtype=np.uint8)
    got = eng.encode_bytes(data, offsets, 2048, out_dtype=torch.float32)
    want = oracle_embeddings(cfg, sd, data, offsets, 2048, batch_size=1)
    max_abs, min_cos = compare_embeddings(got, want)
    (out_dir / "encoder_full_depth_2048.json").write_text(json.dumps({"max_abs": max_abs, "min_cos": min_cos, "byte_lens": lens}))
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos)
    # the truncated string equals its first 2047 bytes encoded on their own (truncation includes the EOS)
    cut = eng.encode_bytes(np.frombuffer(strs[3][:2047], dtype=np.uint8), np.array([0, 2047], dtype=np.int64), 2048,
                           out_dtype=torch.float32)
    assert torch.equal(cut[0], got[3])


@pytest.mark.parametrize("n_tok", [1, 17, 64, 65, 128, 129, 256, 257, 300, 384, 385, 512, 513, 700, 768, 1024, 1025])
def test_latency_path_matches_oracle_and_throughput_path(rpx_lib, cuda_device, n_tok):
    """`rpx_encoder_set_latency_tokens`: the narrow-tile kernels used for one proof state per call
    (retrieval/model.py:348-357) against the HF fp32 oracle and against the throughput tiles."""
    cfg = dict(synth.BYT5_SMALL)
    cfg["num_layers"] = 3
    sd = synth.random_t5_state_dict(cfg, seed=5)
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    data, offsets = synth.synth_states(2 if n_tok < 300 else 1, seed=n_tok, min_len=max(n_tok - 1, 3), max_len=max(n_tok - 1, 3))
    a = eng.encode_bytes(data, offsets, 2048, out_dtype=torch.float32)
    eng.set_latency_tokens(4096)
    b = eng.encode_bytes(data, offsets, 2048, out_dtype=torch.float32)
    eng.set_latency_tokens(0)
    c = eng.encode_bytes(data, offsets, 2048, out_dtype=torch.float32)
    assert torch.equal(a, c)
    # same arithmetic, other tile shapes: the RMSNorm statistics are summed in another grouping, which flips the
    # odd bf16 rounding of an intermediate — a few 1e-4 on unit-norm embeddings, an order below the oracle tolerance
    assert (a - b).abs().max().item() <= 5e-4 and torch.nn.functional.cosine_similarity(a, b, dim=1).min().item() >= 0.99999
    want = oracle_embeddings(cfg, sd, data, offsets, 2048)
    max_abs, min_cos = compare_embeddings(b, want)
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos)


def test_latency_path_batch_equals_single(rpx_lib, cuda_device):
    """A state's embedding on the latency path does not depend on what it is batched with, although the tile
    shapes do (32- vs 64-wide residual tiles at 256 tokens, 32 vs 64 hidden units per FFN-up tile at 128): the
    RMSNorm partial sums, the attention and the pooling are grouped per sequence, not per call."""
    cfg = dict(synth.BYT5_SMALL)
    cfg["num_layers"] = 3
    eng = T5EncoderEngine(cfg, synth.random_t5_state_dict(cfg, seed=6), cuda_device)
    eng.set_latency_tokens(4096)
    data, offsets = synth.synth_states(7, seed=31, min_len=5, max_len=250)
    together = eng.encode_bytes(data, offsets, 2048, out_dtype=torch.float32)      # ~900 tokens in one call
    strs = synth.split_strings(data, offsets)
    for i, sbytes in enumerate(strs):
        alone = eng.encode_bytes(np.frombuffer(sbytes, dtype=np.uint8), np.array([0, len(sbytes)], dtype=np.int64), 2048,
                                 out_dtype=torch.float32)
        assert torch.equal(alone[0], together[i]), (i, len(sbytes))
    # sequences of 40, 300 and 620 tokens (1, 5 and 10 of the kernel's 64-key steps) in the same call
    parts = [synth.split_strings(*synth.synth_states(1, seed=40 + i, min_len=n, max_len=n))[0] for i, n in enumerate((40, 300, 620))]
    offs = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    mixed = eng.encode_bytes(np.frombuffer(b"".join(parts), dtype=np.uint8), offs, 2048, out_dtype=torch.float32)
    for i, sbytes in enumerate(parts):
        alone = eng.encode_bytes(np.frombuffer(sbytes, dtype=np.uint8), np.array([0, len(sbytes)], dtype=np.int64), 2048,
                                 out_dtype=torch.float32)
        assert torch.equal(alone[0], mixed[i]), (i, len(sbytes))
    pair = eng.encode_bytes(*synth.synth_states(2, seed=32, min_len=100, max_len=120), 2048, out_dtype=torch.float32)
    d2, o2 = synth.synth_states(2, seed=32, min_len=100, max_len=120)
    for i, sbytes in enumerate(synth.split_strings(d2, o2)):
        alone = eng.encode_bytes(np.frombuffer(sbytes, dtype=np.uint8), np.array([0, len(sbytes)], dtype=np.int64), 2048,
                                 out_dtype=torch.float32)
        assert torch.equal(alone[0], pair[i])


def test_many_short_sequences_and_chunking(rpx_lib, cuda_device, tiny):
    """Hundreds of sequences split over several engine calls (token-budget chunking) == one call."""
    cfg, sd = tiny
    data, offsets = synth.synth_premises(700, seed=12, min_len=1, max_len=40)
    big = T5EncoderEngine(cfg, sd, cuda_device)
    small = T5EncoderEngine(cfg, sd, cuda_device, max_tokens_per_call=1000)
    a = big.encode_bytes(data, offsets, 64, out_dtype=torch.float32)
    b = small.encode_bytes(data, offsets, 64, out_dtype=torch.float32)
    assert torch.equal(a, b)
    want = oracle_embeddings(cfg, sd, data[: offsets[40]], offsets[:41], 64, batch_size=40)
    max_abs, min_cos = compare_embeddings(a[:40], want)
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos)


def test_byt5_small_full_size_batch_invariance(rpx_lib, cuda_device):
    """BASELINE config 2 geometry at a size where every pipelined path is busy: 1500 premises = one
    full 262,144-token engine call (many tiles per persistent CTA: the operand ring and the accumulator
    hand-off run across many tile boundaries) plus a ragged tail call.  An
    embedding must not depend on what else is in the batch — bit for bit: every output row sums its
    products in an order fixed by the kernel shapes, not by the tile, the pair or the call it lands
    in — and the sampled rows must still match the fp32 oracle."""
    cfg = dict(synth.BYT5_SMALL)
    sd = synth.random_t5_state_dict(cfg, seed=synth.SEED)
    eng = T5EncoderEngine(cfg, sd, cuda_device)
    n = 1500
    data, offsets = synth.synth_premises(n, seed=synth.SEED + 5)
    tokens = np.minimum(np.diff(offsets) + 1, 512)
    assert tokens.sum() > eng.max_tokens_per_call, "the batch must span more than one engine call"
    big = eng.encode_bytes(data, offsets, 512, out_dtype=torch.float32)
    assert torch.isfinite(big).all()
    norms = big.norm(dim=1)
    assert torch.allclose(norms, torch.ones_like(norms), atol=2e-3)
    # rows around the call boundary, the first and last rows, and a stride through the middle
    cut = int(np.searchsorted(np.cumsum(tokens), eng.max_tokens_per_call, side="right"))
    picks = sorted({0, 1, 2, cut - 2, cut - 1, cut, cut + 1, n - 2, n - 1, *range(97, n, 211)})
    blobs = [bytes(data[offsets[i]:offsets[i + 1]]) for i in picks]
    sub_off = np.concatenate([[0], np.cumsum([len(b) for b in blobs])]).astype(np.int64)
    sub_data = np.frombuffer(b"".join(blobs), dtype=np.uint8)
    alone = eng.encode_bytes(sub_data, sub_off, 512, out_dtype=torch.float32)
    assert torch.equal(alone, big[torch.tensor(picks, device=big.device)])
    want = oracle_embeddings(cfg, sd, sub_data[: sub_off[6]], sub_off[:7], 512, batch_size=6)
    max_abs, min_cos = compare_embeddings(alone[:6], want)
    assert max_abs <= EMB_MAX_ABS and min_cos >= EMB_MIN_COS, (max_abs, min_cos)
