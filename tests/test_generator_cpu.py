"""CPU checks of the tactic generator's forward: the unidirectional bucket the decoder's bias table uses, the
decoder-length and shift-right rules, the config rules of `T5GeneratorEngine`, and the float64 restatement
(tests/seq2seq_ref.py) against HF `T5ForConditionalGeneration` in fp32."""
import types

import pytest
import torch

from reprover_b200 import generator, synth
from tests import seq2seq_ref as S


@pytest.mark.parametrize("num_buckets,max_distance", [(32, 128), (16, 32), (64, 512)])
def test_unidirectional_bucket_matches_hf(rpx_lib, num_buckets, max_distance):
    from transformers.models.t5.modeling_t5 import T5Attention

    delta = torch.arange(-3000, 3001, dtype=torch.long)
    want = T5Attention._relative_position_bucket(delta, bidirectional=False, num_buckets=num_buckets,
                                                 max_distance=max_distance)
    got = [rpx_lib.rpx_t5_relative_bucket_unidirectional(int(d), num_buckets, max_distance) for d in delta]
    assert got == want.tolist()
    assert torch.equal(S.relative_bucket(delta, False, num_buckets, max_distance), want)
    # the kernel's LUT clamps key - query at -max_distance: every delta below it is in the last bucket
    assert set(want[delta <= -max_distance].tolist()) == {num_buckets - 1}


def test_bidirectional_restatement_matches_hf():
    from transformers.models.t5.modeling_t5 import T5Attention

    delta = torch.arange(-3000, 3001, dtype=torch.long)
    want = T5Attention._relative_position_bucket(delta, bidirectional=True, num_buckets=32, max_distance=128)
    assert torch.equal(S.relative_bucket(delta, True, 32, 128), want)


def _hf_shift_right(labels, start=0, pad=0):
    from transformers.models.t5.modeling_t5 import T5PreTrainedModel

    fake = types.SimpleNamespace(config=types.SimpleNamespace(decoder_start_token_id=start, pad_token_id=pad))
    return T5PreTrainedModel._shift_right(fake, labels)


def test_shift_right_and_decoder_lengths_edge_cases():
    I = S.IGNORE
    labels = torch.tensor([
        [5, 6, I, 8, 1, I, I],   # -100 inside the length: fed as pad, not counted
        [I, I, I, I, I, I, I],   # nothing counts: length 0
        [9, I, I, I, I, I, I],   # length 1
        [3, 4, 5, 6, 7, 8, 1],   # full row
        [I, I, I, I, I, I, 2],   # only the last position counts: full length
    ])
    assert S.decoder_lengths(labels).tolist() == [5, 0, 1, 7, 7]
    assert torch.equal(S.shift_right(labels), _hf_shift_right(labels))
    assert S.shift_right(labels)[0].tolist() == [0, 5, 6, 0, 8, 1, 0]


def test_config_rules():
    cfg = dict(synth.tiny_config(2), num_decoder_layers=3)
    g = generator.generator_config(cfg)                          # ByT5: untied, unscaled
    assert (g.num_decoder_layers, g.head_key, g.scale_decoder_outputs, g.start_token_id) == (3, "lm_head.weight", False, 0)
    tied = dict(cfg)
    tied.pop("tie_word_embeddings")
    assert generator.generator_config(tied)[1:3] == ("shared.weight", True)
    assert generator.generator_config(dict(cfg, tie_word_embeddings=True))[1:3] == ("shared.weight", True)
    assert "lm_head.weight" not in generator.required_generator_keys(tied)
    with pytest.raises(NotImplementedError, match="decoder_start_token_id"):
        generator.generator_config(dict(cfg, decoder_start_token_id=1))
    assert generator.generator_config(dict(cfg, decoder_start_token_id=0)).start_token_id == 0
    with pytest.raises(NotImplementedError, match="gated-gelu"):
        generator.generator_config(dict(cfg, feed_forward_proj="relu"))
    sd = synth.random_t5_seq2seq_state_dict(dict(cfg, d_model=64, d_ff=128, num_heads=1, num_layers=1,
                                                 num_decoder_layers=1))
    generator.check_generator_checkpoint(dict(cfg, num_decoder_layers=1), sd)
    del sd["decoder.block.0.layer.1.EncDecAttention.k.weight"], sd["lm_head.weight"]
    with pytest.raises(KeyError) as ei:
        generator.check_generator_checkpoint(dict(cfg, num_decoder_layers=1), sd)
    assert "decoder.block.0.layer.1.EncDecAttention.k.weight" in str(ei.value) and "lm_head.weight" in str(ei.value)


def test_synthetic_checkpoint_keeps_encoder_and_separates_tables():
    cfg = dict(synth.tiny_config(1), d_model=64, d_ff=128, num_heads=1, num_decoder_layers=2)
    enc = synth.random_t5_state_dict(cfg, seed=5)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=5)
    for k, v in enc.items():
        assert torch.equal(sd[k], v), k
    assert not torch.equal(sd["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"],
                           sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"])
    assert not torch.equal(sd["lm_head.weight"], sd["shared.weight"])


# Tolerance of the float64 restatement against HF fp32 ("highest"): fp32 rounding through 2 + 2 layers of width
# 128 and a softmax over 384 logits of size ~1 leaves errors of a few 1e-6; 2e-5 on logits and 1e-5 on the loss.
LOGIT_TOL = 2e-5
LOSS_TOL = 1e-5


@pytest.mark.parametrize("tied", [False, True])
def test_restatement_matches_hf(tmp_path, tied):
    torch.set_float32_matmul_precision("highest")
    cfg = dict(synth.tiny_config(2), d_model=128, d_ff=256, num_heads=2, num_decoder_layers=2,
               relative_attention_max_distance=16, relative_attention_num_buckets=8, decoder_start_token_id=0)
    if tied:
        cfg.pop("tie_word_embeddings")
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=11)
    synth.save_hf_checkpoint(str(tmp_path), cfg, sd)
    model = S.hf_model_from_dir(str(tmp_path))
    if not tied:
        assert S.untied_head_is_distinct(model, sd), "HF oracle runs with a tied head"
    I = S.IGNORE
    rows = [[7, 8, 9, I, 11, 1], [I] * 6, [40], [50 + j for j in range(30)], [I, I, 5, 6]]
    ids, mask, labels = S.random_batch(cfg, [20, 7, 1, 33, 12], rows, seed=3)
    with torch.no_grad():
        out = model(input_ids=ids, attention_mask=mask, labels=labels)
    ref = S.forward(cfg, sd, ids, mask, labels)
    lens = S.decoder_lengths(labels)
    for b in range(len(rows)):
        n = int(lens[b])
        err = (out.logits[b, :n].double() - ref["logits"][b, :n]).abs().max() if n else torch.tensor(0.0)
        assert float(err) < LOGIT_TOL, (b, float(err))
    assert abs(float(out.loss) - float(ref["loss"])) < LOSS_TOL
    # per-row log-likelihoods from HF's logits
    lp = torch.log_softmax(out.logits.double(), -1).gather(2, labels.clamp_min(0)[..., None])[..., 0]
    hf_seq = torch.where(labels != I, lp, torch.zeros_like(lp)).sum(1)
    assert torch.allclose(hf_seq, ref["sequence_log_probs"], atol=LOSS_TOL * 30, rtol=0)


def test_decoder_packed_bytes_rejects_unsupported_configs(rpx_lib):
    import ctypes as C

    from reprover_b200 import _native

    def cfg(**kw):
        base = dict(vocab_size=384, d_model=1472, d_kv=64, d_ff=3584, num_layers=4, num_heads=6, rel_buckets=32,
                    rel_max_distance=128, ln_eps=1e-6)
        base.update(kw)
        return _native.T5Config(**base)

    n = rpx_lib.rpx_t5_decoder_packed_bytes(C.byref(cfg()))
    # 4 decoder blocks (self qkv + o, cross q + o, FFN) + the cross K/V of all 4 + head, in bf16
    per_layer = 3 * 384 * 1472 + 1472 * 384 + 384 * 1472 + 1472 * 384 + 3 * 3584 * 1472
    assert 2 * (4 * per_layer + 4 * 2 * 384 * 1472 + 384 * 1472) <= n <= 2 * (4 * per_layer + 4 * 2 * 384 * 1472) + 6_000_000
    assert rpx_lib.rpx_t5_decoder_packed_bytes(C.byref(cfg(d_kv=32))) == 0 and "d_kv" in _native.last_error()
    assert rpx_lib.rpx_t5_decoder_packed_bytes(C.byref(cfg(vocab_size=390))) == 0
    assert rpx_lib.rpx_t5_decoder_packed_bytes(C.byref(cfg(rel_max_distance=16))) == 0  # must exceed buckets / 2
    assert rpx_lib.rpx_seq2seq_workspace_bytes(None, None, 1, 1, 1) == 0
