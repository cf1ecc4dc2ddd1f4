"""CPU checks of generation: the search restatement (tests/beam_ref.py) against HF `generate` on HF's own tiny T5,
the decode-attention reference (tests/decode_attention_ref.py) against an fp32 model of the kernel and injected
defects, and the generation-settings rules of `T5GeneratorEngine.generate`."""
import pytest
import torch

from reprover_b200.generator import GENERATION_DEFAULTS, generation_settings
from tests import beam_ref
from tests import decode_attention_ref as DA

EOS, PAD = 1, 0


@pytest.fixture(scope="module")
def tiny_t5():
    """HF's T5 at toy size, fp32, with the EOS head row pointed along the mean final hidden state (twice the mean row
    norm) so that hypotheses finish at many lengths (a random head almost never emits EOS)."""
    from transformers import T5Config, T5ForConditionalGeneration

    torch.manual_seed(0)
    cfg = T5Config(vocab_size=48, d_model=32, d_kv=8, d_ff=64, num_layers=2, num_decoder_layers=2, num_heads=4,
                   feed_forward_proj="gated-gelu", tie_word_embeddings=False, decoder_start_token_id=0,
                   pad_token_id=PAD, eos_token_id=EOS, relative_attention_num_buckets=8,
                   relative_attention_max_distance=20)
    m = T5ForConditionalGeneration(cfg).eval()
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(2, 48, (6, 12), generator=g)
    dec = torch.randint(2, 48, (6, 10), generator=g)
    with torch.no_grad():
        h = m(input_ids=ids, decoder_input_ids=dec, output_hidden_states=True).decoder_hidden_states[-1]
        h = m.decoder.final_layer_norm(h)
        mean = h.reshape(-1, 32).mean(0)
        row = m.lm_head.weight
        row[EOS] = mean / mean.norm() * row.norm(dim=1).mean() * 2.0
    return m


def _states(seed, lens, vocab=48):
    g = torch.Generator().manual_seed(seed)
    L = max(lens)
    ids = torch.zeros(len(lens), L, dtype=torch.int64)
    mask = torch.zeros(len(lens), L, dtype=torch.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(2, vocab, (n,), generator=g)
        ids[i, n - 1] = EOS
        mask[i, :n] = 1
    return ids, mask


def _hf_generate(model, ids, mask, nb, n_ret, max_length, lp):
    with torch.no_grad():
        return model.generate(input_ids=ids, attention_mask=mask, num_beams=nb, num_return_sequences=n_ret,
                              max_length=max_length, length_penalty=lp, do_sample=False, early_stopping=False,
                              output_scores=True, return_dict_in_generate=True)


def _replay(model, ids, mask, nb, scores):
    """The step function: HF's own recorded step scores, after checking that the prefixes asked for are the ones a
    teacher-forced pass of HF scores the same way."""
    enc_ids = ids.repeat_interleave(nb, 0)
    enc_mask = mask.repeat_interleave(nb, 0)

    def step(t, prefixes):
        with torch.no_grad():
            lg = model(input_ids=enc_ids, attention_mask=enc_mask, decoder_input_ids=prefixes).logits[:, -1].float()
        want = torch.log_softmax(lg, -1) if nb > 1 else lg
        got = scores[t]
        live = got.isfinite().all(-1)
        assert torch.allclose(got[live], want[live], atol=1e-4, rtol=1e-4), f"step {t}: prefixes differ from HF's"
        return got

    return step


CASES = [(1, 1, 0.0), (2, 1, 1.0), (2, 2, 0.0), (4, 1, -0.5), (4, 4, 1.0), (8, 8, 0.0), (8, 1, 1.0), (8, 8, -0.5)]


@pytest.mark.parametrize("nb,n_ret,lp", CASES)
def test_restatement_matches_hf_generate(tiny_t5, nb, n_ret, lp):
    ids, mask = _states(3 + nb, [7, 12, 3])
    max_length = 40
    hf = _hf_generate(tiny_t5, ids, mask, nb, n_ret, max_length, lp)
    step = _replay(tiny_t5, ids, mask, nb, hf.scores)
    if nb == 1:
        seqs = beam_ref.greedy(step, 3, max_length, EOS, PAD, 0)
        assert torch.equal(seqs, hf.sequences)
        return
    seqs, scores = beam_ref.beam_search(step, 3, nb, n_ret, max_length, lp, EOS, PAD, 0)
    assert torch.equal(seqs, hf.sequences)
    assert torch.equal(scores, hf.sequences_scores)


def test_fixture_exercises_every_ending(tiny_t5):
    """Across the beam cases: hypotheses finish at three or more lengths, one search ends by the early-stop
    heuristic and one by max_length."""
    lengths, endings = set(), set()
    for nb, n_ret, lp in CASES[1:]:
        for max_length in (40, 6):
            ids, mask = _states(3 + nb, [7, 12, 3])
            hf = _hf_generate(tiny_t5, ids, mask, nb, n_ret, max_length, lp)
            st = beam_ref.SearchStats()
            seqs, scores = beam_ref.beam_search(_replay(tiny_t5, ids, mask, nb, hf.scores), 3, nb, n_ret, max_length,
                                                lp, EOS, PAD, 0, stats=st)
            assert torch.equal(seqs, hf.sequences) and torch.equal(scores, hf.sequences_scores)
            lengths |= st.finish_lengths
            endings.add(st.ended_by)
    assert len(lengths) >= 3, lengths
    assert {"heuristic", "max_length"} <= endings, endings


def test_output_fill_value_is_hf_s(tiny_t5):
    """Past a beam hypothesis' end HF writes `pad_token_id or eos_token_id[0]`: the EOS id for T5's pad id 0."""
    ids, mask = _states(11, [7, 12, 3])
    hf = _hf_generate(tiny_t5, ids, mask, 2, 2, 40, 0.0)
    seqs = hf.sequences
    short = [r for r in range(seqs.shape[0]) if (seqs[r, 1:] == EOS).any() and int((seqs[r, 1:] == EOS).nonzero()[0]) + 2 < seqs.shape[1]]
    assert short, "no hypothesis shorter than the output"
    for r in short:
        end = int((seqs[r, 1:] == EOS).nonzero()[0]) + 1
        assert bool((seqs[r, end:] == EOS).all())


# ------------------------------------------------------------------------------------------ decode attention ref
def test_decode_attention_reference_accepts_fp32_model_and_catches_defects():
    for t, R in ((0, 3), (1, 4), (40, 6), (130, 5)):
        case = DA.random_case(t, R, H=2, ML=t + 3, max_distance=20, seed=t + R)
        model = DA.fp32_model(case)
        assert DA.check(model, case) == 0, (t, R)
        if t == 0:
            continue
        for defect in DA.DEFECTS:
            bad = DA.fp32_model(case, defect=defect)
            assert DA.check(bad, case) > 0, (defect, t, R)


# ------------------------------------------------------------------------------------------ settings
CFG = {"vocab_size": 384, "eos_token_id": 1, "pad_token_id": 0, "decoder_start_token_id": 0}


def test_settings_defaults_and_precedence():
    s = generation_settings(CFG)
    assert (s.max_length, s.num_beams, s.num_return_sequences, s.length_penalty) == (
        GENERATION_DEFAULTS["max_length"], 1, 1, 1.0)
    assert (s.eos_token_id, s.pad_token_id, s.decoder_start_token_id) == (1, 0, 0)
    assert not s.output_scores and not s.return_dict_in_generate
    s = generation_settings(CFG, {"max_length": 50, "num_beams": 4, "eos_token_id": [1]})
    assert (s.max_length, s.num_beams, s.eos_token_id) == (50, 4, 1)
    s = generation_settings(CFG, {"max_length": 50}, max_length=512, num_beams=64, num_return_sequences=64,
                            length_penalty=0.0, output_scores=True, return_dict_in_generate=True, do_sample=False,
                            early_stopping=False, temperature=0.7)
    assert (s.max_length, s.num_beams, s.num_return_sequences, s.length_penalty) == (512, 64, 64, 0.0)
    assert s.output_scores and s.return_dict_in_generate


@pytest.mark.parametrize("kw,name", [({"do_sample": True}, "do_sample"), ({"early_stopping": True}, "early_stopping"),
                                     ({"early_stopping": "never"}, "early_stopping"),
                                     ({"max_new_tokens": 5}, "max_new_tokens"), ({"min_length": 3}, "min_length"),
                                     ({"no_repeat_ngram_size": 2}, "no_repeat_ngram_size"),
                                     ({"repetition_penalty": 1.2}, "repetition_penalty"),
                                     ({"bad_words_ids": [[5]]}, "bad_words_ids"),
                                     ({"forced_bos_token_id": 2}, "forced_bos_token_id"),
                                     ({"forced_eos_token_id": 1}, "forced_eos_token_id"),
                                     ({"suppress_tokens": [3]}, "suppress_tokens"),
                                     ({"eos_token_id": [1, 2]}, "eos_token_id"), ({"foo": 1}, "foo")])
def test_settings_refusals(kw, name):
    with pytest.raises(NotImplementedError, match=name):
        generation_settings(CFG, **kw)


def test_settings_refuse_checkpoint_processors_and_bad_counts():
    with pytest.raises(NotImplementedError, match="no_repeat_ngram_size"):
        generation_settings(CFG, {"no_repeat_ngram_size": 3})
    generation_settings(CFG, {"min_length": 0, "repetition_penalty": 1.0, "transformers_version": "5.5.0"})
    with pytest.raises(ValueError, match="num_return_sequences"):
        generation_settings(CFG, num_beams=4, num_return_sequences=5)
    with pytest.raises(ValueError, match="max_length"):
        generation_settings(CFG, max_length=1)
