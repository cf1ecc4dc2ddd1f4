"""The generator's validation path without a GPU: reading generator checkpoints (Lightning stand-ins, the retriever
keys a module trained with `ret_ckpt_path` carries, config from shapes and the tied-head rule, a disagreeing cached
config, missing keys, ZeRO without deepspeed), the converter's round trip through HF, `generator_cli`'s settings, and
the epoch-end metrics against a hand-computed example."""
import json
import sys
import types

import pytest
import torch

from reprover_b200 import synth
from reprover_b200.checkpoint import (ZERO_CONVERSION, StandIn, heads_tied, load_generator_checkpoint,
                                      read_lightning_checkpoint)
from reprover_b200.engine import load_hf_checkpoint

# a small T5 v1.1 geometry: nothing here builds an engine
CFG = dict(vocab_size=384, d_model=32, d_kv=8, d_ff=48, num_layers=2, num_decoder_layers=1, num_heads=4,
           relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
           feed_forward_proj="gated-gelu", tie_word_embeddings=False, pad_token_id=0, eos_token_id=1,
           decoder_start_token_id=0)
HPARAMS = {"model_name": "not-cached/byt5-nowhere", "lr": 5e-4, "warmup_steps": 2000, "num_beams": 2,
           "length_penalty": 0.0, "eval_num_retrieved": 100, "eval_num_workers": 1, "eval_num_gpus": 1,
           "eval_num_theorems": 0, "max_inp_seq_len": 2300, "max_oup_seq_len": 512, "ret_ckpt_path": "r.ckpt"}


@pytest.fixture(scope="module")
def weights():
    return synth.random_t5_seq2seq_state_dict(CFG, seed=61)


def _module_state(sd):
    state = {f"generator.{k}": v for k, v in sd.items()}
    enc = synth.random_t5_state_dict(dict(CFG, num_layers=1), seed=62)
    state.update({f"retriever.encoder.{k}": v for k, v in enc.items()})
    return state


@pytest.fixture
def attribute_dict(monkeypatch):
    """A `pytorch_lightning.utilities.parsing.AttributeDict` to pickle; the module is gone before loading."""
    names = ["pytorch_lightning", "pytorch_lightning.utilities", "pytorch_lightning.utilities.parsing"]
    mods = {n: types.ModuleType(n) for n in names}

    class AttributeDict(dict):
        pass

    AttributeDict.__module__ = "pytorch_lightning.utilities.parsing"
    AttributeDict.__qualname__ = "AttributeDict"
    mods[names[-1]].AttributeDict = AttributeDict
    for n, m in mods.items():
        monkeypatch.setitem(sys.modules, n, m)
    return AttributeDict


def _write_ckpt(path, sd, hparams):
    torch.save({"epoch": 1, "global_step": 10, "state_dict": _module_state(sd), "hyper_parameters": hparams}, path)


def test_lightning_checkpoint_keys_hparams_and_config(tmp_path, weights, attribute_dict):
    path = tmp_path / "epoch=1.ckpt"
    _write_ckpt(path, weights, attribute_dict(HPARAMS))
    for n in ("pytorch_lightning.utilities.parsing", "pytorch_lightning.utilities", "pytorch_lightning"):
        del sys.modules[n]
    assert isinstance(read_lightning_checkpoint(str(path))["hyper_parameters"], StandIn)
    cfg, sd, hp = load_generator_checkpoint(str(path))
    assert hp == HPARAMS
    assert not any(k.startswith("retriever") for k in sd)
    for k, v in weights.items():
        assert torch.equal(sd[k], v), k
    for key in ("vocab_size", "d_model", "d_kv", "d_ff", "num_layers", "num_decoder_layers", "num_heads",
                "relative_attention_num_buckets", "relative_attention_max_distance", "layer_norm_epsilon",
                "feed_forward_proj", "tie_word_embeddings", "pad_token_id", "eos_token_id", "decoder_start_token_id"):
        assert cfg[key] == CFG[key], key


def test_tied_head_rule(weights):
    sd = dict(weights)
    assert heads_tied(sd) is False                        # lm_head present and different
    sd["lm_head.weight"] = sd["shared.weight"].clone()
    assert heads_tied(sd) is True                         # present and equal
    del sd["lm_head.weight"]
    assert heads_tied(sd) is True                         # absent


def test_tied_checkpoint_without_lm_head(tmp_path, weights):
    sd = {k: v for k, v in weights.items() if k != "lm_head.weight"}
    path = tmp_path / "tied.ckpt"
    _write_ckpt(path, sd, HPARAMS)
    cfg, got, _ = load_generator_checkpoint(str(path))
    assert cfg["tie_word_embeddings"] is True and "lm_head.weight" not in got


def test_cached_or_given_config_that_disagrees(tmp_path, weights):
    hf = tmp_path / "model"
    synth.save_hf_checkpoint(str(hf), CFG, weights)
    path = tmp_path / "last.ckpt"
    _write_ckpt(path, weights, dict(HPARAMS, model_name=str(hf)))
    cfg, _, _ = load_generator_checkpoint(str(path))
    assert cfg["architectures"] == ["T5ForConditionalGeneration"] and cfg["d_model"] == 32   # the cached one
    (hf / "config.json").write_text(json.dumps(dict(CFG, num_decoder_layers=3)))
    with pytest.raises(ValueError, match="num_decoder_layers"):
        load_generator_checkpoint(str(path))
    with pytest.raises(ValueError, match="tie_word_embeddings"):
        load_generator_checkpoint(str(path), config=dict(CFG, tie_word_embeddings=True))
    with pytest.raises(ValueError, match="d_ff"):
        load_generator_checkpoint(str(path), config=dict(CFG, d_ff=64))


def test_missing_keys(tmp_path, weights):
    sd = {k: v for k, v in weights.items() if k != "decoder.block.0.layer.1.EncDecAttention.k.weight"}
    path = tmp_path / "broken.ckpt"
    _write_ckpt(path, sd, HPARAMS)
    with pytest.raises(KeyError, match="EncDecAttention.k.weight"):
        load_generator_checkpoint(str(path))
    torch.save({"state_dict": {f"encoder.{k}": v for k, v in weights.items()}}, path)   # a retriever's
    with pytest.raises(KeyError, match="'generator.'"):
        load_generator_checkpoint(str(path))


def test_zero_directory_without_deepspeed(tmp_path, monkeypatch):
    d = tmp_path / "epoch=0-step=10.ckpt"
    d.mkdir()
    (d / "zero_to_fp32.py").write_text("")
    monkeypatch.setitem(sys.modules, "deepspeed", None)
    with pytest.raises(RuntimeError, match="deepspeed") as err:
        load_generator_checkpoint(str(d))
    assert ZERO_CONVERSION in str(err.value) and "generator.ckpt" in str(err.value)


def test_converter_round_trip(tmp_path, weights):
    from transformers import ByT5Tokenizer, T5EncoderModel, T5ForConditionalGeneration

    from reprover_b200 import convert_cli

    path = tmp_path / "generator.ckpt"
    _write_ckpt(path, weights, HPARAMS)
    dst = tmp_path / "hf-generator"
    convert_cli.main(["generator", "--src", str(path), "--dst", str(dst)])
    model = T5ForConditionalGeneration.from_pretrained(str(dst))
    got = model.state_dict()
    for k, v in weights.items():
        assert torch.equal(got[k], v), k
    cfg, sd = load_hf_checkpoint(str(dst))
    assert cfg["tie_word_embeddings"] is False
    for k, v in sd.items():
        assert torch.equal(v, weights[k]), k
    assert set(sd) == set(weights) - {"encoder.embed_tokens.weight", "decoder.embed_tokens.weight"}
    assert ByT5Tokenizer.from_pretrained(str(dst))("ab").input_ids == [100, 101, 1]

    ret = tmp_path / "retriever.ckpt"
    enc = synth.random_t5_state_dict(dict(CFG, num_layers=1), seed=63)
    torch.save({"state_dict": {f"encoder.{k}": v for k, v in enc.items()}, "hyper_parameters": {}}, ret)
    convert_cli.main(["retriever", "--src", str(ret), "--dst", str(tmp_path / "hf-retriever")])
    got = T5EncoderModel.from_pretrained(str(tmp_path / "hf-retriever")).state_dict()
    for k, v in enc.items():
        assert torch.equal(got[k], v), k


def test_cli_settings_precedence_and_ignored_keys(tmp_path):
    from reprover_b200.generator_cli import parse_args, resolve_settings

    cfg = tmp_path / "cli.yaml"
    cfg.write_text("seed_everything: 3407\ntrainer:\n  devices: 1\nmodel:\n  model_name: google/byt5-small\n"
                   "  num_beams: 4\n  eval_num_theorems: 250\n  ret_ckpt_path: null\n"
                   "data:\n  data_path: d/random/\n  preds_path: null\n  eval_batch_size: 64\n  max_inp_seq_len: 2300\n"
                   "  p_drop: 0.5\n")
    args, settings, ignored = parse_args(["validate", "--config", str(cfg), "--ckpt_path", "g.ckpt",
                                          "--data.preds_path", "p.pickle", "--data.eval_batch_size=8"])
    assert args.ckpt_path == "g.ckpt" and args.hf_ckpt is None
    assert ignored == ["data.p_drop", "model.eval_num_theorems", "model.model_name", "model.ret_ckpt_path",
                       "seed_everything", "trainer.devices"]
    s = resolve_settings(settings, {"num_beams": 1, "max_inp_seq_len": 999, "max_oup_seq_len": 77})
    assert s == {"data.data_path": "d/random/", "data.eval_batch_size": 8, "model.num_beams": 4,
                 "data.max_inp_seq_len": 2300, "data.max_oup_seq_len": 77, "data.preds_path": "p.pickle"}
    with pytest.raises(SystemExit):
        resolve_settings(settings, {})                         # max_oup_seq_len set nowhere
    with pytest.raises(SystemExit):
        parse_args(["validate", "--config", str(cfg)])         # no checkpoint
    with pytest.raises(SystemExit):
        parse_args(["predict", "--ckpt_path", "g.ckpt"])       # no such subcommand


def test_metrics_by_hand_with_a_partial_last_batch():
    from reprover_b200.generator_eval import ValidationMetrics

    m = ValidationMetrics(3)
    # batch 1, 3 examples, loss 2.0: hits at rank 1, rank 3 (after removing marks), none
    m.update(2.0, [["a", "b", "c"], ["x", "y", "<a>z</a>"], ["p", "q", "r"]], ["<a>a</a>", "z", "s"])
    # batch 2 (the partial last one), 1 example, loss 6.0: hit at rank 2
    m.update(6.0, [["u", "v", "w"]], ["v"])
    got = m.compute()
    assert got == {"loss_val": (2.0 * 3 + 6.0 * 1) / 4, "top1_acc_val": 1 / 4, "top2_acc_val": 2 / 4,
                   "top3_acc_val": 3 / 4}


def test_collate_tokenizes_pads_and_masks_labels():
    from reprover_b200.generator_eval import collate

    ex = [{"state": "⊢ ab", "tactic": "simp", "file_path": "F.lean"}, {"state": "x", "tactic": "rfl<pad>",
                                                                      "file_path": "G.lean"}]
    b = collate(ex, 4, 16)
    assert b["state_ids"].tolist() == [[229, 141, 165, 1], [123, 1, 0, 0]]      # 3 bytes then EOS: truncated
    assert b["state_mask"].tolist() == [[1, 1, 1, 1], [1, 1, 0, 0]]
    # the tactic's own <pad> literal (id 0) becomes -100 too, as `tactic_ids[tactic_ids == pad] = -100` does
    assert b["tactic_ids"].tolist() == [[118, 108, 112, 115, 1], [117, 105, 111, -100, 1]]
    assert b["file_path"] == ["F.lean", "G.lean"] and b["tactic"] == ["simp", "rfl<pad>"]
