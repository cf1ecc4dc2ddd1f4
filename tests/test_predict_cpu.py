"""Dataset-level predict / validate without a GPU: the examples `load_examples` builds against a restatement of the
reference's `RetrievalDataset._load_data(is_train=False)`, reading the checkpoints the reference's training writes,
the CLI's argument handling, and the metrics against a restatement of `retrieval/evaluate.py::_eval`."""
import json
import logging
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from reprover_b200 import synth
from reprover_b200.checkpoint import (ZERO_CONVERSION, StandIn, encoder_state_dict, load_retriever_checkpoint,
                                      read_lightning_checkpoint)
from reprover_b200.corpus import Context, Corpus, Pos
from reprover_b200.evaluation import load_examples, recall_and_mrr


# ------------------------------------------------------------------------------------------------ load_examples
def _write_three_file_dataset(root):
    files = [
        {"path": "A.lean", "imports": [], "premises": [
            {"full_name": "A.one", "code": "theorem one : 1 = 1", "start": [1, 1], "end": [2, 10]},
            {"full_name": "A.two", "code": "theorem two : 2 = 2", "start": [4, 1], "end": [5, 10]}]},
        {"path": "B.lean", "imports": ["A.lean"], "premises": [
            {"full_name": "B.add", "code": "theorem add : a + 0 = a", "start": [1, 1], "end": [3, 5]}]},
        {"path": "C.lean", "imports": ["B.lean"], "premises": [
            {"full_name": "C.mul", "code": "theorem mul : a * 1 = a", "start": [1, 1], "end": [2, 5]},
            {"full_name": "C.sub", "code": "theorem sub : a - 0 = a", "start": [6, 1], "end": [8, 5]}]},
    ]
    (root / "corpus.jsonl").write_text("\n".join(json.dumps(f) for f in files) + "\n")
    data = root / "random"
    data.mkdir()

    def prov(path, line, name):
        return {"full_name": name, "def_path": path, "def_pos": [line, 1], "def_end_pos": [line, 2]}

    def thm(path, name, start, tactics):
        return {"url": "https://example.org/r", "commit": "c" * 40, "file_path": path, "full_name": name,
                "start": start, "end": [start[0] + 9, 1],
                "traced_tactics": [{"tactic": "t", "annotated_tactic": ["t", p], "state_before": s, "state_after": "x"}
                                   for s, p in tactics]}

    splits = {
        "train": [thm("C.lean", "C.t0", [10, 1], [("⊢ a", [prov("A.lean", 1, "A.one"), prov("C.lean", 7, "C.sub")]),
                                                   ("h : p\n⊢ q", [prov("B.lean", 2, "B.add"), prov("B.lean", 2, "B.add")])]),
                  thm("B.lean", "B.t1", [5, 1], [("⊢ b", [])])],
        "val": [thm("A.lean", "A.v0", [7, 1], [("⊢ c", [prov("A.lean", 99, "A.gone")]),   # locates nothing
                                               ("⊢ d", [prov("A.lean", 4, "A.two"), prov("A.lean", 5, "A.two")])])],
        "test": [thm("C.lean", "C.s0", [3, 1], [("⊢ e", [prov("C.lean", 1, "C.mul"), prov("A.lean", 2, "A.one")])])],
    }
    for split, thms in splits.items():
        (data / f"{split}.json").write_text(json.dumps(thms))
    return data


def _restated_load_data(data_path, corpus, split):
    """`RetrievalDataset._load_data` with is_train=False (retrieval/datamodule.py:44-90), positives as sets."""
    out = []
    with open(os.path.join(data_path, f"{split}.json")) as fh:
        theorems = json.load(fh)
    for thm in theorems:
        for i, tac in enumerate(thm["traced_tactics"]):
            positives = set()
            for prov in tac["annotated_tactic"][1]:
                p = corpus.locate_premise(prov["def_path"], Pos(*prov["def_pos"]))
                if p is not None:
                    positives.add(p)
            out.append({"url": thm["url"], "commit": thm["commit"], "file_path": thm["file_path"],
                        "full_name": thm["full_name"], "start": thm["start"], "tactic_idx": i,
                        "context": Context(thm["file_path"], thm["full_name"], Pos(*thm["start"]), tac["state_before"]),
                        "all_pos_premises": positives})
    return out


def test_load_examples_equals_the_reference_dataset(tmp_path):
    data = _write_three_file_dataset(tmp_path)
    corpus = Corpus(str(tmp_path / "corpus.jsonl"))
    got = load_examples(str(data), corpus)
    want = [ex for split in ("train", "val", "test") for ex in _restated_load_data(str(data), corpus, split)]
    assert len(got) == len(want) == 6
    for g, w in zip(got, want):
        assert list(g) == ["url", "commit", "file_path", "full_name", "start", "tactic_idx", "context", "all_pos_premises"]
        assert {k: v for k, v in g.items() if k != "all_pos_premises"} == {k: v for k, v in w.items() if k != "all_pos_premises"}
        assert set(g["all_pos_premises"]) == w["all_pos_premises"]
        assert len(g["all_pos_premises"]) == len(w["all_pos_premises"])     # a premise named twice is listed once
        assert g["context"].theorem_pos == Pos(*w["start"])
    # order: the first provenance first
    assert [p.full_name for p in got[0]["all_pos_premises"]] == ["A.one", "C.sub"]
    # the tactic without a locatable premise is still an example, with no positives
    assert got[3]["full_name"] == "A.v0" and got[3]["tactic_idx"] == 0 and got[3]["all_pos_premises"] == []
    assert [ex["full_name"] for ex in load_examples(str(data), corpus, ("val",))] == ["A.v0", "A.v0"]


# ------------------------------------------------------------------------------------------------ checkpoints
CFG = synth.tiny_config(num_layers=2)


@pytest.fixture(scope="module")
def hf_weights():
    """The state dict of a seeded, randomly initialised HF `T5EncoderModel` of ByT5 geometry (2 layers)."""
    from transformers import T5Config, T5EncoderModel

    torch.manual_seed(44)
    model = T5EncoderModel(T5Config(**{k: v for k, v in CFG.items() if k != "num_decoder_layers"}))
    return {k: v.detach().clone() for k, v in model.state_dict().items()}


def _lightning_ckpt(sd, model_name, hparams_cls=None):
    hp = {"model_name": model_name, "lr": 1e-4, "warmup_steps": 2000, "max_seq_len": 512, "num_retrieved": 37}
    if hparams_cls is not None:
        obj = hparams_cls()
        obj.update(hp)
        hp = obj
    return {"epoch": 3, "global_step": 1200, "pytorch-lightning_version": "2.1.0",
            "state_dict": {f"encoder.{k}": v for k, v in sd.items()}, "hyper_parameters": hp,
            "loops": {"fit_loop": {"epoch_progress": {"current": 3}}}, "callbacks": {}}


@pytest.fixture
def lightning_module(monkeypatch):
    """A `pytorch_lightning.utilities.parsing.AttributeDict` to pickle; the module is gone again before loading."""
    names = ["pytorch_lightning", "pytorch_lightning.utilities", "pytorch_lightning.utilities.parsing"]
    mods = {n: types.ModuleType(n) for n in names}

    class AttributeDict(dict):
        pass

    AttributeDict.__module__ = "pytorch_lightning.utilities.parsing"
    AttributeDict.__qualname__ = "AttributeDict"
    mods["pytorch_lightning.utilities.parsing"].AttributeDict = AttributeDict
    for n, m in mods.items():
        monkeypatch.setitem(sys.modules, n, m)
    return AttributeDict, names


def _same_weights(got, want):
    assert set(got) == set(want)
    for k, v in want.items():
        assert torch.equal(got[k], v), k


def test_lightning_checkpoint_with_resolvable_model_name(tmp_path, hf_weights):
    hf_dir = tmp_path / "hf"
    synth.save_hf_checkpoint(str(hf_dir), CFG, hf_weights)
    path = tmp_path / "last.ckpt"
    torch.save(_lightning_ckpt(hf_weights, str(hf_dir)), path)
    cfg, sd, hp = load_retriever_checkpoint(str(path))
    _same_weights(sd, hf_weights)
    assert cfg["num_layers"] == 2 and cfg["d_model"] == 1472 and cfg["architectures"] == ["T5EncoderModel"]  # cached
    assert hp["max_seq_len"] == 512 and hp["num_retrieved"] == 37


def test_lightning_checkpoint_with_pickled_lightning_class(tmp_path, hf_weights, lightning_module, monkeypatch):
    attr_dict, names = lightning_module
    path = tmp_path / "epoch=3.ckpt"
    torch.save(_lightning_ckpt(hf_weights, "not-cached/byt5-nowhere", attr_dict), path)
    for n in names:
        monkeypatch.delitem(sys.modules, n)
    raw = read_lightning_checkpoint(str(path))
    assert isinstance(raw["hyper_parameters"], StandIn)
    assert raw["hyper_parameters"]._pickled_class == "pytorch_lightning.utilities.parsing.AttributeDict"
    cfg, sd, hp = load_retriever_checkpoint(str(path))
    _same_weights(sd, hf_weights)
    assert hp["num_retrieved"] == 37 and hp["model_name"] == "not-cached/byt5-nowhere"
    # the model name resolves nowhere: the config comes from the shapes, with ByT5's epsilon and max distance
    for key in ("vocab_size", "d_model", "d_kv", "d_ff", "num_layers", "num_heads", "relative_attention_num_buckets",
                "relative_attention_max_distance", "layer_norm_epsilon", "feed_forward_proj"):
        assert cfg[key] == CFG[key], key


def test_config_override_and_disagreement(tmp_path, hf_weights):
    path = tmp_path / "x.ckpt"
    torch.save(_lightning_ckpt(hf_weights, "not-cached/byt5-nowhere"), path)
    cfg, _, _ = load_retriever_checkpoint(str(path), config=dict(CFG, layer_norm_epsilon=1e-5))
    assert cfg["layer_norm_epsilon"] == 1e-5
    with pytest.raises(ValueError, match="num_heads"):
        load_retriever_checkpoint(str(path), config=dict(CFG, num_heads=12, d_kv=32))
    wrong = tmp_path / "hf_wrong"
    synth.save_hf_checkpoint(str(wrong), dict(CFG, d_ff=1024), synth.random_t5_state_dict(dict(CFG, d_ff=1024), seed=1))
    torch.save(_lightning_ckpt(hf_weights, str(wrong)), path)
    with pytest.raises(ValueError, match="d_ff"):
        load_retriever_checkpoint(str(path))


def test_missing_and_malformed_encoder_keys(tmp_path, hf_weights):
    ckpt = _lightning_ckpt(hf_weights, "x")
    del ckpt["state_dict"]["encoder.encoder.final_layer_norm.weight"]
    torch.save(ckpt, tmp_path / "a.ckpt")
    with pytest.raises(KeyError, match=r"encoder\.encoder\.final_layer_norm\.weight") as err:
        load_retriever_checkpoint(str(tmp_path / "a.ckpt"))
    assert "encoder.encoder.block.0.layer.0.SelfAttention.q.weight" in str(err.value)   # the keys that are there
    # the HF weights without the LightningModule's `encoder.` prefix
    torch.save({"state_dict": dict(hf_weights), "hyper_parameters": {}}, tmp_path / "b.ckpt")
    with pytest.raises(KeyError, match="shared.weight"):
        load_retriever_checkpoint(str(tmp_path / "b.ckpt"))
    torch.save({"model": 1}, tmp_path / "c.ckpt")
    with pytest.raises(KeyError, match="state_dict"):
        load_retriever_checkpoint(str(tmp_path / "c.ckpt"))
    with pytest.raises(KeyError):
        encoder_state_dict({"encoder.shared.weight": torch.zeros(3, 4)})


def test_unknown_pickled_classes_are_refused(tmp_path, hf_weights):
    ckpt = _lightning_ckpt(hf_weights, "x")
    ckpt["callbacks"] = {"logger": logging.getLogger("some.logger")}
    torch.save(ckpt, tmp_path / "evil.ckpt")
    with pytest.raises(Exception, match="logging"):
        read_lightning_checkpoint(str(tmp_path / "evil.ckpt"))


def test_zero_directory_without_deepspeed(tmp_path):
    try:
        import deepspeed  # noqa: F401
        pytest.skip("deepspeed is importable here: the directory would be converted")
    except ImportError:
        pass
    d = tmp_path / "epoch=0-step=1.ckpt"
    (d / "checkpoint").mkdir(parents=True)
    (d / "zero_to_fp32.py").write_text("# written by DeepSpeed\n")
    with pytest.raises(RuntimeError) as err:
        load_retriever_checkpoint(str(d))
    assert ZERO_CONVERSION in str(err.value) and "DeepSpeed ZeRO" in str(err.value)
    with pytest.raises(FileNotFoundError):
        load_retriever_checkpoint(str(tmp_path / "absent.ckpt"))


# ------------------------------------------------------------------------------------------------ CLI arguments
def test_cli_config_overrides_and_ignored_keys(tmp_path, caplog):
    from reprover_b200 import predict_cli

    cfg = tmp_path / "cli.yaml"
    cfg.write_text("seed_everything: 3407\n"
                   "trainer:\n  accelerator: gpu\n  strategy:\n    class_path: x.DeepSpeedStrategy\n    init_args:\n      stage: 2\n"
                   "model:\n  model_name: google/byt5-small\n  lr: 1e-4\n  num_retrieved: 100\n"
                   "data:\n  data_path: data/random/\n  corpus_path: data/corpus.jsonl\n  eval_batch_size: 64\n"
                   "  max_seq_len: 1024\n")
    args, settings, ignored = predict_cli.parse_args(
        ["predict", "--config", str(cfg), "--ckpt_path", "r.ckpt", "--data.eval_batch_size=8", "--model.num_retrieved",
         "10", "--data.data_path", "other/random", "--trainer.devices", "2", "--output-path", "out.pickle"])
    assert args.subcommand == "predict" and args.ckpt_path == "r.ckpt" and args.output_path == "out.pickle"
    assert settings["data.eval_batch_size"] == 8 and settings["model.num_retrieved"] == 10
    assert settings["data.data_path"] == "other/random" and settings["data.max_seq_len"] == 1024
    assert settings["data.corpus_path"] == "data/corpus.jsonl"
    assert "trainer.devices" in ignored and "trainer.strategy.init_args.stage" in ignored and "seed_everything" in ignored
    assert "model.model_name" in ignored and not set(ignored) & set(predict_cli.USED_KEYS)
    args, _, _ = predict_cli.parse_args(["validate", "--hf-ckpt", "some/dir", "--data.max_seq_len", "256"])
    assert args.subcommand == "validate" and args.hf_ckpt == "some/dir" and args.output_path == "predictions.pickle"
    with pytest.raises(SystemExit):
        predict_cli.parse_args(["predict", "--config", str(cfg)])               # no checkpoint
    with pytest.raises(SystemExit):
        predict_cli.parse_args(["predict", "--ckpt_path", "a", "--hf-ckpt", "b"])
    with pytest.raises(SystemExit):
        predict_cli.parse_args(["predict", "--ckpt_path", "a", "--data.max_seq_len"])   # override without a value
    # the ignored keys are named in one log line before anything is loaded
    with caplog.at_level(logging.INFO, logger="reprover_b200.predict"), pytest.raises(Exception):
        predict_cli.main(["predict", "--config", str(cfg), "--ckpt_path", str(tmp_path / "absent.ckpt")])
    lines = [r.getMessage() for r in caplog.records if "ignoring" in r.getMessage()]
    assert len(lines) == 1 and "trainer.accelerator" in lines[0] and "model.lr" in lines[0]


# ------------------------------------------------------------------------------------------------ metrics
def _restated_eval(data, preds_map):
    """`retrieval/evaluate.py::_eval` restated: (R@1, R@10, MRR)."""
    r1, r10, mrr = [], [], []
    for thm in data:
        for i, _ in enumerate(thm["traced_tactics"]):
            pred = preds_map[(thm["file_path"], thm["full_name"], tuple(thm["start"]), i)]
            positives = set(pred["all_pos_premises"])
            if not positives:
                continue
            got = pred["retrieved_premises"]
            r1.append(float(got[0] in positives) / len(positives))
            r10.append(float(len(positives.intersection(got[:10]))) / len(positives))
            for j, p in enumerate(got):
                if p in positives:
                    mrr.append(1.0 / (j + 1))
                    break
            else:
                mrr.append(0.0)
    return 100 * np.mean(r1), 100 * np.mean(r10), np.mean(mrr)


def test_metrics_equal_the_reference_evaluation(tmp_path):
    data = synth.write_leandojo_dataset(str(tmp_path), n_files=4, premises_per_file=30, theorems=(5, 4, 4),
                                        min_accessible=20, seed=9)
    corpus = Corpus(os.path.join(data, "../corpus.jsonl"))
    examples = load_examples(data, corpus)
    rng = np.random.default_rng(3)
    records = []
    for ex in examples:
        acc = corpus.get_accessible_premise_indexes(ex["context"].path, ex["context"].theorem_pos)
        order = rng.permutation(acc)[:20].tolist()
        pos = [i for i in range(len(corpus)) if corpus[i] in ex["all_pos_premises"]]
        if pos and rng.random() < 0.6:                       # put a positive somewhere in the first 20
            order = [i for i in order if i != pos[0]]
            order.insert(int(rng.integers(0, 20)), pos[0])
        records.append(dict(ex, retrieved_premises=[corpus[i] for i in order[:20]]))
    preds_map = {(r["file_path"], r["full_name"], tuple(r["start"]), r["tactic_idx"]): r for r in records}
    thms = [t for s in ("train", "val", "test") for t in json.load(open(os.path.join(data, f"{s}.json")))]
    want_r1, want_r10, want_mrr = _restated_eval(thms, preds_map)
    recall, mrr, n = recall_and_mrr([r["all_pos_premises"] for r in records], [r["retrieved_premises"] for r in records], 20)
    assert n == sum(1 for r in records if r["all_pos_premises"]) and 0 < n < len(records)
    assert abs(recall[0] - want_r1) <= 1e-12 and abs(recall[9] - want_r10) <= 1e-12
    assert 0 < want_r10 < 100
    assert abs(mrr - want_mrr) <= 1e-12 and not math.isnan(mrr)
