"""Replays tests/golden/reference_generation.json (the reference's own `format_augmented_state`,
`GeneratorDataset.__getitem__` / `collate`, HF `ByT5Tokenizer` and `TopkAccuracy`; see
tests/golden/make_reference_generation_goldens.py) against this package's restatements."""
import json
import os
from pathlib import Path

import pytest

from reprover_b200.corpus import Context, Premise, format_augmented_state
from reprover_b200.generator_eval import ValidationMetrics, collate, load_examples, predictions_by_key
from reprover_b200.tokenizer import decode, encode_ids

GOLD = json.loads((Path(__file__).resolve().parent / "golden" / "reference_generation.json").read_text())


def _premise(p):
    return Premise(p[0], p[1], tuple(p[2]), tuple(p[3]), p[4])


@pytest.mark.parametrize("case", GOLD["format_augmented_state"], ids=lambda c: f"max_len={c['max_len']}")
def test_format_augmented_state(case):
    got = format_augmented_state(case["state"], [_premise(p) for p in case["premises"]], case["max_len"])
    assert got == case["out"]


def test_encode_and_decode():
    for c in GOLD["encode"]:
        assert encode_ids(c["text"], c["max_length"]) == c["ids"], c
    for c in GOLD["decode"]:
        assert decode(c["ids"]) == c["text"], c


def _write_val(tmp_path):
    path = tmp_path / "val.json"
    path.write_text(json.dumps(GOLD["dataset"]["theorems"]))
    return str(path)


def test_examples_and_collate_with_preds(tmp_path):
    d = GOLD["dataset"]
    records = []
    for key, premises in d["preds"].items():
        path, name, state = key.split("\x00")
        records.append({"context": Context(path, name, (1, 0), state),
                        "retrieved_premises": [_premise(p) for p in premises]})
    examples = load_examples(_write_val(tmp_path), predictions_by_key(records), d["max_inp_seq_len"])
    assert examples == d["examples"]
    batch = collate(examples, d["max_inp_seq_len"], d["max_oup_seq_len"])
    assert list(batch) == list(d["batch"])
    for key, want in d["batch"].items():
        got = batch[key]
        assert (got.tolist() if hasattr(got, "tolist") else got) == want, key


def test_examples_without_preds_and_missing_key(tmp_path):
    d = GOLD["dataset"]
    path = _write_val(tmp_path)
    assert load_examples(path) == d["examples_without_preds"]
    with pytest.raises(KeyError):
        load_examples(path, {}, d["max_inp_seq_len"])


def test_topk_accuracy():
    t = GOLD["topk"]
    m = ValidationMetrics(3)
    for preds, gt in t["batches"]:
        m.update(0.0, preds, gt)
    got = m.compute()
    assert [got[f"top{k}_acc_val"] for k in (1, 2, 3)] == t["acc"]
