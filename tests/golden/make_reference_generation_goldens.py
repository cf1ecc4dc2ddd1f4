"""Golden vectors from the REFERENCE'S OWN CODE for the generator's validation data path.

    python tests/golden/make_reference_generation_goldens.py <reference checkout>

Imports the reference's `common.py` and `generation/datamodule.py` unmodified and runs, with the installed HF
`ByT5Tokenizer` (which needs no files):
  - `format_augmented_state` (p_drop 0) on cases at its edges: the state alone over `max_len`; augmented states of
    exactly `max_len` and `max_len` +- 1 bytes; a large premise skipped and a later small one kept; multibyte UTF-8
    at the cut; marks in premises; special-token literals;
  - `GeneratorDataset._load_data`, `__getitem__(is_train=False)` and `collate` on a small dataset with retrieval
    predictions;
  - the tokenizer with truncation, and `batch_decode(..., skip_special_tokens=True)` on invalid UTF-8 and
    `<extra_id_N>` ids;
  - `TopkAccuracy.update` / `compute` over two batches, the last one partial.  `TopkAccuracy` (generation/model.py)
    subclasses torchmetrics' `Metric`, and torchmetrics is not installed here, so `restated_topk_accuracy` below
    restates its `update` and `compute` line for line: it is the one computation in this file that is not the
    reference's own code.
The inputs and outputs go to `tests/golden/reference_generation.json`, which `tests/test_generation_golden_cpu.py`
replays against `reprover_b200.generator_eval`, `corpus.format_augmented_state`, `tokenizer.encode_ids` and
`tokenizer.decode` on any machine.

`common.py` and `datamodule.py` import packages that are not installed here (lean_dojo, pytorch_lightning,
deepspeed, loguru); `tests/golden/make_reference_goldens.py`'s inert stubs stand in for them, with lean_dojo's `Pos`.
"""
import json
import os
import sys
import tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
OUT = HERE / "reference_generation.json"
sys.path.insert(0, str(HERE))


def restated_topk_accuracy(k, batches, remove_marks):
    """generation/model.py `TopkAccuracy(k)`: `update(batch_preds, batch_gt)` per batch, then `compute()`."""
    correct, total = 0, 0
    for batch_preds, batch_gt in batches:
        assert len(batch_preds) == len(batch_gt)
        for preds, gt in zip(batch_preds, batch_gt):
            gt = remove_marks(gt)
            preds = [remove_marks(p) for p in preds]
            correct += gt in preds[:k]
        total += len(batch_gt)
    return correct / total


def premise_json(p):
    return [p.path, p.full_name, list(p.start), list(p.end), p.code]


def main():
    from make_reference_goldens import _stub_modules

    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    Pos = _stub_modules()
    import types

    import pytorch_lightning as pl

    pl.LightningDataModule = type("LightningDataModule", (), {})
    sys.modules.setdefault("loguru", types.SimpleNamespace(logger=types.SimpleNamespace(
        info=lambda *a, **k: None, warning=lambda *a, **k: None, debug=lambda *a, **k: None)))
    sys.path.insert(0, sys.argv[1])
    import common as refc  # the reference, unmodified
    from generation import datamodule as refdm  # the reference, unmodified
    from transformers import ByT5Tokenizer

    tok = ByT5Tokenizer()

    def P(name, code, line=1):
        return refc.Premise("Gold/A.lean", name, Pos(line, 0), Pos(line + 1, 0), code)

    small = P("Gold.small", "theorem small : a = a")                     # 21 bytes + 2
    big = P("Gold.big", "theorem big : " + "x" * 80, 5)                  # 94 bytes + 2
    marked = P("Gold.mk", "theorem mk (h : p) : mk h := by\n  exact mk h", 9)
    multi = P("Gold.uni", "theorem uni : ∀ α, α → α ⊢ β", 13)        # multibyte
    special = P("Gold.sp", "def sp := \"</s> <pad> <extra_id_7> <unk>\"", 17)
    state = "h : p\n⊢ q ∧ r"
    sl = len(state.encode())
    fas = []

    def case(s, premises, max_len):
        fas.append({"state": s, "premises": [premise_json(p) for p in premises], "max_len": max_len,
                    "out": refc.format_augmented_state(s, premises, max_len, 0.0)})

    unit = len((small.serialize() + "\n\n").encode())
    case(state, [small, big], sl - 1)                         # the state alone is over max_len
    case(state, [small], sl + unit)                           # exactly max_len
    case(state, [small], sl + unit - 1)                       # one byte short: skipped
    case(state, [small], sl + unit + 1)                       # one byte to spare
    case(state, [big, small, marked], sl + unit + 10)         # big skipped, small kept, marked skipped
    case(state, [marked, big, small], None)                   # no budget: everything, top-ranked farthest
    mu = len((multi.serialize() + "\n\n").encode())
    for d in (-2, -1, 0, 1):                                  # the cut inside / at the end of a multibyte premise
        case(state, [multi, small], sl + mu + d)
    case("⊢ <a>x</a> ∧ y", [marked, special], 400)             # marks and special-token literals
    case(state, [], 5)

    with tempfile.TemporaryDirectory() as tmp:
        thms = [{"url": "u", "commit": "c", "file_path": "Gold/A.lean", "full_name": "Gold.t1", "start": [30, 0],
                 "end": [40, 0], "traced_tactics": [
                     {"tactic": "simp [<a>small</a>]", "state_before": state, "state_after": "no goals"},
                     {"tactic": "exact <a>Gold.mk</a> h", "state_before": "h : p\n⊢ mk h", "state_after": "x"}]},
                {"url": "u", "commit": "c", "file_path": "Gold/B.lean", "full_name": "Gold.t2", "start": [1, 0],
                 "end": [9, 0], "traced_tactics": [
                     {"tactic": "rfl</s>", "state_before": "⊢ é = é" + " z" * 60, "state_after": "no goals"},
                     {"tactic": "x" * 40, "state_before": "⊢ <pad> ok", "state_after": "no goals"}]}]
        path = os.path.join(tmp, "val.json")
        with open(path, "w") as fh:
            json.dump(thms, fh)
        order = {"Gold/A.lean": [big, small, marked, multi], "Gold/B.lean": [special, multi, small]}
        preds = {}
        for thm in thms:
            for tac in thm["traced_tactics"]:
                preds[thm["file_path"], thm["full_name"], tac["state_before"]] = {
                    "retrieved_premises": order[thm["file_path"]]}
        max_inp, max_oup = 160, 24
        ds = refdm.GeneratorDataset(path, None, preds, max_inp, max_oup, 0.5, tok, is_train=False)
        items = [dict(ds[i]) for i in range(len(ds))]
        batch = ds.collate(items)
        dataset = {"theorems": thms, "max_inp_seq_len": max_inp, "max_oup_seq_len": max_oup,
                   "preds": {f"{k[0]}\x00{k[1]}\x00{k[2]}": [premise_json(p) for p in v["retrieved_premises"]]
                             for k, v in preds.items()},
                   "examples": items,
                   "batch": {k: (v.tolist() if hasattr(v, "tolist") else v) for k, v in batch.items()}}
        plain = refdm.GeneratorDataset(path, None, None, max_inp, max_oup, 0.5, tok, is_train=False)
        dataset["examples_without_preds"] = [dict(plain[i]) for i in range(len(plain))]

    texts = ["", "abc", "é" * 5, "a" * 10, "x </s> y", "<pad>z", "<extra_id_0>q<extra_id_124>", "<extra_id_125>"]
    encode = [{"text": t, "max_length": m, "ids": tok(t, max_length=m, truncation=True).input_ids}
              for t in texts for m in (4, 7, 64)]
    rows = [[3 + 0xC3, 3 + 0xA9, 1, 0, 0], [3 + 0xC3, 3 + 65, 2], [3 + 0xE2, 3 + 0x8A, 3 + 0xA2, 3 + 0x20],
            [259, 3 + 104, 300, 383, 3 + 105, 1], [0, 0, 0], [3 + 0xFF, 3 + 0x80, 3 + 108]]
    decode = [{"ids": r, "text": t} for r, t in zip(rows, tok.batch_decode(rows, skip_special_tokens=True))]

    batches = [([["a", "b", "c"], ["x", "<a>z</a>", "y"], ["p", "q", "r"]], ["<a>a</a>", "z", "s"]),
               ([["u", "v", "w"]], ["v"])]
    topk = {"batches": batches, "acc": [restated_topk_accuracy(k, batches, refc.remove_marks) for k in (1, 2, 3)]}

    OUT.write_text(json.dumps({"generator": "tests/golden/make_reference_generation_goldens.py (reference common.py "
                                            "and generation/datamodule.py imported unmodified; see its docstring)",
                               "format_augmented_state": fas, "dataset": dataset, "encode": encode, "decode": decode,
                               "topk": topk}, indent=1, ensure_ascii=False) + "\n")
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
