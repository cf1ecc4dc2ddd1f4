"""The tactic generator's validation over a LeanDojo dataset on the engine: what the reference's
`generation/main.py validate` computes with `GeneratorDataModule` and `RetrievalAugmentedGenerator.validation_step`.

    examples = load_examples(os.path.join(data_path, "val.json"), preds, max_inp_seq_len)
    metrics = validate(engine, examples, batch_size=64, num_beams=1, max_inp_seq_len=2300, max_oup_seq_len=512)

Each piece restates the reference's rule:
  - `load_examples` is `GeneratorDataset._load_data` then `__getitem__(is_train=False)`: one example per traced
    tactic, its tactic without marks; with retrieval predictions, the state augmented by `format_augmented_state`
    with the premises the predictions record for (file_path, full_name, state_before), a missing key being a
    KeyError; then the state without marks.
  - `collate` is `GeneratorDataset.collate`: HF ByT5 tokenization with truncation (`tokenizer.encode_ids`),
    padding to the longest, label pads (id 0) as -100.
  - `validation_step` runs the loss and the search on one encoder pass (`T5GeneratorEngine.evaluate`) with the
    reference's keyword arguments; `length_penalty` is not passed, so it comes from the generation config.
  - `ValidationMetrics` is what Lightning reports at the epoch's end: `loss_val`, the mean of the batches' losses
    weighted by their size, and `top{k}_acc_val`, `TopkAccuracy`'s correct / total over all examples.
"""
from __future__ import annotations

import json
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

from .corpus import format_augmented_state, remove_marks
from .tokenizer import PAD_ID, decode, encode_ids, pad_batch

IGNORE_INDEX = -100


def predictions_by_key(preds: Sequence[Dict[str, Any]]) -> Dict[Tuple[str, str, str], Dict[str, Any]]:
    """`GeneratorDataModule`'s lookup table: each record of a retrieval predictions file under
    (context.path, context.theorem_full_name, context.state)."""
    return {(p["context"].path, p["context"].theorem_full_name, p["context"].state): p for p in preds}


def load_predictions(preds_path: str) -> Dict[Tuple[str, str, str], Dict[str, Any]]:
    """A retrieval predictions pickle, written by the reference or by `predict_cli` in either layout, as
    `predictions_by_key`'s table."""
    from .compat import load_reference_predictions

    return predictions_by_key(load_reference_predictions(preds_path))


def load_examples(json_path: str, preds: Optional[Dict[Tuple[str, str, str], Dict[str, Any]]] = None,
                  max_inp_seq_len: Optional[int] = None) -> List[Dict[str, Any]]:
    """The validation examples of one split file (`val.json`), as `GeneratorDataset.__getitem__(is_train=False)`
    returns them; `preds` is `predictions_by_key`'s table, or None for the plain states."""
    with open(json_path) as fh:
        theorems = json.load(fh)
    examples = []
    for thm in theorems:
        for tac in thm["traced_tactics"]:
            ex = {"url": thm["url"], "commit": thm["commit"], "file_path": thm["file_path"],
                  "full_name": thm["full_name"], "state": tac["state_before"], "tactic": remove_marks(tac["tactic"])}
            if preds is not None:
                pred = preds[(ex["file_path"], ex["full_name"], ex["state"])]
                ex["state"] = format_augmented_state(ex["state"], pred["retrieved_premises"], max_inp_seq_len)
            ex["state"] = remove_marks(ex["state"])
            examples.append(ex)
    return examples


def collate(examples: Sequence[Dict[str, Any]], max_inp_seq_len: int, max_oup_seq_len: int) -> Dict[str, Any]:
    """`GeneratorDataset.collate`: int64 CPU tensors `state_ids`, `state_mask`, `tactic_ids` (pads as -100) and
    `tactic_mask`, the `state` and `tactic` strings, and every other field as a list."""
    state = [ex["state"] for ex in examples]
    tactic = [ex["tactic"] for ex in examples]
    state_ids, state_mask = pad_batch([encode_ids(s, max_inp_seq_len) for s in state])
    tactic_ids, tactic_mask = pad_batch([encode_ids(t, max_oup_seq_len) for t in tactic])
    tactic_ids[tactic_ids == PAD_ID] = IGNORE_INDEX
    batch: Dict[str, Any] = {"state": state, "state_ids": torch.from_numpy(state_ids),
                             "state_mask": torch.from_numpy(state_mask), "tactic": tactic,
                             "tactic_ids": torch.from_numpy(tactic_ids), "tactic_mask": torch.from_numpy(tactic_mask)}
    for key in examples[0]:
        if key not in batch:
            batch[key] = [ex[key] for ex in examples]
    return batch


def validation_step(engine, batch: Dict[str, Any], num_beams: int, max_oup_seq_len: int
                    ) -> Tuple[float, List[List[str]]]:
    """(the batch's loss, each example's `num_beams` decoded tactics, best first), as `validation_step` computes
    them, with the loss and the search sharing one encoder pass."""
    out, sequences = engine.evaluate(batch["state_ids"], batch["state_mask"], batch["tactic_ids"],
                                     max_length=max_oup_seq_len, num_beams=num_beams, do_sample=False,
                                     num_return_sequences=num_beams, early_stopping=False)
    texts = [decode(row) for row in sequences.cpu().tolist()]
    batch_size = batch["state_ids"].size(0)
    assert len(texts) == batch_size * num_beams
    return float(out.loss), [texts[i * num_beams:(i + 1) * num_beams] for i in range(batch_size)]


class ValidationMetrics:
    """The epoch-end values Lightning logs for `validation_step`: `loss_val` = sum(loss_b * size_b) / sum(size_b)
    (Lightning infers a batch's size from its first tensor, `state_ids`), and `top{k}_acc_val` for k = 1..num_beams
    = the examples whose ground truth is among their first k predictions, marks removed on both sides, over all
    examples (`TopkAccuracy`)."""

    def __init__(self, num_beams: int) -> None:
        self.num_beams = num_beams
        self.loss_sum = 0.0
        self.total = 0
        self.correct = [0] * num_beams

    def update(self, loss: float, batch_preds: Sequence[Sequence[str]], batch_gt: Sequence[str]) -> None:
        assert len(batch_preds) == len(batch_gt)
        self.loss_sum += loss * len(batch_gt)
        self.total += len(batch_gt)
        for preds, gt in zip(batch_preds, batch_gt):
            gt = remove_marks(gt)
            preds = [remove_marks(p) for p in preds]
            for k in range(1, self.num_beams + 1):
                self.correct[k - 1] += gt in preds[:k]

    def compute(self) -> Dict[str, float]:
        out = {"loss_val": self.loss_sum / self.total}
        out.update({f"top{k}_acc_val": self.correct[k - 1] / self.total for k in range(1, self.num_beams + 1)})
        return out


def validate(engine, examples: Sequence[Dict[str, Any]], *, batch_size: int, num_beams: int, max_inp_seq_len: int,
             max_oup_seq_len: int) -> Dict[str, float]:
    """`ValidationMetrics` over `examples`, taken in order in batches of `batch_size` (the last one may be
    partial), as the reference's validation dataloader takes them."""
    if not examples:
        raise ValueError("no validation examples")
    metrics = ValidationMetrics(num_beams)
    for lo in range(0, len(examples), batch_size):
        batch = collate(examples[lo:lo + batch_size], max_inp_seq_len, max_oup_seq_len)
        loss, preds = validation_step(engine, batch, num_beams, max_oup_seq_len)
        metrics.update(loss, preds, batch["tactic"])
    return metrics.compute()
