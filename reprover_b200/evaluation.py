"""Batched validate / predict path around the hot path (SURVEY.md §8f rank 4).

Host-side mirror of the retrieval half of `PremiseRetriever.validation_step` (reference
retrieval/model.py:215-268: Recall@1..num_retrieved and MRR over a batch of contexts) and
`predict_step` (:281-327: per-example prediction records).  The encode + nearest-premise search
underneath run on the GPU through `B200PremiseRetriever`; the Lightning loop and logging are out
of scope.

`load_examples`, `predict` and `validate` are the dataset-level drivers (`retrieval/main.py predict` /
`validate`): the examples of `RetrievalDataset(is_train=False)` and every one of them ranked, batch
after batch, with the host building batch i's records while the GPU ranks batch i+1.
"""
from __future__ import annotations

from typing import Any, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .corpus import Context, Corpus, Pos, Premise


def recall_and_mrr(all_pos_premises: Sequence[Sequence[Premise]], retrieved: Sequence[Sequence[Premise]],
                   num_retrieved: int) -> Tuple[List[float], float, int]:
    """(Recall@1..num_retrieved in percent, MRR, number of examples with >= 1 positive premise).

    Same arithmetic as the reference: examples without positives are skipped; Recall@j is the
    fraction of an example's positives among its first j retrieved premises, averaged over
    examples; MRR uses the first hit (0 if none within num_retrieved)."""
    recall: List[List[float]] = [[] for _ in range(num_retrieved)]
    mrr: List[float] = []
    n = 0
    assert len(all_pos_premises) == len(retrieved)
    for positives, premises in zip(all_pos_premises, retrieved):
        positives = set(positives)
        if not positives:
            continue
        n += 1
        first = False
        hits = 0
        for j in range(num_retrieved):
            hits += premises[j] in positives   # premises are distinct, so a running count == |intersection|
            recall[j].append(hits / len(positives))
            if premises[j] in positives and not first:
                mrr.append(1.0 / (j + 1))
                first = True
        if not first:
            mrr.append(0.0)
    if n == 0:
        return [float("nan")] * num_retrieved, float("nan"), 0
    return [100.0 * float(np.mean(r)) for r in recall], float(np.mean(mrr)), n


def validation_step(retriever, batch: Dict[str, Any]) -> Dict[str, float]:
    """Retrieve `retriever.num_retrieved` premises for `batch["context"]` (a list of `Context`) and score
    them against `batch["all_pos_premises"]`.  Returns {"Recall@k_val": ..., "MRR": ...}."""
    ctxs: List[Context] = batch["context"]
    k = retriever.num_retrieved
    premises, _ = retriever.retrieve_batch([c.state for c in ctxs], [c.path for c in ctxs],
                                           [c.theorem_full_name for c in ctxs], [c.theorem_pos for c in ctxs], k)
    recall, mrr, n = recall_and_mrr(batch["all_pos_premises"], premises, k)
    out = {f"Recall@{j + 1}_val": recall[j] for j in range(k)}
    out["MRR"] = mrr
    out["num_with_premises"] = n
    return out


_PREDICT_KEYS = ("url", "commit", "file_path", "full_name", "start", "tactic_idx")


def predict_step(retriever, batch: Dict[str, Any]) -> List[Dict[str, Any]]:
    """Prediction records in the format the reference pickles to `predictions.pickle`."""
    ctxs: List[Context] = batch["context"]
    k = retriever.num_retrieved
    premises, scores = retriever.retrieve_batch([c.state for c in ctxs], [c.path for c in ctxs],
                                                [c.theorem_full_name for c in ctxs], [c.theorem_pos for c in ctxs], k)
    records = []
    for i, ctx in enumerate(ctxs):
        rec = {key: batch[key][i] for key in _PREDICT_KEYS if key in batch}
        rec.update(context=ctx, all_pos_premises=batch["all_pos_premises"][i], retrieved_premises=premises[i],
                   scores=scores[i])
        records.append(rec)
    return records


# ---------------------------------------------------------------------------------------------- dataset level
def load_examples(data_path: str, corpus: Corpus, splits: Sequence[str] = ("train", "val", "test")) -> List[Dict[str, Any]]:
    """The evaluation examples of `RetrievalDataset(is_train=False)` over `<data_path>/<split>.json` for each split
    (reference retrieval/datamodule.py:44-90): one per traced tactic, in file (split) order, then theorem order,
    then tactic order, with keys `url, commit, file_path, full_name, start, tactic_idx, context, all_pos_premises`.
    A tactic whose provenances locate no premise is an example with an empty `all_pos_premises`.  Positives are
    the reference's set, listed in the order of their first provenance (`bm25.all_pos_premises`)."""
    from .bm25 import all_pos_premises, load_theorems

    examples: List[Dict[str, Any]] = []
    for thm in load_theorems(data_path, splits):
        for i, tac in enumerate(thm["traced_tactics"]):
            examples.append({
                "url": thm["url"],
                "commit": thm["commit"],
                "file_path": thm["file_path"],
                "full_name": thm["full_name"],
                "start": thm["start"],
                "tactic_idx": i,
                "context": Context(thm["file_path"], thm["full_name"], Pos(*thm["start"]), tac["state_before"]),
                "all_pos_premises": all_pos_premises(tac["annotated_tactic"], corpus),
            })
    return examples


def ranked_batches(retriever, examples: Sequence[Dict[str, Any]], k: int, batch_size: int = 64
                   ) -> Iterator[Tuple[Sequence[Dict[str, Any]], List[List[Premise]], List[List[float]]]]:
    """(examples, retrieved premises, fp32 scores as Python floats) per batch of `batch_size` examples, in order.

    Re-indexes the corpus if it is stale.  Each batch is one `encode_texts` (cut into engine calls by the encoder's
    token budget) and one masked top-k, the steps of `retrieve_batch`.  The next batch is put on the stream before
    this one's results are read back, so the GPU works while the caller turns a batch into records.  Contexts are
    always encoded on the throughput tiles (never the latency path `retrieve` uses for a few states), so every
    result is independent of `batch_size` and of the token budget."""
    from .retrieval_ops import nearest_premises_collect, nearest_premises_enqueue, result_staging

    if batch_size < 1:
        raise ValueError(f"batch_size={batch_size}: must be positive")
    retriever.reindex_corpus(batch_size)
    handle = retriever.index_handle()
    corpus = retriever.corpus
    stream = torch.cuda.current_stream(retriever.device)
    pending = None

    def collect(batch, stage, done):
        done.synchronize()
        try:
            premises, scores = nearest_premises_collect(corpus, stage, len(batch), k)
        except ValueError:
            short = [ex["context"] for ex, c in zip(batch, stage[0].tolist()) if c < k]
            raise ValueError(f"{len(short)} contexts have fewer than k={k} accessible premises, the first in "
                             f"{short[0].path} ({short[0].theorem_full_name})") from None
        return batch, premises, scores

    for lo in range(0, len(examples), batch_size):
        batch = examples[lo:lo + batch_size]
        ctxs = [ex["context"] for ex in batch]
        emb = retriever.encode_texts([c.serialize() for c in ctxs])
        stage = result_staging(len(batch), k)
        nearest_premises_enqueue(corpus, handle, ctxs, emb, k, stage)
        done = torch.cuda.Event()
        done.record(stream)
        if pending is not None:
            yield collect(*pending)
        pending = (batch, stage, done)
    if pending is not None:
        yield collect(*pending)


def prediction_records(batch: Sequence[Dict[str, Any]], premises: List[List[Premise]],
                       scores: List[List[float]]) -> List[Dict[str, Any]]:
    """The records `PremiseRetriever.predict_step` appends (retrieval/model.py:301-325), one per example."""
    return [{key: ex[key] for key in _PREDICT_KEYS} | {"context": ex["context"], "all_pos_premises": ex["all_pos_premises"],
                                                        "retrieved_premises": p, "scores": s}
            for ex, p, s in zip(batch, premises, scores)]


def predict(retriever, examples: Sequence[Dict[str, Any]], k: Optional[int] = None,
            batch_size: int = 64) -> List[Dict[str, Any]]:
    """`trainer.predict` of the reference's retriever over `examples` (`load_examples`): one record per example, in
    order, with the keys and values of `predict_step`.  `k` defaults to `retriever.num_retrieved`."""
    k = retriever.num_retrieved if k is None else k
    records: List[Dict[str, Any]] = []
    for batch, premises, scores in ranked_batches(retriever, examples, k, batch_size):
        records += prediction_records(batch, premises, scores)
    return records


def validate(retriever, examples: Sequence[Dict[str, Any]], k: Optional[int] = None,
             batch_size: int = 64) -> Dict[str, float]:
    """`trainer.validate`'s metrics over a whole split: `Recall@1_val` .. `Recall@{k}_val` in percent and `MRR`, over
    the examples with at least one positive premise (their number in `num_with_premises`).  The reference logs
    per-batch means weighted by each batch's number of such examples, which is this mean over the split."""
    k = retriever.num_retrieved if k is None else k
    positives: List[Sequence[Premise]] = []
    retrieved: List[List[Premise]] = []
    for batch, premises, _ in ranked_batches(retriever, examples, k, batch_size):
        positives += [ex["all_pos_premises"] for ex in batch]
        retrieved += premises
    recall, mrr, n = recall_and_mrr(positives, retrieved, k)
    out = {f"Recall@{j + 1}_val": recall[j] for j in range(k)}
    out["MRR"] = mrr
    out["num_with_premises"] = n
    return out
