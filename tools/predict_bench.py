"""Throughput of the dense retriever's dataset-level predict (`reprover_b200.evaluation.predict`) on a seeded synthetic
LeanDojo-shaped dataset, and where its time goes.

    python tools/predict_bench.py [--files 40] [--premises-per-file 500] [--theorems 1500 150 150] [--k 100]

Workload (assumptions about the real benchmark, not measurements of it): a ByT5-small-geometry encoder (12 layers,
random weights: timing does not depend on the values), premises of 16-600 bytes, proof states of 16-1024 bytes,
lengths uniform in those ranges, 1-8 traced tactics per theorem, every file importing the one before it.  The real
LeanDojo benchmark has about 150 k premises and 260 k traced tactics of other length distributions; the script prints
what it generated so a run on real data can be compared.

Prints one JSON line: GPU name and power limit; the time to re-index the corpus; `predict` end to end, host to host,
with the pickle written to memory (examples/s); and the same work run stage by stage with a device synchronise after
each stage (encoding the contexts, ranking them under their masks, building records, pickling), which splits the
time and, against the end-to-end figure, shows how much of the host work runs under the GPU's.
"""
from __future__ import annotations

import argparse
import io
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def staged(retriever, examples, k, batch_size):
    """predict's work without overlap: seconds spent encoding, ranking, building records."""
    from reprover_b200.evaluation import prediction_records
    from reprover_b200.retrieval_ops import nearest_premises_collect, nearest_premises_enqueue, result_staging

    handle = retriever.index_handle()
    corpus = retriever.corpus
    t_enc = t_rank = t_rec = 0.0
    records = []
    for lo in range(0, len(examples), batch_size):
        batch = examples[lo:lo + batch_size]
        ctxs = [ex["context"] for ex in batch]
        t0 = time.perf_counter()
        emb = retriever.encode_texts([c.serialize() for c in ctxs])
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        stage = result_staging(len(batch), k)
        nearest_premises_enqueue(corpus, handle, ctxs, emb, k, stage)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        premises, scores = nearest_premises_collect(corpus, stage, len(batch), k)
        records += prediction_records(batch, premises, scores)
        t3 = time.perf_counter()
        t_enc, t_rank, t_rec = t_enc + t1 - t0, t_rank + t2 - t1, t_rec + t3 - t2
    return records, t_enc, t_rank, t_rec


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=40)
    ap.add_argument("--premises-per-file", type=int, default=500)
    ap.add_argument("--theorems", type=int, nargs=3, default=[1500, 150, 150])
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--max-seq-len", type=int, default=1024)
    ap.add_argument("--layers", type=int, default=12)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("predict_bench measures the GPU path: no CUDA device")
    from reprover_b200 import synth
    from reprover_b200.corpus import Corpus
    from reprover_b200.evaluation import load_examples, predict
    from reprover_b200.retriever import B200PremiseRetriever

    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        data = synth.write_leandojo_dataset(tmp, n_files=args.files, premises_per_file=args.premises_per_file,
                                            theorems=tuple(args.theorems), tactics_per_theorem=(1, 8),
                                            state_len=(16, 1024), premise_len=(16, 600), min_accessible=args.k)
        corpus = Corpus(os.path.join(data, "../corpus.jsonl"))
        examples = load_examples(data, corpus)
        load_s = time.perf_counter() - t
        cfg = synth.tiny_config(num_layers=args.layers)
        synth.save_hf_checkpoint(os.path.join(tmp, "hf"), cfg, synth.random_t5_state_dict(cfg))
        retr = B200PremiseRetriever.load_hf(os.path.join(tmp, "hf"), args.max_seq_len, dev)
    retr.num_retrieved = args.k
    retr.load_corpus(corpus)
    context_tokens = sum(min(len(ex["context"].state.encode()) + 1, args.max_seq_len) for ex in examples)
    premise_tokens = sum(min(len(p.serialize().encode()) + 1, args.max_seq_len) for p in corpus.all_premises)

    predict(retr, examples[:256], batch_size=args.batch_size)          # warm-up: modules, workspaces, index
    retr.embeddings_staled = True
    torch.cuda.synchronize()
    t = time.perf_counter()
    retr.reindex_corpus(args.batch_size)
    torch.cuda.synchronize()
    reindex_s = time.perf_counter() - t

    e2e = []
    for _ in range(2):
        t = time.perf_counter()
        preds = predict(retr, examples, batch_size=args.batch_size)
        pickle.dump(preds, io.BytesIO())
        e2e.append(time.perf_counter() - t)
    e2e_s = min(e2e)

    records, enc_s, rank_s, rec_s = staged(retr, examples, args.k, args.batch_size)
    t = time.perf_counter()
    pickle.dump(records, io.BytesIO())
    pickle_s = time.perf_counter() - t
    same = pickle.dumps(records) == pickle.dumps(preds)
    split = {"encode_contexts_s": enc_s, "rank_s": rank_s, "records_s": rec_s, "pickle_s": pickle_s}
    serial_s = sum(split.values())
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(), "power_limit": power_limit(),
        "assumed_workload": {"premises": len(corpus), "premise_tokens": premise_tokens, "examples": len(examples),
                             "context_tokens": context_tokens, "k": args.k, "batch_size": args.batch_size,
                             "max_seq_len": args.max_seq_len, "layers": args.layers},
        "dataset_load_s": round(load_s, 3),
        "reindex_s": round(reindex_s, 3), "reindex_premises_per_s": round(len(corpus) / reindex_s, 1),
        "predict_e2e_s": round(e2e_s, 3), "predict_examples_per_s": round(len(examples) / e2e_s, 1),
        "staged": {key: round(v, 3) for key, v in split.items()} | {"total_s": round(serial_s, 3)},
        "staged_share": {key: round(v / serial_s, 3) for key, v in split.items()},
        "dominant": max(split, key=split.get),
        "overlap_saves_s": round(serial_s - e2e_s, 3),
        "staged_equals_pipelined": same,
    }))


if __name__ == "__main__":
    main()
