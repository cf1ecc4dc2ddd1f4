"""Throughput of the BM25 retriever (`reprover_b200.bm25`) on a seeded synthetic workload.

    python tools/bm25_bench.py [--premises 200000] [--queries 4000] [--k 100]

Workload (assumptions, not measurements of a real dataset): premises of 8-120 tokens and proof states of 16-1500
tokens, lengths uniform in those ranges, token ids Zipf-distributed (exponent 1.1) over a 30 000-entry vocabulary
(train_tokenizer.py's default size).  The real corpus's postings count and the states' token counts are not known
here; the script prints what it generated (tokens, postings) so a run on real data can be compared.

Prints one JSON line: GPU name and power limit, index build time and device bytes, queries/s and postings visited/s
for all premises and for per-theorem accessibility masks (8 states per theorem, about half the premises each), and
the float64 CPU oracle's queries/s (tests/bm25_ref.py, one thread, vectorised over documents) on a sample.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def zipf_ids(rng, n, vocab):
    p = 1.0 / np.arange(1, vocab + 1) ** 1.1
    return rng.choice(vocab, size=n, p=p / p.sum())


def power_limit() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, reps=3):
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t)
    return best


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--premises", type=int, default=200_000)
    ap.add_argument("--queries", type=int, default=4000)
    ap.add_argument("--vocab", type=int, default=30_000)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--oracle-sample", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bm25_bench measures the GPU path: no CUDA device")
    from reprover_b200.bm25 import BM25Index

    rng = np.random.default_rng(args.seed)
    d_len = rng.integers(8, 121, args.premises)
    flat = zipf_ids(rng, int(d_len.sum()), args.vocab)
    cut = np.cumsum(d_len)[:-1]
    docs = [a.tolist() for a in np.split(flat, cut)]
    q_len = rng.integers(16, 1501, args.queries)
    qflat = zipf_ids(rng, int(q_len.sum()), args.vocab)
    queries = [a.tolist() for a in np.split(qflat, np.cumsum(q_len)[:-1])]

    t = time.perf_counter()
    index = BM25Index(docs, vocab_size=args.vocab)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t
    df = np.diff(index.term_ptr)
    postings = int(df[qflat].sum())      # what the kernels visit: every posting of every query token

    words_per = (args.premises + 31) // 32
    n_thm = (args.queries + 7) // 8
    bits = rng.random((n_thm, words_per * 32)) < 0.5
    words = np.packbits(bits.reshape(n_thm, -1, 8), axis=2, bitorder="little").reshape(n_thm, -1).view("<u4")
    rows = [i // 8 for i in range(args.queries)]

    index.topk_indexes(queries[:64], args.k)                     # warm-up: module load, allocations
    index.topk_indexes(queries[:64], args.k, words, rows[:64])
    all_s = timed(lambda: index.topk_indexes(queries, args.k))
    mask_s = timed(lambda: index.topk_indexes(queries, args.k, words, rows))

    from tests.bm25_ref import BM25Okapi, rank

    oracle = BM25Okapi(docs)
    sample = queries[: args.oracle_sample]
    t = time.perf_counter()
    for q in sample:
        rank(oracle.get_batch_scores(q, range(args.premises)), range(args.premises), args.k)
    cpu_s = time.perf_counter() - t
    got = index.topk_indexes(sample, args.k)
    agree = all(gi == rank(oracle.get_batch_scores(q, range(args.premises)), range(args.premises), args.k)[0]
                for q, gi in zip(sample, got[0]))

    print(json.dumps({
        "gpu": torch.cuda.get_device_name(), "power_limit": power_limit(),
        "premises": args.premises, "premise_tokens": int(d_len.sum()), "vocab": args.vocab, "nnz": index.nnz,
        "index_device_mb": round(index.device_bytes / 2**20, 1), "index_build_s": round(build_s, 2),
        "queries": args.queries, "query_tokens": int(q_len.sum()), "postings_visited": postings, "k": args.k,
        "all_premises": {"s": round(all_s, 4), "queries_per_s": round(args.queries / all_s, 1),
                         "postings_per_s": round(postings / all_s / 1e9, 3)},
        "masked": {"s": round(mask_s, 4), "queries_per_s": round(args.queries / mask_s, 1),
                   "postings_per_s": round(postings / mask_s / 1e9, 3)},
        "postings_per_s_unit": "1e9",
        "cpu_oracle": {"queries": len(sample), "queries_per_s": round(len(sample) / cpu_s, 2)},
        "oracle_agrees_on_sample": agree,
    }))


if __name__ == "__main__":
    main()
