"""Run the BM25 premise retriever over a LeanDojo dataset on the GPU.  Same flags and output as the reference's
`retrieval/bm25/main.py`:

    python -m reprover_b200.bm25_cli --tokenizer-path tokenizer.json --data-path <dataset>/random \\
        --output-path predictions.pickle [--num-retrieved 100] [--use-all-premises]

The corpus is `<data-path>/../corpus.jsonl`; the theorems are those of `train.json`, `val.json` and `test.json`.  The
output is a pickled list of prediction records that the reference's `retrieval/evaluate.py` and
`generation/datamodule.py` (`preds_path`) read.  Tied scores are ordered by corpus index.
"""
from __future__ import annotations

import argparse
import logging
import os
import pickle

from .bm25 import BM25Index, load_theorems, predict
from .compat import dump_reference_predictions
from .corpus import Corpus

logger = logging.getLogger("reprover_b200.bm25")


def main(argv=None) -> None:
    parser = argparse.ArgumentParser(description="BM25 premise retrieval on the H100 engine.")
    parser.add_argument("--tokenizer-path", type=str, required=True)
    parser.add_argument("--data-path", type=str, required=True)
    parser.add_argument("--output-path", type=str, required=True)
    parser.add_argument("--num-retrieved", type=int, default=100)
    parser.add_argument("--use-all-premises", action="store_true")
    parser.add_argument("--num-cpus", type=int, default=32,
                        help="accepted for compatibility and ignored: scoring runs on one GPU, not in CPU workers")
    parser.add_argument("--native-layout", action="store_true",
                        help="pickle this package's own classes instead of the reference's layout")
    args = parser.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    logger.info(args)
    from tokenizers import Tokenizer

    tokenizer = Tokenizer.from_file(args.tokenizer_path)
    corpus = Corpus(os.path.join(args.data_path, "../corpus.jsonl"))
    theorems = load_theorems(args.data_path)
    index = BM25Index.from_corpus(corpus, tokenizer)
    preds = predict(index, theorems, args.num_retrieved, args.use_all_premises)
    with open(args.output_path, "wb") as fh:
        if args.native_layout:
            pickle.dump(preds, fh)
        else:
            dump_reference_predictions(preds, fh)
    logger.info("Saved predictions to %s", args.output_path)


if __name__ == "__main__":
    main()
