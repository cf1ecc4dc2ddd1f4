"""Run a trained dense retriever over a LeanDojo dataset on the GPU: the `predict` and `validate` subcommands of the
reference's `retrieval/main.py` (LightningCLI), with the same config file and flags.

    python -m reprover_b200.predict_cli predict --config retrieval/confs/cli_lean4_random.yaml \\
        --ckpt_path $PATH_TO_RETRIEVER_CHECKPOINT [--output-path predictions.pickle] [--native-layout]
    python -m reprover_b200.predict_cli validate --config ... --ckpt_path ...

`--ckpt_path` is a Lightning `.ckpt` or a DeepSpeed ZeRO directory (`B200PremiseRetriever.load`); `--hf-ckpt` takes
an HF checkpoint directory or hub id instead (`load_hf`).  Settings come from the YAML config and from
`--data.<key> <value>` / `--model.<key> <value>` overrides, later ones winning; the keys read are
`model.num_retrieved`, `data.data_path`, `data.corpus_path`, `data.max_seq_len` and `data.eval_batch_size`.  Other
LightningCLI keys (trainer, optimizer, logger, ...) are accepted and ignored.

`predict` ranks every traced tactic of `train.json`, `val.json` and `test.json` and writes the records of
`PremiseRetriever.predict_step`, by default in the reference's class layout (what `retrieval/evaluate.py` and
`generation/datamodule.py` read).  `validate` ranks `val.json` and prints Recall@1..k and MRR.
"""
from __future__ import annotations

import argparse
import json
import logging
import os
import pickle
from typing import Any, Dict, List, Optional, Tuple

from .cli_args import parse_cli

logger = logging.getLogger("reprover_b200.predict")

USED_KEYS = ("model.num_retrieved", "data.data_path", "data.corpus_path", "data.max_seq_len", "data.eval_batch_size")
SPLITS = {"predict": ("train", "val", "test"), "validate": ("val",)}


def parse_args(argv: Optional[List[str]] = None) -> Tuple[argparse.Namespace, Dict[str, Any], List[str]]:
    """(fixed flags, settings by dotted key, ignored keys), as `cli_args.parse_cli` reads them."""
    parser = argparse.ArgumentParser(description="Dense premise retrieval (predict / validate) on the H100 engine.")
    parser.add_argument("--output-path", type=str, default="predictions.pickle")
    parser.add_argument("--native-layout", action="store_true",
                        help="pickle this package's own classes instead of the reference's layout")
    return parse_cli(parser, SPLITS, USED_KEYS, argv)


def _load_retriever(args: argparse.Namespace, settings: Dict[str, Any]):
    import torch

    from .retriever import B200PremiseRetriever

    device = torch.device("cuda", torch.cuda.current_device())
    if args.ckpt_path is not None:
        retriever = B200PremiseRetriever.load(args.ckpt_path, device, freeze=True)
    else:
        if "data.max_seq_len" not in settings:
            raise SystemExit("--hf-ckpt needs data.max_seq_len (in --config or as --data.max_seq_len)")
        retriever = B200PremiseRetriever.load_hf(args.hf_ckpt, int(settings["data.max_seq_len"]), device)
    # LightningCLI builds the model from the config and links data.max_seq_len -> model.max_seq_len
    if "data.max_seq_len" in settings:
        retriever.max_seq_len = int(settings["data.max_seq_len"])
    if "model.num_retrieved" in settings:
        retriever.num_retrieved = int(settings["model.num_retrieved"])
    return retriever


def main(argv: Optional[List[str]] = None):
    """Runs the subcommand; returns the records (`predict`) or the metrics dict (`validate`)."""
    from .corpus import Corpus
    from .evaluation import load_examples, predict, validate

    args, settings, ignored = parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    if ignored:
        logger.info("ignoring settings this command does not use: %s", ", ".join(ignored))
    for key in ("data.data_path", "data.corpus_path"):
        if key not in settings:
            raise SystemExit(f"{key} is not set (in --config or as --{key})")
    batch_size = int(settings.get("data.eval_batch_size", 64))
    retriever = _load_retriever(args, settings)
    corpus = Corpus(settings["data.corpus_path"])
    retriever.load_corpus(corpus)
    examples = load_examples(settings["data.data_path"], corpus, SPLITS[args.subcommand])
    logger.info("%d examples, %d premises, k = %d", len(examples), len(corpus), retriever.num_retrieved)
    if args.subcommand == "validate":
        metrics = validate(retriever, examples, batch_size=batch_size)
        print(json.dumps(metrics))
        return metrics
    preds = predict(retriever, examples, batch_size=batch_size)
    os.makedirs(os.path.dirname(os.path.abspath(args.output_path)), exist_ok=True)
    with open(args.output_path, "wb") as fh:
        if args.native_layout:
            pickle.dump(preds, fh)
        else:
            from .compat import dump_reference_predictions

            dump_reference_predictions(preds, fh)
    logger.info("Retrieval predictions saved to %s", args.output_path)
    return preds


if __name__ == "__main__":
    main()
