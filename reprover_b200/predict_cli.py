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

logger = logging.getLogger("reprover_b200.predict")

USED_KEYS = ("model.num_retrieved", "data.data_path", "data.corpus_path", "data.max_seq_len", "data.eval_batch_size")
SPLITS = {"predict": ("train", "val", "test"), "validate": ("val",)}


def _flatten(tree: Dict[str, Any], prefix: str = "") -> Dict[str, Any]:
    """{"data": {"max_seq_len": 1024}} -> {"data.max_seq_len": 1024}."""
    out: Dict[str, Any] = {}
    for key, value in tree.items():
        if isinstance(value, dict):
            out.update(_flatten(value, f"{prefix}{key}."))
        else:
            out[f"{prefix}{key}"] = value
    return out


def parse_args(argv: Optional[List[str]] = None) -> Tuple[argparse.Namespace, Dict[str, Any], List[str]]:
    """(fixed flags, settings by dotted key, ignored keys).  Settings are the config files' in order, then the
    dotted command-line overrides; override values are read as YAML scalars, as LightningCLI reads them."""
    import yaml

    parser = argparse.ArgumentParser(description="Dense premise retrieval (predict / validate) on the H100 engine.")
    parser.add_argument("subcommand", choices=sorted(SPLITS))
    parser.add_argument("--config", action="append", default=[], help="LightningCLI YAML config (repeatable)")
    parser.add_argument("--ckpt_path", type=str, default=None, help="Lightning .ckpt file or DeepSpeed ZeRO directory")
    parser.add_argument("--hf-ckpt", type=str, default=None, help="HF checkpoint directory or hub id")
    parser.add_argument("--output-path", type=str, default="predictions.pickle")
    parser.add_argument("--native-layout", action="store_true",
                        help="pickle this package's own classes instead of the reference's layout")
    args, rest = parser.parse_known_args(argv)
    if (args.ckpt_path is None) == (args.hf_ckpt is None):
        parser.error("pass exactly one of --ckpt_path and --hf-ckpt")
    settings: Dict[str, Any] = {}
    for path in args.config:
        with open(path) as fh:
            settings.update(_flatten(yaml.safe_load(fh) or {}))
    i = 0
    while i < len(rest):
        tok = rest[i]
        if not tok.startswith("--"):
            parser.error(f"unexpected argument {tok!r}")
        if "=" in tok:
            key, value = tok[2:].split("=", 1)
            i += 1
        else:
            if i + 1 >= len(rest):
                parser.error(f"{tok} needs a value")
            key, value = tok[2:], rest[i + 1]
            i += 2
        settings[key] = yaml.safe_load(value)
    ignored = sorted({k for k in settings if k not in USED_KEYS})
    return args, settings, ignored


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
