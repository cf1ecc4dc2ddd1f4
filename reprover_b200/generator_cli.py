"""Validate a trained tactic generator over a LeanDojo dataset on the GPU: the `validate` subcommand of the
reference's `generation/main.py` (LightningCLI), with the same config file and flags.

    python -m reprover_b200.generator_cli validate --config generation/confs/cli_lean4_random.yaml \\
        --ckpt_path $PATH_TO_GENERATOR_CHECKPOINT [--data.preds_path predictions.pickle]

`--ckpt_path` is a Lightning `.ckpt` or a DeepSpeed ZeRO directory (`T5GeneratorEngine.load`); `--hf-ckpt` takes an
HF checkpoint directory instead (`T5GeneratorEngine.from_hf_dir`).  Settings come from the YAML config and from
`--data.<key> <value>` / `--model.<key> <value>` overrides, later ones winning; the keys read are
`model.num_beams`, `data.data_path`, `data.preds_path`, `data.eval_batch_size`, `data.max_inp_seq_len` and
`data.max_oup_seq_len`.  A setting wins over the checkpoint's hyper-parameter of the same name, since LightningCLI
builds the module from the config and only loads the weights from `--ckpt_path`.  Other keys (trainer, optimizer,
`model.eval_num_theorems`, whose Pass@1 needs Lean, `model.ret_ckpt_path`, ...) are accepted and ignored.

`data.preds_path` is a retrieval predictions pickle (`predict_cli predict`'s, in either layout, or the reference's);
null means plain states.  Prints one JSON line: `loss_val` and `top{k}_acc_val` for k = 1..num_beams.
"""
from __future__ import annotations

import argparse
import json
import logging
import os
from typing import Any, Dict, List, Optional, Tuple

from .cli_args import parse_cli

logger = logging.getLogger("reprover_b200.generator")

USED_KEYS = ("model.num_beams", "data.data_path", "data.preds_path", "data.eval_batch_size", "data.max_inp_seq_len",
             "data.max_oup_seq_len")
SUBCOMMANDS = ("validate",)
# setting -> the reference module's hyper-parameter it sets
_HPARAMS = {"model.num_beams": "num_beams", "data.max_inp_seq_len": "max_inp_seq_len",
            "data.max_oup_seq_len": "max_oup_seq_len"}


def parse_args(argv: Optional[List[str]] = None) -> Tuple[argparse.Namespace, Dict[str, Any], List[str]]:
    """(fixed flags, settings by dotted key, ignored keys), as `cli_args.parse_cli` reads them."""
    parser = argparse.ArgumentParser(description="Tactic generator validation on the H100 engine.")
    return parse_cli(parser, SUBCOMMANDS, USED_KEYS, argv)


def resolve_settings(settings: Dict[str, Any], hparams: Dict[str, Any]) -> Dict[str, Any]:
    """The validation settings: each from the config when it is set there, else from the checkpoint's
    hyper-parameters; `data.eval_batch_size` and `data.data_path` must be set."""
    out = {}
    for key in ("data.data_path", "data.eval_batch_size"):
        if settings.get(key) is None:
            raise SystemExit(f"{key} is not set (in --config or as --{key})")
        out[key] = settings[key]
    for key, hp in _HPARAMS.items():
        value = settings.get(key, hparams.get(hp))
        if value is None:
            raise SystemExit(f"{key} is set neither in the config nor in the checkpoint's hyper-parameters")
        out[key] = int(value)
    out["data.eval_batch_size"] = int(out["data.eval_batch_size"])
    out["data.preds_path"] = settings.get("data.preds_path")
    return out


def _load_engine(args: argparse.Namespace):
    import torch

    from .generator import T5GeneratorEngine

    device = torch.device("cuda", torch.cuda.current_device())
    if args.ckpt_path is not None:
        return T5GeneratorEngine.load(args.ckpt_path, device, freeze=True)
    return T5GeneratorEngine.from_hf_dir(args.hf_ckpt, device)


def main(argv: Optional[List[str]] = None) -> Dict[str, float]:
    """Runs the subcommand; returns the metrics dict it prints."""
    from .generator_eval import load_examples, load_predictions, validate

    args, settings, ignored = parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    if ignored:
        logger.info("ignoring settings this command does not use: %s", ", ".join(ignored))
    engine = _load_engine(args)
    s = resolve_settings(settings, engine.hparams)
    preds = None
    if s["data.preds_path"] is not None:
        preds = load_predictions(s["data.preds_path"])
    examples = load_examples(os.path.join(s["data.data_path"], "val.json"), preds, s["data.max_inp_seq_len"])
    logger.info("%d examples, %s retrieval data, num_beams = %d", len(examples), "with" if preds else "without",
                s["model.num_beams"])
    metrics = validate(engine, examples, batch_size=s["data.eval_batch_size"], num_beams=s["model.num_beams"],
                       max_inp_seq_len=s["data.max_inp_seq_len"], max_oup_seq_len=s["data.max_oup_seq_len"])
    print(json.dumps(metrics))
    return metrics


if __name__ == "__main__":
    main()
