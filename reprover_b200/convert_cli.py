"""Convert a checkpoint the reference's training writes into an HF checkpoint directory, as the reference's
`scripts/convert_checkpoint.py` does, on the CPU and without pytorch_lightning:

    python -m reprover_b200.convert_cli generator --src CKPT --dst DIR
    python -m reprover_b200.convert_cli retriever --src CKPT --dst DIR

`--src` is a Lightning `.ckpt` file or a DeepSpeed ZeRO directory.  `DIR` gets `config.json`, fp32
`model.safetensors` (`T5ForConditionalGeneration` names for a generator, `T5EncoderModel` names for a retriever) and
the ByT5 tokenizer files.  This is how the prover's `gen_ckpt_path` / `ret_ckpt_path` are made from training output,
and what `T5GeneratorEngine.from_hf_dir` / `B200PremiseRetriever.load_hf` read.
"""
from __future__ import annotations

import argparse
import logging
from typing import List, Optional

logger = logging.getLogger("reprover_b200.convert")


def convert(model_type: str, src: str, dst: str) -> None:
    from .checkpoint import load_generator_checkpoint, load_retriever_checkpoint
    from .engine import save_hf_dir

    if model_type == "generator":
        cfg, sd, _ = load_generator_checkpoint(src)
        save_hf_dir(dst, cfg, sd, "T5ForConditionalGeneration")
    elif model_type == "retriever":
        cfg, sd, _ = load_retriever_checkpoint(src)
        save_hf_dir(dst, cfg, sd, "T5EncoderModel")
    else:
        raise ValueError(f"model_type={model_type!r}: generator or retriever")
    from transformers import ByT5Tokenizer

    ByT5Tokenizer().save_pretrained(dst)


def main(argv: Optional[List[str]] = None) -> None:
    parser = argparse.ArgumentParser(description="Lightning / DeepSpeed checkpoint -> HF checkpoint directory.")
    parser.add_argument("model_type", choices=["generator", "retriever"])
    parser.add_argument("--src", type=str, required=True)
    parser.add_argument("--dst", type=str, required=True)
    args = parser.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    logger.info("Loading the model from %s", args.src)
    convert(args.model_type, args.src, args.dst)
    logger.info("The model saved in Hugging Face format to %s", args.dst)


if __name__ == "__main__":
    main()
