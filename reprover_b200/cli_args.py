"""The command-line settings of the LightningCLI-style commands (`predict_cli`, `generator_cli`): YAML config files
plus dotted `--section.key value` overrides, flattened to one dict by dotted key."""
from __future__ import annotations

import argparse
from typing import Any, Dict, Iterable, List, Optional, Tuple


def flatten(tree: Dict[str, Any], prefix: str = "") -> Dict[str, Any]:
    """{"data": {"max_seq_len": 1024}} -> {"data.max_seq_len": 1024}."""
    out: Dict[str, Any] = {}
    for key, value in tree.items():
        if isinstance(value, dict):
            out.update(flatten(value, f"{prefix}{key}."))
        else:
            out[f"{prefix}{key}"] = value
    return out


def parse_cli(parser: argparse.ArgumentParser, subcommands: Iterable[str], used_keys: Iterable[str],
              argv: Optional[List[str]] = None) -> Tuple[argparse.Namespace, Dict[str, Any], List[str]]:
    """Parses `argv` with `parser`, to which this adds the subcommand, `--config`, `--ckpt_path` and `--hf-ckpt`.
    Returns (fixed flags, settings by dotted key, ignored keys: the settings not in `used_keys`).  Settings are the
    config files' in order, then the dotted command-line overrides; override values are read as YAML scalars, as
    LightningCLI reads them.  Exactly one of `--ckpt_path` and `--hf-ckpt` must be given."""
    import yaml

    parser.add_argument("subcommand", choices=sorted(subcommands))
    parser.add_argument("--config", action="append", default=[], help="LightningCLI YAML config (repeatable)")
    parser.add_argument("--ckpt_path", type=str, default=None, help="Lightning .ckpt file or DeepSpeed ZeRO directory")
    parser.add_argument("--hf-ckpt", type=str, default=None, help="HF checkpoint directory or hub id")
    args, rest = parser.parse_known_args(argv)
    if (args.ckpt_path is None) == (args.hf_ckpt is None):
        parser.error("pass exactly one of --ckpt_path and --hf-ckpt")
    settings: Dict[str, Any] = {}
    for path in args.config:
        with open(path) as fh:
            settings.update(flatten(yaml.safe_load(fh) or {}))
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
    used = set(used_keys)
    ignored = sorted({k for k in settings if k not in used})
    return args, settings, ignored
