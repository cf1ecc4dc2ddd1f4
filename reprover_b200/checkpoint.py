"""Reading the checkpoints the reference's training writes: the retriever's (`PremiseRetriever.load`,
retrieval/model.py:49-50 -> common.py:load_checkpoint) and the tactic generator's (`RetrievalAugmentedGenerator.load`,
generation/model.py, the same `load_checkpoint`).

A Lightning `.ckpt` is a `torch.save` of a dict whose `state_dict` holds the LightningModule's parameters (the HF
encoder sits under the module attribute `encoder.`, so its keys read `encoder.shared.weight`,
`encoder.encoder.block.{i}...`; the generator's HF `T5ForConditionalGeneration` sits under `generator.`) and whose
`hyper_parameters` holds `save_hyperparameters()`'s dict (`model_name`,
`max_seq_len`, `num_retrieved`, ...).  The same layout comes out of `convert_zero_checkpoint_to_fp32_state_dict`, which
the reference applies to a DeepSpeed ZeRO directory before loading it.

The pickle may name classes of `pytorch_lightning`, `lightning` or `deepspeed` (an `AttributeDict` of hyper-parameters,
callback and loop state).  Neither package is needed here: a restricted unpickler turns those classes into inert
stand-ins, loads tensors and plain containers, and refuses every other class.
"""
from __future__ import annotations

import json
import os
import pickle
import tempfile
from typing import Any, Dict, Optional, Tuple

import torch

_FOREIGN = ("pytorch_lightning", "lightning", "lightning_fabric", "deepspeed")
_BUILTINS = {"set", "frozenset", "slice", "range", "complex", "bytearray", "bytes", "int", "float", "str", "bool",
             "list", "tuple", "dict"}
_OTHER = {("collections", "OrderedDict"), ("collections", "defaultdict"), ("_codecs", "encode"),
          ("argparse", "Namespace"), ("copyreg", "_reconstructor"), ("pathlib", "PosixPath"),
          ("pathlib", "WindowsPath"), ("pathlib", "PurePosixPath"), ("datetime", "datetime"),
          ("datetime", "timedelta"), ("numpy.core.multiarray", "_reconstruct"),
          ("numpy._core.multiarray", "_reconstruct"), ("numpy.core.multiarray", "scalar"),
          ("numpy._core.multiarray", "scalar"), ("numpy", "ndarray"), ("numpy", "dtype")}
# ByT5's values for what the tensors cannot show (google/byt5-small config.json)
BYT5_LN_EPS = 1e-6
BYT5_MAX_DISTANCE = 128
ZERO_CONVERSION = "pytorch_lightning.utilities.deepspeed.convert_zero_checkpoint_to_fp32_state_dict"


class StandIn(dict):
    """What a pickled `pytorch_lightning` / `lightning` / `deepspeed` object becomes: its items (an `AttributeDict`
    is a dict) and its attributes, with the original class name in `_pickled_class`."""

    _pickled_class = ""

    def __init__(self, *args, **kwargs) -> None:
        super().__init__()
        self._args = args

    def __setstate__(self, state) -> None:
        if isinstance(state, tuple) and len(state) == 2:   # (dict, slots)
            state = {**(state[0] or {}), **(state[1] or {})}
        if isinstance(state, dict):
            self.__dict__.update(state)
        else:
            self.__dict__["_state"] = state


def _stand_in(module: str, name: str) -> type:
    return type(name, (StandIn,), {"_pickled_class": f"{module}.{name}", "__module__": __name__})


class _Unpickler(pickle.Unpickler):
    def find_class(self, module: str, name: str):
        root = module.split(".")[0]
        if root in _FOREIGN:
            return _stand_in(module, name)
        if root == "torch":
            obj = super().find_class(module, name)
            if isinstance(obj, (type, torch.dtype, torch.device)) or name.startswith("_rebuild") or name == "_get_layout":
                return obj
        elif (module == "builtins" and name in _BUILTINS) or (module, name) in _OTHER \
                or (module == "numpy.dtypes" and name.endswith("DType")):
            return super().find_class(module, name)
        raise pickle.UnpicklingError(f"checkpoint pickles {module}.{name}, which this reader does not load")


class _PickleModule:
    """What `torch.load(pickle_module=...)` needs: an `Unpickler` class and `load`."""

    __name__ = "reprover_b200.checkpoint"
    Unpickler = _Unpickler

    @staticmethod
    def load(fh, **kw):
        return _Unpickler(fh, **kw).load()


def read_lightning_checkpoint(path: str) -> Dict[str, Any]:
    """The dict a Lightning `.ckpt` file holds, tensors on the CPU, foreign classes as `StandIn`s."""
    return torch.load(path, map_location="cpu", pickle_module=_PickleModule, weights_only=False)


def is_deepspeed_checkpoint(path: str) -> bool:
    """A DeepSpeed ZeRO checkpoint directory (reference common.py:_is_deepspeed_checkpoint)."""
    if not os.path.exists(path):
        raise FileNotFoundError(f"checkpoint {path} does not exist")
    return os.path.isdir(path) and os.path.exists(os.path.join(path, "zero_to_fp32.py"))


def _convert_zero_checkpoint(ckpt_dir: str, out_file: str, example_name: str = "retriever.ckpt") -> None:
    try:
        import deepspeed  # noqa: F401
        try:
            from pytorch_lightning.utilities.deepspeed import convert_zero_checkpoint_to_fp32_state_dict
        except ImportError:
            from lightning.pytorch.utilities.deepspeed import convert_zero_checkpoint_to_fp32_state_dict
    except ImportError as exc:
        raise RuntimeError(
            f"{ckpt_dir} is a DeepSpeed ZeRO checkpoint directory, and converting it needs the `deepspeed` and "
            f"`pytorch_lightning` packages, which are not importable here.  Convert it where they are, with "
            f"`{ZERO_CONVERSION}({ckpt_dir!r}, {example_name!r})`, and pass the resulting file.") from exc
    convert_zero_checkpoint_to_fp32_state_dict(ckpt_dir, out_file)


def _encoder_keys(num_layers: int) -> list:
    from .engine import required_weight_keys

    return ["shared.weight"] + required_weight_keys({"num_layers": num_layers})


def encoder_state_dict(state_dict: Dict[str, torch.Tensor], prefix: str = "encoder.") -> Dict[str, torch.Tensor]:
    """The HF `T5EncoderModel` state dict inside a LightningModule's: keys under `prefix`, prefix stripped, fp32.
    Raises KeyError naming the missing keys and the keys that are there when it is not a T5 encoder's."""
    sd = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix) and torch.is_tensor(v)}
    if "shared.weight" not in sd and "encoder.embed_tokens.weight" in sd:
        sd["shared.weight"] = sd["encoder.embed_tokens.weight"]
    layers = 0
    while f"encoder.block.{layers}.layer.0.SelfAttention.q.weight" in sd:
        layers += 1
    missing = [k for k in _encoder_keys(max(layers, 1)) if k not in sd]
    if missing:
        raise KeyError(f"checkpoint has no T5/ByT5 encoder under {prefix!r}: {len(missing)} keys missing "
                       f"({[prefix + k for k in missing[:6]]}...); its state_dict keys are "
                       f"{sorted(state_dict)[:12]}{'...' if len(state_dict) > 12 else ''}")
    return {k: v.float() for k, v in sd.items()}


_SHAPE_KEYS = ("vocab_size", "d_model", "num_heads", "d_kv", "d_ff", "num_layers", "relative_attention_num_buckets")


def config_from_shapes(sd: Dict[str, torch.Tensor]) -> Dict[str, Any]:
    """A ByT5 encoder config read off the weights of `encoder_state_dict`'s result; what the weights do not show
    (layer-norm epsilon, relative-position max distance) takes ByT5's values."""
    vocab, d_model = sd["shared.weight"].shape
    buckets, heads = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"].shape
    inner = sd["encoder.block.0.layer.0.SelfAttention.q.weight"].shape[0]
    if inner % heads:
        raise ValueError(f"attention width {inner} is not a multiple of the {heads} heads of the relative bias")
    layers = 0
    while f"encoder.block.{layers}.layer.0.SelfAttention.q.weight" in sd:
        layers += 1
    return dict(vocab_size=int(vocab), d_model=int(d_model), num_heads=int(heads), d_kv=int(inner // heads),
                d_ff=int(sd["encoder.block.0.layer.1.DenseReluDense.wi_0.weight"].shape[0]), num_layers=layers,
                relative_attention_num_buckets=int(buckets), relative_attention_max_distance=BYT5_MAX_DISTANCE,
                layer_norm_epsilon=BYT5_LN_EPS, feed_forward_proj="gated-gelu", model_type="t5")


def cached_config(model_name: str, filename: str = "config.json") -> Optional[Dict[str, Any]]:
    """`filename` (a JSON file: `config.json`, `generation_config.json`) of `model_name` from a local checkpoint
    directory or the local HF cache; None when neither has it.  Never goes to the network."""
    path = os.path.join(model_name, filename) if os.path.isdir(model_name) else None
    if path is None:
        try:
            from huggingface_hub import try_to_load_from_cache

            found = try_to_load_from_cache(model_name, filename)
            path = found if isinstance(found, str) else None
        except Exception:   # not a repo id, or no huggingface_hub
            path = None
    if path is None or not os.path.exists(path):
        return None
    with open(path) as fh:
        return json.load(fh)


def resolve_config(model_name: Optional[str], sd: Dict[str, torch.Tensor],
                   config: Optional[Dict[str, Any]] = None) -> Dict[str, Any]:
    """The encoder config for the weights `sd`: `config` when given, else `model_name`'s cached config, else the one
    derived from the shapes.  A given or cached config that disagrees with the shapes is an error."""
    derived = config_from_shapes(sd)
    chosen, source = config, "the config passed in"
    if chosen is None and model_name:
        chosen, source = cached_config(model_name), f"the cached config of {model_name!r}"
    if chosen is None:
        return derived
    diff = {k: (chosen.get(k), derived[k]) for k in _SHAPE_KEYS if chosen.get(k) != derived[k]}
    if diff:
        raise ValueError(f"{source} disagrees with the checkpoint's weights (config, weights): {diff}")
    return dict(chosen)


def _read_module_checkpoint(ckpt_path: str) -> Tuple[Dict[str, Any], Dict[str, Any]]:
    """(LightningModule state dict, hyper-parameters) of a Lightning `.ckpt` file."""
    ckpt = read_lightning_checkpoint(ckpt_path)
    if not isinstance(ckpt, dict) or not isinstance(ckpt.get("state_dict"), dict):
        raise KeyError(f"{ckpt_path} is not a Lightning checkpoint: no `state_dict` entry "
                       f"(top-level keys: {sorted(ckpt) if isinstance(ckpt, dict) else type(ckpt).__name__})")
    return ckpt["state_dict"], dict(ckpt.get("hyper_parameters") or {})


def load_retriever_checkpoint(ckpt_path: str, config: Optional[Dict[str, Any]] = None
                              ) -> Tuple[Dict[str, Any], Dict[str, torch.Tensor], Dict[str, Any]]:
    """(encoder config, fp32 encoder state dict, hyper-parameters) of a retriever checkpoint: a Lightning `.ckpt`
    file or a DeepSpeed ZeRO directory (converted as the reference converts it)."""
    if is_deepspeed_checkpoint(ckpt_path):
        with tempfile.TemporaryDirectory() as tmp:
            out = os.path.join(tmp, "lightning.ckpt")
            _convert_zero_checkpoint(ckpt_path, out)
            return load_retriever_checkpoint(out, config)
    state_dict, hparams = _read_module_checkpoint(ckpt_path)
    sd = encoder_state_dict(state_dict)
    return resolve_config(hparams.get("model_name"), sd, config), sd, hparams


# ------------------------------------------------------------------------------------------ the generator
_TIED_ALIASES = ("encoder.embed_tokens.weight", "decoder.embed_tokens.weight")


def _count_blocks(sd: Dict[str, torch.Tensor], stack: str) -> int:
    n = 0
    while f"{stack}.block.{n}.layer.0.SelfAttention.q.weight" in sd:
        n += 1
    return n


def heads_tied(sd: Dict[str, torch.Tensor]) -> bool:
    """Whether the head is the embedding: False when `lm_head.weight` is present and differs from `shared.weight`,
    True otherwise.  The shapes alone cannot tell: ByT5's untied head has the embedding's shape, and a tied module's
    state dict lists `lm_head.weight` as the embedding itself."""
    head = sd.get("lm_head.weight")
    return head is None or (head.shape == sd["shared.weight"].shape and torch.equal(head, sd["shared.weight"]))


def generator_state_dict(state_dict: Dict[str, Any], prefix: str = "generator.") -> Dict[str, torch.Tensor]:
    """The HF `T5ForConditionalGeneration` state dict inside a LightningModule's: keys under `prefix`, prefix
    stripped, fp32.  Everything else (`retriever.*`: the frozen retriever a module trained with `ret_ckpt_path`
    carries) is dropped.  Raises KeyError naming the missing keys when it is not a T5 encoder-decoder's."""
    from .generator import required_generator_keys

    sd = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix) and torch.is_tensor(v)}
    if "shared.weight" not in sd:
        for alias in _TIED_ALIASES:
            if alias in sd:
                sd["shared.weight"] = sd[alias]
                break
    n_enc, n_dec = max(_count_blocks(sd, "encoder"), 1), max(_count_blocks(sd, "decoder"), 1)
    need = _encoder_keys(n_enc)
    if "shared.weight" in sd:
        need += required_generator_keys({"num_layers": n_enc, "num_decoder_layers": n_dec,
                                         "feed_forward_proj": "gated-gelu", "tie_word_embeddings": heads_tied(sd)})
    missing = [k for k in dict.fromkeys(need) if k not in sd]
    if missing:
        raise KeyError(f"checkpoint has no T5/ByT5 encoder-decoder under {prefix!r}: {len(missing)} keys missing "
                       f"({[prefix + k for k in missing[:6]]}...); its state_dict keys are "
                       f"{sorted(state_dict)[:12]}{'...' if len(state_dict) > 12 else ''}")
    return {k: v.float() for k, v in sd.items()}


_SEQ2SEQ_SHAPE_KEYS = _SHAPE_KEYS + ("num_decoder_layers", "tie_word_embeddings")


def seq2seq_config_from_shapes(sd: Dict[str, torch.Tensor]) -> Dict[str, Any]:
    """A ByT5 encoder-decoder config read off the weights of `generator_state_dict`'s result: `config_from_shapes`
    for the encoder, the decoder's layer count from `decoder.block.*`, and `tie_word_embeddings` by `heads_tied`.
    Ids (pad 0 = decoder start, EOS 1), the layer-norm epsilon and the relative-position maximum distance take
    ByT5's values.  A decoder whose attention geometry differs from the encoder's is an error."""
    cfg = config_from_shapes(sd)
    dec_buckets, dec_heads = sd["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"].shape
    dec_inner = sd["decoder.block.0.layer.0.SelfAttention.q.weight"].shape[0]
    dec_ff = sd["decoder.block.0.layer.2.DenseReluDense.wi_0.weight"].shape[0]
    enc = (cfg["relative_attention_num_buckets"], cfg["num_heads"], cfg["num_heads"] * cfg["d_kv"], cfg["d_ff"])
    if (dec_buckets, dec_heads, dec_inner, dec_ff) != enc:
        raise ValueError(f"decoder (buckets, heads, attention width, d_ff) = {(dec_buckets, dec_heads, dec_inner, dec_ff)}"
                         f" differs from the encoder's {enc}")
    cfg.update(num_decoder_layers=_count_blocks(sd, "decoder"), tie_word_embeddings=heads_tied(sd),
               is_encoder_decoder=True, pad_token_id=0, eos_token_id=1, decoder_start_token_id=0,
               architectures=["T5ForConditionalGeneration"])
    return cfg


def resolve_seq2seq_config(model_name: Optional[str], sd: Dict[str, torch.Tensor],
                           config: Optional[Dict[str, Any]] = None) -> Dict[str, Any]:
    """`resolve_config` for an encoder-decoder: `config` when given, else `model_name`'s cached config, else
    `seq2seq_config_from_shapes`.  A given or cached config that disagrees with the shapes (the encoder's keys, the
    decoder's layer count, or the tied-head rule) is an error."""
    derived = seq2seq_config_from_shapes(sd)
    chosen, source = config, "the config passed in"
    if chosen is None and model_name:
        chosen, source = cached_config(model_name), f"the cached config of {model_name!r}"
    if chosen is None:
        return derived
    norm = dict(chosen)
    norm["num_decoder_layers"] = chosen.get("num_decoder_layers") or chosen.get("num_layers")
    norm["tie_word_embeddings"] = chosen.get("tie_word_embeddings", True) is not False
    diff = {k: (norm.get(k), derived[k]) for k in _SEQ2SEQ_SHAPE_KEYS if norm.get(k) != derived[k]}
    if diff:
        raise ValueError(f"{source} disagrees with the checkpoint's weights (config, weights): {diff}")
    return dict(chosen)


def load_generator_checkpoint(ckpt_path: str, config: Optional[Dict[str, Any]] = None
                              ) -> Tuple[Dict[str, Any], Dict[str, torch.Tensor], Dict[str, Any]]:
    """(model config, fp32 `T5ForConditionalGeneration` state dict, hyper-parameters) of a tactic-generator
    checkpoint: a Lightning `.ckpt` file or a DeepSpeed ZeRO directory (converted as the reference converts it).
    The hyper-parameters are what `save_hyperparameters()` stored (`model_name`, `num_beams`, `length_penalty`,
    `max_inp_seq_len`, `max_oup_seq_len`, ...)."""
    if is_deepspeed_checkpoint(ckpt_path):
        with tempfile.TemporaryDirectory() as tmp:
            out = os.path.join(tmp, "lightning.ckpt")
            _convert_zero_checkpoint(ckpt_path, out, "generator.ckpt")
            return load_generator_checkpoint(out, config)
    state_dict, hparams = _read_module_checkpoint(ckpt_path)
    sd = generator_state_dict(state_dict)
    return resolve_seq2seq_config(hparams.get("model_name"), sd, config), sd, hparams
