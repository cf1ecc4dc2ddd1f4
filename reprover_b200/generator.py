"""The tactic generator's teacher-forced forward on the engine.

`T5GeneratorEngine` stands where the reference holds `self.generator =
T5ForConditionalGeneration.from_pretrained(...)` (generation/model.py), the way `T5EncoderEngine` stands for the
retriever's `self.encoder`.  Called as the reference calls it in `forward` (generation/model.py:101-111),

    gen(input_ids=state_ids, attention_mask=state_mask, labels=tactic_ids).loss

it returns HF's loss, the logits and the per-row log-likelihoods of the labels, all computed by `rpx_seq2seq_forward`
(encoder, cross K / V, decoder layers, head and log-softmax in sm_90a CUDA).  `generate` runs HF's beam search
(or greedy search) over an incremental decoder with a KV cache (`rpx_seq2seq_generate`), as the reference calls it in
`HuggingFaceGenerator.generate` (prover/tactic_generator.py) and `validation_step` (generation/model.py).
"""
from __future__ import annotations

import ctypes as C
import json
import os
from typing import Any, Dict, NamedTuple, Optional, Union

import torch

from . import _native
from .engine import EncoderConfig, T5EncoderEngine, _stream_ptr, load_hf_checkpoint, resolve_checkpoint_dir

_DEC_LAYER_KEYS = {
    "h_q": "decoder.block.{i}.layer.0.SelfAttention.q.weight",
    "h_k": "decoder.block.{i}.layer.0.SelfAttention.k.weight",
    "h_v": "decoder.block.{i}.layer.0.SelfAttention.v.weight",
    "h_o": "decoder.block.{i}.layer.0.SelfAttention.o.weight",
    "h_ln0": "decoder.block.{i}.layer.0.layer_norm.weight",
    "h_cq": "decoder.block.{i}.layer.1.EncDecAttention.q.weight",
    "h_ck": "decoder.block.{i}.layer.1.EncDecAttention.k.weight",
    "h_cv": "decoder.block.{i}.layer.1.EncDecAttention.v.weight",
    "h_co": "decoder.block.{i}.layer.1.EncDecAttention.o.weight",
    "h_ln1": "decoder.block.{i}.layer.1.layer_norm.weight",
    "h_wi0": "decoder.block.{i}.layer.2.DenseReluDense.wi_0.weight",
    "h_wi1": "decoder.block.{i}.layer.2.DenseReluDense.wi_1.weight",
    "h_wo": "decoder.block.{i}.layer.2.DenseReluDense.wo.weight",
    "h_ln2": "decoder.block.{i}.layer.2.layer_norm.weight",
}
_DEC_REL_BIAS_KEY = "decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"
IGNORE_INDEX = -100


class GeneratorConfig(NamedTuple):
    """What the config rules decide (`generator_config`)."""

    num_decoder_layers: int
    head_key: str                # "lm_head.weight" (untied, ByT5) or "shared.weight" (tied)
    scale_decoder_outputs: bool  # logits scaled by d_model ** -0.5
    start_token_id: int


def generator_config(config: Dict) -> GeneratorConfig:
    """The HF T5 config rules the engine implements, checked:
      - `feed_forward_proj` must be "gated-gelu" (T5 v1.1 / ByT5);
      - `decoder_start_token_id` must equal `pad_token_id` (`_shift_right` feeds both);
      - `tie_word_embeddings: false` (ByT5): the head is `lm_head.weight` and outputs are not scaled;
        absent or true: the head is `shared.weight` and outputs are scaled by d_model ** -0.5
        (transformers 5.5 `T5Config.scale_decoder_outputs`)."""
    if config.get("feed_forward_proj", "relu") != "gated-gelu":
        raise NotImplementedError(f"feed_forward_proj={config.get('feed_forward_proj', 'relu')!r}: only the gated-gelu "
                                  f"T5 v1.1 / ByT5 feed-forward is implemented")
    pad = int(config.get("pad_token_id", 0))
    start = config.get("decoder_start_token_id")
    start = pad if start is None else int(start)
    if start != pad:
        raise NotImplementedError(f"decoder_start_token_id={start} != pad_token_id={pad}: HF `_shift_right` feeds both "
                                  f"and the engine implements them as one id")
    tied = config.get("tie_word_embeddings", True) is not False
    n_dec = int(config.get("num_decoder_layers") or config["num_layers"])
    return GeneratorConfig(n_dec, "shared.weight" if tied else "lm_head.weight", tied, start)


def required_generator_keys(config: Dict) -> list:
    """Every state-dict key the decoder half reads (HF T5ForConditionalGeneration names)."""
    g = generator_config(config)
    keys = [_DEC_REL_BIAS_KEY, "decoder.final_layer_norm.weight", "encoder.final_layer_norm.weight", "shared.weight",
            g.head_key]
    for i in range(g.num_decoder_layers):
        keys += [pattern.format(i=i) for pattern in _DEC_LAYER_KEYS.values()]
    return list(dict.fromkeys(keys))


def check_generator_checkpoint(config: Dict, state_dict: Dict[str, torch.Tensor]) -> GeneratorConfig:
    """The config rules (`generator_config`), and a KeyError listing every decoder-side key the state dict lacks."""
    g = generator_config(config)
    missing = [k for k in required_generator_keys(config) if k not in state_dict]
    if missing:
        raise KeyError(f"checkpoint is not a T5/ByT5 encoder-decoder state dict: {len(missing)} weights missing: "
                       f"{missing}")
    return g


# HF `GenerationConfig` defaults of the settings `generate` reads (transformers 5.5)
GENERATION_DEFAULTS = {"max_length": 20, "num_beams": 1, "num_return_sequences": 1, "length_penalty": 1.0,
                       "early_stopping": False, "do_sample": False}
# Settings whose value, other than the one listed, makes HF add a logits processor, a stopping criterion or a
# decoding mode the engine does not run.
_NEUTRAL = {"min_length": 0, "min_new_tokens": None, "max_new_tokens": None, "no_repeat_ngram_size": 0,
            "encoder_no_repeat_ngram_size": 0, "repetition_penalty": 1.0, "encoder_repetition_penalty": 1.0,
            "bad_words_ids": None, "force_words_ids": None, "forced_bos_token_id": None, "forced_eos_token_id": None,
            "suppress_tokens": None, "begin_suppress_tokens": None, "sequence_bias": None,
            "exponential_decay_length_penalty": None, "renormalize_logits": False, "num_beam_groups": 1,
            "diversity_penalty": 0.0, "constraints": None, "max_time": None, "stop_strings": None,
            "logits_processor": None, "stopping_criteria": None, "prefix_allowed_tokens_fn": None,
            "guidance_scale": None, "low_memory": None, "output_attentions": False, "output_hidden_states": False,
            "output_logits": False, "assistant_model": None, "streamer": None, "synced_gpus": None,
            "decoder_input_ids": None, "use_cache": True, "watermarking_config": None, "epsilon_cutoff": 0.0,
            "eta_cutoff": 0.0}
# Sampling settings: HF ignores them when do_sample is False, and so does the engine.
_IGNORED = {"temperature", "top_k", "top_p", "min_p", "typical_p", "top_h"}


class GenerationSettings(NamedTuple):
    """What `generation_settings` decides for one `generate` call."""

    max_length: int
    num_beams: int
    num_return_sequences: int
    length_penalty: float
    eos_token_id: int
    pad_token_id: int
    decoder_start_token_id: int
    output_scores: bool
    return_dict_in_generate: bool


def generation_settings(config: Dict, generation_config: Optional[Dict] = None, **kwargs: Any) -> GenerationSettings:
    """HF `generate`'s settings as the engine runs them: a keyword argument wins over the checkpoint's
    `generation_config.json` (`generation_config`), which wins over HF's `GenerationConfig` defaults.  `eos_token_id`,
    `pad_token_id` and `decoder_start_token_id` come from the same chain, ending at the model config.
    Raises NotImplementedError naming each setting the engine does not run: `do_sample=True`, `early_stopping` other
    than False, `max_new_tokens`, a list of EOS ids, and any setting that would make HF add a logits processor or a
    stopping criterion (`min_length`, `no_repeat_ngram_size`, `repetition_penalty`, `bad_words_ids`, ...)."""
    gen = dict(generation_config or {})
    given = {k: v for k, v in kwargs.items() if v is not None}

    def pick(name, fallback=None):
        if name in given:
            return given[name]
        if gen.get(name) is not None:
            return gen[name]
        if name in GENERATION_DEFAULTS:
            return GENERATION_DEFAULTS[name]
        return config.get(name, fallback)

    refused = []
    if bool(pick("do_sample")):
        refused.append("do_sample=True")
    if pick("early_stopping") is not False:
        refused.append(f"early_stopping={pick('early_stopping')!r}")
    known = set(GENERATION_DEFAULTS) | {"eos_token_id", "pad_token_id", "decoder_start_token_id", "output_scores",
                                        "return_dict_in_generate"}
    for source in (gen, given):
        for name, value in source.items():
            if name in known or name in _IGNORED or value is None:
                continue
            if name not in _NEUTRAL:
                if source is given:
                    refused.append(name)
                continue
            if value != _NEUTRAL[name] and f"{name}={value!r}" not in refused:
                refused.append(f"{name}={value!r}")
    eos = pick("eos_token_id")
    if isinstance(eos, (list, tuple)):
        if len(eos) != 1:
            refused.append(f"eos_token_id={list(eos)!r} (one EOS id only)")
        else:
            eos = eos[0]
    if eos is None:
        refused.append("eos_token_id=None (the engine stops on one EOS id)")
    if refused:
        raise NotImplementedError(f"T5GeneratorEngine.generate runs beam or greedy search with one EOS id and no "
                                  f"logits processor; not supported: {refused}")
    num_beams = int(pick("num_beams"))
    n_ret = int(pick("num_return_sequences"))
    max_length = int(pick("max_length"))
    if num_beams < 1:
        raise ValueError(f"num_beams={num_beams} must be at least 1")
    if not 1 <= n_ret <= num_beams:
        raise ValueError(f"num_return_sequences={n_ret} must be in [1, num_beams={num_beams}]")
    if max_length < 2:
        raise ValueError(f"max_length={max_length}: the engine generates at least one token after the start token")
    pad = int(pick("pad_token_id", 0))
    start = pick("decoder_start_token_id")
    start = pad if start is None else int(start)
    return GenerationSettings(max_length, num_beams, n_ret, float(pick("length_penalty")), int(eos), pad, start,
                              bool(kwargs.get("output_scores") or gen.get("output_scores") or False),
                              bool(kwargs.get("return_dict_in_generate") or gen.get("return_dict_in_generate")
                                   or False))


class GenerateOutput(NamedTuple):
    """HF `generate(..., return_dict_in_generate=True)`'s output as far as the reference reads it.  The per-step
    `.scores` tuple is not produced."""

    sequences: torch.Tensor                   # int64 [B * num_return_sequences, L_out], state-major, best first
    sequences_scores: Optional[torch.Tensor]  # fp32 [B * num_return_sequences]; None for greedy or without output_scores


class Seq2SeqOutput(NamedTuple):
    """What HF `T5ForConditionalGeneration` returns, as far as the reference reads it (`.loss`, `.logits`), plus
    the per-row sums the loss is made of."""

    loss: torch.Tensor                # fp64 scalar: -sum(sequence_log_probs) / sum(num_tokens); NaN if nothing counts
    logits: Optional[torch.Tensor]    # [B, L_out, V] fp32; zeros at and past a row's decoder length
    sequence_log_probs: torch.Tensor  # [B] fp64: sum of log p(label) over the row's counted positions
    num_tokens: torch.Tensor          # [B] int32: the counted positions (labels != -100)


class T5GeneratorEngine:
    """ByT5/T5 encoder-decoder on one GPU: the teacher-forced forward (`rpx_seq2seq_forward`), `generate`
    (`rpx_seq2seq_generate`), and both on one encoder pass (`evaluate`, `rpx_seq2seq_evaluate`)."""

    def __init__(self, config: Dict, state_dict: Dict[str, torch.Tensor], device: Union[int, str, torch.device],
                 generation_config: Optional[Dict] = None) -> None:
        g = check_generator_checkpoint(config, state_dict)
        self.generation_config = dict(generation_config or {})
        self.lib = _native.load()
        self.device = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if self.device.type != "cuda":
            raise RuntimeError(f"T5GeneratorEngine needs a CUDA device (got {self.device}); this engine has no CPU path")
        self.config = EncoderConfig(config)
        self.gen_config = g
        self.vocab_size = int(config["vocab_size"])
        # the encoder half: its own handle from the encoder.* keys (validates them)
        self.encoder = T5EncoderEngine(config, state_dict, self.device)
        self._handle = C.c_void_p()
        self._ws: Optional[torch.Tensor] = None
        self.hparams: Dict[str, Any] = {}
        self.last_steps = 0  # decoder steps of the last `evaluate`'s search (HF's count)
        with torch.cuda.device(self.device):
            cfg = _native.T5Config(
                vocab_size=config["vocab_size"], d_model=config["d_model"], d_kv=config["d_kv"], d_ff=config["d_ff"],
                num_layers=g.num_decoder_layers, num_heads=config["num_heads"],
                rel_buckets=config.get("relative_attention_num_buckets", 32),
                rel_max_distance=config.get("relative_attention_max_distance", 128),
                ln_eps=config.get("layer_norm_epsilon", 1e-6))
            nbytes = self.lib.rpx_t5_decoder_packed_bytes(C.byref(cfg))
            if nbytes == 0:
                raise _native.RpxError(_native.RPX_ERR_UNSUPPORTED, _native.last_error())
            self._packed = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            keep = []  # device copies of the raw fp32 weights, alive until packing has run

            def dev(t: torch.Tensor) -> int:
                d = t.to(device=self.device, dtype=torch.float32).contiguous()
                keep.append(d)
                return d.data_ptr()

            w = _native.T5DecoderWeights()
            w.d_shared = dev(state_dict["shared.weight"])
            w.d_rel_bias = dev(state_dict[_DEC_REL_BIAS_KEY])
            w.d_final_ln = dev(state_dict["decoder.final_layer_norm.weight"])
            w.d_enc_final_ln = dev(state_dict["encoder.final_layer_norm.weight"])
            w.d_head = dev(state_dict[g.head_key])
            arrays = []
            for field, pattern in _DEC_LAYER_KEYS.items():
                arr = (C.c_void_p * g.num_decoder_layers)(
                    *[dev(state_dict[pattern.format(i=i)]) for i in range(g.num_decoder_layers)])
                arrays.append(arr)
                setattr(w, field, C.cast(arr, _native._PP))
            _native.check(self.lib.rpx_t5_decoder_create(
                C.byref(cfg), C.byref(w), int(g.scale_decoder_outputs), g.start_token_id, self._packed.data_ptr(),
                nbytes, _stream_ptr(self.device), C.byref(self._handle)))
            torch.cuda.current_stream(self.device).synchronize()
            del keep

    @classmethod
    def from_hf_dir(cls, path: str, device, **kw) -> "T5GeneratorEngine":
        cfg, sd = load_hf_checkpoint(path)
        gc_path = os.path.join(resolve_checkpoint_dir(path), "generation_config.json")
        if "generation_config" not in kw and os.path.exists(gc_path):
            with open(gc_path) as fh:
                kw["generation_config"] = json.load(fh)
        return cls(cfg, sd, device, **kw)

    @classmethod
    def load(cls, ckpt_path: str, device, freeze: bool = True, config: Optional[Dict] = None) -> "T5GeneratorEngine":
        """The reference's `RetrievalAugmentedGenerator.load` (generation/model.py, common.py:load_checkpoint): a
        Lightning `.ckpt` written by the reference's training, or a DeepSpeed ZeRO checkpoint directory.  The model
        config is `config`, else `model_name`'s cached config, else the one the weights' shapes give
        (`checkpoint.load_generator_checkpoint`); `generation_config.json` is `model_name`'s cached one when there
        is one.  `engine.hparams` holds the checkpoint's hyper-parameters.  `freeze` is accepted for parity: the
        engine keeps no gradients."""
        from .checkpoint import cached_config, load_generator_checkpoint

        cfg, sd, hp = load_generator_checkpoint(ckpt_path, config)
        gen_cfg = cached_config(hp["model_name"], "generation_config.json") if hp.get("model_name") else None
        engine = cls(cfg, sd, device, generation_config=gen_cfg)
        engine.hparams = hp
        return engine

    def close(self) -> None:
        if getattr(self, "_handle", None) and self._handle.value:
            self.lib.rpx_t5_decoder_destroy(self._handle)
            self._handle = C.c_void_p()
        if getattr(self, "encoder", None) is not None:
            self.encoder.close()

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    @property
    def dtype(self) -> torch.dtype:
        return torch.bfloat16

    def _workspace(self, B: int, L_in: int, L_out: int) -> torch.Tensor:
        need = self.lib.rpx_seq2seq_workspace_bytes(self._handle, self.encoder._handle, B, L_in, L_out)
        if need == 0:
            raise _native.RpxError(_native.RPX_ERR_INVALID, f"no workspace size for batch={B} {L_in}x{L_out}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(int(need * 1.1) + 4096, dtype=torch.uint8, device=self.device)
        return self._ws

    def __call__(self, input_ids: torch.Tensor = None, attention_mask: Optional[torch.Tensor] = None,
                 labels: torch.Tensor = None, return_logits: bool = True, *, decoder_input_ids=None,
                 decoder_attention_mask=None, encoder_outputs=None, past_key_values=None, head_mask=None,
                 decoder_head_mask=None, cross_attn_head_mask=None, inputs_embeds=None, decoder_inputs_embeds=None,
                 use_cache: Optional[bool] = None, output_attentions: Optional[bool] = None,
                 output_hidden_states: Optional[bool] = None, return_dict: Optional[bool] = None) -> Seq2SeqOutput:
        """HF `T5ForConditionalGeneration.forward(input_ids, attention_mask, labels)` with teacher forcing.
        `attention_mask` must be a right-padded prefix mask (None: every position is a token).  `labels` [B, L_out]
        holds ids or -100.  `return_logits=False` skips writing the [B, L_out, V] logits."""
        unsupported = {"decoder_input_ids": decoder_input_ids is not None,
                       "decoder_attention_mask": decoder_attention_mask is not None,
                       "encoder_outputs": encoder_outputs is not None, "past_key_values": past_key_values is not None,
                       "head_mask": head_mask is not None, "decoder_head_mask": decoder_head_mask is not None,
                       "cross_attn_head_mask": cross_attn_head_mask is not None,
                       "inputs_embeds": inputs_embeds is not None,
                       "decoder_inputs_embeds": decoder_inputs_embeds is not None, "use_cache": bool(use_cache),
                       "output_attentions": bool(output_attentions),
                       "output_hidden_states": bool(output_hidden_states)}
        asked = [k for k, v in unsupported.items() if v]
        if asked:
            raise NotImplementedError(f"T5GeneratorEngine runs the teacher-forced forward from labels only; "
                                      f"not supported: {asked}")
        ids, mask = self._states(input_ids, attention_mask)
        lab = self._labels(labels, ids.shape[0])
        B, L_in = ids.shape
        L_out = lab.shape[1]
        logits, seq_lp, seq_n = self._loss_outputs(B, L_out, return_logits)
        with torch.cuda.device(self.device):
            ws = self._workspace(B, L_in, L_out)
            _native.check(self.lib.rpx_seq2seq_forward(
                self._handle, self.encoder._handle, ids.data_ptr(), None if mask is None else mask.data_ptr(), B, L_in,
                lab.data_ptr(), L_out, None if logits is None else logits.data_ptr(), seq_lp.data_ptr(),
                seq_n.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr(self.device)))
        return self._seq2seq_output(logits, seq_lp, seq_n)

    forward = __call__

    def _states(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor]):
        """Device int64 ids and mask (or None) of a [batch, seq_len] batch of states."""
        if input_ids is None or input_ids.dim() != 2:
            raise ValueError("input_ids must be a [batch, seq_len] tensor")
        ids = input_ids.to(device=self.device, dtype=torch.int64).contiguous()
        mask = None
        if attention_mask is not None:
            if attention_mask.shape != input_ids.shape:
                raise ValueError(f"attention_mask {tuple(attention_mask.shape)} != input_ids {tuple(input_ids.shape)}")
            mask = attention_mask.to(device=self.device, dtype=torch.int64).contiguous()
        return ids, mask

    def _labels(self, labels: torch.Tensor, batch: int) -> torch.Tensor:
        if labels is None or labels.dim() != 2 or labels.shape[0] != batch:
            raise ValueError("labels must be a [batch, tgt_len] tensor with input_ids' batch")
        return labels.to(device=self.device, dtype=torch.int64).contiguous()

    def _loss_outputs(self, B: int, L_out: int, return_logits: bool):
        logits = torch.empty(B, L_out, self.vocab_size, dtype=torch.float32, device=self.device) if return_logits else None
        seq_lp = torch.empty(B, dtype=torch.float64, device=self.device)
        seq_n = torch.empty(B, dtype=torch.int32, device=self.device)
        return logits, seq_lp, seq_n

    @staticmethod
    def _seq2seq_output(logits, seq_lp: torch.Tensor, seq_n: torch.Tensor) -> Seq2SeqOutput:
        loss = -seq_lp.sum() / seq_n.sum().double()  # 0 / 0 = NaN when nothing counts, as HF's empty mean
        return Seq2SeqOutput(loss, logits, seq_lp, seq_n)

    def to(self, device=None, *args: Any, **kwargs: Any) -> "T5GeneratorEngine":
        """HF's `model.to(device)`, as the reference calls it after loading a generator: the engine is bound to the
        GPU it was built on, so this returns it unchanged for that device (or no device) and raises for another."""
        if device is not None and not isinstance(device, torch.dtype):
            d = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
            same = d.type == "cuda" and (d.index is None or d.index == self.device.index
                                         or (self.device.index is None and d.index == torch.cuda.current_device()))
            if not same:
                raise ValueError(f"T5GeneratorEngine lives on {self.device}; it cannot move to {d}")
        return self

    def eval(self) -> "T5GeneratorEngine":
        """HF's `model.eval()`: the engine only evaluates, so it is returned unchanged."""
        return self

    def generate(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, *,
                 max_length: Optional[int] = None, num_beams: Optional[int] = None, do_sample: Optional[bool] = None,
                 num_return_sequences: Optional[int] = None, length_penalty: Optional[float] = None,
                 early_stopping: Optional[Union[bool, str]] = None, output_scores: bool = False,
                 return_dict_in_generate: bool = False, _trace_steps: int = 0, **unsupported: Any):
        """HF `T5ForConditionalGeneration.generate` for beam search (`num_beams > 1`) and greedy search, as the
        reference calls it.  Returns the sequences [B * num_return_sequences, L_out] (int64, on the engine's device),
        or with `return_dict_in_generate` a `GenerateOutput` with `.sequences` and `.sequences_scores` (None for greedy
        or without `output_scores`, as HF).  Settings follow `generation_settings`; a `pad_token_id` other than the
        decoder start id is refused (the engine fills with the start id, or EOS when that is 0, as HF's
        `output_fill_value` does for T5).  `_trace_steps` (tests) records each of the first that many steps and returns
        `(output, trace)`: "scores" [steps, R, V] (log-probs; logits for greedy), "parents" and "tokens" [steps, R],
        and "steps", the decoder steps HF runs for this call (the step at which the last search ended)."""
        s = self._generation_settings(max_length=max_length, num_beams=num_beams, do_sample=do_sample,
                                      num_return_sequences=num_return_sequences, length_penalty=length_penalty,
                                      early_stopping=early_stopping, output_scores=output_scores,
                                      return_dict_in_generate=return_dict_in_generate, **unsupported)
        ids, mask = self._states(input_ids, attention_mask)
        seqs, scores, trace = self._search(ids, mask, s, int(_trace_steps))
        if not s.return_dict_in_generate:
            if trace is not None:
                return GenerateOutput(seqs, scores), trace
            return seqs
        out = self._generate_output(s, seqs, scores)
        return (out, trace) if trace is not None else out

    def _generation_settings(self, **kwargs: Any) -> GenerationSettings:
        """`generation_settings` for this engine, and the refusals of ids the engine does not run."""
        s = generation_settings(self.config, self.generation_config, **kwargs)
        if s.decoder_start_token_id != self.gen_config.start_token_id:
            raise NotImplementedError(f"decoder_start_token_id={s.decoder_start_token_id}: the engine starts every "
                                      f"hypothesis with the config's {self.gen_config.start_token_id}")
        if s.pad_token_id != self.gen_config.start_token_id:
            raise NotImplementedError(f"pad_token_id={s.pad_token_id}: the engine pads with the decoder start id "
                                      f"{self.gen_config.start_token_id}, as `_shift_right` does")
        return s

    @staticmethod
    def _generate_output(s: GenerationSettings, seqs: torch.Tensor, scores: Optional[torch.Tensor]):
        if not s.return_dict_in_generate:
            return seqs
        return GenerateOutput(seqs, scores if s.output_scores else None)

    def evaluate(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor], labels: torch.Tensor, *,
                 return_logits: bool = False, **generate_kwargs: Any):
        """`self(input_ids, attention_mask, labels)` and `self.generate(input_ids, attention_mask, **generate_kwargs)`
        in one call, as the reference's `validation_step` runs them on one batch, with the encoder and the
        cross-attention K / V computed once for both (`rpx_seq2seq_evaluate`).  Returns `(Seq2SeqOutput, generate
        output)`, each equal bit for bit to what the two calls return; the settings and refusals are `generate`'s."""
        s = self._generation_settings(**generate_kwargs)
        ids, mask = self._states(input_ids, attention_mask)
        lab = self._labels(labels, ids.shape[0])
        B, L_in = ids.shape
        L_out = lab.shape[1]
        nb, n_ret, ML = s.num_beams, s.num_return_sequences, s.max_length
        logits, seq_lp, seq_n = self._loss_outputs(B, L_out, return_logits)
        seqs = torch.empty(B * n_ret, ML, dtype=torch.int64, device=self.device)
        scores = torch.empty(B * n_ret, dtype=torch.float32, device=self.device) if nb > 1 else None
        out_len, steps = C.c_int32(0), C.c_int32(0)
        with torch.cuda.device(self.device):
            need = self.lib.rpx_seq2seq_evaluate_workspace_bytes(self._handle, self.encoder._handle, B, L_in, L_out, nb,
                                                                 ML)
            if need == 0:
                raise _native.RpxError(_native.RPX_ERR_INVALID, f"no evaluate workspace for batch={B} {L_in}x{L_out} "
                                       f"num_beams={nb} max_length={ML}")
            ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            _native.check(self.lib.rpx_seq2seq_evaluate(
                self._handle, self.encoder._handle, ids.data_ptr(), None if mask is None else mask.data_ptr(), B, L_in,
                lab.data_ptr(), L_out, None if logits is None else logits.data_ptr(), seq_lp.data_ptr(),
                seq_n.data_ptr(), nb, n_ret, ML, s.length_penalty, s.eos_token_id, seqs.data_ptr(),
                None if scores is None else scores.data_ptr(), C.byref(out_len), C.byref(steps), ws.data_ptr(),
                ws.numel(), _stream_ptr(self.device)))
        self.last_steps = steps.value
        return (self._seq2seq_output(logits, seq_lp, seq_n),
                self._generate_output(s, seqs[:, :out_len.value].contiguous(), scores))

    def _search(self, ids: torch.Tensor, mask: Optional[torch.Tensor], s: GenerationSettings, trace_steps: int):
        """rpx_seq2seq_generate on device ids / mask: (sequences [B * n_ret, L_out], scores or None, trace or None)."""
        B, L_in = ids.shape
        nb, n_ret, ML = s.num_beams, s.num_return_sequences, s.max_length
        R = B * nb
        seqs = torch.empty(B * n_ret, ML, dtype=torch.int64, device=self.device)
        scores = torch.empty(B * n_ret, dtype=torch.float32, device=self.device) if nb > 1 else None
        trace = None
        if trace_steps:
            n = min(trace_steps, ML - 1)
            trace = {"scores": torch.full((n, R, self.vocab_size), float("nan"), device=self.device),
                     "parents": torch.full((n, R), -1, dtype=torch.int32, device=self.device),
                     "tokens": torch.full((n, R), -1, dtype=torch.int32, device=self.device)}
            c_trace = _native.GenerateTrace(trace["scores"].data_ptr(), trace["parents"].data_ptr(),
                                            trace["tokens"].data_ptr(), n)
        out_len, steps = C.c_int32(0), C.c_int32(0)
        with torch.cuda.device(self.device):
            need = self.lib.rpx_seq2seq_generate_workspace_bytes(self._handle, self.encoder._handle, B, L_in, nb, ML)
            if need == 0:
                raise _native.RpxError(_native.RPX_ERR_INVALID, f"no generate workspace for batch={B} in_len={L_in} "
                                       f"num_beams={nb} max_length={ML}")
            ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            _native.check(self.lib.rpx_seq2seq_generate(
                self._handle, self.encoder._handle, ids.data_ptr(), None if mask is None else mask.data_ptr(), B, L_in,
                nb, n_ret, ML, s.length_penalty, s.eos_token_id, seqs.data_ptr(),
                None if scores is None else scores.data_ptr(), C.byref(out_len), C.byref(steps),
                None if trace is None else C.byref(c_trace), ws.data_ptr(), ws.numel(), _stream_ptr(self.device)))
        if trace is not None:
            trace["steps"] = steps.value
        return seqs[:, :out_len.value].contiguous(), scores, trace
