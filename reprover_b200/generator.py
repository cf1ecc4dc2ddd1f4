"""The tactic generator's teacher-forced forward on the engine.

`T5GeneratorEngine` stands where the reference holds `self.generator =
T5ForConditionalGeneration.from_pretrained(...)` (generation/model.py), the way `T5EncoderEngine` stands for the
retriever's `self.encoder`.  Called as the reference calls it in `forward` (generation/model.py:101-111),

    gen(input_ids=state_ids, attention_mask=state_mask, labels=tactic_ids).loss

it returns HF's loss, the logits and the per-row log-likelihoods of the labels, all computed by `rpx_seq2seq_forward`
(encoder, cross K / V, decoder layers, head and log-softmax in sm_90a CUDA).  Beam search / `generate` is not here.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, NamedTuple, Optional, Union

import torch

from . import _native
from .engine import EncoderConfig, T5EncoderEngine, _stream_ptr, load_hf_checkpoint

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


class Seq2SeqOutput(NamedTuple):
    """What HF `T5ForConditionalGeneration` returns, as far as the reference reads it (`.loss`, `.logits`), plus
    the per-row sums the loss is made of."""

    loss: torch.Tensor                # fp64 scalar: -sum(sequence_log_probs) / sum(num_tokens); NaN if nothing counts
    logits: Optional[torch.Tensor]    # [B, L_out, V] fp32; zeros at and past a row's decoder length
    sequence_log_probs: torch.Tensor  # [B] fp64: sum of log p(label) over the row's counted positions
    num_tokens: torch.Tensor          # [B] int32: the counted positions (labels != -100)


class T5GeneratorEngine:
    """ByT5/T5 encoder-decoder, teacher-forced, on one GPU (`rpx_seq2seq_forward`)."""

    def __init__(self, config: Dict, state_dict: Dict[str, torch.Tensor], device: Union[int, str, torch.device]) -> None:
        g = check_generator_checkpoint(config, state_dict)
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
        return cls(cfg, sd, device, **kw)

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
        if input_ids is None or input_ids.dim() != 2:
            raise ValueError("input_ids must be a [batch, seq_len] tensor")
        if labels is None or labels.dim() != 2 or labels.shape[0] != input_ids.shape[0]:
            raise ValueError("labels must be a [batch, tgt_len] tensor with input_ids' batch")
        ids = input_ids.to(device=self.device, dtype=torch.int64).contiguous()
        mask = None
        if attention_mask is not None:
            if attention_mask.shape != input_ids.shape:
                raise ValueError(f"attention_mask {tuple(attention_mask.shape)} != input_ids {tuple(input_ids.shape)}")
            mask = attention_mask.to(device=self.device, dtype=torch.int64).contiguous()
        lab = labels.to(device=self.device, dtype=torch.int64).contiguous()
        B, L_in = ids.shape
        L_out = lab.shape[1]
        logits = torch.empty(B, L_out, self.vocab_size, dtype=torch.float32, device=self.device) if return_logits else None
        seq_lp = torch.empty(B, dtype=torch.float64, device=self.device)
        seq_n = torch.empty(B, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            ws = self._workspace(B, L_in, L_out)
            _native.check(self.lib.rpx_seq2seq_forward(
                self._handle, self.encoder._handle, ids.data_ptr(), None if mask is None else mask.data_ptr(), B, L_in,
                lab.data_ptr(), L_out, None if logits is None else logits.data_ptr(), seq_lp.data_ptr(),
                seq_n.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr(self.device)))
        loss = -seq_lp.sum() / seq_n.sum().double()  # 0 / 0 = NaN when nothing counts, as HF's empty mean
        return Seq2SeqOutput(loss, logits, seq_lp, seq_n)

    forward = __call__
