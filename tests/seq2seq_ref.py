"""Float64 restatement of HF `T5ForConditionalGeneration.forward(input_ids, attention_mask, labels)` (T5 v1.1 /
ByT5: gated-gelu FFN, RMSNorm without mean subtraction, no attention scaling) and of the label rules the engine
implements, written from the model's definition rather than by calling HF, so that the CPU suite can pin it against
HF and the GPU suite can use it where HF fp32 is too slow to call.

Per row b (the rows never interact):
    encoder over the first len_enc(b) state tokens (bidirectional bias), final RMSNorm -> e
    decoder inputs  _shift_right(labels[b]) over the first dec_len(b) positions (`decoder_lengths`)
    per decoder layer: h += O(causal_attn(RMS(h)) + unidirectional bias);  h += O_c(attn(Q_c RMS(h), K_c e, V_c e));
                       h += wo(gelu_new(wi_0 n) * (wi_1 n))
    logits = RMS_final(h) W_head^T (* d_model ** -0.5 when the embeddings are tied)
    log p(label_p) = log_softmax(logits_p)[label_p] for the positions whose label is not -100.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch

IGNORE = -100


def relative_bucket(rel: torch.Tensor, bidirectional: bool, num_buckets: int, max_distance: int) -> torch.Tensor:
    """T5's relative-position bucket (key - query), float32 log-spaced part as in the model code."""
    ret = torch.zeros_like(rel)
    nb = num_buckets
    if bidirectional:
        nb //= 2
        ret = ret + (rel > 0).long() * nb
        n = rel.abs()
    else:
        n = -torch.clamp(rel, max=0)
    max_exact = nb // 2
    large = max_exact + (torch.log(n.float().clamp_min(1) / max_exact) / math.log(max_distance / max_exact)
                         * (nb - max_exact)).long()
    large = torch.clamp(large, max=nb - 1)
    return ret + torch.where(n < max_exact, n, large)


def decoder_lengths(labels: torch.Tensor) -> torch.Tensor:
    """Row b's decoder length: 1 + the last position whose label is not -100 (0 for a row of -100 only)."""
    L = labels.shape[1]
    pos = torch.arange(1, L + 1).expand_as(labels)
    return torch.where(labels != IGNORE, pos, torch.zeros_like(pos)).amax(1)


def shift_right(labels: torch.Tensor, start_id: int = 0, pad_id: int = 0) -> torch.Tensor:
    """HF `_shift_right`: start token, then labels[:, :-1], -100 replaced by the pad id."""
    out = torch.full_like(labels, start_id)
    out[:, 1:] = labels[:, :-1]
    return out.masked_fill(out == IGNORE, pad_id)


def _rms(x, w, eps):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def _gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x.pow(3))))


def _attend(xq, xkv, w, pre, H, bias=None, causal=False):
    q = (xq @ w[pre + "q.weight"].t()).reshape(xq.shape[0], H, -1).transpose(0, 1)
    k = (xkv @ w[pre + "k.weight"].t()).reshape(xkv.shape[0], H, -1).transpose(0, 1)
    v = (xkv @ w[pre + "v.weight"].t()).reshape(xkv.shape[0], H, -1).transpose(0, 1)
    s = q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    if causal:
        Lq = xq.shape[0]
        s = s.masked_fill(torch.ones(Lq, Lq, dtype=torch.bool).triu(1), -math.inf)
    o = torch.softmax(s, -1) @ v
    return o.transpose(0, 1).reshape(xq.shape[0], -1) @ w[pre + "o.weight"].t()


def _bias(table, L_q, L_k, bidirectional, nb, R):
    rel = torch.arange(L_k)[None, :] - torch.arange(L_q)[:, None]
    return table[relative_bucket(rel, bidirectional, nb, R)].permute(2, 0, 1)  # [H, Lq, Lk]


def _ffn(x, w, pre):
    return (_gelu_new(x @ w[pre + "wi_0.weight"].t()) * (x @ w[pre + "wi_1.weight"].t())) @ w[pre + "wo.weight"].t()


def forward_row(cfg: Dict, w: Dict[str, torch.Tensor], ids: torch.Tensor, labels: torch.Tensor
                ) -> Tuple[torch.Tensor, torch.Tensor]:
    """One row: ids [len_enc] (the state's tokens), labels [L_out].  Returns (logits [dec_len, V], log p [dec_len])
    in float64; log p is 0 where the label is -100."""
    H, eps = cfg["num_heads"], cfg.get("layer_norm_epsilon", 1e-6)
    nb, R = cfg.get("relative_attention_num_buckets", 32), cfg.get("relative_attention_max_distance", 128)
    n_dec = int(cfg.get("num_decoder_layers") or cfg["num_layers"])
    tied = cfg.get("tie_word_embeddings", True) is not False
    emb = w["shared.weight"]
    x = emb[ids]
    Le = x.shape[0]
    eb = _bias(w["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], Le, Le, True, nb, R)
    for i in range(cfg["num_layers"]):
        p = f"encoder.block.{i}."
        x = x + _attend(_rms(x, w[p + "layer.0.layer_norm.weight"], eps), _rms(x, w[p + "layer.0.layer_norm.weight"], eps),
                        w, p + "layer.0.SelfAttention.", H, eb)
        x = x + _ffn(_rms(x, w[p + "layer.1.layer_norm.weight"], eps), w, p + "layer.1.DenseReluDense.")
    e = _rms(x, w["encoder.final_layer_norm.weight"], eps)
    Ld = int(decoder_lengths(labels[None])[0])
    if Ld == 0:
        return torch.zeros(0, emb.shape[0], dtype=torch.float64), torch.zeros(0, dtype=torch.float64)
    y = emb[shift_right(labels[None])[0, :Ld]]
    db = _bias(w["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], Ld, Ld, False, nb, R)
    for i in range(n_dec):
        p = f"decoder.block.{i}."
        n = _rms(y, w[p + "layer.0.layer_norm.weight"], eps)
        y = y + _attend(n, n, w, p + "layer.0.SelfAttention.", H, db, causal=True)
        y = y + _attend(_rms(y, w[p + "layer.1.layer_norm.weight"], eps), e, w, p + "layer.1.EncDecAttention.", H)
        y = y + _ffn(_rms(y, w[p + "layer.2.layer_norm.weight"], eps), w, p + "layer.2.DenseReluDense.")
    y = _rms(y, w["decoder.final_layer_norm.weight"], eps)
    if tied:
        y = y * cfg["d_model"] ** -0.5
    logits = y @ (w["shared.weight"] if tied else w["lm_head.weight"]).t()
    lab = labels[:Ld]
    lp = torch.log_softmax(logits, -1).gather(1, lab.clamp_min(0)[:, None])[:, 0]
    return logits, torch.where(lab != IGNORE, lp, torch.zeros_like(lp))


def forward(cfg: Dict, sd: Dict[str, torch.Tensor], input_ids: torch.Tensor, attention_mask: torch.Tensor,
            labels: torch.Tensor) -> Dict[str, torch.Tensor]:
    """The whole batch: logits [B, L_out, V] (zeros past each row's decoder length), sequence_log_probs [B],
    num_tokens [B], loss (float64; NaN when no label counts)."""
    w = {k: v.double() for k, v in sd.items()}
    B, L_out = labels.shape
    V = cfg["vocab_size"]
    logits = torch.zeros(B, L_out, V, dtype=torch.float64)
    seq_lp = torch.zeros(B, dtype=torch.float64)
    lens = attention_mask.sum(1) if attention_mask is not None else torch.full((B,), input_ids.shape[1])
    for b in range(B):
        lg, lp = forward_row(cfg, w, input_ids[b, :int(lens[b])], labels[b])
        logits[b, :lg.shape[0]] = lg
        seq_lp[b] = lp.sum()
    n = (labels != IGNORE).sum(1)
    return {"logits": logits, "sequence_log_probs": seq_lp, "num_tokens": n,
            "loss": -seq_lp.sum() / n.sum().double()}


def hf_model_from_dir(path: str):
    """HF T5ForConditionalGeneration in fp32 from a checkpoint directory, loaded by `from_pretrained`: constructing
    the model and calling load_state_dict would tie `lm_head.weight` to `shared.weight` (transformers 5.5 shares
    their storage) and silently overwrite the embedding with the head."""
    from transformers import T5ForConditionalGeneration

    m = T5ForConditionalGeneration.from_pretrained(path, torch_dtype=torch.float32)
    return m.eval()


def untied_head_is_distinct(model, sd: Dict[str, torch.Tensor]) -> bool:
    """The loaded model's head and embedding are the checkpoint's own, distinct tensors."""
    return (not torch.equal(model.lm_head.weight, model.shared.weight)
            and torch.equal(model.lm_head.weight.detach().float(), sd["lm_head.weight"].float())
            and torch.equal(model.shared.weight.detach().float(), sd["shared.weight"].float()))


def random_batch(cfg: Dict, in_lens: List[int], label_rows: List[List[int]], seed: int):
    """input_ids / attention_mask [B, max in_len] (right-padded) and labels [B, max out_len] (-100-padded) from row
    lengths; label_rows gives each row's labels, None entries drawn at random."""
    g = torch.Generator().manual_seed(seed)
    B = len(in_lens)
    L_in = max(in_lens)
    ids = torch.randint(3, cfg["vocab_size"], (B, L_in), generator=g)
    mask = (torch.arange(L_in)[None, :] < torch.tensor(in_lens)[:, None]).long()
    ids = ids * mask
    L_out = max(len(r) for r in label_rows)
    labels = torch.full((B, L_out), IGNORE, dtype=torch.long)
    for b, r in enumerate(label_rows):
        labels[b, :len(r)] = torch.tensor(r, dtype=torch.long)
    return ids, mask, labels
