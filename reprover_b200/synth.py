"""Deterministic synthetic inputs and checkpoints (there is no network: no real
corpus, no `google/byt5-small` weights).  Shapes / distributions follow SURVEY.md §8d.

Used by the tests, `bench.py` and `__graft_entry__.smoke()`; both the engine and the
oracle load the *same* synthetic checkpoint, so parity does not depend on how the
weights were drawn.
"""
from __future__ import annotations

import json
import os
from typing import Dict, List, Tuple

import numpy as np

SEED = 3407  # the reference's own seed (retrieval/confs/cli_lean4_random.yaml:1)

BYT5_SMALL = dict(
    vocab_size=384,
    d_model=1472,
    d_kv=64,
    d_ff=3584,
    num_layers=12,
    num_decoder_layers=4,
    num_heads=6,
    relative_attention_num_buckets=32,
    relative_attention_max_distance=128,
    dropout_rate=0.1,
    layer_norm_epsilon=1e-6,
    feed_forward_proj="gated-gelu",
    tie_word_embeddings=False,
    pad_token_id=0,
    eos_token_id=1,
)

# printable ASCII without '<' (0x3C): no ByT5 special-token literal can form, so
# tokenisation is exactly bytes + 3 (SURVEY.md §8 a5).
_ALPHABET = np.array([b for b in range(0x20, 0x7F) if b != 0x3C], dtype=np.uint8)
_TURNSTILE = "⊢ ".encode("utf-8")


def tiny_config(num_layers: int = 2) -> Dict:
    """ByT5-small geometry with fewer layers (fast CPU oracle runs)."""
    cfg = dict(BYT5_SMALL)
    cfg["num_layers"] = num_layers
    return cfg


def synth_byte_strings(n: int, seed: int = SEED, min_len: int = 16, max_len: int = 511,
                       prefix: bytes = b"") -> Tuple[np.ndarray, np.ndarray]:
    """n random byte strings; returns (bytes uint8 [total], offsets int64 [n+1]).

    Lengths ~ UniformInt[min_len, max_len] (bytes, before the EOS the tokenizer appends),
    bytes ~ Uniform(printable ASCII minus '<'); `prefix` is prepended to every string and
    counts towards its length.
    """
    rng = np.random.Generator(np.random.PCG64(seed))
    lens = rng.integers(min_len, max_len + 1, size=n, dtype=np.int64)
    lens = np.maximum(lens, len(prefix))
    offsets = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    data = _ALPHABET[rng.integers(0, len(_ALPHABET), size=int(offsets[-1]))]
    if prefix:
        pre = np.frombuffer(prefix, dtype=np.uint8)
        idx = offsets[:-1, None] + np.arange(len(pre))[None, :]
        data[idx] = pre[None, :]
    return data, offsets


def synth_premises(n: int, seed: int = SEED, **kw) -> Tuple[np.ndarray, np.ndarray]:
    return synth_byte_strings(n, seed, **kw)


def synth_states(n: int, seed: int = SEED + 100003, **kw) -> Tuple[np.ndarray, np.ndarray]:
    """Proof-state-like queries: every string starts with the turnstile (Context asserts it)."""
    return synth_byte_strings(n, seed, prefix=_TURNSTILE, **kw)


def split_strings(data: np.ndarray, offsets: np.ndarray) -> List[bytes]:
    return [data[offsets[i]:offsets[i + 1]].tobytes() for i in range(len(offsets) - 1)]


def random_t5_state_dict(cfg: Dict, seed: int = SEED) -> Dict[str, "torch.Tensor"]:
    """fp32 encoder weights under HF key names.

    Standard deviations follow HF `T5PreTrainedModel._init_weights` (factor 1.0) except
    that the RMSNorm weights are 1 + 0.1 N(0,1) and the relative-attention bias has std
    0.5: with the stock init (norm weights exactly 1, bias std 0.026) a kernel that
    dropped either would still pass a tolerance check.
    """
    import torch

    g = torch.Generator().manual_seed(seed)
    D, F = cfg["d_model"], cfg["d_ff"]
    H, dk = cfg["num_heads"], cfg["d_kv"]
    inner = H * dk

    def normal(shape, std):
        return torch.randn(shape, generator=g, dtype=torch.float32) * std

    sd = {"shared.weight": normal((cfg["vocab_size"], D), 1.0)}
    sd["encoder.embed_tokens.weight"] = sd["shared.weight"]
    sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"] = normal(
        (cfg["relative_attention_num_buckets"], H), 0.5)
    for i in range(cfg["num_layers"]):
        a = f"encoder.block.{i}.layer.0."
        f = f"encoder.block.{i}.layer.1."
        sd[a + "SelfAttention.q.weight"] = normal((inner, D), (D * dk) ** -0.5)
        sd[a + "SelfAttention.k.weight"] = normal((inner, D), D ** -0.5)
        sd[a + "SelfAttention.v.weight"] = normal((inner, D), D ** -0.5)
        sd[a + "SelfAttention.o.weight"] = normal((D, inner), inner ** -0.5)
        sd[a + "layer_norm.weight"] = 1.0 + normal((D,), 0.1)
        sd[f + "DenseReluDense.wi_0.weight"] = normal((F, D), D ** -0.5)
        sd[f + "DenseReluDense.wi_1.weight"] = normal((F, D), D ** -0.5)
        sd[f + "DenseReluDense.wo.weight"] = normal((D, F), F ** -0.5)
        sd[f + "layer_norm.weight"] = 1.0 + normal((D,), 0.1)
    sd["encoder.final_layer_norm.weight"] = 1.0 + normal((D,), 0.1)
    return sd


def random_t5_seq2seq_state_dict(cfg: Dict, seed: int = SEED) -> Dict[str, "torch.Tensor"]:
    """fp32 encoder-decoder weights under HF `T5ForConditionalGeneration` key names: `random_t5_state_dict`'s
    encoder plus the decoder (`num_decoder_layers`, default `num_layers`) and, unless the config ties the embeddings,
    `lm_head.weight`.  Drawn from a second generator, so the encoder keys equal `random_t5_state_dict(cfg, seed)`.
    The decoder's relative-attention bias is drawn apart from the encoder's, and the head apart from `shared`."""
    import torch

    sd = random_t5_state_dict(cfg, seed)
    g = torch.Generator().manual_seed(seed + 7919)
    D, F = cfg["d_model"], cfg["d_ff"]
    H, dk = cfg["num_heads"], cfg["d_kv"]
    inner = H * dk

    def normal(shape, std):
        return torch.randn(shape, generator=g, dtype=torch.float32) * std

    sd["decoder.embed_tokens.weight"] = sd["shared.weight"]
    sd["decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"] = normal(
        (cfg["relative_attention_num_buckets"], H), 0.5)
    for i in range(int(cfg.get("num_decoder_layers") or cfg["num_layers"])):
        for j, att in ((0, "SelfAttention"), (1, "EncDecAttention")):
            a = f"decoder.block.{i}.layer.{j}."
            sd[a + att + ".q.weight"] = normal((inner, D), (D * dk) ** -0.5)
            sd[a + att + ".k.weight"] = normal((inner, D), D ** -0.5)
            sd[a + att + ".v.weight"] = normal((inner, D), D ** -0.5)
            sd[a + att + ".o.weight"] = normal((D, inner), inner ** -0.5)
            sd[a + "layer_norm.weight"] = 1.0 + normal((D,), 0.1)
        f = f"decoder.block.{i}.layer.2."
        sd[f + "DenseReluDense.wi_0.weight"] = normal((F, D), D ** -0.5)
        sd[f + "DenseReluDense.wi_1.weight"] = normal((F, D), D ** -0.5)
        sd[f + "DenseReluDense.wo.weight"] = normal((D, F), F ** -0.5)
        sd[f + "layer_norm.weight"] = 1.0 + normal((D,), 0.1)
    sd["decoder.final_layer_norm.weight"] = 1.0 + normal((D,), 0.1)
    if cfg.get("tie_word_embeddings", True) is False:
        sd["lm_head.weight"] = normal((cfg["vocab_size"], D), D ** -0.5)
    return sd


def save_hf_checkpoint(path: str, cfg: Dict, state_dict: Dict) -> None:
    """Writes `config.json` + `model.safetensors` the way `save_pretrained` lays them out."""
    from safetensors.torch import save_file

    os.makedirs(path, exist_ok=True)
    hf_cfg = dict(cfg)
    arch = "T5ForConditionalGeneration" if "decoder.final_layer_norm.weight" in state_dict else "T5EncoderModel"
    hf_cfg.update(architectures=[arch], model_type="t5", is_encoder_decoder=True)
    with open(os.path.join(path, "config.json"), "w") as fh:
        json.dump(hf_cfg, fh, indent=1)
    tensors = {k: v.contiguous() for k, v in state_dict.items()
               if k not in ("encoder.embed_tokens.weight", "decoder.embed_tokens.weight")}
    save_file(tensors, os.path.join(path, "model.safetensors"), metadata={"format": "pt"})


def random_unit_rows(n: int, d: int, seed: int, device, dtype=None, chunk: int = 1 << 16):
    """[n, d] rows drawn N(0,1) then L2-normalised (a synthetic embedding index)."""
    import torch

    dtype = dtype or torch.bfloat16
    out = torch.empty(n, d, device=device, dtype=dtype)
    g = torch.Generator(device=device).manual_seed(seed)
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        x = torch.randn(hi - lo, d, generator=g, device=device, dtype=torch.float32)
        out[lo:hi] = torch.nn.functional.normalize(x, dim=1).to(dtype)
    return out


def write_leandojo_dataset(root: str, n_files: int = 8, premises_per_file: int = 40, theorems: Tuple[int, int, int] = (6, 3, 3),
                           tactics_per_theorem: Tuple[int, int] = (1, 4), state_len: Tuple[int, int] = (16, 400),
                           premise_len: Tuple[int, int] = (16, 300), min_accessible: int = 0, seed: int = SEED) -> str:
    """A seeded LeanDojo-layout dataset under `root`: `corpus.jsonl` and `random/{train,val,test}.json`; returns the
    split directory (`data_path`; the corpus is `<data_path>/../corpus.jsonl`).

    File i imports file i-1, so it sees every earlier file.  Premise j of a file spans lines 10j+1 .. 10j+5.
    `theorems` is the number of theorems per split, each in a file whose imports hold at least `min_accessible`
    premises, with `tactics_per_theorem` (inclusive range) traced tactics.  States and premise code are random
    printable ASCII (`synth_byte_strings`, lengths in the given inclusive ranges); states start with the turnstile.
    Every tactic's provenances name 0-3 premises its theorem can see, located at a position inside them, and about
    one tactic in four also names a position no premise covers (the reference skips it when collecting positives)."""
    rng = np.random.default_rng(seed)
    pdata, poff = synth_premises(n_files * premises_per_file, seed=seed + 1, min_len=premise_len[0],
                                 max_len=premise_len[1])
    bodies = [s.decode() for s in split_strings(pdata, poff)]
    os.makedirs(os.path.join(root, "random"), exist_ok=True)
    with open(os.path.join(root, "corpus.jsonl"), "w") as fh:
        for f in range(n_files):
            premises = [{"full_name": f"Synth.F{f}.p{j}", "code": f"theorem p{j} : {bodies[f * premises_per_file + j]}",
                         "start": [10 * j + 1, 1], "end": [10 * j + 5, 1], "kind": "theorem"}
                        for j in range(premises_per_file)]
            fh.write(json.dumps({"path": f"Synth/F{f}.lean", "imports": [f"Synth/F{f - 1}.lean"] if f else [],
                                 "premises": premises}) + "\n")
    first_file = min(n_files - 1, -(-min_accessible // premises_per_file))
    n_tac = rng.integers(tactics_per_theorem[0], tactics_per_theorem[1] + 1, size=sum(theorems))
    sdata, soff = synth_states(int(n_tac.sum()), seed=seed + 2, min_len=state_len[0], max_len=state_len[1])
    states = iter(s.decode() for s in split_strings(sdata, soff))
    t_all = 0
    for split, count in zip(("train", "val", "test"), theorems):
        thms = []
        for t in range(count):
            f = int(rng.integers(first_file, n_files))
            line = 10 * int(rng.integers(0, premises_per_file + 1)) + 3
            visible = f * premises_per_file + (line - 3) // 10     # imported files + own premises ending before line
            tactics = []
            for _ in range(int(n_tac[t_all])):
                prov = []
                for g in rng.choice(visible, size=min(visible, int(rng.integers(0, 4))), replace=False).tolist():
                    gf, gj = divmod(int(g), premises_per_file)
                    prov.append({"full_name": f"Synth.F{gf}.p{gj}", "def_path": f"Synth/F{gf}.lean",
                                 "def_pos": [10 * gj + 2, 1], "def_end_pos": [10 * gj + 5, 1]})
                if rng.random() < 0.25:
                    prov.append({"full_name": "Synth.missing", "def_path": f"Synth/F{f}.lean",
                                 "def_pos": [10 * premises_per_file + 50, 1], "def_end_pos": [10 * premises_per_file + 51, 1]})
                tactics.append({"tactic": "simp", "annotated_tactic": ["simp [<a>x</a>]", prov],
                                "state_before": next(states), "state_after": "no goals"})
            t_all += 1
            thms.append({"url": "https://example.org/synth", "commit": "0" * 40, "file_path": f"Synth/F{f}.lean",
                         "full_name": f"Synth.{split}{t}", "start": [line, 1], "end": [line + 8, 1],
                         "traced_tactics": tactics})
        with open(os.path.join(root, "random", f"{split}.json"), "w") as fh:
            json.dump(thms, fh)
    return os.path.join(root, "random")
