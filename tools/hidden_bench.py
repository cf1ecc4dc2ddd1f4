"""Device-side timing (CUDA events) of the encoder's per-token output, `engine(ids, mask)` (rpx_encode_ids_hidden),
against the pooled embedding of the same batch (`encode_ids`) and against HF `T5EncoderModel` in bf16 on the same
GPU, on a synthetic ByT5-small checkpoint.  Rows are right-padded: the longest row of a batch is L tokens, the
others are uniform in [L/2, L].  `store_ms` is the final-norm store alone (profiling class 6 of the hidden call,
`pool` of the pooled one), `store_bytes` what it has to move: T D 4 + T P 4 read, B L D 2 written (bf16 output).

    python tools/hidden_bench.py [--shapes 1x256,64x512,64x2048] [--reps R] [--warmup W] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from reprover_b200 import synth  # noqa: E402
from reprover_b200.engine import T5EncoderEngine  # noqa: E402


def board():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True)
        name, power = (s.strip() for s in out.stdout.strip().split(","))
        return {"name": name, "power_limit_w": float(power)}
    except (OSError, subprocess.CalledProcessError, ValueError):
        return {"name": torch.cuda.get_device_name(), "power_limit_w": None}


def hf_encoder(cfg, sd, dev):
    """HF `T5EncoderModel` holding the synthetic weights, bf16 on the GPU (the reference's model after load_hf)."""
    from transformers import T5Config, T5EncoderModel

    keys = ("vocab_size", "d_model", "d_kv", "d_ff", "num_layers", "num_heads", "relative_attention_num_buckets",
            "relative_attention_max_distance", "layer_norm_epsilon", "feed_forward_proj")
    model = T5EncoderModel(T5Config(**{k: cfg[k] for k in keys}, dropout_rate=0.0))
    weights = dict(sd)
    weights.setdefault("encoder.embed_tokens.weight", weights["shared.weight"])
    model.load_state_dict(weights, strict=False)
    return model.to(dev, torch.bfloat16).eval()


def batch(B, L, vocab_lo, vocab_hi, dev, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    lens[0] = L
    ids = torch.randint(vocab_lo, vocab_hi, (B, L), generator=g)
    mask = (torch.arange(L)[None, :] < lens[:, None]).long()
    return (ids * mask).to(dev), mask.to(dev), int(lens.sum())


def time_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def store_ms(eng, fn, reps):
    eng.set_profiling(True)
    eng.read_profile()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    prof = eng.read_profile()["pool"]
    eng.set_profiling(False)
    return prof["ms"] / max(prof["launches"], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1x256,64x512,64x2048")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    cfg = dict(synth.BYT5_SMALL)
    sd = synth.random_t5_state_dict(cfg, seed=synth.SEED)
    eng = T5EncoderEngine(cfg, sd, dev)
    hf = hf_encoder(cfg, sd, dev)
    D, P = cfg["d_model"], -(-cfg["d_model"] // 128)
    rows = []
    for i, shape in enumerate(args.shapes.split(",")):
        B, L = (int(x) for x in shape.split("x"))
        ids, mask, T = batch(B, L, 3, 259, dev, seed=i)

        def hidden():
            return eng(ids, mask)

        def pooled():
            return eng.encode_ids(ids, mask)

        def reference():
            with torch.no_grad():
                return hf(input_ids=ids, attention_mask=mask).last_hidden_state

        row = {"batch": B, "seq_len": L, "tokens": T,
               "hidden_ms": time_ms(hidden, args.reps, args.warmup),
               "encode_ids_ms": time_ms(pooled, args.reps, args.warmup),
               "hf_bf16_ms": time_ms(reference, max(args.reps // 4, 2), 1),
               "store_ms": store_ms(eng, hidden, args.reps),
               "pool_ms": store_ms(eng, pooled, args.reps),
               "store_bytes": T * D * 4 + T * P * 4 + B * L * D * 2}
        row["store_tb_per_s"] = row["store_bytes"] / (row["store_ms"] * 1e-3) / 1e12
        row["speedup_vs_hf"] = row["hf_bf16_ms"] / row["hidden_ms"]
        rows.append(row)
        torch.cuda.empty_cache()
    result = {"board": board(), "checkpoint": "synthetic ByT5-small (12 layers, d_model 1472)", "shapes": rows}
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
