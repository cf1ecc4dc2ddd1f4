"""Throughput of the tactic generator's teacher-forced forward (`T5GeneratorEngine`, rpx_seq2seq_forward) at the
generator's validation shape, against HF `T5ForConditionalGeneration` in bf16 on the same GPU.

Shape (generation/confs/cli_lean4_random.yaml): eval_batch_size 64, states of up to max_inp_seq_len = 2300 bytes,
tactics of up to 512, the full 12 + 4 layer ByT5-small geometry; weights and lengths seeded and synthetic.
Prints one JSON line: decoder tokens/s and examples/s of both, the losses, the card and its power limit.

    python tools/generator_bench.py [--steps 5] [--warmup 2] [--batch 64] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from reprover_b200 import synth  # noqa: E402
from reprover_b200.generator import T5GeneratorEngine  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # no nvidia-smi
        return f"unknown ({exc})"


def batch(cfg, B, seed):
    g = torch.Generator().manual_seed(seed)
    in_lens = torch.randint(200, 2301, (B,), generator=g)
    out_lens = torch.randint(16, 513, (B,), generator=g)
    L_in, L_out = int(in_lens.max()), int(out_lens.max())
    ids = torch.randint(3, cfg["vocab_size"], (B, L_in), generator=g)
    mask = (torch.arange(L_in)[None, :] < in_lens[:, None]).long()
    ids = ids * mask
    labels = torch.randint(3, cfg["vocab_size"], (B, L_out), generator=g)
    labels = torch.where(torch.arange(L_out)[None, :] < out_lens[:, None], labels, torch.full_like(labels, -100))
    return ids.cuda(), mask.cuda(), labels.cuda()


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps, out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--no-hf", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("generator_bench needs a CUDA device (H100); nothing is measured without one")
    cfg = dict(synth.BYT5_SMALL, decoder_start_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=synth.SEED)
    ids, mask, labels = batch(cfg, args.batch, synth.SEED)
    n_dec = int((labels != -100).sum())
    res = {"card": card(), "batch": args.batch, "max_in": int(mask.sum(1).max()), "decoder_tokens": n_dec}
    with tempfile.TemporaryDirectory() as tmp:
        synth.save_hf_checkpoint(tmp, cfg, sd)
        gen = T5GeneratorEngine.from_hf_dir(tmp, torch.device("cuda:0"))
        t, out = timed(lambda: gen(input_ids=ids, attention_mask=mask, labels=labels, return_logits=False),
                       args.steps, args.warmup)
        res.update(engine_s=t, engine_dec_tokens_per_s=n_dec / t, engine_examples_per_s=args.batch / t,
                   engine_loss=float(out.loss))
        gen.close()
        del gen
        torch.cuda.empty_cache()
        if not args.no_hf:
            from transformers import T5ForConditionalGeneration

            m = T5ForConditionalGeneration.from_pretrained(tmp, dtype=torch.bfloat16).cuda().eval()
            with torch.no_grad():
                t, o = timed(lambda: m(input_ids=ids, attention_mask=mask, labels=labels), args.steps, args.warmup)
            res.update(hf_bf16_s=t, hf_bf16_dec_tokens_per_s=n_dec / t, hf_bf16_examples_per_s=args.batch / t,
                       hf_bf16_loss=float(o.loss), speedup=res["engine_s"] and t / res["engine_s"])
            res["loss_abs_diff"] = abs(res["engine_loss"] - res["hf_bf16_loss"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
