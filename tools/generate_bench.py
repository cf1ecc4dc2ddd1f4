"""Tactic generation on the engine (`T5GeneratorEngine.generate`, rpx_seq2seq_generate) against HF
`T5ForConditionalGeneration.generate` in bf16 on the same GPU, at the reference's two call shapes:

  prover      one 2300-byte state, num_beams = num_return_sequences = 64, max_length 512, length_penalty 0.0
              (prover/tactic_generator.py `HuggingFaceGenerator.generate` with prover/evaluate.py's defaults)
  validation  64 states of up to 2300 bytes, greedy (num_beams 1), max_length 512 (generation/model.py
              `validation_step`)

The checkpoint is the seeded synthetic 12 + 4 layer ByT5-small geometry.  Its random head would end searches at
arbitrary points, so both arms run with the EOS row of `lm_head` set to zero: its logit is then 0 against 383 random
logits of either sign, so EOS never reaches the top candidates and every search runs to max_length in both arms.  The
script counts HF's decoder calls (a forward hook) and the engine's steps and prints both.

Prints one JSON line per workload: steps, time per step, total time of each arm, the card and its power limit, and
the per-step byte floor from shapes (decoder weights, the head, the cross K / V and the self K / V read at the mean
step).

    python tools/generate_bench.py [--repeats 2] [--no-hf]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from reprover_b200 import synth  # noqa: E402
from reprover_b200.generator import T5GeneratorEngine  # noqa: E402
from tools.generator_bench import card  # noqa: E402

EOS = 1


def states(cfg, n, seed, fixed=None):
    g = torch.Generator().manual_seed(seed)
    lens = [fixed] * n if fixed else torch.randint(200, 2301, (n,), generator=g).tolist()
    L = max(lens)
    ids = torch.randint(3, cfg["vocab_size"], (n, L), generator=g)
    mask = (torch.arange(L)[None, :] < torch.tensor(lens)[:, None]).long()
    ids = ids * mask
    for i, k in enumerate(lens):
        ids[i, k - 1] = EOS
    return ids.cuda(), mask.cuda(), lens


def byte_floor(cfg, n_states, enc_tokens, R, steps):
    """Bytes one decoder step must read at least, from shapes: bf16 decoder weights, the head, the cross K / V of
    every state, and the self K / V of all rows at the mean step."""
    D, F, inner, L, V = cfg["d_model"], cfg["d_ff"], cfg["num_heads"] * cfg["d_kv"], cfg["num_decoder_layers"], \
        cfg["vocab_size"]
    per_layer = (3 * inner * D + inner * D + inner * D + inner * D + 2 * F * D + F * D) * 2
    weights = L * per_layer
    head = V * D * 2
    cross = enc_tokens * L * 2 * inner * 2
    mean_t = (steps - 1) / 2
    self_kv = R * (mean_t + 1) * L * 2 * inner * 2
    return {"weights_B": weights, "head_B": head, "cross_kv_B": cross, "self_kv_mean_step_B": int(self_kv),
            "floor_mean_step_B": int(weights + head + cross + self_kv)}


def run(fn, repeats):
    best, out = None, None
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--max-length", type=int, default=512)
    ap.add_argument("--no-hf", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("generate_bench needs a CUDA device (H100); nothing is measured without one")
    cfg = dict(synth.BYT5_SMALL, decoder_start_token_id=0, eos_token_id=EOS, pad_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=synth.SEED)
    head = sd["lm_head.weight"]
    head[EOS] = 0.0
    workloads = {"prover": dict(n=1, fixed=2300, num_beams=64, num_return_sequences=64, length_penalty=0.0),
                 "validation": dict(n=64, fixed=None, num_beams=1, num_return_sequences=1, length_penalty=1.0)}
    ML = args.max_length
    with tempfile.TemporaryDirectory() as tmp:
        synth.save_hf_checkpoint(tmp, cfg, sd)
        gen = T5GeneratorEngine.from_hf_dir(tmp, torch.device("cuda:0"))
        results = {}
        for name, w in workloads.items():
            ids, mask, lens = states(cfg, w["n"], synth.SEED + 7, w["fixed"])
            kw = dict(num_beams=w["num_beams"], num_return_sequences=w["num_return_sequences"], max_length=ML,
                      length_penalty=w["length_penalty"], output_scores=True, return_dict_in_generate=True)
            gen.generate(ids, mask, **dict(kw, max_length=8))  # warm-up: modules, workspace
            t, (out, trace) = run(lambda: gen.generate(ids, mask, _trace_steps=1, **kw), args.repeats)
            steps = trace["steps"]
            R = w["n"] * w["num_beams"]
            results[name] = {"workload": name, "card": card(), "states": w["n"], "num_beams": w["num_beams"],
                             "max_length": ML, "engine_steps": steps, "engine_s": t, "engine_ms_per_step": 1e3 * t / steps,
                             "engine_out_len": int(out.sequences.shape[1]),
                             **byte_floor(cfg, w["n"], sum(lens), R, steps)}
        gen.close()
        del gen
        torch.cuda.empty_cache()
        if not args.no_hf:
            from transformers import T5ForConditionalGeneration

            m = T5ForConditionalGeneration.from_pretrained(tmp, dtype=torch.bfloat16).cuda().eval()
            calls = [0]
            m.decoder.register_forward_hook(lambda *a: calls.__setitem__(0, calls[0] + 1))
            for name, w in workloads.items():
                ids, mask, _ = states(cfg, w["n"], synth.SEED + 7, w["fixed"])
                kw = dict(num_beams=w["num_beams"], num_return_sequences=w["num_return_sequences"], max_length=ML,
                          length_penalty=w["length_penalty"], do_sample=False, early_stopping=False,
                          output_scores=True, return_dict_in_generate=True)
                with torch.no_grad():
                    m.generate(input_ids=ids, attention_mask=mask, **dict(kw, max_length=8))
                    calls[0] = 0
                    t, out = run(lambda: m.generate(input_ids=ids, attention_mask=mask, **kw), args.repeats)
                steps = calls[0] // args.repeats
                r = results[name]
                r.update(hf_bf16_steps=steps, hf_bf16_s=t, hf_bf16_ms_per_step=1e3 * t / steps,
                         hf_bf16_out_len=int(out.sequences.shape[1]), speedup=t / r["engine_s"])
    for r in results.values():
        print(json.dumps(r))


if __name__ == "__main__":
    main()
