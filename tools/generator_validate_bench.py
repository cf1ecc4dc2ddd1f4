"""The tactic generator's dataset-level validation on the engine (`generator_eval.validate`, what the reference's
`generation/main.py validate` computes), and the shared prefill of `T5GeneratorEngine.evaluate` against `__call__` +
`generate` on the same batches.

The val set is synthetic and seeded in the LeanDojo layout (`synth.write_leandojo_dataset`): states of 200..2300
bytes, tactics of 8..160 printable bytes.  The checkpoint is the seeded 12 + 4 layer ByT5-small geometry with the EOS
row of `lm_head` set to zero, so no search ends early and every batch runs max_length - 1 decoder steps (as in
tools/generate_bench.py).  The reference's validation shape: eval_batch_size 64, max_inp_seq_len 2300,
max_oup_seq_len 512, num_beams 1; plus one run at num_beams 8.

For each num_beams it prints one JSON line:
  validate_examples_per_s  `validate` over the whole val set, host to host (tokenization, decoding and metrics
                           included), after one warm-up batch;
  evaluate_s / separate_s  per batch, `evaluate` and `__call__` + `generate`, alternated in one run (median of the
                           repeats of each batch, summed over batches); every output is checked equal bit for bit;
  card                     the GPU's name and power limit, read in the same run.

    python tools/generator_validate_bench.py [--examples 256] [--repeats 3] [--beam-examples 64]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from reprover_b200 import synth  # noqa: E402
from reprover_b200.generator import T5GeneratorEngine  # noqa: E402
from reprover_b200.generator_eval import collate, load_examples, validate  # noqa: E402
from tools.generator_bench import card  # noqa: E402

EOS = 1
BATCH, MAX_INP, MAX_OUP = 64, 2300, 512


def write_val_set(root: str, n_examples: int) -> str:
    """A LeanDojo-layout dataset whose val split holds about `n_examples` tactics, with random tactic strings."""
    n_thm = max(1, n_examples // 4)
    data = synth.write_leandojo_dataset(root, n_files=4, premises_per_file=10, theorems=(1, n_thm, 1),
                                        tactics_per_theorem=(4, 4), state_len=(200, 2300), seed=synth.SEED + 11)
    rng = np.random.default_rng(synth.SEED + 12)
    path = os.path.join(data, "val.json")
    with open(path) as fh:
        thms = json.load(fh)
    alphabet = [chr(c) for c in range(0x20, 0x7F) if c != 0x3C]
    for thm in thms:
        for tac in thm["traced_tactics"]:
            tac["tactic"] = "".join(rng.choice(alphabet, size=int(rng.integers(8, 161))).tolist())
    with open(path, "w") as fh:
        json.dump(thms, fh)
    return path


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def same(a, b) -> bool:
    if a is None or b is None:
        return a is None and b is None
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


def run_beams(gen, examples, nb: int, repeats: int):
    kw = dict(max_length=MAX_OUP, num_beams=nb, num_return_sequences=nb, do_sample=False, early_stopping=False,
              output_scores=True, return_dict_in_generate=True)
    batches = [collate(examples[lo:lo + BATCH], MAX_INP, MAX_OUP) for lo in range(0, len(examples), BATCH)]
    warm = collate(examples[:2], MAX_INP, MAX_OUP)
    gen.evaluate(warm["state_ids"], warm["state_mask"], warm["tactic_ids"], **dict(kw, max_length=8))
    t_val, metrics = timed(lambda: validate(gen, examples, batch_size=BATCH, num_beams=nb, max_inp_seq_len=MAX_INP,
                                            max_oup_seq_len=MAX_OUP))
    ev_s, sep_s, equal = 0.0, 0.0, True
    for b in batches:
        args = (b["state_ids"].cuda(), b["state_mask"].cuda())
        lab = b["tactic_ids"].cuda()
        ev, sep = [], []
        for _ in range(repeats):
            t, (loss_a, gen_a) = timed(lambda: gen.evaluate(*args, lab, **kw))
            ev.append(t)
            t, (loss_b, gen_b) = timed(lambda: (gen(*args, lab, return_logits=False), gen.generate(*args, **kw)))
            sep.append(t)
            equal &= all(same(x, y) for x, y in zip(loss_a, loss_b)) and all(same(x, y) for x, y in zip(gen_a, gen_b))
        ev_s += statistics.median(ev)
        sep_s += statistics.median(sep)
    return {"num_beams": nb, "examples": len(examples), "batches": len(batches), "eval_batch_size": BATCH,
            "max_inp_seq_len": MAX_INP, "max_oup_seq_len": MAX_OUP, "validate_s": t_val,
            "validate_examples_per_s": len(examples) / t_val, "evaluate_s": ev_s, "separate_s": sep_s,
            "prefill_saving": 1.0 - ev_s / sep_s, "outputs_equal": bool(equal), "repeats": repeats,
            "metrics": metrics}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--examples", type=int, default=256, help="val examples at num_beams 1")
    ap.add_argument("--beam-examples", type=int, default=64, help="val examples at num_beams 8")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("generator_validate_bench needs a CUDA device (H100); nothing is measured without one")
    cfg = dict(synth.BYT5_SMALL, decoder_start_token_id=0, eos_token_id=EOS, pad_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=synth.SEED)
    sd["lm_head.weight"][EOS] = 0.0
    gen = T5GeneratorEngine(cfg, sd, torch.device("cuda:0"))
    with tempfile.TemporaryDirectory() as tmp:
        examples = load_examples(write_val_set(os.path.join(tmp, "ds"), max(args.examples, args.beam_examples)))
    for nb, n in ((1, args.examples), (8, args.beam_examples)):
        r = run_beams(gen, examples[:n], nb, args.repeats)
        print(json.dumps({"card": card(), **r}), flush=True)
    gen.close()


if __name__ == "__main__":
    main()
