"""The REFERENCE'S OWN `HuggingFaceGenerator` (prover/tactic_generator.py) running on `T5GeneratorEngine` after the
one-line swap INTEGRATION.md documents:

    prover/tactic_generator.py:188
    - self.generator = AutoModelForSeq2SeqLM.from_pretrained(self.model_path)
    + self.generator = T5GeneratorEngine.from_hf_dir(self.model_path, self.device)

    python tests/golden/check_generate_with_reference.py [<reference checkout>]    # default /root/reference

Imports `prover/tactic_generator.py` unmodified (lean_dojo, pytorch_lightning, deepspeed stubbed as in
make_reference_retriever_golden.py; ray and openai as empty modules), makes the swap by giving the module's
`AutoModelForSeq2SeqLM` name a `from_pretrained` that builds the engine for the generator's device, and lets
`initialize()` (which then calls `.to(self.device).eval()` on the engine) and `generate(state, ...)` run as the prover
runs them, decoding `.sequences` with the reference's own tokenizer call.  It checks that generate returns
(tactic, score) pairs with distinct tactics and non-increasing scores, and compares them with the unmodified
reference's HF generator on the same synthetic checkpoint.

With a CUDA device the engine is the real one, and the scores are compared within 0.05 per token (bf16 against HF's
fp32; a near-tie that bf16 decides the other way fails the check and is worth a look).  Without one, the engine's
native search is stood in for by tests/beam_ref.py over HF's fp32 step log-probs and `.to()` returns the engine on any
device (everything else — settings, the output layout, the swap, `.eval()`, decoding — is the engine's own code), and
the pairs must equal the reference's within 1e-4.  Prints one JSON line; exit code 0 = every check passed.
"""
import asyncio
import json
import sys
import tempfile
import types
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent.parent))

import make_reference_retriever_golden as gold  # noqa: E402


def _host_engine_class():
    from reprover_b200.generator import GeneratorConfig, T5GeneratorEngine, generator_config
    from reprover_b200.engine import load_hf_checkpoint
    from tests import beam_ref

    class HostEngine(T5GeneratorEngine):
        """T5GeneratorEngine with its native search replaced by beam_ref over HF fp32 step log-probs."""

        def __init__(self, config, state_dict, device, generation_config=None):
            self.config = dict(config)
            self.generation_config = dict(generation_config or {})
            self.gen_config: GeneratorConfig = generator_config(config)
            self.vocab_size = int(config["vocab_size"])
            self.device = torch.device("cpu")
            self._hf = None

        @classmethod
        def from_hf_dir(cls, path, device, **kw):
            cfg, sd = load_hf_checkpoint(path)
            eng = cls(cfg, sd, device, **kw)
            eng._hf = cls_model(path)
            return eng

        def to(self, device=None, *a, **k):  # the real `to` accepts only the engine's GPU
            return self

        def close(self):
            pass

        def _search(self, ids, mask, s, trace_steps):
            nb = s.num_beams
            enc_ids, enc_mask = ids.repeat_interleave(nb, 0), (None if mask is None else mask.repeat_interleave(nb, 0))

            def step(t, prefixes):
                with torch.no_grad():
                    lg = self._hf(input_ids=enc_ids, attention_mask=enc_mask, decoder_input_ids=prefixes).logits[:, -1]
                return torch.log_softmax(lg.float(), -1) if nb > 1 else lg.float()

            if nb == 1:
                return beam_ref.greedy(step, ids.shape[0], s.max_length, s.eos_token_id, s.pad_token_id, 0), None, None
            seqs, scores = beam_ref.beam_search(step, ids.shape[0], nb, s.num_return_sequences, s.max_length,
                                                s.length_penalty, s.eos_token_id, s.pad_token_id,
                                                s.decoder_start_token_id)
            return seqs, scores, None

    def cls_model(path):
        from tests import seq2seq_ref

        return seq2seq_ref.hf_model_from_dir(path)

    return HostEngine


def main() -> int:
    ref_root = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    Pos = gold._stub_modules()
    for name in ("ray", "openai"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, ref_root)
    import prover.tactic_generator as tg  # the reference, unmodified
    from transformers import ByT5Tokenizer

    from reprover_b200 import synth

    torch.set_float32_matmul_precision("highest")
    on_gpu = torch.cuda.is_available()
    if on_gpu:
        from reprover_b200.generator import T5GeneratorEngine as Engine
    else:
        Engine = _host_engine_class()
    cfg = dict(synth.tiny_config(2), num_decoder_layers=2, decoder_start_token_id=0, eos_token_id=1, pad_token_id=0)
    sd = synth.random_t5_seq2seq_state_dict(cfg, seed=synth.SEED)
    state = "n : ℕ\n⊢ gcd n n = n"
    num_samples, max_len = 4, 24
    checks = {}
    with tempfile.TemporaryDirectory() as tmp:
        synth.save_hf_checkpoint(tmp, cfg, sd)
        ByT5Tokenizer().save_pretrained(tmp)
        device = "cuda" if on_gpu else "cpu"

        def run(swapped):
            g = tg.HuggingFaceGenerator(tmp, device, max_inp_seq_len=2300, max_oup_seq_len=max_len,
                                        length_penalty=0.0)
            original = tg.AutoModelForSeq2SeqLM
            if swapped:
                tg.AutoModelForSeq2SeqLM = types.SimpleNamespace(
                    from_pretrained=lambda path: Engine.from_hf_dir(path, g.device))
            try:
                g.initialize()
                pairs = asyncio.run(g.generate(state, "Foo.lean", "foo", Pos(1, 0), num_samples))
            finally:
                tg.AutoModelForSeq2SeqLM = original
            return g, pairs

        g_eng, eng_pairs = run(True)
        _, ref_pairs = run(False)
        checks["engine_is_the_generator"] = isinstance(g_eng.generator, Engine)
        checks["pairs"] = bool(eng_pairs) and all(isinstance(t, str) and isinstance(s, float) for t, s in eng_pairs)
        checks["distinct_tactics"] = len({t for t, _ in eng_pairs}) == len(eng_pairs)
        checks["scores_non_increasing"] = all(a[1] >= b[1] for a, b in zip(eng_pairs, eng_pairs[1:]))
        tol = 0.05 * max_len if on_gpu else 1e-4
        same_tactics = [t for t, _ in eng_pairs] == [t for t, _ in ref_pairs]
        checks["matches_reference"] = same_tactics and all(abs(a[1] - b[1]) <= tol for a, b in zip(eng_pairs, ref_pairs))
        g_eng.generator.close()
    ok = all(bool(v) for v in checks.values())
    print(json.dumps({"ok": ok, "engine": "cuda" if on_gpu else "host search stand-in", "checks": checks,
                      "engine_pairs": eng_pairs, "reference_pairs": ref_pairs}, ensure_ascii=False))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
