"""Dense-retriever predictions written by THIS package's CLI (`python -m reprover_b200.predict_cli predict`, reference
layout) read by the REFERENCE'S OWN evaluation script.

    python tests/golden/check_predict_with_reference.py [<reference checkout>]    # default /root/reference

Writes a small synthetic LeanDojo-layout dataset (`synth.write_leandojo_dataset`), runs the CLI's host side on it
with a seeded host ranking standing in for the GPU retriever (the examples, records, their classes and the pickle are
the CLI's own; only the encoder and the top-k are swapped, so this runs without a GPU), then imports
`retrieval/evaluate.py` unmodified (lean_dojo stubbed as in make_reference_retriever_golden.py) and lets its `main()`
load the pickle and compute R@1, R@10 and MRR for every split.  Prints one JSON line; exit code 0 = every check passed.
"""
import io
import json
import os
import pickle
import sys
import tempfile
from contextlib import redirect_stderr
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent.parent))

import make_reference_retriever_golden as gold  # noqa: E402


class _HostRetriever:
    """The attributes `predict_cli` touches; ranking by a seeded score over the accessible premises."""

    num_retrieved = 20

    def load_corpus(self, corpus):
        self.corpus = corpus


def _host_ranked_batches(retriever, examples, k, batch_size=64):
    import numpy as np

    corpus = retriever.corpus
    rng = np.random.default_rng(0)
    scores = rng.random(len(corpus))
    for lo in range(0, len(examples), batch_size):
        batch = examples[lo:lo + batch_size]
        premises, values = [], []
        for ex in batch:
            acc = corpus.get_accessible_premise_indexes(ex["context"].path, ex["context"].theorem_pos)
            best = sorted(acc, key=lambda i: (-scores[i], i))[:k]
            premises.append([corpus[i] for i in best])
            values.append([float(np.float32(scores[i])) for i in best])
        yield batch, premises, values


def main() -> int:
    ref_root = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    from reprover_b200 import evaluation, predict_cli, synth

    predict_cli._load_retriever = lambda args, settings: _HostRetriever()
    evaluation.ranked_batches = _host_ranked_batches
    checks = {}
    with tempfile.TemporaryDirectory() as tmp:
        data = synth.write_leandojo_dataset(tmp, min_accessible=20)
        out = Path(tmp) / "predictions.pickle"
        predict_cli.main(["predict", "--ckpt_path", "unused.ckpt", "--data.data_path", data, "--data.corpus_path",
                          os.path.join(data, "../corpus.jsonl"), "--output-path", str(out)])
        assert "common" not in sys.modules and "lean_dojo" not in sys.modules

        Pos = gold._stub_modules()
        sys.path.insert(0, ref_root)
        import common as refc
        from retrieval import evaluate

        with open(out, "rb") as fh:
            preds = pickle.load(fh)
        checks["contexts_are_reference_class"] = all(type(p["context"]) is refc.Context for p in preds)
        checks["premises_are_reference_class"] = all(type(q) is refc.Premise for p in preds
                                                     for q in p["retrieved_premises"] + p["all_pos_premises"])
        checks["positions_are_lean_dojo_pos"] = all(type(p["context"].theorem_pos) is Pos for p in preds)
        checks["context_serializes"] = all(p["context"].serialize() == p["context"].state for p in preds)
        checks["record_keys"] = all(list(p) == ["url", "commit", "file_path", "full_name", "start", "tactic_idx",
                                                "context", "all_pos_premises", "retrieved_premises", "scores"]
                                    for p in preds)
        log = io.StringIO()
        from loguru import logger

        logger.remove()
        logger.add(log, format="{message}")
        sys.argv = ["evaluate.py", "--preds-file", str(out), "--data-path", data]
        with redirect_stderr(io.StringIO()):
            evaluate.main()
        lines = [l for l in log.getvalue().splitlines() if l.startswith("R@1")]
        checks["evaluate_reports_every_split"] = len(lines) == 3
    ok = all(bool(v) for v in checks.values())
    print(json.dumps({"ok": ok, "checks": {k: bool(v) for k, v in checks.items()}, "metrics": lines}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
