"""BM25 predictions written by THIS package's CLI (`python -m reprover_b200.bm25_cli`, reference layout) read by
the REFERENCE'S OWN evaluation script.

    python tests/golden/check_bm25_with_reference.py [<reference checkout>]    # default /root/reference

Writes the tiny LeanDojo-layout dataset of the BM25 tests, runs the CLI's host side on it with the float64 oracle
standing in for the GPU index (the records, their classes and the pickle are the CLI's own; only the scoring is
swapped, so this runs without a GPU), then imports `retrieval/evaluate.py` unmodified (lean_dojo stubbed as in
make_reference_retriever_golden.py) and lets its `main()` load the pickle and compute R@1, R@10 and MRR for every split.
Prints one JSON line; exit code 0 = every check passed.
"""
import io
import json
import pickle
import sys
import tempfile
from contextlib import redirect_stderr
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent.parent))

import make_reference_retriever_golden as gold  # noqa: E402


def main() -> int:
    ref_root = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    from reprover_b200 import bm25_cli
    from tests.bm25_data import write_dataset
    from tests.test_bm25_cpu import _OracleIndex

    bm25_cli.BM25Index.from_corpus = classmethod(lambda cls, c, t, device=None: _OracleIndex(c, t))
    checks = {}
    with tempfile.TemporaryDirectory() as tmp:
        data, tok_path = write_dataset(Path(tmp))
        out = Path(tmp) / "bm25_predictions.pickle"
        bm25_cli.main(["--tokenizer-path", str(tok_path), "--data-path", str(data), "--output-path", str(out)])
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
        log = io.StringIO()
        from loguru import logger

        logger.remove()
        logger.add(log, format="{message}")
        sys.argv = ["evaluate.py", "--preds-file", str(out), "--data-path", str(data)]
        with redirect_stderr(io.StringIO()):
            evaluate.main()
        lines = [l for l in log.getvalue().splitlines() if l.startswith("R@1")]
        checks["evaluate_reports_every_split"] = len(lines) == 3
    ok = all(bool(v) for v in checks.values())
    print(json.dumps({"ok": ok, "checks": {k: bool(v) for k, v in checks.items()}, "metrics": lines}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
