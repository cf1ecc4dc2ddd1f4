"""A tiny LeanDojo-layout dataset for the BM25 tests: `corpus.jsonl` next to a split directory holding
`train.json`, `val.json` and `test.json`, and a BPE tokenizer trained on it offline the way the reference's
`retrieval/bm25/train_tokenizer.py` trains one (Whitespace pre-tokenizer, the same special tokens)."""
from __future__ import annotations

import json
import random
from pathlib import Path
from typing import Tuple

WORDS = ["Nat", "add", "mul", "comm", "assoc", "zero", "succ", "le", "lt", "List", "map", "foldl", "length", "rfl",
         "simp", "Eq", "trans", "symm", "Function", "comp", "id", "Prod", "fst", "snd", "Option", "some", "none",
         "Finset", "sum", "card", "Real", "sqrt", "abs", "pow", "two", "Int", "neg", "sub", "div", "mod"]


def _code(rng: random.Random, name: str) -> str:
    body = " ".join(rng.choice(WORDS) for _ in range(rng.randint(2, 14)))
    return f"theorem {name} (a b : Nat) : {body} := by simp"


def write_dataset(root: Path, seed: int = 0, n_files: int = 4, per_file: int = 6) -> Tuple[Path, Path]:
    """Writes the dataset under `root`; returns (data path, tokenizer path)."""
    from tokenizers import Tokenizer
    from tokenizers.models import BPE
    from tokenizers.pre_tokenizers import Whitespace
    from tokenizers.trainers import BpeTrainer

    rng = random.Random(seed)
    lines, names = [], []
    for f in range(n_files):
        path = f"Toy/F{f}.lean"
        premises = []
        for j in range(per_file):
            name = f"Toy.F{f}.thm{j}"
            line = 10 * j + 1
            premises.append({"full_name": name, "code": _code(rng, name), "start": [line, 1], "end": [line + 5, 20],
                             "kind": "theorem"})
            names.append((path, name, line))
        lines.append({"path": path, "imports": [f"Toy/F{i}.lean" for i in range(f)], "premises": premises})
    root.mkdir(parents=True, exist_ok=True)
    (root / "corpus.jsonl").write_text("\n".join(json.dumps(l) for l in lines) + "\n")
    data = root / "random"
    data.mkdir(exist_ok=True)
    states = []
    for split, n_thm in (("train", 3), ("val", 2), ("test", 2)):
        thms = []
        for t in range(n_thm):
            f = rng.randrange(n_files)
            tactics = []
            for i in range(rng.randint(1, 3)):
                used = rng.sample(names, 2)
                prov = [{"full_name": nm, "def_path": p, "def_pos": [ln + 1, 1], "def_end_pos": [ln + 5, 20]}
                        for p, nm, ln in used]
                prov.append({"full_name": "Missing.x", "def_path": "Toy/F0.lean", "def_pos": [999, 1],
                             "def_end_pos": [999, 2]})   # not locatable: left out of all_pos_premises
                state = "a b : Nat\n⊢ " + " ".join(rng.choice(WORDS) for _ in range(rng.randint(0, 12)))
                if i == 0 and t == 0 and split == "val":
                    state = "⊢ zzz qqq"   # only tokens no premise contains
                states.append(state)
                tactics.append({"tactic": "simp", "annotated_tactic": ["simp [<a>x</a>]", prov],
                                "state_before": state, "state_after": "no goals"})
            thms.append({"url": "https://example.org/toy", "commit": "0" * 40, "file_path": f"Toy/F{f}.lean",
                         "full_name": f"Toy.{split}{t}", "start": [10 * rng.randrange(per_file) + 3, 1],
                         "end": [200, 1], "traced_tactics": tactics})
        (data / f"{split}.json").write_text(json.dumps(thms))
    tok = Tokenizer(BPE(unk_token="[UNK]"))
    tok.pre_tokenizer = Whitespace()
    trainer = BpeTrainer(vocab_size=300, special_tokens=["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"],
                         show_progress=False)
    codes = [p["code"] for l in lines for p in l["premises"]]
    tok.train_from_iterator(codes + states, trainer=trainer)
    tok_path = root / "tokenizer.json"
    tok.save(str(tok_path))
    return data, tok_path
