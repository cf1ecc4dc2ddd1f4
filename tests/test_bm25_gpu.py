"""BM25 on the H100 against the float64 oracle (tests/bm25_ref.py): every score equal with `==`, every ranking
equal to the oracle's stable (score desc, index asc) ranking, on a corpus that spans ten 4096-premise tiles."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_DOCS = 40_000
VOCAB = 3000
EVERYWHERE = VOCAB - 1        # a term that occurs in every premise
NO_POSTINGS = VOCAB + 50      # inside the index's vocabulary, in no premise
OUT_OF_VOCAB = VOCAB + 500    # beyond it


def _zipf(rng, n, vocab):
    p = 1.0 / np.arange(1, vocab + 1) ** 1.1
    return rng.choice(vocab, size=n, p=p / p.sum())


@pytest.fixture(scope="module")
def setup(cuda_device):
    from reprover_b200.bm25 import BM25Index
    from tests.bm25_ref import BM25Okapi

    rng = np.random.default_rng(7)
    docs = []
    for _ in range(N_DOCS):
        d = _zipf(rng, int(rng.integers(0, 60)), VOCAB - 1).tolist()
        d.insert(int(rng.integers(0, len(d) + 1)), EVERYWHERE)
        docs.append(d)
    queries = {
        "one_token": [int(_zipf(rng, 1, 200)[0])],
        "everywhere": [EVERYWHERE, EVERYWHERE],
        "long": _zipf(rng, 2048, VOCAB).tolist(),
        "repeats": [3, 3, 17, 3, EVERYWHERE, 17],
        "unknown": [NO_POSTINGS, OUT_OF_VOCAB, NO_POSTINGS],
        "mixed_unknown": [5, OUT_OF_VOCAB, 40, NO_POSTINGS, 5],
    }
    for i in range(10):
        queries[f"rand{i}"] = _zipf(rng, int(rng.integers(1, 400)), VOCAB).tolist()
    index = BM25Index(docs, device=cuda_device, vocab_size=VOCAB + 100)
    oracle = BM25Okapi(docs)
    want = {name: np.asarray(oracle.get_batch_scores(q, range(N_DOCS))) for name, q in queries.items()}
    return index, oracle, queries, want


def test_dense_scores_equal_the_oracle_bit_for_bit(setup):
    index, oracle, queries, want = setup
    for name, q in queries.items():
        got = index.get_scores(q)
        assert got.dtype == np.float64 and got.shape == (N_DOCS,)
        assert np.all(got == want[name]), (name, int(np.sum(got != want[name])))
    assert not np.any(want["unknown"]) and np.all(want["everywhere"] > 0)
    sub = [5, 4099, 0, N_DOCS - 1, 8192]
    assert index.get_batch_scores(queries["long"], sub) == oracle.get_batch_scores(queries["long"], sub)


def _masks(rng):
    """Per-'theorem' accessibility rows: dense, sparse, a prefix, one with fewer premises than k, and an empty one."""
    bits = np.zeros((5, N_DOCS), dtype=bool)
    bits[0] = rng.random(N_DOCS) < 0.9
    bits[1] = rng.random(N_DOCS) < 0.05
    bits[2, : 20_000] = True
    bits[3, rng.choice(N_DOCS, 50, replace=False)] = True
    padded = np.zeros((5, (N_DOCS + 31) // 32 * 32), dtype=bool)
    padded[:, :N_DOCS] = bits
    words = np.packbits(padded.reshape(5, -1, 8), axis=2, bitorder="little").reshape(5, -1).view("<u4")
    return bits, words


@pytest.mark.parametrize("k", [1, 100, 1024])
def test_topk_equals_the_oracle_ranking(setup, k):
    from tests.bm25_ref import rank

    index, oracle, queries, want = setup
    bits, words = _masks(np.random.default_rng(11))
    names = list(queries)
    rows = [i % len(bits) for i in range(len(names))]
    idx, scores = index.topk_indexes([queries[n] for n in names], k, words, rows)
    for n, r, gi, gs in zip(names, rows, idx, scores):
        acc = np.flatnonzero(bits[r])
        wi, ws = rank(want[n][acc], acc, k)
        assert gi == wi, (n, r)
        assert gs == ws, (n, r)
        assert len(gi) == min(k, len(acc))
    idx, scores = index.topk_indexes([queries[n] for n in names], k)       # use_all_premises
    for n, gi, gs in zip(names, idx, scores):
        wi, ws = rank(want[n], np.arange(N_DOCS), k)
        assert gi == wi and gs == ws, n


def test_query_without_known_tokens_returns_first_accessible_indexes(setup):
    index, _, queries, _ = setup
    bits, words = _masks(np.random.default_rng(11))
    idx, scores = index.topk_indexes([queries["unknown"]] * 2, 300, words, [1, 3])
    assert idx[0] == np.flatnonzero(bits[1])[:300].tolist() and scores[0] == [0.0] * 300
    assert idx[1] == np.flatnonzero(bits[3]).tolist() and scores[1] == [0.0] * 50
    idx, scores = index.topk_indexes([queries["unknown"]], 10)
    assert idx[0] == list(range(10)) and scores[0] == [0.0] * 10


def test_batch_invariance(setup):
    index, _, queries, _ = setup
    bits, words = _masks(np.random.default_rng(11))
    alone = index.topk_indexes([queries["long"]], 100, words[:1], [0])
    names = list(queries)
    batch = index.topk_indexes([queries[n] for n in names], 100, words, [0] * len(names))
    assert batch[0][names.index("long")] == alone[0][0] and batch[1][names.index("long")] == alone[1][0]
    split = index.topk_indexes([queries[n] for n in names], 100, words, [0] * len(names), max_batch_tokens=300)
    assert split == batch


def test_cli_end_to_end_equals_the_oracle(tmp_path, cuda_device):
    import pickle

    from tokenizers import Tokenizer

    from reprover_b200 import bm25_cli
    from reprover_b200.bm25 import load_theorems
    from reprover_b200.corpus import Corpus
    from tests.bm25_data import write_dataset
    from tests.bm25_ref import BM25Okapi, process_theorem

    data, tok_path = write_dataset(tmp_path, seed=5, n_files=5, per_file=8)
    tok = Tokenizer.from_file(str(tok_path))
    corpus = Corpus(str(data / "../corpus.jsonl"))
    oracle = BM25Okapi([tok.encode(p.serialize()).tokens for p in corpus.all_premises])
    for use_all in (False, True):
        out = tmp_path / f"preds{int(use_all)}.pickle"
        bm25_cli.main(["--tokenizer-path", str(tok_path), "--data-path", str(data), "--output-path", str(out),
                       "--native-layout"] + (["--use-all-premises"] if use_all else []))
        with open(out, "rb") as fh:
            got = pickle.load(fh)
        want = [r for thm in load_theorems(str(data))
                for r in process_theorem(thm, corpus, lambda s: tok.encode(s).tokens, oracle, 100, use_all)]
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert g["retrieved_premises"] == w["retrieved_premises"]
            assert g["scores"] == w["scores"]
            assert all(type(s) is float for s in g["scores"])
            assert set(g["all_pos_premises"]) == set(w["all_pos_premises"])
            assert {k: g[k] for k in ("url", "commit", "file_path", "full_name", "start", "tactic_idx", "context")} == \
                {k: w[k] for k in ("url", "commit", "file_path", "full_name", "start", "tactic_idx", "context")}
