"""BM25 without a GPU: the float64 oracle and the host-side index construction on hand-computed cases, the
prediction records and pickle layout of the CLI, and the C ABI's argument checks."""
import ctypes as C
import math
import pickle

import numpy as np
import pytest
import torch

from reprover_b200 import _native
from reprover_b200.bm25 import okapi_postings

needs_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")

# a: in every document; b, c, d, e: in one each.  N = 3, avgdl = 8 / 3
THREE = [["a", "b", "a"], ["a", "c"], ["a", "d", "e"]]
IDS = {w: i for i, w in enumerate("abcde")}
IDF_RARE = 0.5108256237659907       # log(3 - 1 + 0.5) - log(1 + 0.5)
IDF_A_RAW = -1.9459101490553135     # log(3 - 3 + 0.5) - log(3 + 0.5) < 0
AVERAGE_IDF = 0.019478469201729888  # (IDF_A_RAW + 4 IDF_RARE) / 5
IDF_A = 0.004869617300432472        # negative idf floored to 0.25 * AVERAGE_IDF
C_B_D0 = 0.4836218923228314         # IDF_RARE * (1 * 2.5 / (1 + 1.5 * (0.25 + 0.75 * 3 / (8 / 3))))
C_A_D0 = 0.006687886421194811       # IDF_A * (2 * 2.5 / (2 + 1.5 * (0.25 + 0.75 * 3 / (8 / 3))))
C_A_D1 = 0.005486892732881659       # IDF_A * (1 * 2.5 / (1 + 1.5 * (0.25 + 0.75 * 2 / (8 / 3))))


def test_three_documents_idf_by_hand():
    from tests.bm25_ref import BM25Okapi

    bm = BM25Okapi(THREE)
    assert bm.avgdl == 8 / 3 and bm.doc_len == [3, 2, 3]
    assert bm.average_idf == pytest.approx(AVERAGE_IDF, rel=1e-14)
    assert bm.idf["a"] == pytest.approx(IDF_A, rel=1e-14) and IDF_A == pytest.approx(0.25 * AVERAGE_IDF, rel=1e-14)
    assert IDF_A_RAW < 0
    for w in "bcde":
        assert bm.idf[w] == pytest.approx(IDF_RARE, rel=1e-15)
    st = okapi_postings([[IDS[w] for w in d] for d in THREE])
    assert st.avgdl == bm.avgdl and st.doc_len == bm.doc_len and st.average_idf == bm.average_idf
    assert {w: st.idf[IDS[w]] for w in "abcde"} == bm.idf
    assert st.term_ptr.tolist() == [0, 3, 4, 5, 6, 7]
    assert st.post_doc.tolist() == [0, 1, 2, 0, 1, 2, 2]
    scores = bm.get_batch_scores(["b"], [0, 1, 2])
    assert scores[0] == pytest.approx(C_B_D0, rel=1e-14) and scores[1:] == [0.0, 0.0]
    assert bm.get_batch_scores(["a"], [0, 1])[0] == pytest.approx(C_A_D0, rel=1e-14)
    assert bm.get_batch_scores(["a"], [1])[0] == pytest.approx(C_A_D1, rel=1e-14)


def test_repeated_query_token_counts_twice():
    from tests.bm25_ref import BM25Okapi

    bm = BM25Okapi(THREE)
    once = bm.get_batch_scores(["b"], [0, 1, 2])
    twice = bm.get_batch_scores(["b", "a", "b"], [0, 1, 2])
    c_b, c_a = bm.contribution("b", 0), bm.contribution("a", 0)
    assert c_b == once[0]
    assert twice[0] == (c_b + c_a) + c_b          # query order, fp64
    assert twice[0] == pytest.approx(2 * C_B_D0 + C_A_D0, rel=1e-14)
    assert twice[1] == bm.contribution("a", 1)


def test_unknown_token_adds_nothing():
    from tests.bm25_ref import BM25Okapi

    bm = BM25Okapi(THREE)
    assert bm.get_batch_scores(["zzz"], [0, 1, 2]) == [0.0, 0.0, 0.0]
    assert bm.get_batch_scores(["zzz", "b", "zzz"], [0, 1, 2]) == bm.get_batch_scores(["b"], [0, 1, 2])


def _zipf_corpus(seed, n_docs, vocab, lo, hi):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, vocab + 1)
    p /= p.sum()
    return [rng.choice(vocab, size=int(rng.integers(lo, hi + 1)), p=p).tolist() for _ in range(n_docs)]


def test_post_c_is_bit_identical_to_the_oracle():
    from tests.bm25_ref import BM25Okapi

    docs = _zipf_corpus(3, 400, 120, 0, 40)   # empty documents included
    bm = BM25Okapi(docs)
    st = okapi_postings(docs, vocab_size=130)
    assert st.vocab_size == 130 and st.term_ptr[-1] == st.nnz == sum(len(set(d)) for d in docs)
    assert list(st.idf) == list(bm.idf) and st.idf == bm.idf            # values and _calc_idf's order
    assert any(v < 0 for v in st.idf.values()) or st.average_idf > 0
    for t in range(st.vocab_size):
        a, b = st.term_ptr[t], st.term_ptr[t + 1]
        docs_t = st.post_doc[a:b]
        assert np.all(np.diff(docs_t) > 0)
        want = [bm.contribution(t, int(d)) for d in docs_t]
        assert st.post_c[a:b].tolist() == want, t
    # a query's score is the plain query-order sum of the postings' contributions
    query = [5, 0, 0, 117, 129, 3, 0]
    got = np.zeros(len(docs))
    for t in query:
        if t < st.vocab_size:
            a, b = st.term_ptr[t], st.term_ptr[t + 1]
            got[st.post_doc[a:b]] += st.post_c[a:b]
    assert got.tolist() == bm.get_batch_scores(query, range(len(docs)))


def test_oracle_ranking_orders_ties_by_index():
    from tests.bm25_ref import rank

    idx, sc = rank([0.0, 2.0, 0.0, 2.0, 1.0], [7, 3, 5, 9, 1], 4)
    assert idx == [3, 9, 1, 5] and sc == [2.0, 2.0, 1.0, 0.0]
    assert rank([1.0], [4], 10) == ([4], [1.0])


def test_index_mask_is_get_accessible_premise_indexes(tmp_path):
    from tests.bm25_data import write_dataset

    from reprover_b200.bm25 import load_theorems
    from reprover_b200.corpus import Corpus

    data, _ = write_dataset(tmp_path)
    corpus = Corpus(str(data / "../corpus.jsonl"))
    for thm in load_theorems(str(data)):
        words = corpus.accessible_index_mask_words(thm["file_path"], thm["start"])
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")[: len(corpus)]
        assert np.flatnonzero(bits).tolist() == corpus.get_accessible_premise_indexes(thm["file_path"], thm["start"])


class _OracleIndex:
    """Stands in for BM25Index (which needs a GPU) with the float64 oracle, to exercise the CLI's host side."""

    def __init__(self, corpus, tokenizer):
        from tests.bm25_ref import BM25Okapi

        self.corpus, self.tokenizer = corpus, tokenizer
        self.bm25 = BM25Okapi([tokenizer.encode(p.serialize()).tokens for p in corpus.all_premises])

    def encode_queries(self, texts):
        return [self.tokenizer.encode(t).tokens for t in texts]

    def topk(self, queries, k, contexts=None, use_all_premises=False):
        from tests.bm25_ref import rank

        prem, scores = [], []
        for i, q in enumerate(queries):
            acc = (range(len(self.corpus)) if use_all_premises else
                   self.corpus.get_accessible_premise_indexes(contexts[i].path, contexts[i].theorem_pos))
            idx, sc = rank(self.bm25.get_batch_scores(q, acc), acc, k)
            prem.append([self.corpus[j] for j in idx])
            scores.append(sc)
        return prem, scores


class _Recorder(pickle.Unpickler):
    def find_class(self, module, name):
        self.seen = getattr(self, "seen", set()) | {(module, name)}
        if module in ("common", "lean_dojo"):
            return type(name, (), {"__setstate__": lambda self, st: self.__dict__.update(st)})
        return super().find_class(module, name)


def _as_plain(p):
    return (p.path, p.full_name, (p.start.line_nb, p.start.column_nb))


@pytest.mark.parametrize("use_all", [False, True])
def test_cli_records_and_reference_layout(tmp_path, monkeypatch, use_all):
    from tests.bm25_data import write_dataset
    from tests.bm25_ref import process_theorem
    from tokenizers import Tokenizer

    from reprover_b200 import bm25_cli
    from reprover_b200.bm25 import load_theorems
    from reprover_b200.corpus import Corpus

    data, tok_path = write_dataset(tmp_path)
    monkeypatch.setattr(bm25_cli.BM25Index, "from_corpus", classmethod(lambda cls, c, t, device=None: _OracleIndex(c, t)))
    out = tmp_path / "preds.pickle"
    argv = ["--tokenizer-path", str(tok_path), "--data-path", str(data), "--output-path", str(out),
            "--num-retrieved", "5", "--num-cpus", "8"] + (["--use-all-premises"] if use_all else [])
    bm25_cli.main(argv)
    with open(out, "rb") as fh:
        rec = _Recorder(fh)
        got = rec.load()
    assert {("common", "Context"), ("common", "Premise"), ("lean_dojo", "Pos")} <= rec.seen
    theorems = load_theorems(str(data))
    tok = Tokenizer.from_file(str(tok_path))
    corpus = Corpus(str(data / "../corpus.jsonl"))
    oracle = _OracleIndex(corpus, tok)
    want = [r for thm in theorems
            for r in process_theorem(thm, corpus, lambda s: tok.encode(s).tokens, oracle.bm25, 5, use_all)]
    assert len(got) == len(want) == sum(len(t["traced_tactics"]) for t in theorems)
    keys = {"url", "commit", "file_path", "full_name", "start", "tactic_idx", "context", "all_pos_premises",
            "retrieved_premises", "scores"}
    for g, w in zip(got, want):
        assert set(g) == keys
        for k in ("url", "commit", "file_path", "full_name", "start", "tactic_idx", "scores"):
            assert g[k] == w[k], k
        assert all(type(s) is float for s in g["scores"])
        assert len(g["retrieved_premises"]) == len(g["scores"]) <= 5
        assert (g["context"].path, g["context"].theorem_full_name, g["context"].state) == \
            (w["context"].path, w["context"].theorem_full_name, w["context"].state)
        assert (g["context"].theorem_pos.line_nb, g["context"].theorem_pos.column_nb) == tuple(w["start"])
        assert [_as_plain(p) for p in g["retrieved_premises"]] == [_as_plain(p) for p in w["retrieved_premises"]]
        assert sorted(map(_as_plain, g["all_pos_premises"])) == sorted(map(_as_plain, w["all_pos_premises"]))
        assert len(g["all_pos_premises"]) == 2          # the unlocatable provenance is left out
    assert [g["tactic_idx"] for g in got[:3]] == list(range(len(theorems[0]["traced_tactics"])))[:3]
    # the query made of tokens no premise contains: every score is 0, so the first accessible premises in index order
    zero = next(g for g in got if g["context"].state == "⊢ zzz qqq")
    assert zero["scores"] == [0.0] * len(zero["scores"])

    bm25_cli.main(argv + ["--native-layout"])
    with open(out, "rb") as fh:
        native = pickle.load(fh)
    assert type(native[0]["context"]).__module__ == "reprover_b200.corpus"
    assert [[_as_plain(p) for p in r["retrieved_premises"]] for r in native] == \
        [[_as_plain(p) for p in r["retrieved_premises"]] for r in got]


def test_abi_workspace_and_argument_checks(rpx_lib):
    ws = rpx_lib.rpx_bm25_topk_workspace_bytes
    assert ws(200_000, 256, 100) >= 49 * 256 * 100 * 16      # one sorted list per 4096-premise tile and query
    assert ws(200_000, 1, 1024) > 0
    assert ws(200_000, 1, 1025) == 0 and ws(200_000, 0, 10) == 0 and ws(200_000, 65536, 10) == 0 and ws(0, 1, 1) == 0
    buf = (C.c_uint8 * 4096)()
    h = C.c_void_p()
    assert rpx_lib.rpx_bm25_create(buf, buf, buf, 10, 0, 5, C.byref(h)) == _native.RPX_ERR_UNSUPPORTED
    assert rpx_lib.rpx_bm25_create(None, buf, buf, 10, 5, 5, C.byref(h)) == _native.RPX_ERR_INVALID
    assert rpx_lib.rpx_bm25_create(buf, None, None, 10, 5, 5, C.byref(h)) == _native.RPX_ERR_INVALID
    assert not h.value
    assert rpx_lib.rpx_bm25_create(buf, buf, buf, 10, 5, 5, C.byref(h)) == _native.RPX_OK and h.value
    try:
        off = (C.c_int64 * 3)(0, 4, 2)       # decreasing
        rows = (C.c_int32 * 2)(0, 1)
        big = 1 << 20
        call = rpx_lib.rpx_bm25_topk
        assert call(h, buf, off, 2, None, 0, None, 0, 10, buf, buf, None, buf, big, None) == _native.RPX_ERR_INVALID
        assert "offsets" in _native.last_error()
        off = (C.c_int64 * 3)(0, 2, 4)
        assert call(h, buf, off, 2, None, 0, None, 0, 1025, buf, buf, None, buf, big, None) == _native.RPX_ERR_UNSUPPORTED
        assert call(h, buf, off, 2, buf, 1, rows, 1, 10, buf, buf, None, buf, big, None) == _native.RPX_ERR_INVALID
        assert "mask row" in _native.last_error()
        assert call(h, buf, off, 2, buf, 0, rows, 2, 10, buf, buf, None, buf, big, None) == _native.RPX_ERR_INVALID
        assert call(h, buf, off, 2, buf, 1, None, 2, 10, buf, buf, None, buf, big, None) == _native.RPX_ERR_INVALID
        assert call(h, buf, off, 2, None, 0, None, 0, 10, buf, buf, None, buf, 1024, None) in (
            _native.RPX_ERR_WORKSPACE, _native.RPX_ERR_INVALID)      # too small (or the stack buffer is unaligned)
    finally:
        assert rpx_lib.rpx_bm25_destroy(h) == _native.RPX_OK


@needs_no_gpu
def test_bm25_refuses_cpu(rpx_lib):
    from reprover_b200.bm25 import BM25Index

    with pytest.raises(RuntimeError, match="CUDA"):
        BM25Index([[1, 2], [2, 3]])
    buf = (C.c_uint8 * 4096)()
    h = C.c_void_p()
    assert rpx_lib.rpx_bm25_create(buf, buf, buf, 10, 5, 5, C.byref(h)) == _native.RPX_OK
    try:
        assert rpx_lib.rpx_bm25_scores(h, buf, 2, buf, None) == _native.RPX_ERR_CUDA and _native.last_error()
    finally:
        rpx_lib.rpx_bm25_destroy(h)


def test_idf_formula_matches_math_log():
    st = okapi_postings([[0], [0, 1], [2]])
    assert st.idf[1] == math.log(3 - 1 + 0.5) - math.log(1 + 0.5)
