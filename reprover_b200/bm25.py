"""The reference's BM25 premise retriever (`retrieval/bm25/main.py`) on the GPU.

`BM25Index` stands where the reference builds `rank_bm25.BM25Okapi(tokenized_premises)` (main.py:154-158): it
tokenises every premise, computes BM25Okapi's statistics on the host (document lengths, document frequencies, idf
with the negative-idf floor, avgdl) and turns them into an inverted index whose postings carry each term's fp64
contribution to each document, computed with exactly the expression `get_batch_scores` evaluates.  Scoring and
ranking run in `rpx_bm25_*` (csrc/rpx_bm25.cu), which adds the contributions in query order, so every score equals
the reference's bit for bit.  Ties are ordered by corpus index (the reference's `np.argsort` leaves them unordered).

`predict` is the per-theorem loop of the script (`_process_theorem`, main.py:24-70) over a whole dataset.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native
from .corpus import Context, Corpus, Pos

K1 = 1.5
B = 0.75
EPSILON = 0.25
MAX_K = 1024


class BM25Index:
    """BM25Okapi (k1 = 1.5, b = 0.75, epsilon = 0.25) over token-id documents, scored on a CUDA device.

    `documents[i]` is the list of token ids of premise i.  `corpus` and `tokenizer` are optional: `from_corpus`
    sets them, and `topk` needs the corpus to return premises and accessibility masks.  Attributes with
    rank_bm25's meaning: `corpus_size`, `avgdl`, `doc_len`, `average_idf`, `idf` (term id -> idf)."""

    def __init__(self, documents: Sequence[Sequence[int]], device: Any = None, corpus: Optional[Corpus] = None,
                 tokenizer: Any = None, vocab_size: Optional[int] = None) -> None:
        device = torch.device(device) if device is not None else torch.device("cuda")
        if device.type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("BM25Index scores on a CUDA device only (no CPU path in this engine)")
        self.corpus, self.tokenizer, self.device = corpus, tokenizer, device
        st = okapi_postings(documents, vocab_size)
        self.corpus_size, self.doc_len, self.avgdl = st.corpus_size, st.doc_len, st.avgdl
        self.idf, self.average_idf, self.vocab_size, self.nnz = st.idf, st.average_idf, st.vocab_size, st.nnz
        self.term_ptr, self.post_doc, self.post_c = st.term_ptr, st.post_doc, st.post_c   # host copies
        vocab, n, term_ptr, post_c = st.vocab_size, st.corpus_size, st.term_ptr, st.post_c
        self._term_ptr = torch.from_numpy(term_ptr).to(device)
        self._post_doc = torch.from_numpy(self.post_doc).to(device)
        self._post_c = torch.from_numpy(post_c).to(device)
        self.lib = _native.load()
        self._handle = C.c_void_p()
        _native.check(self.lib.rpx_bm25_create(self._term_ptr.data_ptr(), self._post_doc.data_ptr() if self.nnz else None,
                                               self._post_c.data_ptr() if self.nnz else None, vocab, n, self.nnz,
                                               C.byref(self._handle)))

    @classmethod
    def from_corpus(cls, corpus: Corpus, tokenizer: Any, device: Any = None) -> "BM25Index":
        """Index `corpus.all_premises` tokenised by a `tokenizers.Tokenizer` (main.py:155-158)."""
        docs = [e.ids for e in tokenizer.encode_batch([p.serialize() for p in corpus.all_premises])]
        return cls(docs, device=device, corpus=corpus, tokenizer=tokenizer, vocab_size=tokenizer.get_vocab_size())

    def close(self) -> None:
        if getattr(self, "_handle", None) is not None and self._handle.value:
            self.lib.rpx_bm25_destroy(self._handle)
            self._handle = C.c_void_p()

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    @property
    def device_bytes(self) -> int:
        """Device memory the index holds (term offsets, postings' documents and contributions)."""
        return sum(t.numel() * t.element_size() for t in (self._term_ptr, self._post_doc, self._post_c))

    def token_ids(self, query: Sequence[Any]) -> np.ndarray:
        """int32 token ids of a query given as ids or as token strings (mapped through the tokenizer's vocabulary; a
        string it does not know is dropped: it scores 0 everywhere, as in BM25Okapi).  Ids outside the index's
        vocabulary become -1, which the kernel skips for the same reason."""
        if not isinstance(query, np.ndarray) and any(isinstance(t, str) for t in query):
            if self.tokenizer is None:
                raise TypeError("token strings need an index built with a tokenizer")
            query = [t for t in (self.tokenizer.token_to_id(t) if isinstance(t, str) else t for t in query) if t is not None]
        ids = np.asarray(query, dtype=np.int64).reshape(-1)
        return np.where((ids >= 0) & (ids < self.vocab_size), ids, -1).astype(np.int32)

    def encode_queries(self, texts: Sequence[str]) -> List[List[int]]:
        """Untruncated token ids of query texts (main.py:46)."""
        return [e.ids for e in self.tokenizer.encode_batch(list(texts))]

    # ---- rank_bm25's interface -------------------------------------------------------------------------------
    def get_scores(self, query: Sequence[Any]) -> np.ndarray:
        """fp64 scores of every document (BM25Okapi.get_scores)."""
        ids = torch.from_numpy(self.token_ids(query)).to(self.device)
        out = torch.empty(self.corpus_size, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _native.check(self.lib.rpx_bm25_scores(self._handle, ids.data_ptr() if ids.numel() else None, ids.numel(),
                                                   out.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream))
        return out.cpu().numpy()

    def get_batch_scores(self, query: Sequence[Any], doc_ids: Sequence[int]) -> List[float]:
        """Scores of `query` on the documents `doc_ids` (BM25Okapi.get_batch_scores)."""
        doc_ids = list(doc_ids)
        assert all(di < self.corpus_size for di in doc_ids)
        return self.get_scores(query)[np.asarray(doc_ids, dtype=np.int64)].tolist()

    # ---- ranking -----------------------------------------------------------------------------------------------
    def topk_indexes(self, queries: Sequence[Sequence[Any]], k: int, mask_words: Optional[np.ndarray] = None,
                     mask_rows: Optional[Sequence[int]] = None, max_batch_tokens: int = 1 << 20,
                     max_workspace_bytes: int = 1 << 29) -> Tuple[List[List[int]], List[List[float]]]:
        """The k best documents of every query under (score desc, index asc), best first, with their scores.

        `mask_words` [R, ceil(N / 32)] uint32 rows in `Corpus.accessible_mask_words`' layout and `mask_rows[q]`, the
        row of query q, restrict each query to its accessible documents; a query with fewer than k of them gets a
        shorter list.  Queries go to the device in batches of at most `max_batch_tokens` tokens; the result does not
        depend on the batching."""
        if not isinstance(k, (int, np.integer)) or not 1 <= k <= MAX_K:
            raise ValueError(f"k={k}: the engine returns between 1 and {MAX_K} documents per query")
        k = int(k)
        ids = [self.token_ids(q) for q in queries]
        if (mask_words is None) != (mask_rows is None):
            raise ValueError("mask_words and mask_rows go together")
        if mask_words is not None:
            mask_words = np.ascontiguousarray(mask_words, dtype=np.uint32).reshape(-1, (self.corpus_size + 31) // 32)
            mask_rows = np.asarray(mask_rows, dtype=np.int64)
            if mask_rows.shape != (len(ids),) or (len(ids) and (mask_rows.min() < 0 or mask_rows.max() >= len(mask_words))):
                raise ValueError("mask_rows must name one row of mask_words per query")
        per_query = int(self.lib.rpx_bm25_topk_workspace_bytes(self.corpus_size, 1, k))
        max_q = max(1, min(65535, max_workspace_bytes // max(per_query, 1)))
        idx_out: List[List[int]] = []
        score_out: List[List[float]] = []
        q0 = 0
        while q0 < len(ids):
            q1, tokens = q0, 0
            while q1 < len(ids) and q1 - q0 < max_q and (q1 == q0 or tokens + len(ids[q1]) <= max_batch_tokens):
                tokens += len(ids[q1])
                q1 += 1
            rows = None if mask_words is None else mask_rows[q0:q1]
            i, s, c = self._topk_batch(ids[q0:q1], k, mask_words, rows)
            for r in range(q1 - q0):
                idx_out.append(i[r, : c[r]].tolist())
                score_out.append(s[r, : c[r]].tolist())
            q0 = q1
        return idx_out, score_out

    def _topk_batch(self, ids: List[np.ndarray], k: int, mask_words: Optional[np.ndarray], rows: Optional[np.ndarray]):
        nq = len(ids)
        offsets = np.zeros(nq + 1, dtype=np.int64)
        np.cumsum([len(a) for a in ids], out=offsets[1:])
        dev = self.device
        tokens = torch.from_numpy(np.concatenate(ids) if offsets[-1] else np.zeros(1, np.int32)).to(dev)
        mask_dev, h_rows, n_rows, stride = None, None, 0, 0
        if mask_words is not None:
            used, local = np.unique(rows, return_inverse=True)   # upload only the rows this batch uses
            mask_dev = torch.from_numpy(mask_words[used].view(np.int32)).to(dev)
            h_rows = np.ascontiguousarray(local, dtype=np.int32)
            n_rows, stride = len(used), mask_words.shape[1]
        out_s = torch.empty(nq, k, dtype=torch.float64, device=dev)
        out_i = torch.empty(nq, k, dtype=torch.int64, device=dev)
        out_c = torch.empty(nq, dtype=torch.int32, device=dev)
        ws_bytes = int(self.lib.rpx_bm25_topk_workspace_bytes(self.corpus_size, nq, k))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _native.check(self.lib.rpx_bm25_topk(
                self._handle, tokens.data_ptr(), offsets.ctypes.data, nq,
                mask_dev.data_ptr() if mask_dev is not None else None, stride,
                h_rows.ctypes.data if h_rows is not None else None, n_rows, k, out_s.data_ptr(), out_i.data_ptr(),
                out_c.data_ptr(), ws.data_ptr(), ws_bytes, torch.cuda.current_stream(dev).cuda_stream))
        return out_i.cpu().numpy(), out_s.cpu().numpy(), out_c.cpu().numpy()

    def topk(self, queries: Sequence[Sequence[Any]], k: int, contexts: Optional[Sequence[Context]] = None,
             use_all_premises: bool = False) -> Tuple[List[List[Any]], List[List[float]]]:
        """Retrieved premises and Python-float scores per query, as the reference's `_process_theorem` produces them:
        over every premise with `use_all_premises`, otherwise over the premises accessible to `contexts[q]`
        (`Corpus.get_accessible_premise_indexes(ctx.path, ctx.theorem_pos)`, shared by contexts of one theorem)."""
        if self.corpus is None:
            raise ValueError("topk returns premises: build the index with from_corpus (or use topk_indexes)")
        if use_all_premises:
            idx, scores = self.topk_indexes(queries, k)
        else:
            if contexts is None or len(contexts) != len(queries):
                raise ValueError("pass one context per query, or use_all_premises=True")
            idx, scores = [], []
            for c0 in range(0, len(queries), self._MASK_CHUNK):   # bounds the host memory the masks take
                keys: Dict[Tuple[str, int, int], int] = {}
                words, rows = [], []
                for ctx in contexts[c0:c0 + self._MASK_CHUNK]:
                    pos = Pos.from_any(ctx.theorem_pos)
                    key = (ctx.path, pos.line_nb, pos.column_nb)
                    if key not in keys:
                        keys[key] = len(words)
                        words.append(self.corpus.accessible_index_mask_words(ctx.path, pos))
                    rows.append(keys[key])
                i, s = self.topk_indexes(queries[c0:c0 + self._MASK_CHUNK], k, np.stack(words), rows)
                idx += i
                scores += s
        return [[self.corpus[i] for i in row] for row in idx], scores

    _MASK_CHUNK = 4096


class OkapiPostings:
    """BM25Okapi's statistics of a tokenised corpus and the inverted index built from them (host arrays)."""

    corpus_size: int
    doc_len: List[int]
    avgdl: float
    idf: Dict[int, float]
    average_idf: float
    vocab_size: int
    nnz: int
    term_ptr: np.ndarray   # [vocab + 1] int64
    post_doc: np.ndarray   # [nnz] int32, ascending within a term
    post_c: np.ndarray     # [nnz] fp64 contribution of the term to the document's score


def okapi_postings(documents: Sequence[Sequence[int]], vocab_size: Optional[int] = None) -> OkapiPostings:
    """BM25Okapi's construction (`_initialize`, `_calc_idf`) on token-id documents, plus every posting's
    contribution computed as `get_batch_scores` computes it.  `vocab_size` widens the id range past the largest id."""
    st = OkapiPostings()
    n = len(documents)
    if n == 0:
        raise ValueError("BM25 needs at least one document")
    st.corpus_size = n
    lens = np.fromiter((len(d) for d in documents), dtype=np.int64, count=n)
    st.doc_len = lens.tolist()
    flat = (np.concatenate([np.asarray(d, dtype=np.int64) for d in documents]) if lens.sum()
            else np.zeros(0, dtype=np.int64))
    if flat.size and flat.min() < 0:
        raise ValueError("token ids must be non-negative")
    vocab = int(flat.max()) + 1 if flat.size else 1
    if vocab_size is not None:
        vocab = max(vocab, int(vocab_size))
    st.vocab_size = vocab
    st.avgdl = int(lens.sum()) / n
    # postings: one (term, document) pair per distinct token of a document, term-major, documents ascending
    doc_of = np.repeat(np.arange(n, dtype=np.int64), lens)
    pairs, tf = np.unique(flat * n + doc_of, return_counts=True)
    terms, docs = pairs // n, pairs % n
    nd = np.bincount(terms, minlength=vocab)
    # idf in BM25Okapi._calc_idf's order: terms by first appearance (documents in order, tokens in order)
    present, first = np.unique(flat, return_index=True)
    idf: Dict[int, float] = {}
    idf_sum = 0
    negative = []
    for t in present[np.argsort(first, kind="stable")].tolist():
        f = int(nd[t])
        v = math.log(n - f + 0.5) - math.log(f + 0.5)
        idf[t] = v
        idf_sum += v
        if v < 0:
            negative.append(t)
    st.average_idf = idf_sum / len(idf) if idf else 0.0
    eps = EPSILON * st.average_idf
    for t in negative:
        idf[t] = eps
    st.idf = idf
    idf_arr = np.zeros(vocab, dtype=np.float64)
    if idf:
        idf_arr[np.fromiter(idf.keys(), dtype=np.int64)] = np.fromiter(idf.values(), dtype=np.float64)
    # get_batch_scores adds `idf * (tf * (k1 + 1) / (tf + k1 * (1 - b + b * doc_len / avgdl)))` per query token;
    # the same numpy float64 operations, in the same order, per posting
    dl = lens[docs]
    post_c = idf_arr[terms] * (tf * (K1 + 1) / (tf + K1 * (1 - B + B * dl / st.avgdl)))
    term_ptr = np.zeros(vocab + 1, dtype=np.int64)
    np.cumsum(nd, out=term_ptr[1:])
    st.nnz = int(tf.size)
    st.post_c = post_c
    st.post_doc = docs.astype(np.int32)
    st.term_ptr = term_ptr
    return st


def load_theorems(data_path: str) -> List[Dict[str, Any]]:
    """The theorems of `train.json`, `val.json` and `test.json` under `data_path`, in that order (main.py:124-129)."""
    import json
    import os

    theorems: List[Dict[str, Any]] = []
    for split in ("train", "val", "test"):
        with open(os.path.join(data_path, f"{split}.json")) as fh:
            theorems.extend(json.load(fh))
    return theorems


def all_pos_premises(annotated_tactic: Any, corpus: Corpus) -> list:
    """Premises used by an annotated tactic that the corpus can locate (reference common.py:341-354)."""
    _, provenances = annotated_tactic
    found = set()
    for prov in provenances:
        p = corpus.locate_premise(prov["def_path"], Pos(*prov["def_pos"]))
        if p is not None:
            found.add(p)
    return list(found)


def predict(index: Any, theorems: Sequence[Dict[str, Any]], num_retrieved: int = 100,
            use_all_premises: bool = False) -> List[Dict[str, Any]]:
    """One prediction record per traced tactic, with the keys of the reference's `_process_theorem`
    (main.py:55-67).  `index` is a `BM25Index` built with `from_corpus`; all tactics are scored in one `topk` call."""
    corpus = index.corpus
    contexts: List[Context] = []
    owners = []
    for thm in theorems:
        for i, tac in enumerate(thm["traced_tactics"]):
            contexts.append(Context(thm["file_path"], thm["full_name"], Pos(*thm["start"]), tac["state_before"]))
            owners.append((thm, i, tac))
    queries = index.encode_queries([c.serialize() for c in contexts])
    premises, scores = index.topk(queries, num_retrieved, contexts=None if use_all_premises else contexts,
                                  use_all_premises=use_all_premises)
    preds = []
    for (thm, i, tac), ctx, prem, sc in zip(owners, contexts, premises, scores):
        preds.append({
            "url": thm["url"],
            "commit": thm["commit"],
            "file_path": thm["file_path"],
            "full_name": thm["full_name"],
            "start": thm["start"],
            "tactic_idx": i,
            "context": ctx,
            "all_pos_premises": all_pos_premises(tac["annotated_tactic"], corpus),
            "retrieved_premises": prem,
            "scores": sc,
        })
    return preds
