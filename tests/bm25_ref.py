"""Float64 oracle of the BM25 baseline: a restatement of `rank_bm25.BM25Okapi` (construction, `_calc_idf`,
`get_batch_scores`) and of the reference script's `_process_theorem` (retrieval/bm25/main.py:24-70), in pure
Python / numpy.  It imports neither the reference nor rank_bm25.  The one deliberate change: rankings use a stable
(score desc, index asc) order where the reference's `np.argsort` leaves ties unordered."""
from __future__ import annotations

import math
from typing import Any, Callable, Dict, List, Sequence

import numpy as np


class BM25Okapi:
    def __init__(self, corpus: Sequence[Sequence[Any]], k1: float = 1.5, b: float = 0.75, epsilon: float = 0.25):
        self.k1, self.b, self.epsilon = k1, b, epsilon
        self.corpus_size = 0
        self.avgdl = 0
        self.doc_freqs: List[Dict[Any, int]] = []
        self.idf: Dict[Any, float] = {}
        self.doc_len: List[int] = []
        nd = self._initialize(corpus)
        self._calc_idf(nd)
        # per term: documents and counts, to build get_batch_scores' q_freq arrays without a dict lookup per document
        self._postings: Dict[Any, tuple] = {}
        for di, freqs in enumerate(self.doc_freqs):
            for w, f in freqs.items():
                self._postings.setdefault(w, ([], []))
                self._postings[w][0].append(di)
                self._postings[w][1].append(f)

    def _initialize(self, corpus):
        nd: Dict[Any, int] = {}
        num_doc = 0
        for document in corpus:
            self.doc_len.append(len(document))
            num_doc += len(document)
            frequencies: Dict[Any, int] = {}
            for word in document:
                frequencies[word] = frequencies.get(word, 0) + 1
            self.doc_freqs.append(frequencies)
            for word in frequencies:
                nd[word] = nd.get(word, 0) + 1
            self.corpus_size += 1
        self.avgdl = num_doc / self.corpus_size
        return nd

    def _calc_idf(self, nd):
        idf_sum = 0
        negative_idfs = []
        for word, freq in nd.items():
            idf = math.log(self.corpus_size - freq + 0.5) - math.log(freq + 0.5)
            self.idf[word] = idf
            idf_sum += idf
            if idf < 0:
                negative_idfs.append(word)
        self.average_idf = idf_sum / len(self.idf)
        eps = self.epsilon * self.average_idf
        for word in negative_idfs:
            self.idf[word] = eps

    def q_freq(self, q, doc_ids: np.ndarray) -> np.ndarray:
        """`np.array([(self.doc_freqs[di].get(q) or 0) for di in doc_ids])`."""
        full = np.zeros(self.corpus_size, dtype=np.int64)
        if q in self._postings:
            docs, freqs = self._postings[q]
            full[docs] = freqs
        return full[doc_ids]

    def get_batch_scores(self, query: Sequence[Any], doc_ids: Sequence[int]) -> List[float]:
        doc_ids = np.asarray(list(doc_ids), dtype=np.int64)
        assert all(di < len(self.doc_freqs) for di in doc_ids)
        score = np.zeros(len(doc_ids))
        doc_len = np.array(self.doc_len)[doc_ids]
        for q in query:
            q_freq = self.q_freq(q, doc_ids)
            score += (self.idf.get(q) or 0) * (q_freq * (self.k1 + 1) /
                                               (q_freq + self.k1 * (1 - self.b + self.b * doc_len / self.avgdl)))
        return score.tolist()

    def contribution(self, q, doc: int) -> float:
        """What `get_batch_scores` adds to document `doc`'s score for one query token `q`."""
        di = np.array([doc])
        f = self.q_freq(q, di)
        return float(((self.idf.get(q) or 0) * (f * (self.k1 + 1) /
                                                (f + self.k1 * (1 - self.b + self.b * np.array(self.doc_len)[di] / self.avgdl))))[0])


def rank(scores: Sequence[float], accessible: Sequence[int], k: int):
    """`np.argsort(scores)[::-1][:k]` with ties ordered by corpus index: (indexes, scores)."""
    s = np.asarray(scores, dtype=np.float64)
    acc = np.asarray(list(accessible), dtype=np.int64)
    order = np.lexsort((acc, -s))[:k]
    return acc[order].tolist(), s[order].tolist()


def process_theorem(thm: Dict[str, Any], corpus, tokenize: Callable[[str], List[Any]], bm25: BM25Okapi,
                    num_retrieved: int, use_all_premises: bool) -> List[Dict[str, Any]]:
    """`_process_theorem` on this package's `Corpus` / `Context`; `tokenize(text)` returns the token list."""
    from reprover_b200.corpus import Context, Pos

    preds = []
    if use_all_premises:
        accessible = list(range(len(corpus)))
    else:
        accessible = corpus.get_accessible_premise_indexes(thm["file_path"], Pos(*thm["start"]))
    for i, tac in enumerate(thm["traced_tactics"]):
        ctx = Context(thm["file_path"], thm["full_name"], Pos(*thm["start"]), tac["state_before"])
        scores = bm25.get_batch_scores(tokenize(ctx.serialize()), accessible)
        idx, sc = rank(scores, accessible, num_retrieved)
        found = set()
        for prov in tac["annotated_tactic"][1]:
            p = corpus.locate_premise(prov["def_path"], Pos(*prov["def_pos"]))
            if p is not None:
                found.add(p)
        preds.append({
            "url": thm["url"], "commit": thm["commit"], "file_path": thm["file_path"], "full_name": thm["full_name"],
            "start": thm["start"], "tactic_idx": i, "context": ctx, "all_pos_premises": list(found),
            "retrieved_premises": [corpus[j] for j in idx], "scores": sc,
        })
    return preds
