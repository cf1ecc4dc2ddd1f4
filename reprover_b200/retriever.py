"""`B200PremiseRetriever` — drop-in for the inference surface of the reference's
`PremiseRetriever` (retrieval/model.py:29): `load_hf`, `load_corpus`,
`embedding_size`, `_encode`, `reindex_corpus`, `retrieve`, and the attributes its
callers touch (`corpus`, `corpus_embeddings`, `embeddings_staled`, `device`,
`max_seq_len`, `num_retrieved`).  Callers in the reference: `retrieval/index.py:33-38`,
`prover/tactic_generator.py:271-292`, `generation/model.py:163-164,224-233`.

Everything numeric is a call into the CUDA engine through the C ABI; torch only owns
the buffers.  Training (`forward`, `training_step`, optimizers) is out of scope.
"""
from __future__ import annotations

import os
import pickle
from typing import Any, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import tokenizer as byt5
from .corpus import Context, Corpus, IndexedCorpus, Pos, Premise
from .engine import T5EncoderEngine, load_hf_checkpoint


class _Serialized:
    """Lazy `[p.serialize() for p in premises]` (one pass, known length)."""

    def __init__(self, premises: Sequence[Premise]) -> None:
        self._premises = premises

    def __len__(self) -> int:
        return len(self._premises)

    def __iter__(self):
        for p in self._premises:
            yield p.serialize()


class B200PremiseRetriever:
    def __init__(self, model_name: str, lr: float = 0.0, warmup_steps: int = 0, max_seq_len: int = 2048,
                 num_retrieved: int = 100, device: Union[int, str, torch.device, None] = None,
                 dtype: Optional[torch.dtype] = None, max_tokens_per_call: int = 1 << 18,
                 output_dtype: Optional[torch.dtype] = None) -> None:
        """`model_name` is an HF checkpoint directory (config.json + model.safetensors) or a hub id that
        is available in the local HF cache."""
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else "cpu"
        device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(
                "B200PremiseRetriever runs on a B200 (sm_100a) only; there is no CPU path. "
                "(The reference warns that CPU indexing is very slow, retrieval/index.py:28-30; this engine refuses.)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.lr = lr
        self.warmup_steps = warmup_steps
        self.num_retrieved = num_retrieved
        self.max_seq_len = max_seq_len
        self.device = device
        # Reference dtype policy (retrieval/model.py:56-66): bf16 on GPUs with cc >= 8 unless told
        # otherwise — on an H100 that is bf16, which is the one compute dtype this engine has (bf16
        # operands, fp32 accumulation, fp32 residual stream; similarity index held in bf16 like the
        # reference's GPU path, :363-366).  `dtype=torch.float32` in the reference means an fp32 MODEL
        # and an fp32 index; quietly running bf16 under that name would misreport what was computed, so
        # it is refused.  `output_dtype=torch.float32` is the separate, honest knob: same computation,
        # embeddings handed back as fp32 tensors.
        if dtype not in (None, torch.bfloat16):
            raise NotImplementedError(
                f"dtype={dtype}: this engine computes in bf16 (fp32 accumulation) only — the reference's own "
                f"default on this GPU. Pass dtype=None / torch.bfloat16; use output_dtype=torch.float32 to get "
                f"the embeddings as fp32 tensors.")
        self.dtype = torch.bfloat16 if output_dtype is None else output_dtype
        if self.dtype not in (torch.bfloat16, torch.float32):
            raise NotImplementedError(f"output dtype {self.dtype} is not supported (bf16 or fp32)")
        self.model_name = model_name
        cfg, sd = load_hf_checkpoint(model_name)
        self.encoder = T5EncoderEngine(cfg, sd, device, max_tokens_per_call=max_tokens_per_call)
        self._index_handle = None      # rpx_index over the bf16 copy of corpus_embeddings
        self._index_source = None      # (tensor identity, version) the handle was built from
        self._corpus_embeddings: Optional[torch.Tensor] = None
        self.corpus: Optional[Corpus] = None
        self.corpus_embeddings = None
        self.embeddings_staled = True
        self.sharded_index = None
        self._tokenizer = None

    # ------------------------------------------------------------------ construction (reference :52-85)
    @classmethod
    def load_hf(cls, ckpt_path: str, max_seq_len: int, device, dtype=None) -> "B200PremiseRetriever":
        return cls(ckpt_path, 0.0, 0, max_seq_len, 100, device=device, dtype=dtype)

    @property
    def corpus_embeddings(self) -> Optional[torch.Tensor]:
        """[N, D] embedding matrix, row i for `corpus.all_premises[i]` (reference attribute of the same name).
        Assigning a new tensor drops the engine's handle on the old one."""
        return self.__dict__.get("_corpus_embeddings")

    @corpus_embeddings.setter
    def corpus_embeddings(self, value: Optional[torch.Tensor]) -> None:
        if value is not self.__dict__.get("_corpus_embeddings"):
            handle = self.__dict__.get("_index_handle")
            if handle is not None:
                handle.close()
            self.__dict__["_index_handle"] = None
            self.__dict__["_index_source"] = None
        self.__dict__["_corpus_embeddings"] = value

    @property
    def tokenizer(self):
        """The HF `ByT5Tokenizer` the reference keeps in `self.tokenizer` (retrieval/model.py:44); its
        callers only persist it (`generation/model.py:224-226`: `retriever.tokenizer.save_pretrained(dir)`).
        The engine itself tokenises on the device (`rpx_encode_bytes`) and never calls this object."""
        if self._tokenizer is None:
            try:
                from transformers import AutoTokenizer, ByT5Tokenizer
            except ImportError as exc:  # pragma: no cover
                raise RuntimeError("`retriever.tokenizer` needs the `transformers` package") from exc
            # The engine tokenises as ByT5 does (bytes + 3, EOS = 1), whatever files the checkpoint ships; use
            # the checkpoint's own tokenizer files only when they exist and are ByT5's
            tok = None
            try:
                from .engine import resolve_checkpoint_dir

                ckpt = resolve_checkpoint_dir(self.model_name)
                if os.path.exists(os.path.join(ckpt, "tokenizer_config.json")):
                    cand = AutoTokenizer.from_pretrained(ckpt)
                    if isinstance(cand, ByT5Tokenizer):
                        tok = cand
            except Exception:
                tok = None
            self._tokenizer = tok if tok is not None else ByT5Tokenizer()
        return self._tokenizer

    def load_corpus(self, path_or_corpus: Union[str, Corpus]) -> None:
        """Attach a corpus: a `Corpus`, a `corpus.jsonl` path (stale index) or a pickled
        `IndexedCorpus` (fresh index)."""
        self.sharded_index = None   # a row-sharded index belongs to the corpus it was built from
        if isinstance(path_or_corpus, Corpus):
            self.corpus = path_or_corpus
            self.corpus_embeddings = None
            self.embeddings_staled = True
            return
        path = path_or_corpus
        if path.endswith(".jsonl"):
            self.corpus = Corpus(path)
            self.corpus_embeddings = None
            self.embeddings_staled = True
        else:
            from .compat import convert_corpus, load_reference_index

            try:
                with open(path, "rb") as fh:
                    indexed = pickle.load(fh)
            except (ModuleNotFoundError, AttributeError):
                # an index in the reference's layout (classes from `common` / `lean_dojo`), read without them
                indexed = load_reference_index(path)
            corpus = indexed.corpus
            if not isinstance(corpus, Corpus):
                # inside the reference tree `common` IS importable and pickle.load hands back the reference's
                # own Corpus: convert it, or retrieval would silently run the reference's torch code
                corpus = convert_corpus(corpus)
            self.corpus = corpus
            self.corpus_embeddings = indexed.embeddings
            self.embeddings_staled = False

    @property
    def embedding_size(self) -> int:
        return self.encoder.hidden_size

    # ------------------------------------------------------------------ encode
    def _encode(self, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
        """Reference `_encode` (retrieval/model.py:92-114): [B, L] ids + mask -> [B, D] unit rows."""
        return self.encoder.encode_ids(input_ids, attention_mask, out_dtype=self.dtype)

    @torch.no_grad()
    def encode_texts(self, texts: Sequence[str], batch_size: int = 64, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """tokenizer(...) + `_encode` for a sequence of strings (reference :199-206), rows in input order.

        Strings without special-token literals (practically all Lean code) go to the device as raw
        bytes; the rest are tokenised on the host with HF semantics and use the ids entry point.
        `texts` is walked once (it may produce its strings lazily): strings are gathered until the
        next one would overflow the engine's token budget for one call, then handed over as ONE
        asynchronous engine call — the host gathers group i+1 while the GPU encodes group i, and every
        call but the last is full."""
        n = len(texts)
        if out is None:
            out = torch.empty(n, self.embedding_size, dtype=self.dtype, device=self.device)
        budget = self.encoder.max_tokens_per_call
        special: List[Tuple[int, str]] = []
        rows: List[int] = []
        blobs: List[bytes] = []
        tokens = 0

        def flush() -> None:
            nonlocal tokens
            if not rows:
                return
            if rows[-1] - rows[0] + 1 == len(rows):     # contiguous: write in place
                self.encoder.encode_strings(blobs, self.max_seq_len, out_dtype=self.dtype, out=out[rows[0]:rows[-1] + 1])
            else:
                emb = self.encoder.encode_strings(blobs, self.max_seq_len, out_dtype=self.dtype)
                out[torch.tensor(rows, device=self.device)] = emb
            rows.clear()
            blobs.clear()
            tokens = 0

        for i, t in enumerate(texts):
            if "<" in t and byt5.needs_id_path(t):
                special.append((i, t))
                continue
            b = t.encode("utf-8")
            tk = min(len(b) + 1, self.max_seq_len)
            if tokens + tk > budget:
                flush()
            rows.append(i)
            blobs.append(b)
            tokens += tk
        flush()
        for lo in range(0, len(special), batch_size):
            part = special[lo:lo + batch_size]
            ids, mask = byt5.pad_batch([byt5.encode_ids(t, self.max_seq_len) for _, t in part])
            emb = self._encode(torch.from_numpy(ids).to(self.device), torch.from_numpy(mask).to(self.device))
            out[torch.tensor([i for i, _ in part], device=self.device)] = emb
        return out

    @torch.no_grad()
    def reindex_corpus(self, batch_size: int) -> None:
        """Reference :183-210.  `batch_size` is kept for signature parity; the engine packs premises by
        token budget instead (results do not depend on batching: padded keys have zero weight)."""
        if not self.embeddings_staled:
            return
        assert self.corpus is not None, "load_corpus first"
        premises = self.corpus.all_premises
        self.corpus_embeddings = torch.empty(len(premises), self.embedding_size, dtype=self.dtype, device=self.device)
        # premises are serialised lazily while encode_texts walks them, so the regex work of group i+1
        # overlaps the GPU's work on group i
        self.encode_texts(_Serialized(premises), batch_size=batch_size, out=self.corpus_embeddings)
        self.embeddings_staled = False

    # ------------------------------------------------------------------ retrieve (reference :338-375)
    @torch.no_grad()
    def retrieve(self, state: str, file_name: str, theorem_full_name: str, theorem_pos: Any,
                 k: int) -> Tuple[List[Premise], List[float]]:
        premises, scores = self.retrieve_batch([state], [file_name], [theorem_full_name], [theorem_pos], k)
        assert len(premises) == len(scores) == 1
        return premises[0], scores[0]

    @torch.no_grad()
    def retrieve_batch(self, states: Sequence[str], file_names: Sequence[str], theorem_full_names: Sequence[str],
                       theorem_poses: Sequence[Any], k: int) -> Tuple[List[List[Premise]], List[List[float]]]:
        """Batched `retrieve` (what validation_step / predict_step do with Q = eval_batch_size,
        reference :215-225, 281-289)."""
        self.reindex_corpus(batch_size=32)
        ctxs = [Context(f, t, Pos.from_any(p), s) for s, f, t, p in zip(states, file_names, theorem_full_names, theorem_poses)]
        if not isinstance(k, int) or k < 1:
            raise ValueError(f"k={k!r}: retrieve() needs a positive number of premises")
        context_emb = self._encode_states([c.serialize() for c in ctxs])
        return self.corpus.get_nearest_premises(self.index_handle(), ctxs, context_emb, k)

    # Proof states are encoded one (or a few) at a time: below this many packed tokens per engine call the
    # encoder's latency path is used (narrow tiles; `rpx_encoder_set_latency_tokens`).  Re-indexing never
    # takes it, so the index stays independent of how premises are batched.
    state_latency_tokens = 768

    def _encode_states(self, texts: Sequence[str]) -> torch.Tensor:
        enc = self.encoder
        if not hasattr(enc, "set_latency_tokens"):
            return self.encode_texts(texts)
        enc.set_latency_tokens(self.state_latency_tokens)
        try:
            return self.encode_texts(texts)
        finally:
            enc.set_latency_tokens(0)

    def index_handle(self):
        """The engine's handle on the similarity index: the bf16 device copy of `corpus_embeddings`
        (the reference moves / casts the index to the query's device and dtype on first use, :363-366 —
        bf16 on this GPU) plus the state derived from it once.  Rebuilt when `corpus_embeddings` is replaced
        or modified in place."""
        from .retrieval_ops import IndexHandle

        emb = self.corpus_embeddings
        assert emb is not None, "no index: load_corpus + reindex_corpus first"
        src = (id(emb), emb._version)
        if self._index_handle is None or self._index_source != src:
            if emb.device != self.device or emb.dtype != torch.bfloat16:
                if self.dtype == torch.bfloat16:
                    # like the reference, keep the index on the query's device in the query's dtype
                    self.corpus_embeddings = emb = emb.to(device=self.device, dtype=torch.bfloat16)
                    bf16 = emb
                else:
                    bf16 = emb.to(device=self.device, dtype=torch.bfloat16)   # fp32 stays what the caller sees
            else:
                bf16 = emb
            if self._index_handle is not None:
                self._index_handle.close()
            self._index_handle = IndexHandle(bf16)
            self._index_source = (id(self.corpus_embeddings), self.corpus_embeddings._version)
        return self._index_handle

    # ------------------------------------------------------------------ row-sharded index (SURVEY §8e)
    # One process per GPU, `torch.distributed` initialised by the caller.  `reindex_corpus_sharded`
    # encodes only this rank's rows (no communication); `retrieve_batch_sharded` needs the same
    # states on every rank and returns the same answer on every rank: local fused sim+top-k under
    # this rank's slice of the accessibility bitmask, one all-gather, device-side merge.
    @torch.no_grad()
    def reindex_corpus_sharded(self, batch_size: int = 64, group=None) -> "ShardedIndex":
        from .dist import ShardedIndex

        assert self.corpus is not None, "load_corpus first"
        index = getattr(self, "sharded_index", None)
        if index is not None and index.embeddings is not None and index.bounds[-1] == len(self.corpus) \
                and index.group is group:
            return index
        index = ShardedIndex(len(self.corpus), group=group)
        premises = self.corpus.all_premises[index.lo:index.hi]
        emb = torch.empty(len(premises), self.embedding_size, dtype=self.dtype, device=self.device)
        if len(premises):
            self.encode_texts(_Serialized(premises), batch_size=batch_size, out=emb)
        index.set_embeddings(emb if emb.dtype == torch.bfloat16 else emb.to(torch.bfloat16))
        self.sharded_index = index
        return index

    @torch.no_grad()
    def retrieve_batch_sharded(self, states: Sequence[str], file_names: Sequence[str], theorem_full_names: Sequence[str],
                               theorem_poses: Sequence[Any], k: int, group=None,
                               **ops) -> Tuple[List[List[Premise]], List[List[float]]]:
        """`retrieve_batch` over the row-sharded index (`ops`: injectable compute steps, see dist.sharded_topk)."""
        index = self.reindex_corpus_sharded(group=group)
        ctxs = [Context(f, t, Pos.from_any(p), s) for s, f, t, p in zip(states, file_names, theorem_full_names, theorem_poses)]
        context_emb = self._encode_states([c.serialize() for c in ctxs]).to(torch.bfloat16)
        words = np.stack([self.corpus.accessible_mask_words_range(c.path, c.theorem_pos, index.lo, index.hi) for c in ctxs])
        if words.shape[1] == 0:     # a rank without rows still takes part in the collective
            words = np.zeros((len(ctxs), 1), dtype=np.uint32)
        mask = torch.from_numpy(words.view(np.int32)).to(context_emb.device)
        scores, idx, counts, _ = index.topk(context_emb, k, access_mask=mask, **ops)
        if any(c < k for c in counts.cpu().tolist()):
            raise ValueError
        idx_h, scores_h = idx.cpu().tolist(), scores.cpu().tolist()
        return [[self.corpus.all_premises[i] for i in row] for row in idx_h], scores_h

    # ------------------------------------------------------------------ index I/O (reference retrieval/index.py:37-40)
    def save_index(self, path: str, reference_layout: bool = True) -> None:
        """Write the indexed corpus (`retrieval/index.py:37-40`: `IndexedCorpus(corpus, fp32 CPU embeddings)`).

        `reference_layout=True` (default): a pickle a STOCK reference checkout loads — classes
        `common.IndexedCorpus / Corpus / File / Premise`, `lean_dojo.Pos`, a networkx transitive-closure
        graph (`reprover_b200.compat.dump_reference_index`); `load_corpus` of this package reads it back
        through the compat loader.  `False`: this package's own (leaner) classes."""
        assert self.corpus is not None and not self.embeddings_staled
        emb = self.corpus_embeddings.to(torch.float32).cpu()
        with open(path, "wb") as fh:
            if reference_layout:
                from .compat import dump_reference_index

                dump_reference_index(self.corpus, emb, fh)
            else:
                pickle.dump(IndexedCorpus(self.corpus, emb), fh)
