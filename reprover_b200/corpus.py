"""Host-side data model of the retrieval corpus.

Mirrors the *interface* of the reference's `common.py` objects that sit on the
retrieval hot path — `Pos` (lean_dojo), `Context` (common.py:34-56), `Premise`
(:59-106), `PremiseSet` (:109-138), `File` (:141-178), `Corpus` (:181-326) and
`IndexedCorpus` (:329-338) — so code written against the reference keeps working,
but the internals are index-based: premises of one file are contiguous in
`all_premises` (the reference builds the list file by file, common.py:202-209),
so accessibility is a union of index ranges plus a prefix of the own file, which is
what the device-side access mask needs (SURVEY.md §8f rank 1).

`Corpus.get_nearest_premises` keeps the reference signature but runs the matmul +
ranking on the GPU through `rpx_sim_topk` (see `reprover_b200.retrieval_ops`).
"""
from __future__ import annotations

import json
import re
from dataclasses import dataclass, field
from functools import total_ordering
from typing import Any, Dict, Generator, Iterable, List, Optional, Sequence, Tuple

import numpy as np

MARK_START_SYMBOL = "<a>"
MARK_END_SYMBOL = "</a>"


@total_ordering
@dataclass(frozen=True)
class Pos:
    """A (line, column) source position; stands in for `lean_dojo.Pos` (absent in this image)."""

    line_nb: int
    column_nb: int

    @classmethod
    def from_any(cls, p: Any) -> "Pos":
        if isinstance(p, Pos):
            return p
        if hasattr(p, "line_nb") and hasattr(p, "column_nb"):
            return cls(int(p.line_nb), int(p.column_nb))
        # the reference asserts isinstance(pos, lean_dojo.Pos): anything that is not position-like
        # fails the same way (AssertionError), not with whatever unpacking happens to raise
        try:
            a, b = p
            return cls(int(a), int(b))
        except (TypeError, ValueError):
            raise AssertionError(f"not a source position: {p!r}") from None

    def _key(self) -> Tuple[int, int]:
        return (self.line_nb, self.column_nb)

    def __lt__(self, other: Any) -> bool:
        return self._key() < Pos.from_any(other)._key()

    def __iter__(self):
        yield self.line_nb
        yield self.column_nb


def remove_marks(s: str) -> str:
    """Strip the `<a>` / `</a>` premise-name marks."""
    return s.replace(MARK_START_SYMBOL, "").replace(MARK_END_SYMBOL, "")


def format_augmented_state(s: str, premises: Sequence["Premise"], max_len: Optional[int] = None) -> str:
    """The reference's `format_augmented_state` (common.py) without `p_drop`, which only training sets: the state
    with retrieved premises prepended, each as `p.serialize() + "\n\n"`.  Lengths are UTF-8 bytes; the premises'
    budget is `max_len` minus the state's length (it may be negative).  A premise that would overrun the budget is
    skipped, and later, shorter ones may still fit.  Each accepted premise goes in front of the text so far, so the
    top-ranked premise ends up farthest from the state.  `max_len=None`: no budget."""
    budget = None if max_len is None else max_len - len(s.encode("utf-8"))
    aug = ""
    length = 0
    for p in premises:
        p_str = f"{p.serialize()}\n\n"
        n = len(p_str.encode("utf-8"))
        if budget is not None and length + n > budget:
            continue
        length += n
        aug = p_str + aug
    return aug + s


@dataclass(unsafe_hash=True)
class Context:
    """A retrieval query: a proof state inside a theorem (reference common.py:34-56)."""

    path: str
    theorem_full_name: str
    theorem_pos: Pos = field(compare=False)
    state: str

    def __post_init__(self) -> None:
        assert isinstance(self.path, str)
        assert isinstance(self.theorem_full_name, str)
        object.__setattr__(self, "theorem_pos", Pos.from_any(self.theorem_pos))
        assert isinstance(self.state, str), "state must be a string"
        assert "⊢" in self.state, "a proof state must contain the turnstile"
        assert MARK_START_SYMBOL not in self.state and MARK_END_SYMBOL not in self.state

    def serialize(self) -> str:
        return self.state


@dataclass(unsafe_hash=True)
class Premise:
    """A retrievable definition / theorem (reference common.py:59-106)."""

    path: str
    full_name: str
    start: Pos = field(repr=False)
    end: Pos = field(repr=False, compare=False)
    code: str = field(compare=False)

    def __post_init__(self) -> None:
        assert isinstance(self.path, str)
        assert isinstance(self.full_name, str)
        self.start = Pos.from_any(self.start)
        self.end = Pos.from_any(self.end)
        assert self.start <= self.end
        assert isinstance(self.code, str) and self.code != ""

    def serialize(self) -> str:
        """Text fed to the encoder: the code with the premise's own name wrapped in marks.

        Same rule as the reference (common.py:93-106): replace `_root_.<full_name>`;
        then, trying the fully qualified name first and successively shorter suffixes,
        wrap the first spelling (optionally «quoted») that occurs after whitespace.

        Like the reference, the name is used as a regex pattern UN-escaped (its dots match any
        character).  Compiling one or two fresh patterns per premise costs ~90 us, which would cap
        re-indexing at ~11 k premises/s per host thread — below what one GPU encodes — so names
        made of ordinary components (no regex metacharacter, quote or space: all but a handful of
        Lean names) take `_sub_plain`, a direct scan with exactly `re.sub`'s semantics for that
        pattern shape (pinned against `re.sub` in tests/test_host_cpu.py)."""
        marked = f"{MARK_START_SYMBOL}{self.full_name}{MARK_END_SYMBOL}"
        text = self.code.replace(f"_root_.{self.full_name}", marked)
        parts = self.full_name.split(".")
        if all(_PLAIN_COMPONENT.match(c) for c in parts):
            if parts[-1] not in text:   # every suffix ends with the last component
                return text
            for first in range(len(parts)):
                replaced = _sub_plain(text, parts[first:], marked)
                if replaced is not None:
                    return replaced
            return text
        for first in range(len(parts)):
            suffix = ".".join(parts[first:])
            replaced = re.sub(f"(?<=\\s)«?{suffix}»?", marked, text)
            if replaced != text:
                return replaced
        return text


_PLAIN_COMPONENT = re.compile(r"[^.^$*+?{}\[\]\\|()«»\s]+\Z")


def _sub_plain(text: str, comps: Sequence[str], repl: str) -> Optional[str]:
    """`re.sub("(?<=\\s)«?" + ".".join(comps) + "»?", repl, text)` for metacharacter-free components
    (so the pattern is: after whitespace, optional «, the components separated by ONE arbitrary
    non-newline character each, optional »).  Returns None when nothing matches or the result
    equals `text` (the caller then tries the next suffix, as the reference does)."""
    head = comps[0]
    out: List[str] = []
    last = 0          # end of the previous match (text[last:] is still to be copied)
    pos = 0
    n = len(text)
    while True:
        j = text.find(head, pos)
        if j < 0:
            break
        # where the match would start: at the « right before the head, else at the head itself
        if j >= 2 and text[j - 1] == "«" and j - 1 >= last and text[j - 2].isspace():
            start = j - 1
        elif j >= 1 and j >= last and text[j - 1].isspace():
            start = j
        else:
            pos = j + 1
            continue
        e = j + len(head)
        ok = True
        for c in comps[1:]:
            if e >= n or text[e] == "\n" or not text.startswith(c, e + 1):
                ok = False
                break
            e += 1 + len(c)
        if not ok:
            pos = j + 1
            continue
        if e < n and text[e] == "»":
            e += 1
        out.append(text[last:start])
        out.append(repl)
        last = e
        pos = e
    if not out:
        return None
    out.append(text[last:])
    result = "".join(out)
    return None if result == text else result


class PremiseSet:
    """Premises keyed by (path, full_name) (reference common.py:109-138)."""

    def __init__(self) -> None:
        self.path2premises: Dict[str, Dict[str, Premise]] = {}

    def __iter__(self) -> Generator[Premise, None, None]:
        for by_name in self.path2premises.values():
            yield from by_name.values()

    def add(self, p: Premise) -> None:
        self.path2premises.setdefault(p.path, {})[p.full_name] = p

    def update(self, premises: Iterable[Premise]) -> None:
        for p in premises:
            self.add(p)

    def __contains__(self, p: Premise) -> bool:
        return p.full_name in self.path2premises.get(p.path, ())

    def __len__(self) -> int:
        return sum(len(v) for v in self.path2premises.values())


@dataclass(frozen=True)
class File:
    """One `*.lean` file and the premises it defines (reference common.py:141-178)."""

    path: str
    premises: List[Premise] = field(repr=False, compare=False)

    @classmethod
    def from_data(cls, file_data: Dict[str, Any]) -> "File":
        path = file_data["path"]
        kept: List[Premise] = []
        for rec in file_data["premises"]:
            name = rec["full_name"]
            if name is None:
                continue
            if "user__.n" in name or rec["code"] == "":
                continue  # ill-formed (AST errors)
            if name.startswith("[") and name.endswith("]"):
                continue  # mutual definitions
            kept.append(Premise(path, name, Pos(*rec["start"]), Pos(*rec["end"]), rec["code"]))
        return cls(path, kept)

    @property
    def is_empty(self) -> bool:
        return len(self.premises) == 0


class Corpus:
    """A DAG of files; every file owns a contiguous slice of `all_premises`.

    Construct from a `corpus.jsonl` path (reference common.py:195-219) or from an
    in-memory list of `(File, imports)` with `Corpus.from_files` (used for synthetic
    corpora).  Files must appear after the files they import.
    """

    def __init__(self, jsonl_path: Optional[str] = None) -> None:
        self.all_premises: List[Premise] = []
        self._files: Dict[str, File] = {}
        self._range: Dict[str, Tuple[int, int]] = {}
        # transitive imports as bit sets over the files' insertion order (bit i = self._order[i]):
        # a Python int per file keeps a mathlib-sized import closure (5 k files, each importing most
        # of its predecessors) at ~3 MB and a union at one big-int OR, where sets of path strings
        # cost ~200 MB and quadratic time
        self._order: List[str] = []
        self._index: Dict[str, int] = {}
        self._dep_bits: Dict[str, int] = {}
        self.imported_premises_cache: Dict[str, List[Premise]] = {}
        if jsonl_path is not None:
            with open(jsonl_path) as fh:
                for line in fh:
                    data = json.loads(line)
                    self._add_file(File.from_data(data), data["imports"])

    def __getstate__(self):
        state = dict(self.__dict__)
        state.pop("_import_words_cache", None)  # derived data: keep index pickles lean
        state.pop("_recent_masks", None)
        state.pop("_recent_masks_dev", None)
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        if "_dep_bits" not in state:  # pickles written before the bit-set representation
            self._order = list(self._files)
            self._index = {p: i for i, p in enumerate(self._order)}
            old = state.get("_deps", {})
            self._dep_bits = {p: sum(1 << self._index[d] for d in old.get(p, ())) for p in self._order}
            self.__dict__.pop("_deps", None)

    def _dep_paths(self, path: str) -> Generator[str, None, None]:
        """Files `path` imports (transitively), in corpus order."""
        bits = self._dep_bits[path]
        while bits:
            low = bits & -bits
            yield self._order[low.bit_length() - 1]
            bits ^= low

    @classmethod
    def from_files(cls, files: Iterable[Tuple[File, Iterable[str]]]) -> "Corpus":
        c = cls()
        for f, imports in files:
            c._add_file(f, list(imports))
        return c

    def _add_file(self, f: File, imports: List[str]) -> None:
        assert f.path not in self._files, f"duplicate file {f.path}"
        closure = 0
        for imp in imports:
            assert imp in self._files, f"{f.path} imports {imp} before it is defined"
            closure |= (1 << self._index[imp]) | self._dep_bits[imp]
        lo = len(self.all_premises)
        self.all_premises.extend(f.premises)
        self._files[f.path] = f
        self._range[f.path] = (lo, len(self.all_premises))
        self._index[f.path] = len(self._order)
        self._order.append(f.path)
        self._dep_bits[f.path] = closure

    # ---- reference-compatible accessors ------------------------------------------------
    def _get_file(self, path: str) -> File:
        return self._files[path]

    def __len__(self) -> int:
        return len(self.all_premises)

    def __contains__(self, path: str) -> bool:
        return path in self._files

    def __getitem__(self, idx: int) -> Premise:
        return self.all_premises[idx]

    @property
    def files(self) -> List[File]:
        return list(self._files.values())

    @property
    def num_files(self) -> int:
        return len(self._files)

    def get_dependencies(self, path: str) -> List[str]:
        return list(self._dep_paths(path))

    def get_premises(self, path: str) -> List[Premise]:
        return self._files[path].premises

    def num_premises(self, path: str) -> int:
        return len(self._files[path].premises)

    def locate_premise(self, path: str, pos: Any) -> Optional[Premise]:
        pos = Pos.from_any(pos)
        for p in self.get_premises(path):
            if p.start <= pos <= p.end:
                return p
        return None

    def fill_cache(self) -> None:
        for path in self._files:
            self._get_imported_premises(path)

    def _get_imported_premises(self, path: str) -> List[Premise]:
        cached = self.imported_premises_cache.get(path)
        if cached is None:
            cached = []
            for dep in self.get_dependencies(path):
                cached.extend(self._files[dep].premises)
            self.imported_premises_cache[path] = cached
        return cached

    def get_accessible_premises(self, path: str, pos: Any) -> PremiseSet:
        """Premises visible at `pos` in `path`: earlier in the file, or (transitively) imported."""
        pos = Pos.from_any(pos)
        out = PremiseSet()
        for p in self.get_premises(path):
            if p.end <= pos:
                out.add(p)
        out.update(self._get_imported_premises(path))
        return out

    def get_accessible_premise_indexes(self, path: str, pos: Any) -> List[int]:
        pos = Pos.from_any(pos)
        lo, hi = self._range[path]
        idx = [i for i in range(lo, hi) if self.all_premises[i].end <= pos]
        for dep in self.get_dependencies(path):
            a, b = self._range[dep]
            idx.extend(range(a, b))
        return sorted(idx)

    # ---- access mask for the device kernel -----------------------------------------------
    def file_range(self, path: str) -> Tuple[int, int]:
        """[lo, hi) slice of `all_premises` owned by `path`."""
        return self._range[path]

    def accessible_mask(self, path: str, pos: Any) -> np.ndarray:
        """Boolean [N] array, True where `all_premises[i] in get_accessible_premises(path, pos)`.

        Membership in the reference is by (path, full_name) (PremiseSet.__contains__), so
        a later same-named duplicate of an accessible premise also tests True; this is
        reproduced here so that the masked device top-k equals the reference walk
        (common.py:313-322) exactly.
        """
        pos = Pos.from_any(pos)
        mask = np.zeros(len(self.all_premises), dtype=bool)
        for dep in self._dep_paths(path):
            a, b = self._range[dep]
            mask[a:b] = True
        lo, hi = self._range[path]
        visible_names = {p.full_name for p in self.all_premises[lo:hi] if p.end <= pos}
        if visible_names:
            for i in range(lo, hi):
                if self.all_premises[i].full_name in visible_names:
                    mask[i] = True
        return mask

    def _import_mask_words(self, path: str) -> np.ndarray:
        """Packed bitmask of the premises `path` imports (transitively); cached per file, like the
        reference's `imported_premises_cache` (common.py:265-278)."""
        cache = self.__dict__.setdefault("_import_words_cache", {})
        words = cache.get(path)
        if words is None or len(words) != (len(self.all_premises) + 31) // 32:
            # files are contiguous in all_premises: expand the file-level bit set by the file sizes
            sizes = cache.get(None)
            if sizes is None or len(sizes) != len(self._order):
                sizes = np.fromiter((len(self._files[p].premises) for p in self._order), dtype=np.int64,
                                    count=len(self._order))
                cache.clear()
                cache[None] = sizes
            nbytes = (len(self._order) + 7) // 8
            file_bits = np.unpackbits(np.frombuffer(self._dep_bits[path].to_bytes(nbytes, "little"), dtype=np.uint8),
                                      bitorder="little")[: len(self._order)].astype(bool)
            mask = np.zeros((len(self.all_premises) + 31) // 32 * 32, dtype=bool)
            mask[: len(self.all_premises)] = np.repeat(file_bits, sizes)
            words = np.packbits(mask.reshape(-1, 8), axis=1, bitorder="little").reshape(-1).view("<u4").copy()
            cache[path] = words
        return words

    def accessible_mask_words(self, path: str, pos: Any) -> np.ndarray:
        """`accessible_mask` packed little-endian into uint32 words (bit i&31 of word i>>5).
        Per query only the own-file prefix is recomputed; the imports part comes from a per-file cache."""
        pos = Pos.from_any(pos)
        # proof search asks for the same (file, theorem position) over and over (one theorem, many states):
        # keep the last few masks
        recent = self.__dict__.setdefault("_recent_masks", {})
        key = (path, pos.line_nb, pos.column_nb)
        hit = recent.get(key)
        if hit is not None and len(hit) == (len(self.all_premises) + 31) // 32:
            return hit
        words = self._import_mask_words(path).copy()
        lo, hi = self._range[path]
        own = self.all_premises[lo:hi]
        visible_names = {p.full_name for p in own if p.end <= pos}
        if visible_names:
            for i, p in enumerate(own, start=lo):
                if p.full_name in visible_names:
                    words[i >> 5] |= np.uint32(1 << (i & 31))
        if len(recent) >= 32:
            recent.pop(next(iter(recent)))
        recent[key] = words
        return words

    def accessible_index_mask_words(self, path: str, pos: Any) -> np.ndarray:
        """The bits of `get_accessible_premise_indexes(path, pos)` in `accessible_mask_words`' layout: premises of the
        (transitively) imported files and premises of `path` that end at or before `pos`, chosen by index.  Unlike
        `accessible_mask_words` it does not add same-named duplicates of visible premises; this is the set the
        reference's BM25 script ranks (retrieval/bm25/main.py:38-40)."""
        pos = Pos.from_any(pos)
        words = self._import_mask_words(path).copy()
        lo, hi = self._range[path]
        for i in range(lo, hi):
            if self.all_premises[i].end <= pos:
                words[i >> 5] |= np.uint32(1 << (i & 31))
        return words

    def accessible_mask_words_range(self, path: str, pos: Any, lo: int, hi: int) -> np.ndarray:
        """The bits [lo, hi) of `accessible_mask_words`, re-packed from bit 0: the bitmask a rank that owns
        rows [lo, hi) of a row-sharded index hands to `rpx_sim_topk` (bit i <=> global row lo + i)."""
        assert 0 <= lo <= hi <= len(self.all_premises)
        words = self.accessible_mask_words(path, pos)
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")[lo:hi]
        padded = np.zeros((hi - lo + 31) // 32 * 32, dtype=np.uint8)
        padded[: hi - lo] = bits
        return np.packbits(padded.reshape(-1, 8), axis=1, bitorder="little").reshape(-1).view("<u4").copy()

    # ---- nearest-neighbour search (signature of reference common.py:299-305) ---------------
    def get_nearest_premises(self, premise_embeddings, batch_context: List[Context], batch_context_emb, k: int):
        """k accessible premises with the highest similarity for every context, best first.

        Same contract as the reference: returns `(List[List[Premise]], List[List[float]])`
        and raises `ValueError` when a context has fewer than `k` accessible premises.
        The matmul and the ranking run in `rpx_sim_topk` on the GPU with the per-query
        accessibility bitmask applied inside the kernel.
        """
        from .retrieval_ops import nearest_premises_device

        return nearest_premises_device(self, premise_embeddings, batch_context, batch_context_emb, k)


@dataclass(frozen=True)
class IndexedCorpus:
    """A corpus plus its premise embeddings: the on-disk index (reference common.py:329-338).

    `embeddings` is a CPU fp32 torch tensor [len(corpus), d_model]; row i belongs to
    `corpus.all_premises[i]`.
    """

    corpus: Corpus
    embeddings: Any

    def __post_init__(self) -> None:
        import torch

        assert self.embeddings.device == torch.device("cpu")
        assert len(self.embeddings) == len(self.corpus)
