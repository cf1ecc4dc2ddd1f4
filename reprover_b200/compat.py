"""Reading indexes written by the *reference* (`retrieval/index.py:37-40`).

A reference index is a pickle of `common.IndexedCorpus(corpus: common.Corpus, embeddings)`, where
`common.Corpus` holds a networkx `transitive_dep_graph` (node attribute "file" = `common.File`) and
`all_premises` of `common.Premise` with `lean_dojo.Pos` positions (common.py:181-219).  Neither
`common` nor `lean_dojo` is importable next to this package, so the unpickler below maps those
classes onto light stand-ins and rebuilds a `reprover_b200.corpus.Corpus` (file order = order of
first appearance in `all_premises`, then remaining nodes; imports = graph successors, which are
already transitive).  networkx must be importable to decode the graph object itself.
"""
from __future__ import annotations

import io
import pickle
from typing import Any, Dict, List

from .corpus import Corpus, File, IndexedCorpus, Pos, Premise


class _Bag:
    """Stand-in that just records the pickled attribute dict."""

    def __setstate__(self, state):
        if isinstance(state, tuple) and len(state) == 2 and isinstance(state[1], dict):  # dataclass with slots
            state = {**(state[0] or {}), **state[1]}
        self.__dict__.update(state)


class _RefPos(_Bag):
    pass


class _RefPremise(_Bag):
    pass


class _RefFile(_Bag):
    pass


class _RefCorpus(_Bag):
    pass


class _RefIndexedCorpus(_Bag):
    pass


class _RefContext(_Bag):
    pass


_MAP = {
    ("common", "IndexedCorpus"): _RefIndexedCorpus,
    ("common", "Corpus"): _RefCorpus,
    ("common", "File"): _RefFile,
    ("common", "Premise"): _RefPremise,
    ("common", "Context"): _RefContext,
}


class _Unpickler(pickle.Unpickler):
    def find_class(self, module: str, name: str):
        if (module, name) in _MAP:
            return _MAP[(module, name)]
        if name == "Pos" and module.split(".")[0] == "lean_dojo":
            return _RefPos
        return super().find_class(module, name)


def _pos(p: Any) -> Pos:
    return Pos(int(p.line_nb), int(p.column_nb))


def _premise(p: Any) -> Premise:
    return Premise(p.path, p.full_name, _pos(p.start), _pos(p.end), p.code)


def _file_order(ref: Any) -> List[str]:
    """File order for the converted corpus: every file after the files it imports, and the files that
    hold premises in the order `all_premises` lists them.

    The reference adds graph nodes in `corpus.jsonl` order, which is an import order (it asserts that every
    import is already a node, common.py:211-213), and networkx keeps insertion order through
    `transitive_closure_dag` — so the graph's own node order is the natural choice and also places files
    WITHOUT premises (which `all_premises` cannot reveal) correctly.  If a pickle's node order has been
    disturbed, fall back to a topological order that keeps the premise-bearing files in sequence."""
    g = ref.transitive_dep_graph
    nodes = list(g.nodes)
    rank = {path: i for i, path in enumerate(nodes)}
    if all(rank[dep] < rank[path] for path in nodes for dep in g.successors(path)):
        return nodes
    seen, with_premises = set(), []
    for p in ref.all_premises:
        if p.path not in seen:
            seen.add(p.path)
            with_premises.append(p.path)
    order: List[str] = []
    placed = set()

    def place(path: str, stack: tuple) -> None:
        if path in placed:
            return
        if path in stack:
            raise ValueError(f"reference corpus has an import cycle through {path}")
        for dep in g.successors(path):        # imports first (empty files are pulled in here)
            place(dep, stack + (path,))
        placed.add(path)
        order.append(path)

    for path in with_premises + [n for n in nodes if n not in seen]:
        place(path, ())
    return order


def convert_corpus(ref: Any) -> Corpus:
    """`common.Corpus` (the reference's own object or the unpickler's stand-in) ->
    `reprover_b200.corpus.Corpus` with the same `all_premises` order."""
    g = ref.transitive_dep_graph
    files = []
    for path in _file_order(ref):
        premises = [_premise(p) for p in g.nodes[path]["file"].premises]
        files.append((File(path, premises), list(g.successors(path))))
    corpus = Corpus.from_files(files)
    got = [(p.path, p.full_name, p.start) for p in corpus.all_premises]
    want = [(p.path, p.full_name, _pos(p.start)) for p in ref.all_premises]
    if got != want:
        raise ValueError("converted corpus does not reproduce the reference's all_premises order")
    return corpus


def load_reference_index(path_or_bytes) -> IndexedCorpus:
    """Load an `IndexedCorpus` pickle produced by the reference and convert it."""
    if isinstance(path_or_bytes, (bytes, bytearray)):
        fh = io.BytesIO(path_or_bytes)
    else:
        fh = open(path_or_bytes, "rb")
    with fh:
        ref = _Unpickler(fh).load()
    return IndexedCorpus(convert_corpus(ref.corpus), ref.embeddings)


def load_reference_predictions(path_or_bytes) -> List[Dict[str, Any]]:
    """Load a retrieval predictions pickle in the reference's layout (`dump_reference_predictions`, or the reference's
    own `predictions.pickle`) with `context` as `reprover_b200.corpus.Context` and premises as `Premise`."""
    from .corpus import Context

    fh = io.BytesIO(path_or_bytes) if isinstance(path_or_bytes, (bytes, bytearray)) else open(path_or_bytes, "rb")
    with fh:
        ref = _Unpickler(fh).load()
    conv: Dict[int, Premise] = {}

    def premise(p: Any) -> Premise:
        q = conv.get(id(p))
        if q is None:
            q = conv[id(p)] = _premise(p)
        return q

    out = []
    for rec in ref:
        c = rec["context"]
        out.append({**rec, "context": Context(c.path, c.theorem_full_name, _pos(c.theorem_pos), c.state),
                    "all_pos_premises": [premise(p) for p in rec["all_pos_premises"]],
                    "retrieved_premises": [premise(p) for p in rec["retrieved_premises"]]})
    return out


# ------------------------------------------------------------------------------------------ export
# The other direction: an index built by this engine, written so that a STOCK checkout of the
# reference loads it — `pickle.load` at retrieval/model.py:81-85 must find `common.IndexedCorpus`,
# `common.Corpus` (attributes `transitive_dep_graph`: networkx DiGraph, transitive closure, node
# attribute "file"; `all_premises`; `imported_premises_cache`, common.py:181-224), `common.File`,
# `common.Premise` and `lean_dojo.Pos` (`from lean_dojo import Pos`, common.py:14), with fp32 CPU
# embeddings (common.py:336-338).  When this process runs inside the reference tree the real classes
# are used; otherwise stand-ins are registered under those module names for the duration of the dump
# (pickle stores classes by module + qualified name, and instances as NEWOBJ + attribute dict, which is
# what the reference's dataclasses produce).
import contextlib
import sys
import types


def _stand_in(module: str, name: str) -> type:
    cls = type(name, (), {})
    cls.__module__, cls.__qualname__ = module, name
    return cls


_COMMON_CLASSES = ("IndexedCorpus", "Corpus", "File", "Premise", "Context")


@contextlib.contextmanager
def _reference_classes():
    """Yield {"IndexedCorpus", "Corpus", "File", "Premise", "Context", "Pos"} -> classes that pickle under the
    reference's names."""
    common = sys.modules.get("common")
    lean_dojo = sys.modules.get("lean_dojo")
    if (common is not None and lean_dojo is not None and hasattr(lean_dojo, "Pos")
            and all(hasattr(common, n) for n in _COMMON_CLASSES)):
        yield {n: getattr(common, n) for n in _COMMON_CLASSES} | {"Pos": lean_dojo.Pos}
        return
    added = []
    try:
        classes = {n: _stand_in("common", n) for n in _COMMON_CLASSES}
        classes["Pos"] = _stand_in("lean_dojo", "Pos")
        for mod_name, names in (("common", _COMMON_CLASSES), ("lean_dojo", ("Pos",))):
            if mod_name in sys.modules:
                raise RuntimeError(f"a module named {mod_name!r} that is not the reference's is loaded; cannot write "
                                   f"the reference index layout from this process")
            m = types.ModuleType(mod_name)
            for n in names:
                setattr(m, n, classes[n])
            sys.modules[mod_name] = m
            added.append(mod_name)
        yield classes
    finally:
        for mod_name in added:
            sys.modules.pop(mod_name, None)


def _raw(cls: type, **attrs) -> Any:
    """An instance of `cls` with exactly these attributes, bypassing __init__ / frozen dataclasses."""
    obj = object.__new__(cls)
    obj.__dict__.update(attrs)
    return obj


def _ref_pos(ref: Dict[str, type], p: Pos) -> Any:
    return _raw(ref["Pos"], line_nb=int(p.line_nb), column_nb=int(p.column_nb))


def _ref_premise(ref: Dict[str, type], p: Premise) -> Any:
    return _raw(ref["Premise"], path=p.path, full_name=p.full_name, start=_ref_pos(ref, p.start),
                end=_ref_pos(ref, p.end), code=p.code)


def dump_reference_index(corpus: Corpus, embeddings, fh) -> None:
    """Write `IndexedCorpus(corpus, embeddings)` to the binary file `fh` in the reference's layout."""
    import networkx as nx
    import torch

    emb = embeddings.detach().to(torch.float32).cpu().contiguous()
    assert emb.shape[0] == len(corpus), "one embedding row per premise"
    with _reference_classes() as ref:
        conv = {}

        def premise(p: Premise):
            q = conv.get(id(p))
            if q is None:
                q = _ref_premise(ref, p)
                conv[id(p)] = q
            return q

        g = nx.DiGraph()
        for f in corpus.files:
            g.add_node(f.path, file=_raw(ref["File"], path=f.path, premises=[premise(p) for p in f.premises]))
        for f in corpus.files:
            for dep in corpus.get_dependencies(f.path):    # already the transitive closure
                g.add_edge(f.path, dep)
        # `imported_premises_cache` is filled lazily by the reference (common.py:262-273): an empty one is a
        # valid state and keeps a mathlib-sized pickle from carrying every file's transitive premise list
        ref_corpus = _raw(ref["Corpus"], transitive_dep_graph=g, all_premises=[premise(p) for p in corpus.all_premises],
                          imported_premises_cache={})
        pickle.dump(_raw(ref["IndexedCorpus"], corpus=ref_corpus, embeddings=emb), fh, protocol=4)


def dump_reference_predictions(preds: List[Dict[str, Any]], fh) -> None:
    """Write retrieval predictions (the records of the reference's BM25 script, retrieval/bm25/main.py:55-67) to the
    binary file `fh` with `context` as `common.Context`, premises as `common.Premise` and positions as `lean_dojo.Pos`,
    so that the reference's `retrieval/evaluate.py` and `generation/datamodule.py` load them."""
    with _reference_classes() as ref:
        conv: Dict[int, Any] = {}

        def premise(p: Premise):
            q = conv.get(id(p))
            if q is None:
                q = conv[id(p)] = _ref_premise(ref, p)
            return q

        out = []
        for rec in preds:
            ctx = rec["context"]
            out.append({**rec,
                        "context": _raw(ref["Context"], path=ctx.path, theorem_full_name=ctx.theorem_full_name,
                                        theorem_pos=_ref_pos(ref, ctx.theorem_pos), state=ctx.state),
                        "all_pos_premises": [premise(p) for p in rec["all_pos_premises"]],
                        "retrieved_premises": [premise(p) for p in rec["retrieved_premises"]]})
        pickle.dump(out, fh)
