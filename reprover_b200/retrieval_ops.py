"""Similarity + top-k on the GPU through the C ABI (`rpx_index_*`, `rpx_topk_merge*`).

`nearest_premises_device` is the body of `Corpus.get_nearest_premises` (reference
common.py:299-326): the matmul, the ranking and the accessibility filter run in one
device pass; only k (index, score) pairs per query come back to the host.

`IndexHandle` stands where the reference keeps `self.corpus_embeddings`
(retrieval/model.py:190, 363-366): a bf16 [N, D] matrix on the device plus the small
device state the engine derives from it once (row-norm bound of the exactness guard).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from . import _native

_ws_cache = {}


def _workspace(device: torch.device, nbytes: int) -> torch.Tensor:
    ws = _ws_cache.get(device)
    if ws is None or ws.numel() < nbytes:
        _ws_cache[device] = None
        ws = torch.empty(nbytes + 4096, dtype=torch.uint8, device=device)
        _ws_cache[device] = ws
    return ws


class IndexHandle:
    """`rpx_index` over a bf16 [N, D] CUDA tensor.  Keeps the tensor alive; re-create after the
    tensor's contents change (`for_tensor` does that by itself through the tensor's version counter)."""

    def __init__(self, embeddings: torch.Tensor) -> None:
        if embeddings.device.type != "cuda":
            raise RuntimeError("the index lives on a CUDA device only (no CPU path in this engine)")
        if embeddings.dtype != torch.bfloat16 or embeddings.dim() != 2:
            raise TypeError("the index is a 2-D bf16 matrix (the dtype the reference's GPU path holds it in)")
        self.lib = _native.load()
        self.embeddings = embeddings.contiguous()
        self.device = embeddings.device
        self.n, self.d = int(self.embeddings.shape[0]), int(self.embeddings.shape[1])
        self._version = embeddings._version
        self._state = torch.empty(int(self.lib.rpx_index_state_bytes()), dtype=torch.uint8, device=self.device)
        self._handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _native.check(self.lib.rpx_index_create(
                self.embeddings.data_ptr() if self.n else None, self.n, self.d, self._state.data_ptr(),
                torch.cuda.current_stream(self.device).cuda_stream, C.byref(self._handle)))

    def close(self) -> None:
        if getattr(self, "_handle", None) is not None and self._handle.value:
            self.lib.rpx_index_destroy(self._handle)
            self._handle = C.c_void_p()

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def stats(self) -> Dict[str, float]:
        """Guard diagnostics (synchronises): row-norm bound, largest |fp32 - fp64| score difference and
        largest epsilon a guard has seen, number of queries that took the exact pass."""
        nm, er, ep, nx = C.c_float(), C.c_float(), C.c_float(), C.c_int64()
        with torch.cuda.device(self.device):
            _native.check(self.lib.rpx_index_stats(self._handle, torch.cuda.current_stream(self.device).cuda_stream,
                                                   C.byref(nm), C.byref(er), C.byref(ep), C.byref(nx)))
        return {"norm_max": nm.value, "max_err": er.value, "max_eps": ep.value, "n_exact": int(nx.value)}

    # one handle per live tensor (keyed by storage address + shape, validated by the version counter)
    _cache: "Dict[tuple, IndexHandle]" = {}

    @classmethod
    def for_tensor(cls, embeddings: torch.Tensor) -> "IndexHandle":
        emb = embeddings if embeddings.is_contiguous() else embeddings.contiguous()
        key = (emb.device.index, emb.data_ptr(), tuple(emb.shape))
        h = cls._cache.get(key)
        if h is not None and h._version == emb._version and h.embeddings.data_ptr() == emb.data_ptr():
            return h
        if h is not None:
            h.close()
        if len(cls._cache) >= 4:   # a process holds a handful of indexes; do not pin old ones forever
            cls._cache.pop(next(iter(cls._cache))).close()
        h = cls(emb)
        cls._cache[key] = h
        return h


def _check_k(k: int) -> None:
    if not isinstance(k, (int, np.integer)) or k < 1 or k > _native.TOPK_MAX_K:
        raise ValueError(f"k={k}: the engine returns between 1 and {_native.TOPK_MAX_K} premises per query "
                         f"(k <= 200 on the fast paths, larger k through the exact pass)")


def sim_topk(queries: torch.Tensor, index: Union[torch.Tensor, IndexHandle], k: int,
             access_mask: Optional[torch.Tensor] = None, idx_offset: int = 0, want_scores64: bool = False,
             want_packed: bool = False, flags: int = _native.RPX_TOPK_AUTO):
    """Top-k rows of `index` for every row of `queries` (both bf16, same CUDA device).

    Returns (scores fp32 [Q,k], indices int64 [Q,k], counts int32 [Q]) and, with
    `want_scores64`, the fp64 scores as a 4th element; with `want_packed` a last element
    [Q,k,2] int64 of (fp64 score bits, index) records.  Order: score desc, index asc.
    `access_mask`: optional uint32 bitmask [Q, ceil(N/32)] (as int32 tensor) on the device.
    `flags`: `_native.RPX_TOPK_FORCE_*` pins the path (parity tests); 0 = automatic.
    """
    lib = _native.load()
    if queries.device.type != "cuda":
        raise RuntimeError("sim_topk runs on a CUDA device only (no CPU path in this engine)")
    handle = index if isinstance(index, IndexHandle) else None
    if queries.dtype != torch.bfloat16 or (handle is None and index.dtype != torch.bfloat16):
        raise TypeError("sim_topk takes bf16 queries and index (the dtype the reference's GPU path holds them in)")
    if handle is None and index.device != queries.device:
        raise RuntimeError("queries and index must live on the same CUDA device")
    _check_k(k)
    if handle is None:
        handle = IndexHandle.for_tensor(index)
    assert queries.dim() == 2 and queries.shape[1] == handle.d and queries.device == handle.device
    queries = queries.contiguous()
    nq, d = queries.shape
    if nq == 0:
        raise ValueError("sim_topk needs at least one query")
    dev = queries.device
    scores = torch.empty(nq, k, dtype=torch.float32, device=dev)
    idx = torch.empty(nq, k, dtype=torch.int64, device=dev)
    counts = torch.empty(nq, dtype=torch.int32, device=dev)
    scores64 = torch.empty(nq, k, dtype=torch.float64, device=dev) if want_scores64 else None
    packed = torch.empty(nq, k, 2, dtype=torch.int64, device=dev) if want_packed else None
    mask_ptr, stride = None, 0
    if access_mask is not None:
        assert access_mask.device == dev and access_mask.dtype == torch.int32 and access_mask.dim() == 2
        assert access_mask.shape[0] == nq
        access_mask = access_mask.contiguous()
        mask_ptr, stride = access_mask.data_ptr(), access_mask.shape[1]
    with torch.cuda.device(dev):
        need = lib.rpx_index_topk_workspace_bytes(handle.n, d, nq, k)
        if need == 0:
            raise _native.RpxError(_native.RPX_ERR_UNSUPPORTED, _native.last_error())
        ws = _workspace(dev, need)
        _native.check(lib.rpx_index_topk(
            handle._handle, queries.data_ptr(), nq, k, mask_ptr, stride, scores.data_ptr(),
            scores64.data_ptr() if want_scores64 else None, idx.data_ptr(), counts.data_ptr(),
            packed.data_ptr() if want_packed else None, idx_offset, flags, ws.data_ptr(), ws.numel(),
            torch.cuda.current_stream(dev).cuda_stream))
    out = [scores, idx, counts]
    if want_scores64:
        out.append(scores64)
    if want_packed:
        out.append(packed)
    return tuple(out)


def topk_merge(scores64: torch.Tensor, idx: torch.Tensor):
    """Merge [n_parts, Q, k] per-shard results into the global top-k (same ordering contract).

    Returns (scores fp32 [Q,k], idx int64 [Q,k], counts int32 [Q], scores fp64 [Q,k])."""
    lib = _native.load()
    assert scores64.dtype == torch.float64 and idx.dtype == torch.int64 and scores64.shape == idx.shape
    scores64 = scores64.contiguous()
    idx = idx.contiguous()
    n_parts, nq, k = scores64.shape
    dev = scores64.device
    out_s = torch.empty(nq, k, dtype=torch.float32, device=dev)
    out_s64 = torch.empty(nq, k, dtype=torch.float64, device=dev)
    out_i = torch.empty(nq, k, dtype=torch.int64, device=dev)
    out_c = torch.empty(nq, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _native.check(lib.rpx_topk_merge(scores64.data_ptr(), idx.data_ptr(), n_parts, nq, k, out_s.data_ptr(),
                                         out_s64.data_ptr(), out_i.data_ptr(), out_c.data_ptr(),
                                         torch.cuda.current_stream(dev).cuda_stream))
    return out_s, out_i, out_c, out_s64


def topk_merge_packed(packed: torch.Tensor, out: Optional[Tuple[torch.Tensor, ...]] = None):
    """Same merge over the gathered [n_parts, Q, k, 2] (fp64 score bits, index) records that
    `sim_topk(..., want_packed=True)` produces — no un-interleaving copies in between.
    `out`: optional preallocated (scores fp32, idx int64, counts int32, scores fp64) to write into."""
    lib = _native.load()
    assert packed.dtype == torch.int64 and packed.dim() == 4 and packed.shape[-1] == 2 and packed.is_contiguous()
    n_parts, nq, k, _ = packed.shape
    dev = packed.device
    if out is None:
        out = (torch.empty(nq, k, dtype=torch.float32, device=dev), torch.empty(nq, k, dtype=torch.int64, device=dev),
               torch.empty(nq, dtype=torch.int32, device=dev), torch.empty(nq, k, dtype=torch.float64, device=dev))
    out_s, out_i, out_c, out_s64 = out
    with torch.cuda.device(dev):
        _native.check(lib.rpx_topk_merge_packed(packed.data_ptr(), n_parts, nq, k, out_s.data_ptr(), out_s64.data_ptr(),
                                                out_i.data_ptr(), out_c.data_ptr(),
                                                torch.cuda.current_stream(dev).cuda_stream))
    return out_s, out_i, out_c, out_s64


def nearest_premises_device(corpus, premise_embeddings: Union[torch.Tensor, IndexHandle], batch_context,
                            batch_context_emb: torch.Tensor, k: int) -> Tuple[List[list], List[List[float]]]:
    """Reference `Corpus.get_nearest_premises` (common.py:299-326) with the heavy half on the GPU.

    Embeddings are used in bf16 (what the reference's GPU path holds them in,
    retrieval/model.py:59-64, 363-366); fp32 inputs are cast.  Raises ValueError when a
    context has fewer than k accessible premises (common.py:323-324).
    """
    dev = batch_context_emb.device
    if dev.type != "cuda":
        raise RuntimeError("get_nearest_premises needs the embeddings on a CUDA device")
    _check_k(k)
    nq = batch_context_emb.shape[0]
    stage = _result_staging(nq, k)
    nearest_premises_enqueue(corpus, premise_embeddings, batch_context, batch_context_emb, k, stage)
    # one synchronisation for the three results (pinned staging, asynchronous copies)
    torch.cuda.current_stream(dev).synchronize()
    return nearest_premises_collect(corpus, stage, nq, k)


def nearest_premises_enqueue(corpus, premise_embeddings: Union[torch.Tensor, IndexHandle], batch_context,
                             batch_context_emb: torch.Tensor, k: int, stage: Tuple[torch.Tensor, ...]) -> None:
    """The device half of `nearest_premises_device`: access masks, the masked top-k, and asynchronous copies of
    (counts, indices, fp32 scores) into the pinned host buffers `stage` (see `result_staging`).  Returns without
    waiting; the results are valid once the current stream has reached this point."""
    dev = batch_context_emb.device
    if dev.type != "cuda":
        raise RuntimeError("get_nearest_premises needs the embeddings on a CUDA device")
    _check_k(k)
    q = batch_context_emb.to(torch.bfloat16)
    e = premise_embeddings
    if not isinstance(e, IndexHandle):
        if e.device != dev or e.dtype != torch.bfloat16:
            e = e.to(device=dev, dtype=torch.bfloat16)
        n_rows = e.shape[0]
    else:
        n_rows = e.n
    assert len(batch_context) == q.shape[0] and n_rows == len(corpus.all_premises)
    mask = _device_mask(corpus, batch_context, dev)
    scores, idx, counts = sim_topk(q, e, k, access_mask=mask)
    nq = q.shape[0]
    stage[0][:nq].copy_(counts, non_blocking=True)
    stage[1][:nq].copy_(idx, non_blocking=True)
    stage[2][:nq].copy_(scores, non_blocking=True)


def nearest_premises_collect(corpus, stage: Tuple[torch.Tensor, ...], nq: int, k: int):
    """The host half: premises and Python-float scores from the staged results of `nq` queries.  Raises ValueError
    when a query had fewer than k accessible premises (common.py:323-324)."""
    if bool((stage[0][:nq] < k).any()):
        raise ValueError
    idx_h = stage[1][:nq].tolist()
    scores_h = stage[2][:nq].tolist()
    premises = corpus.all_premises
    results = [[premises[i] for i in row] for row in idx_h]
    return results, scores_h


def result_staging(nq: int, k: int) -> Tuple[torch.Tensor, ...]:
    """Fresh pinned host buffers (counts, indices, fp32 scores) for `nq` queries of `nearest_premises_enqueue`."""
    return (torch.empty(nq, dtype=torch.int32, pin_memory=True), torch.empty(nq, k, dtype=torch.int64, pin_memory=True),
            torch.empty(nq, k, dtype=torch.float32, pin_memory=True))


_staging = {}


def _result_staging(nq: int, k: int):
    """Pinned host buffers for (counts, indices, scores) of up to nq queries, reused call after call."""
    st = _staging.get(k)
    if st is None or st[0].shape[0] < nq:
        cap = max(nq, 8)
        st = (torch.empty(cap, dtype=torch.int32).pin_memory(), torch.empty(cap, k, dtype=torch.int64).pin_memory(),
              torch.empty(cap, k, dtype=torch.float32).pin_memory())
        _staging[k] = st
    return st


def _device_mask(corpus, batch_context, dev: torch.device) -> torch.Tensor:
    """[Q, words] int32 access bitmask on the device.  The rows of the last few (file, position) pairs stay
    on the device: proof search retrieves for many states of one theorem, i.e. with the same mask."""
    cache = corpus.__dict__.setdefault("_recent_masks_dev", {})
    rows = []
    for ctx in batch_context:
        pos = ctx.theorem_pos
        key = (ctx.path, pos.line_nb, pos.column_nb, dev.index)
        words = corpus.accessible_mask_words(ctx.path, pos)
        hit = cache.get(key)
        if hit is None or hit[0] is not words:     # (the host array is the cache token: same object, same bits)
            if len(cache) >= 32:
                cache.pop(next(iter(cache)))
            hit = (words, torch.from_numpy(words.view(np.int32)).to(dev))
            cache[key] = hit
        rows.append(hit[1])
    return rows[0].unsqueeze(0) if len(rows) == 1 else torch.stack(rows)
