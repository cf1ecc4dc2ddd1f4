"""Host mirror of the ByT5 tokenizer the reference obtains from `AutoTokenizer`
(retrieval/model.py:44; HF `ByT5Tokenizer`, tokenization_byt5.py).

The engine tokenises on the device (`rpx_encode_bytes`: id = byte + 3, EOS appended,
truncation including the EOS).  That is the whole tokenizer *unless* the text contains
one of the special-token literals, which HF's added-token splitter turns into single
ids (`</s>` -> 1, `<pad>` -> 0, `<unk>` -> 2, `<extra_id_N>` -> 383 - N ... see below)
with whitespace stripping around pad/eos/unk (`AddedToken(lstrip=True, rstrip=True)`,
tokenization_byt5.py:81-85).  `needs_id_path` detects those strings; `encode_ids`
reproduces HF's ids for them so they can be routed through `rpx_encode_ids`.
Pinned against the installed `transformers.ByT5Tokenizer` in tests/test_host_cpu.py.
"""
from __future__ import annotations

import re
from typing import List, Sequence, Tuple

PAD_ID, EOS_ID, UNK_ID = 0, 1, 2
BYTE_OFFSET = 3
NUM_EXTRA_IDS = 125
VOCAB_BYTES = 256

# `<extra_id_i>` ids: HF appends the 125 sentinels after the 259 base ids, in the order
# the list [f"<extra_id_{i}>" for i in range(125)] is added -> id = 259 + i.
_SPECIAL = re.compile(r"</s>|<pad>|<unk>|<extra_id_(?:\d+)>")
_STRIPPING = {"</s>": EOS_ID, "<pad>": PAD_ID, "<unk>": UNK_ID}


def _extra_id(tok: str):
    n = int(tok[len("<extra_id_"):-1])
    # only the canonical spelling (no leading zeros) of 0..124 is a token
    if n < NUM_EXTRA_IDS and tok == f"<extra_id_{n}>":
        return VOCAB_BYTES + BYTE_OFFSET + n
    return None


def needs_id_path(text: str) -> bool:
    """True when `text` holds a special-token literal, i.e. tokenisation != bytes + 3."""
    if "<" not in text:
        return False
    for m in _SPECIAL.finditer(text):
        tok = m.group(0)
        if tok in _STRIPPING or _extra_id(tok) is not None:
            return True
    return False


def _segments(text: str) -> List[Tuple[str, object]]:
    """Split into ('text', str) / ('tok', id, strips) pieces the way HF's trie splitter does
    (leftmost-longest literal match)."""
    out: List[Tuple[str, object]] = []
    pos = 0
    for m in _SPECIAL.finditer(text):
        tok = m.group(0)
        if tok in _STRIPPING:
            tid, strips = _STRIPPING[tok], True
        else:
            tid, strips = _extra_id(tok), False
            if tid is None:
                continue
        if m.start() > pos:
            out.append(("text", text[pos:m.start()]))
        out.append(("tok", (tid, strips)))
        pos = m.end()
    if pos < len(text):
        out.append(("text", text[pos:]))
    return out


def encode_ids(text: str, max_length: int) -> List[int]:
    """ids HF's `tokenizer(text, max_length=max_length, truncation=True)` yields (with the EOS)."""
    segs = _segments(text)
    ids: List[int] = []
    for i, (kind, val) in enumerate(segs):
        if kind == "tok":
            ids.append(val[0])
            continue
        piece: str = val  # type: ignore[assignment]
        # a stripping token (pad/eos/unk) eats the whitespace on both of its sides
        if i + 1 < len(segs) and segs[i + 1][0] == "tok" and segs[i + 1][1][1]:
            piece = piece.rstrip()
        if i > 0 and segs[i - 1][0] == "tok" and segs[i - 1][1][1]:
            piece = piece.lstrip()
        ids.extend(b + BYTE_OFFSET for b in piece.encode("utf-8"))
    ids = ids[: max(max_length - 1, 0)]
    # HF `_add_eos_if_not_present`: no second EOS when the text already ends with one
    if not ids or ids[-1] != EOS_ID:
        ids.append(EOS_ID)
    return ids


def pad_batch(id_lists: Sequence[Sequence[int]]):
    """Right-pad with PAD_ID to the longest (padding="longest"); returns (ids, mask) int64 numpy arrays."""
    import numpy as np

    L = max(len(x) for x in id_lists)
    ids = np.zeros((len(id_lists), L), dtype=np.int64)
    mask = np.zeros((len(id_lists), L), dtype=np.int64)
    for r, x in enumerate(id_lists):
        ids[r, : len(x)] = x
        mask[r, : len(x)] = 1
    return ids, mask


def decode(ids: Sequence[int]) -> str:
    """HF `ByT5Tokenizer.batch_decode(..., skip_special_tokens=True)` of one row: the ids below 3 (pad, EOS, unk) and
    from 259 on (the `<extra_id_N>` sentinels) are dropped, every other id is the byte id - 3, and the bytes are
    decoded as UTF-8 with `errors="ignore"`."""
    data = bytes(int(i) - BYTE_OFFSET for i in ids if BYTE_OFFSET <= int(i) < BYTE_OFFSET + VOCAB_BYTES)
    return data.decode("utf-8", errors="ignore")
