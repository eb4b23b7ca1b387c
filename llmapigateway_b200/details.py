"""The error detail of a failed streaming attempt, as the text the client's 503 carries.

The engine keeps at most `detail_cap` bytes of the failing first event (`save_detail`, stream_machine.cuh) and sets
`SF_DETAIL_TRUNC` when the event was longer.  The reference puts the whole event into the detail
(request_handler.py:51,87, then chat.py:155/185/198), so a truncated one is rebuilt here from the attempt's own chunks, which
the caller still holds.  This is host work on failed attempts only: `detail_cap` stays the memory bound of the common case.
"""
from __future__ import annotations

from . import _abi

_SEP = "\n\n"
_REAL_PREFIX = "data: {"


def first_event(chunks) -> str | None:
    """The first `data: {` piece of an attempt's chunks, the way the priming loop finds it (request_handler.py:74-91): every
    chunk is decoded on its own and dropped when that fails (an empty chunk is never yielded), and the text is split on
    "\\n\\n", the unterminated tail carried into the next chunk.  None when no such piece is complete."""
    carry = ""
    for raw in chunks:
        if not len(raw):
            continue
        try:
            carry += bytes(raw).decode("utf-8")
        except UnicodeDecodeError:
            continue
        pieces = carry.split(_SEP)
        carry = "" if carry.endswith(_SEP) else pieces.pop()
        for piece in pieces:
            if piece.startswith(_REAL_PREFIX):
                return piece
    return None


def attempt_detail(detail: bytes, verdict: int, flags: int, chunks) -> str:
    """The error detail of one failed streaming attempt: the engine's bytes, decoded; the whole first event when the engine
    truncated it (`VERDICT_FAIL_EVENT` with `SF_DETAIL_TRUNC`).  `chunks` = every chunk the attempt fed while priming.
    (A `VERDICT_FAIL_PARSE` detail is cut to 200 characters by its callers, far below `detail_cap`.)"""
    if verdict == _abi.VERDICT_FAIL_EVENT and flags & _abi.SF_DETAIL_TRUNC:
        whole = first_event(chunks)
        if whole is not None:
            return whole
    return bytes(detail).decode("utf-8", errors="replace")
