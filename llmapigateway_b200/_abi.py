"""ctypes mirror of include/llmgw_b200.h (structs, enums) and value decoding helpers."""
from __future__ import annotations

import ctypes as C
import struct

KIND_ABSENT, KIND_INT, KIND_FLOAT, KIND_NULL, KIND_TRUE, KIND_FALSE, KIND_STR, KIND_BIGINT, KIND_OBJECT, KIND_ARRAY, KIND_FLOAT_INEXACT = range(11)
PHASE_FREE, PHASE_PRIMING, PHASE_COMMITTED, PHASE_FAILED = range(4)
VERDICT_NONE, VERDICT_OK, VERDICT_FAIL_EVENT, VERDICT_FAIL_PARSE, VERDICT_FAIL_HTTP = range(5)
SF_A_USAGE_BOUND, SF_EMITTED_ANY, SF_CARRY_OVERFLOW, SF_EXOTIC_SEEN, SF_SYNCED, SF_REC_VALID, SF_DETAIL_TRUNC, SF_ROWQ_OVERFLOW, SF_PENDING = (1 << i for i in range(9))

# TopKey | PartFlag bits returned by the part parser (json_machine.cuh)
TK_ERROR, TK_DETAIL, TK_CODE, TK_USAGE, TK_CHOICES, TK_MODEL, TK_PROVIDER = (1 << i for i in range(7))
PF_VALID_A, PF_VALID_B, PF_TYPE_ERROR, PF_EXOTIC, PF_TOO_DEEP, PF_CONTENT = (1 << i for i in range(8, 14))

STR_CAP = 120


class Val(C.Structure):
    _fields_ = [("bits", C.c_int64), ("kind", C.c_uint8), ("_pad", C.c_uint8 * 7)]


class UsageRec(C.Structure):
    _fields_ = [("prompt_tokens", Val), ("completion_tokens", Val), ("total_tokens", Val),
                ("reasoning_tokens", Val), ("cached_tokens", Val), ("cost", Val),
                ("model_val", Val), ("provider_val", Val),
                ("model_len", C.c_uint8), ("provider_len", C.c_uint8), ("str_flags", C.c_uint8), ("exotic", C.c_uint8),
                ("model", C.c_char * STR_CAP), ("provider", C.c_char * STR_CAP)]


class StreamState(C.Structure):
    _fields_ = [("phase", C.c_uint8), ("verdict", C.c_uint8), ("flags", C.c_uint16),
                ("carry_a_len", C.c_uint32), ("carry_b_len", C.c_uint32), ("detail_len", C.c_uint32),
                ("n_events_a", C.c_uint32), ("n_events_b", C.c_uint32), ("n_usage_b", C.c_uint32),
                ("n_exotic", C.c_uint32), ("n_error_rows", C.c_uint32),
                ("n_chunks_in", C.c_uint32), ("n_chunks_emitted", C.c_uint32), ("pending_len", C.c_uint32),
                ("bytes_in", C.c_uint64), ("bytes_emitted", C.c_uint64), ("rec", UsageRec)]


class RowEvent(C.Structure):
    _fields_ = [("slot", C.c_uint32), ("seq", C.c_uint32), ("rec", UsageRec)]


class TextMark(C.Structure):
    """lgw_text_mark: a mid-stream write_log call (chat_logging.py:139): the transcript written there is the stream's text[:text_pos]."""
    _fields_ = [("slot", C.c_uint32), ("seq", C.c_uint32), ("text_pos", C.c_uint64)]


TF_LONE_SURROGATE, TF_EXOTIC, TF_CARRY_OVERFLOW, TF_MARKQ_OVERFLOW, TF_SEQUENTIAL = 1, 2, 4, 8, 16
TF_DOC_ERROR_LOG = 32          # lgw_documents_text: the document's top-level "error" made write_log run at chat_logging.py:139 too


class SegResult(C.Structure):
    _fields_ = [("emit_chunk_begin", C.c_uint32), ("phase", C.c_uint8), ("verdict", C.c_uint8),
                ("flags", C.c_uint16), ("detail_len", C.c_uint32)]


class DocUsage(C.Structure):
    _fields_ = [("flags", C.c_uint32), ("rec_valid", C.c_uint8), ("error_row", C.c_uint8), ("exotic", C.c_uint8), ("_pad", C.c_uint8), ("rec", UsageRec)]


class Limits(C.Structure):
    _fields_ = [("max_streams", C.c_uint32), ("carry_cap", C.c_uint32), ("detail_cap", C.c_uint32),
                ("rowq_cap", C.c_uint32), ("max_step_chunks", C.c_uint32), ("max_step_bytes", C.c_uint64)]


class Unrepresentable:
    """A JSON value the device reports but cannot carry (big integer, string where a number
    belongs, container ...).  Only its kind is known."""

    def __init__(self, kind: int):
        self.kind = kind

    def __repr__(self):
        return f"Unrepresentable(kind={self.kind})"


def val_to_py(v: Val):
    k = v.kind
    if k == KIND_INT:
        return int(v.bits)
    if k == KIND_FLOAT:
        return struct.unpack("<d", struct.pack("<q", v.bits))[0]
    if k == KIND_NULL:
        return None
    if k == KIND_TRUE:
        return True
    if k == KIND_FALSE:
        return False
    return Unrepresentable(k)


def _rec_text(rec: UsageRec, field: str, n: int) -> str:
    raw = C.string_at(C.addressof(rec) + getattr(UsageRec, field).offset, n)
    return raw.decode("utf-8", errors="surrogatepass")


def usage_rec_to_dict(rec: UsageRec) -> dict:
    """The dict chat_logging.py:233-272 (get_token_usage) would have returned."""
    out = {name: val_to_py(getattr(rec, name)) for name in
           ("prompt_tokens", "completion_tokens", "total_tokens", "reasoning_tokens", "cached_tokens", "cost")}
    for name, val, ln, shift in (("provider", rec.provider_val, rec.provider_len, 2), ("model", rec.model_val, rec.model_len, 0)):
        if val.kind == KIND_ABSENT:
            continue
        if val.kind == KIND_STR and (rec.str_flags >> shift) & 3:      # truncated / lone surrogate: reported, not guessed
            out[name] = Unrepresentable(KIND_STR)
        else:
            out[name] = _rec_text(rec, name, ln) if val.kind == KIND_STR else val_to_py(val)
    return out


class DocError(C.Structure):          # == lgw_doc_error
    _fields_ = [("result", C.c_uint8), ("error_kind", C.c_uint8), ("message_kind", C.c_uint8), ("detail_kind", C.c_uint8), ("text_len", C.c_uint32)]


EDR_NONE, EDR_TEXT, EDR_TRUE, EDR_FALSE, EDR_ERROR_NOT_OBJECT, EDR_EXOTIC, EDR_ZERO = range(7)
ED_TYPE_NAMES = {1: "str", 2: "NoneType", 3: "bool", 4: "bool", 5: "int", 6: "int", 9: "list", 10: "list"}   # (numbers: int or float, see responses.py)
