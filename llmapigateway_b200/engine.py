"""Python face of the engine: thin ctypes calls into the C ABI, numpy in / numpy out.

Mirrors the seams of the reference (SURVEY.md 8(b)):
  Engine.step      <- the per-chunk bodies of request_handler.py:34-63, :69-98, :109-142 and
                      chat_logging.py:90-147 for every stream at once
  Engine.close     <- end of stream: the final tokens_usage row of chat_logging.py:150
  Engine.detail    <- error_detail of a failed attempt (request_handler.py:51,87,98)
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _abi, _native

SEG_DTYPE = np.dtype([("emit_chunk_begin", "<u4"), ("phase", "u1"), ("verdict", "u1"), ("flags", "<u2"), ("detail_len", "<u4")])
assert SEG_DTYPE.itemsize == C.sizeof(_abi.SegResult)


class EngineError(RuntimeError):
    pass


@dataclass
class StepResult:
    out: np.ndarray            # uint8, same size as the input bytes (re-emitted stream)
    segs: np.ndarray           # SEG_DTYPE per segment
    rows: list                 # list[_abi.RowEvent] mid-stream row events

    def keep_mask(self, seg_chunk: np.ndarray, n_chunks: int) -> np.ndarray:
        """Per-chunk keep flags derived from the per-segment suffix rule."""
        keep = np.zeros(n_chunks, dtype=bool)
        for s in range(len(self.segs)):
            keep[int(self.segs["emit_chunk_begin"][s]):int(seg_chunk[s + 1])] = True
        return keep


@dataclass
class StepText:
    """What the transcript tap appended in one step (chat_logging.py:124-139)."""
    text: np.ndarray           # uint8: the appended text of every segment, packed in segment order (UTF-8, surrogates as 'surrogatepass')
    seg_off: np.ndarray        # uint64 [n_segs + 1]: segment s appended text[seg_off[s]:seg_off[s+1]]
    flags: np.ndarray          # uint32 per segment: _abi.TF_* bits
    marks: list                # [(slot, seq, text_pos)] mid-stream write_log calls: transcript = stream text[:text_pos]

    def segment(self, s: int) -> bytes:
        return self.text[int(self.seg_off[s]):int(self.seg_off[s + 1])].tobytes()


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class Engine:
    def __init__(self, device: int = 0, max_streams: int = 8192, carry_cap: int = 65536, detail_cap: int = 4096,
                 rowq_cap: int = 4096, max_step_chunks: int = 1 << 22, max_step_bytes: int = 1 << 28):
        self._lib = _native.load()
        self.limits = _abi.Limits(max_streams, carry_cap, detail_cap, rowq_cap, max_step_chunks, max_step_bytes)
        h = C.c_void_p()
        rc = self._lib.lgw_engine_create(device, C.byref(self.limits), C.byref(h))
        if rc != 0:
            raise EngineError(f"lgw_engine_create failed ({rc}): {self._lib.lgw_last_error(None).decode()}")
        self._h = h
        self.device = device

    # -- plumbing -------------------------------------------------------------------------------
    def _ck(self, rc: int, what: str):
        if rc != 0:
            raise EngineError(f"{what} failed ({rc}): {self._lib.lgw_last_error(self._h).decode()}")

    def close_engine(self):
        if getattr(self, "_h", None):
            self._lib.lgw_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close_engine()
        except Exception:
            pass

    def alloc_pinned(self, nbytes: int) -> np.ndarray:
        """Page-locked host memory (lgw_alloc_pinned) as a uint8 array.  The engine keeps no record of it and closing the
        engine does not free it: it is the caller's until lgw_free_pinned, so arrays that view it stay valid."""
        p = C.c_void_p()
        self._ck(self._lib.lgw_alloc_pinned(self._h, nbytes, C.byref(p)), "alloc_pinned")
        return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p.value))

    def set_stream(self, cuda_stream_ptr: int | None):
        self._ck(self._lib.lgw_engine_set_stream(self._h, C.c_void_p(cuda_stream_ptr or 0)), "set_stream")

    def set_mode(self, mode: int):
        """0: bulk kernel + fix-up (default); 1: exact sequential path only (tests)."""
        self._ck(self._lib.lgw_engine_set_mode(self._h, mode), "set_mode")

    # -- streams ----------------------------------------------------------------------------------
    def open(self, slots, http_status=None):
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        st = np.full(len(slots), 200, dtype=np.int32) if http_status is None else np.ascontiguousarray(http_status, dtype=np.int32)
        self._ck(self._lib.lgw_streams_open(self._h, _ptr(slots), _ptr(st), len(slots)), "streams_open")

    def _states(self, fn, slots):
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        if len(slots) == 0:
            return []
        out = (_abi.StreamState * len(slots))()
        self._ck(fn(self._h, _ptr(slots), len(slots), out), "streams_state")
        return out                            # a ctypes array: len(), indexing and iteration like a list, no per-element views built

    def state(self, slots):
        return self._states(self._lib.lgw_streams_state, slots)

    def close(self, slots):
        return self._states(self._lib.lgw_streams_close, slots)

    def detail(self, slot: int) -> bytes:
        buf = C.create_string_buffer(self.limits.detail_cap)
        n = C.c_uint32(0)
        self._ck(self._lib.lgw_stream_detail(self._h, slot, buf, self.limits.detail_cap, C.byref(n)), "stream_detail")
        return buf.raw[:n.value]

    def details(self, slots, stride: int | None = None) -> list:
        """Error details of many failed attempts in one round trip (lgw_streams_details)."""
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        n = len(slots)
        if n == 0:
            return []
        stride = stride or min(self.limits.detail_cap, 1024)       # (a detail longer than the stride is cut: pass stride=detail_cap for the full text)
        buf = np.empty(n * stride, dtype=np.uint8)
        lens = np.zeros(n, dtype=np.uint32)
        self._ck(self._lib.lgw_streams_details(self._h, _ptr(slots), n, _ptr(buf), stride, _ptr(lens)), "streams_details")
        if int(lens.max()) >= stride and stride < self.limits.detail_cap:        # something was cut: once more with the full capacity
            return self.details(slots, self.limits.detail_cap)
        raw = buf.tobytes()
        return [raw[i * stride:i * stride + int(lens[i])] for i in range(n)]

    # -- the hot path --------------------------------------------------------------------------------
    def step(self, data: np.ndarray, chunk_off: np.ndarray, seg_chunk: np.ndarray, seg_slot: np.ndarray,
             out: np.ndarray | None = None, relay_from_host: bool = False) -> StepResult:
        """Host-buffer step: H2D, kernels, D2H inside the call.  relay_from_host=True: "verdicts only" -- the re-emitted bytes are
        not downloaded; `StepResult.out` is then the caller's own `data` (the relayed bytes are the original bytes at the same
        offsets, request_handler.py:141-142), everything else is the same."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        chunk_off = np.ascontiguousarray(chunk_off, dtype=np.uint32)
        seg_chunk = np.ascontiguousarray(seg_chunk, dtype=np.uint32)
        seg_slot = np.ascontiguousarray(seg_slot, dtype=np.uint32)
        n_bytes, n_chunks, n_segs = data.size, chunk_off.size - 1, seg_slot.size
        if relay_from_host:
            out = None
        elif out is None:
            out = np.empty(max(n_bytes, 1), dtype=np.uint8)
        segs = np.zeros(max(n_segs, 1), dtype=SEG_DTYPE)
        cap = self.limits.rowq_cap
        rows = getattr(self, "_rows_buf", None)
        if rows is None:
            rows = self._rows_buf = (_abi.RowEvent * max(cap, 1))()       # reused from step to step; the events returned are copies
        n_rows = C.c_uint32(0)
        self._last_n_segs = n_segs
        self._ck(self._lib.lgw_sse_step(self._h, _ptr(data), n_bytes, _ptr(chunk_off), n_chunks, _ptr(seg_chunk), _ptr(seg_slot),
                                        n_segs, _ptr(out) if out is not None else None, _ptr(segs), rows, cap, C.byref(n_rows)), "sse_step")
        return StepResult((out if out is not None else data)[:n_bytes], segs[:n_segs], [_abi.RowEvent.from_buffer_copy(rows[i]) for i in range(n_rows.value)])

    def step_device(self, d_data: int, n_bytes: int, d_chunk_off: int, n_chunks: int, d_seg_chunk: int, d_seg_slot: int,
                    n_segs: int, d_out: int, d_segs: int):
        """Device-pointer step (asynchronous on the engine stream)."""
        self._last_n_segs = n_segs
        self._ck(self._lib.lgw_sse_step_device(self._h, d_data, n_bytes, d_chunk_off, n_chunks, d_seg_chunk, d_seg_slot,
                                               n_segs, d_out, d_segs), "sse_step_device")

    def fetch_rows(self):
        cap = self.limits.rowq_cap
        rows = (_abi.RowEvent * max(cap, 1))()
        n_rows = C.c_uint32(0)
        self._ck(self._lib.lgw_fetch_rows(self._h, rows, cap, C.byref(n_rows)), "fetch_rows")
        return [rows[i] for i in range(n_rows.value)]

    # -- transcript tap (SURVEY 8(f) rank 3) -----------------------------------------------------------
    def enable_transcripts(self):
        """Allocate the per-stream transcript tap (the reference taps only with LOG_CHAT_ENABLED, chat_logging.py:166-168);
        streams opened afterwards are tapped."""
        self._ck(self._lib.lgw_transcripts_enable(self._h), "transcripts_enable")
        self._text_on = True

    def step_transcript(self) -> StepText:
        """The text the tap appended for the chunks the LAST step relayed (run once per step, before the next one)."""
        total, n_marks = C.c_uint64(0), C.c_uint32(0)
        self._ck(self._lib.lgw_step_transcript_run(self._h, C.byref(total), C.byref(n_marks)), "step_transcript_run")
        n_segs = self._last_n_segs
        text = np.empty(max(total.value, 1), dtype=np.uint8)
        seg_off = np.zeros(n_segs + 1, dtype=np.uint64)
        flags = np.zeros(max(n_segs, 1), dtype=np.uint32)
        marks = (_abi.TextMark * max(n_marks.value, 1))()
        self._ck(self._lib.lgw_step_transcript_fetch(self._h, _ptr(text), _ptr(seg_off), _ptr(flags), marks), "step_transcript_fetch")
        return StepText(text[:total.value], seg_off, flags[:n_segs], [(marks[i].slot, marks[i].seq, marks[i].text_pos) for i in range(n_marks.value)])

    def transcript_last_ms(self) -> float:
        ms = C.c_float(0)
        self._ck(self._lib.lgw_transcript_last_ms(self._h, C.byref(ms)), "transcript_last_ms")
        return ms.value

    def last_step_direct(self) -> bool:
        """True when the last host-buffer step moved the bytes with the kernel itself (pinned host buffers, no staging copies)."""
        return bool(self._lib.lgw_last_step_direct(self._h))

    def sync(self):
        self._ck(self._lib.lgw_sync(self._h), "sync")

    def last_step_ms(self):
        """Device time of the four kernels of the last step (CUDA events on the launching stream) and of the whole host-buffer call."""
        ms, k = (C.c_float * 4)(), (C.c_float * 4)()
        self._ck(self._lib.lgw_last_step_ms(self._h, C.byref(ms)), "last_step_ms")
        self._ck(self._lib.lgw_last_step_kernel_ms(self._h, C.byref(k)), "last_step_kernel_ms")
        return dict(prime=k[0], relay=k[1], commit=k[2], host_step=ms[3])

    def set_kernel_timing(self, on: bool):
        """True: CUDA events between the kernels of a step (per-kernel times, back-to-back launches); False (default): the kernels
        are chained with programmatic dependent launches and only their total is timed."""
        self._ck(self._lib.lgw_engine_set_kernel_timing(self._h, 1 if on else 0), "set_kernel_timing")

    def debug_counters(self):
        out = (C.c_uint32 * 4)()
        self._ck(self._lib.lgw_debug_counters(self._h, out), "debug_counters")
        return dict(sequential=out[0], bulk=out[1], from_template=out[2], stashed=out[3])

    def launch_count(self) -> int:
        n = C.c_uint64(0)
        self._ck(self._lib.lgw_launch_count(self._h, C.byref(n)), "launch_count")
        return n.value

    # ---- request-body rewrite (rows a1-a4) -------------------------------------------------------
    def load_rules(self, plans) -> None:
        """Upload a compiled plan table (`rewrite.RulePlans`).  chat.py reads the rule dicts per request;
        here they are compiled once per config load."""
        from . import rewrite as rw
        p, o, blob = plans.packed()
        assert p.dtype == rw.PLAN_DTYPE and o.dtype == rw.OP_DTYPE
        self._ck(self._lib.lgw_rules_load(self._h, _ptr(p) if len(p) else None, len(p), _ptr(o) if len(o) else None, len(o),
                                          _ptr(blob), len(blob)), "rules_load")
        self._plan_growth = plans.max_growth()

    def scan_packed(self, buf: np.ndarray, off: np.ndarray, model_cap: int = 256):
        """chat.py:31-45 for n packed bodies: (SCAN_DTYPE[n], uint8 [n, model_cap] model bytes, zero padded)."""
        from . import rewrite as rw
        n = len(off) - 1
        scans = np.zeros(max(n, 1), dtype=rw.SCAN_DTYPE)
        models = np.zeros((max(n, 1), model_cap), dtype=np.uint8)
        self._ck(self._lib.lgw_bodies_scan(self._h, _ptr(buf), _ptr(off), n, model_cap, _ptr(scans), _ptr(models)), "bodies_scan")
        return scans[:n], models[:n]

    def scan_bodies(self, bodies, model_cap: int = 256):
        """chat.py:31-45 for a batch: (SCAN_DTYPE array, list of model bytes)."""
        from . import rewrite as rw
        buf, off = rw.pack_bodies(bodies)
        scans, models = self.scan_packed(buf, off, model_cap)
        lens = np.minimum(scans["model_len"], model_cap)
        return scans, [bytes(models[i, :int(lens[i])]) for i in range(len(bodies))]

    def rewrite_packed(self, buf: np.ndarray, off: np.ndarray, plan_idx: np.ndarray, slot_cap: int, out: np.ndarray | None = None):
        """One upstream attempt for n packed bodies -> (out bytes, out_off[n+1], RESULT_DTYPE[n])."""
        from . import rewrite as rw
        n = len(off) - 1
        plan_idx = np.ascontiguousarray(plan_idx, dtype=np.uint32)
        assert len(plan_idx) == n and off.dtype == np.uint64 and buf.dtype == np.uint8
        if out is None:
            growth = getattr(self, "_plan_growth", 0) + 64
            out = np.empty(min(n * slot_cap, 6 * int(off[n]) + n * growth) + 64, dtype=np.uint8)
        out_off = np.zeros(n + 1, dtype=np.uint64)
        res = np.zeros(max(n, 1), dtype=rw.RESULT_DTYPE)
        self._ck(self._lib.lgw_bodies_rewrite(self._h, _ptr(buf), _ptr(off), n, _ptr(plan_idx), slot_cap,
                                              _ptr(out), out.nbytes, _ptr(out_off), _ptr(res)), "bodies_rewrite")
        return out, out_off, res[:n]

    def rewrite_bodies(self, bodies, plan_idx, slot_cap: int | None = None, with_matched: bool = False):
        """list[bytes] in -> list[(status, payload bytes)] (payload empty unless status == BODY_OK);
        with_matched adds the bit mask of plan keys present at the top level and the kind of the root value."""
        from . import rewrite as rw
        buf, off = rw.pack_bodies(bodies)
        if slot_cap is None:
            longest = max((len(b) for b in bodies), default=0)
            slot_cap = 6 * longest + getattr(self, "_plan_growth", 0) + 64      # worst case: every byte becomes \u00XX
            slot_cap = (slot_cap + 15) & ~15
        out, out_off, res = self.rewrite_packed(buf, off, np.asarray(plan_idx, dtype=np.uint32), slot_cap)
        rows = [(int(res["status"][i]), bytes(out[int(out_off[i]):int(out_off[i + 1])]) if res["status"][i] == rw.BODY_OK else b"")
                for i in range(len(bodies))]
        if with_matched:
            return [(st, b, int(res["matched"][i]), int(res["root_kind"][i])) for i, (st, b) in enumerate(rows)]
        return rows

    def documents_usage(self, docs):
        """Response tap of non-streaming responses (chat_logging.py:98-150 with is_real_streaming=False): for every document the
        list of usage rows the tap thread writes -- the extra row of a top-level "error" (:139), then the final row (:150).
        -> list of (rows: list[dict], exotic: bool)"""
        from . import rewrite as rw
        buf, off = rw.pack_bodies(docs)
        n = len(docs)
        out = (_abi.DocUsage * max(n, 1))()
        self._ck(self._lib.lgw_documents_usage(self._h, _ptr(buf), _ptr(off), n, out), "documents_usage")
        res = []
        for i in range(n):
            row = _abi.usage_rec_to_dict(out[i].rec)
            res.append(([dict(row), row] if out[i].error_row else [row], bool(out[i].exotic)))
        return res

    def documents_text(self, docs):
        """The text the same tap accumulates for every document (chat_logging.py:124-139): what both of its write_log calls write.
        -> list of (text bytes: UTF-8, a lone surrogate in 'surrogatepass' form; flags: _abi.TF_* bits, TF_DOC_ERROR_LOG when the
        document has the extra row of documents_usage)"""
        from . import rewrite as rw
        buf, off = rw.pack_bodies(docs)
        n = len(docs)
        text = np.empty(max(2 * int(off[n] - off[0]), 1), dtype=np.uint8)
        text_off = np.zeros(n + 1, dtype=np.uint64)
        flags = np.zeros(max(n, 1), dtype=np.uint32)
        self._ck(self._lib.lgw_documents_text(self._h, _ptr(buf), _ptr(off), n, _ptr(text), text.size, _ptr(text_off), _ptr(flags)),
                 "documents_text")
        return [(text[int(text_off[i]):int(text_off[i + 1])].tobytes(), int(flags[i])) for i in range(n)]

    def documents_text_last_ms(self) -> float:
        ms = C.c_float(0)
        self._ck(self._lib.lgw_documents_text_last_ms(self._h, C.byref(ms)), "documents_text_last_ms")
        return ms.value

    def documents_error_detail(self, docs, text_stride: int = 4096):
        """request_handler.py:167-169 for failing non-streaming responses -> list of (DocError, text bytes)."""
        from . import rewrite as rw
        buf, off = rw.pack_bodies(docs)
        n = len(docs)
        out = (_abi.DocError * max(n, 1))()
        text = np.zeros(max(n, 1) * text_stride, dtype=np.uint8)
        self._ck(self._lib.lgw_documents_error_detail(self._h, _ptr(buf), _ptr(off), n, out, _ptr(text), text_stride), "documents_error_detail")
        return [(out[i], bytes(text[i * text_stride:i * text_stride + out[i].text_len])) for i in range(n)]

    def bodies_last_ms(self):
        ms = (C.c_float * 3)()
        self._ck(self._lib.lgw_bodies_last_ms(self._h, C.byref(ms)), "bodies_last_ms")
        return dict(rewrite=ms[0], offsets=ms[1], pack=ms[2])
