"""Host-side mirror of the reference's streaming seam, backed by the engine.

  make_llm_request(...)   <- llm_gateway_core/services/request_handler.py:8   (same signature, same
                             (response, error_detail) return convention, never raises)
  StreamBatcher           <- the per-chunk bodies of request_handler.py:34-142 and the response tap of
                             chat_logging.py:165-231, turned into batched engine steps (SURVEY 8(b) threading)
  shard_of(stream_id, n)  <- SURVEY 8(e): stream -> GPU by hash, no cross-GPU dependency

The upstream HTTP I/O stays httpx exactly as in the reference (request_handler.py:15,23); only the
byte work moves to the GPU.  Non-streaming requests go through the engine too: the attempt's body is the
bytes `rewrite_bodies` rendered (rows a3/a4), the response is checked and re-rendered by the response plan
(row a12) and tapped by `log_chat_completions` (row a8, non-streaming mode).
"""
from __future__ import annotations

import asyncio
import concurrent.futures
import zlib
from dataclasses import dataclass, field

import numpy as np

from . import _abi


def shard_of(stream_id, n_gpus: int) -> int:
    """Stable stream -> GPU map (crc32, not Python's salted hash)."""
    return zlib.crc32(str(stream_id).encode("utf-8")) % max(1, n_gpus)


@dataclass
class FeedResult:
    emitted: bytes | None        # the chunk to relay now (original bytes), or None when dropped
    phase: int
    verdict: int
    flags: int = 0               # lgw_stream_flag bits after the step (SF_CARRY_OVERFLOW: an event outgrew carry_cap)


@dataclass
class _Pending:
    slot: int
    gen: int                     # generation of the slot when the chunk was fed: entries of an earlier user of the slot are dropped
    chunk: bytes
    fut: asyncio.Future


class StreamBatcher:
    """One per engine/GPU.  Coroutines call feed(); a pump task packs everything that arrived during
    `window_s` into one engine step (run in a worker thread: ctypes releases the GIL).

    Slots are handed out first-in first-out and carry a generation counter: a chunk that is still queued when its
    request goes away (client disconnect cancels the awaiting feed()) can never be packed into the next stream that
    gets the slot, and a slot only returns to the free list once no step that contains it is in flight."""

    def __init__(self, engine, window_s: float = 0.002, usage_sink=None, arena_bytes: int = 8 << 20, transcript_log=None,
                 relay_from: str = "device"):
        import collections
        self.eng = engine
        self.window_s = window_s
        self.usage_sink = usage_sink
        # relay_from="device": the bytes handed to the client are the ones the engine re-emitted (downloaded with the step).
        # relay_from="host": "verdicts only" (lgw_sse_step with out_bytes = NULL) -- the relayed chunk is the very chunk object
        # the upstream delivered, as in the reference (`yield chunk`, request_handler.py:141-142); the engine decides WHICH chunks
        # are relayed and everything else, and the step's download shrinks to the per-segment results.
        if relay_from not in ("device", "host"):
            raise ValueError("relay_from must be 'device' or 'host'")
        self.relay_from = relay_from
        # chat transcripts (SURVEY 8(f) rank 3): with a `transcripts.TranscriptLog` the engine's transcript tap runs after every
        # step and every row goes through write_log (file, THEN the usage row, chat_logging.py:47-56) instead of straight to the sink
        self.transcript_log = transcript_log
        self._book = None
        self._req: dict[int, tuple] = {}                      # slot -> (request headers, request body text) for the log file
        if transcript_log is not None:
            from .transcripts import TranscriptBook
            engine.enable_transcripts()
            self._book = TranscriptBook()
            if transcript_log.usage_sink is None:
                transcript_log.usage_sink = usage_sink
        self._free = collections.deque(range(engine.limits.max_streams))
        self._gen = [0] * engine.limits.max_streams
        self._pending: list[_Pending] = []
        self._inflight: dict[int, asyncio.Future] = {}        # slot -> done-future of the step that currently holds chunks of it
        self._wake = asyncio.Event()
        self._task: asyncio.Task | None = None
        self._closed = False
        self.steps = 0
        self.dropped_stale = 0
        self.overflowed = 0                                   # streams that reported SF_CARRY_OVERFLOW (logged, see feed())
        self.rows_lost = 0                                    # segments that reported SF_ROWQ_OVERFLOW (raise Engine(rowq_cap=...))
        # the engine handle is not thread-safe: every call into it goes through this one worker thread
        self._worker = concurrent.futures.ThreadPoolExecutor(max_workers=1, thread_name_prefix="lgw-engine")
        # pinned ingress/egress arenas (SURVEY 8(f) rank 4): chunks are packed straight into page-locked memory the engine
        # owns (lgw_alloc_pinned), so the step's H2D/D2H copies are DMA transfers, not staged pageable copies
        self._arena_in = self._arena_out = None
        alloc = getattr(engine, "alloc_pinned", None)
        if alloc is not None and arena_bytes:
            try:
                self._arena_in, self._arena_out = alloc(arena_bytes), alloc(arena_bytes)
            except Exception:
                self._arena_in = self._arena_out = None

    # -- slots ---------------------------------------------------------------------------------------
    async def open_stream(self, http_status: int = 200, req_headers=None, req_body_str: str = "") -> int:
        if not self._free:
            raise RuntimeError("no free stream slot on this engine")
        slot = self._free.popleft()
        self._gen[slot] += 1
        if self._book is not None:
            self._book.open(slot)
            self._req[slot] = (req_headers if req_headers is not None else {}, req_body_str)
        try:
            await asyncio.get_running_loop().run_in_executor(self._worker, self.eng.open, [slot], [http_status])
        except BaseException:
            self._free.append(slot)
            raise
        return slot

    async def close_stream(self, slot: int):
        """End of upstream: returns (final StreamState, usage dict or None).  The usage dict is the
        last DB row of chat_logging.py:150 and goes to the usage sink (TokensUsageDB.insert_usage seam)."""
        self._gen[slot] += 1                                   # whatever is still queued for this slot is stale from now on
        self._pending = [p for p in self._pending if p.slot != slot or self._cancel(p)]
        fut = self._inflight.get(slot)
        if fut is not None:                                    # a step that contains chunks of this slot is running: let it finish
            try:
                await asyncio.shield(fut)
            except Exception:
                pass
        try:
            st = (await asyncio.get_running_loop().run_in_executor(self._worker, self.eng.close, [slot]))[0]
        finally:
            self._free.append(slot)                            # (open() initialises the slot's state again: a failed close does not poison it)
        usage = None
        text = None
        if self._book is not None:
            text, _tflags = self._book.close(slot)
        if st.flags & _abi.SF_EMITTED_ANY:
            usage = _abi.usage_rec_to_dict(st.rec)
            self._row(slot, usage, text)                        # the final write_log (chat_logging.py:150)
        self._req.pop(slot, None)
        return st, usage

    @staticmethod
    def _cancel(p: _Pending) -> bool:
        if not p.fut.done():
            p.fut.cancel()
        return False

    def _row(self, slot: int, usage: dict, text):
        """One write_log call of the tap (chat_logging.py:139,150): with transcripts on, the log file and then the row; else the row."""
        if self.transcript_log is None or text is None:
            self._sink(usage)
            return
        headers, body = self._req.get(slot, ({}, ""))
        self.transcript_log.write_log(headers, body, text, usage)

    def _sink(self, usage: dict):
        if self.usage_sink is None:
            return
        try:                                                   # the reference swallows insert errors (tokens_usage_db.py:155-159)
            self.usage_sink.insert_usage(usage)
        except Exception:
            pass

    # -- request bodies / non-streaming responses (rows a1-a4, a12): same worker thread, same engine ---------
    def load_rules(self, plans) -> None:
        """Compiled plan table (rewrite.RulePlans); call at config load / hot reload, before serving."""
        self._worker.submit(self.eng.load_rules, plans).result()
        self.plans = plans

    async def rewrite_bodies(self, bodies, plan_idx):
        return await asyncio.get_running_loop().run_in_executor(self._worker, self.eng.rewrite_bodies, list(bodies), list(plan_idx))

    async def rewrite_bodies_matched(self, bodies, plan_idx):
        return await asyncio.get_running_loop().run_in_executor(self._worker, lambda: self.eng.rewrite_bodies(list(bodies), list(plan_idx), with_matched=True))

    async def scan_bodies(self, bodies):
        return await asyncio.get_running_loop().run_in_executor(self._worker, self.eng.scan_bodies, list(bodies))

    async def normalise_responses(self, contents, http_status, target_url: str, strict: bool = True):
        from .responses import normalise_responses
        return await asyncio.get_running_loop().run_in_executor(
            self._worker, lambda: normalise_responses(self.eng, self.plans, list(contents), list(http_status), target_url, strict))

    async def documents_usage(self, docs):
        """Response tap of non-streaming responses (chat_logging.py:98-150): the usage rows of each document."""
        return await asyncio.get_running_loop().run_in_executor(self._worker, self.eng.documents_usage, list(docs))

    async def documents_tap(self, docs):
        """The whole non-streaming tap of each document, in one worker call: [((rows, exotic), (text, text flags))] -- the rows
        of documents_usage and the text every one of those write_log calls writes (Engine.documents_text)."""
        def _both(docs):
            return list(zip(self.eng.documents_usage(docs), self.eng.documents_text(docs)))
        return await asyncio.get_running_loop().run_in_executor(self._worker, _both, list(docs))

    async def detail(self, slot: int) -> str:
        raw = await asyncio.get_running_loop().run_in_executor(self._worker, self.eng.detail, slot)
        return raw.decode("utf-8", errors="replace")

    # -- data ------------------------------------------------------------------------------------------
    async def feed(self, slot: int, chunk: bytes) -> FeedResult:
        loop = asyncio.get_running_loop()
        fut = loop.create_future()
        self._pending.append(_Pending(slot, self._gen[slot], bytes(chunk), fut))
        if self._task is None or self._task.done():
            self._task = loop.create_task(self._pump())
        self._wake.set()
        return await fut

    def _pack(self, blobs, total):
        """All chunks back to back: in the pinned arena when they fit, else in ordinary memory."""
        if self._arena_in is not None and total <= self._arena_in.size:
            pos = 0
            for b in blobs:
                self._arena_in[pos:pos + len(b)] = np.frombuffer(b, dtype=np.uint8)
                pos += len(b)
            return self._arena_in[:total], self._arena_out[:max(total, 1)]
        return (np.frombuffer(b"".join(blobs), dtype=np.uint8) if blobs else np.zeros(0, np.uint8)), None

    async def _pump(self):
        loop = asyncio.get_running_loop()
        while self._pending:
            await asyncio.sleep(self.window_s)
            batch, self._pending = self._pending, []
            by_slot: dict[int, list[_Pending]] = {}
            for p in batch:
                if p.fut.cancelled() or p.gen != self._gen[p.slot]:      # the request went away / the slot has a new user
                    self.dropped_stale += 1
                    continue
                by_slot.setdefault(p.slot, []).append(p)
            slots = list(by_slot)
            if not slots:
                continue
            blobs, offs, segc = [], [0], [0]
            for s in slots:
                for p in by_slot[s]:
                    blobs.append(p.chunk); offs.append(offs[-1] + len(p.chunk))
                segc.append(segc[-1] + len(by_slot[s]))
            data, out = self._pack(blobs, offs[-1])
            done = loop.create_future()
            for s in slots:
                self._inflight[s] = done
            def _step():
                kw = {"relay_from_host": True} if self.relay_from == "host" else ({"out": out} if out is not None else {})
                r = self.eng.step(data, np.array(offs, np.uint32), np.array(segc, np.uint32), np.array(slots, np.uint32), **kw)
                return r, (self.eng.step_transcript() if self._book is not None else None)
            try:
                res, step_text = await loop.run_in_executor(self._worker, _step)
            except Exception as exc:                      # engine failure: the endpoint answers 500/503 like chat.py:26,198
                for ps in by_slot.values():
                    for p in ps:
                        if not p.fut.done():
                            p.fut.set_exception(exc)
                continue
            finally:
                for s in slots:
                    if self._inflight.get(s) is done:
                        del self._inflight[s]
                if not done.done():
                    done.set_result(None)
            self.steps += 1
            try:
                snaps = {}
                if step_text is not None:                                       # what the tap appended this step + the text at each mark
                    snaps = {(sl, seq): t for sl, seq, t in self._book.apply(slots, step_text)}
                for ev in sorted(res.rows, key=lambda r: (r.slot, r.seq)):      # mid-stream rows, chat_logging.py:139
                    self._row(ev.slot, _abi.usage_rec_to_dict(ev.rec), snaps.get((ev.slot, ev.seq)))
            except Exception:
                pass
            for k, s in enumerate(slots):
                try:
                    eb = int(res.segs["emit_chunk_begin"][k])
                    flags = int(res.segs["flags"][k])
                    if flags & _abi.SF_CARRY_OVERFLOW:
                        self.overflowed += 1
                    if flags & getattr(_abi, "SF_ROWQ_OVERFLOW", 0):          # more mid-stream rows in one step than rowq_cap: rows were dropped
                        self.rows_lost += 1
                    for j, p in enumerate(by_slot[s]):
                        c = segc[k] + j
                        emitted = None
                        if c >= eb and len(p.chunk):
                            # the re-emitted bytes (host mode: the upstream's own chunk object, no copy)
                            emitted = p.chunk if self.relay_from == "host" else res.out[offs[c]:offs[c + 1]].tobytes()
                        if not p.fut.done():
                            p.fut.set_result(FeedResult(emitted, int(res.segs["phase"][k]), int(res.segs["verdict"][k]), flags))
                except Exception as exc:                                         # never leave a future of the batch unresolved
                    for p in by_slot[s]:
                        if not p.fut.done():
                            p.fut.set_exception(exc)


async def make_llm_request(target_url: str, headers: dict, payload: dict, is_streaming: bool, *, batcher: StreamBatcher,
                           client_factory=None, exotic_fallback=None, log_request: dict | None = None):
    """Drop-in for request_handler.py:8.  Returns (response, None) on success and (None, error_detail) on
    failure; never raises (request_handler.py:178-187).  `payload` is the attempt's body: the bytes
    `StreamBatcher.rewrite_bodies` produced (rows a3/a4) -- a dict is still accepted on the streaming branch
    and encoded by httpx as in the reference.  Non-streaming success is a ready `Response` whose body is
    byte-identical to what FastAPI renders from the reference's returned dict (row a12).
    `log_request` = dict(req_headers=..., req_body_str=...) of the CLIENT request: what write_log prints above the transcript
    (chat_logging.py:176-186) when the batcher keeps transcripts."""
    import httpx
    from fastapi.responses import Response, StreamingResponse
    client = (client_factory or (lambda **kw: httpx.AsyncClient(**kw)))(timeout=httpx.Timeout(300.0, connect=60.0))
    slot = None
    ctx = None

    async def _release(close_slot: bool = True):
        """Give back whatever this attempt still holds -- the stream slot, the upstream response, the client (the reference
        leaves its AsyncClient to the garbage collector, request_handler.py:15).  Every resource is released at most once and
        no error of one release keeps the others from running."""
        nonlocal slot, ctx
        s_, c_ = slot, ctx
        slot = ctx = None
        try:
            if s_ is not None and close_slot:
                await batcher.close_stream(s_)
        except Exception:
            pass
        try:
            if c_ is not None:
                await c_.__aexit__(None, None, None)
        except Exception:
            pass
        try:
            aclose = getattr(client, "aclose", None)
            if aclose is not None:
                await aclose()
        except Exception:
            pass
    body_kw = {"content": bytes(payload)} if isinstance(payload, (bytes, bytearray, memoryview)) else {"json": payload}
    if not is_streaming:                                                  # request_handler.py:152-176
        try:
            if "json" in body_kw:
                raise TypeError("non-streaming payloads must be the bytes produced by rewrite_bodies (no CPU serialiser in this package)")
            response = await client.post(target_url, headers=headers, timeout=None, **body_kw)
            body, detail = (await batcher.normalise_responses([response.content], [response.status_code], target_url, False))[0]
            if body == "exotic":
                # a document the engine reports but does not model (duplicate keys, floats with more than 15 significant digits,
                # nesting beyond 16 ...): NOT a failed attempt -- the integrator's own code path decides (INTEGRATION.md 3(b)
                # passes the reference's make_llm_request here); without one the attempt fails loudly with the reason
                if exotic_fallback is not None:
                    return await exotic_fallback(target_url, headers, payload, False, response)
                return None, f"Unexpected error during request to {target_url}: response not modelled by the engine ({detail}); pass exotic_fallback="
            if body is None:
                return None, detail
            resp = Response(content=body, status_code=200, media_type="application/json")
            resp.lgw_tapped = False                                          # log_chat_completions (below) taps it like chat_logging.py does
            return resp, None
        except httpx.RequestError as e:                                   # request_handler.py:178-182
            return None, f"RequestError connecting to {target_url}: {str(e)}"
        except Exception as e:                                            # request_handler.py:183-187
            return None, f"Unexpected error during request to {target_url}: {str(e)}"
        finally:
            await _release()
    try:
        ctx = client.stream("POST", target_url, headers=headers, timeout=None, **body_kw)
        response = await ctx.__aenter__()
        if response.status_code >= 400:                                   # request_handler.py:25-30
            body = await response.aread()
            detail = body.decode("utf-8")
            await _release()
            return None, detail
        slot = await batcher.open_stream(response.status_code, **(log_request or {}))
        chunks = response.aiter_bytes()
        first_kept: list[bytes] = []
        committed = False
        async for chunk in chunks:                                        # priming: request_handler.py:69-95
            r = await batcher.feed(slot, chunk)
            if r.phase == _abi.PHASE_FAILED:
                detail = await batcher.detail(slot)
                if r.verdict == _abi.VERDICT_FAIL_PARSE:                  # :183-187 (message tail is the JSON library's text: unpinned)
                    detail = f"Unexpected error during request to {target_url}: first event is not valid JSON: {detail[:200]}"
                await _release()
                return None, detail
            if r.emitted is not None:
                first_kept.append(r.emitted)
            if r.phase == _abi.PHASE_COMMITTED:
                committed = True
                break

        async def relay():                                                # combined_generator, request_handler.py:100-144
            try:
                for c in first_kept:
                    yield c
                if committed:
                    async for chunk in chunks:
                        r = await batcher.feed(slot, chunk)
                        if r.emitted is not None:
                            yield r.emitted
            finally:
                # (shielded: a client disconnect cancels this generator, the slot and the upstream connection must still be released)
                await asyncio.shield(_release())

        resp = StreamingResponse(relay(), media_type="text/event-stream", headers={"Transfer-Encoding": "chunked", "X-Accel-Buffering": "no"})
        resp.lgw_tapped = True            # the engine's tap already saw every relayed chunk: log_chat_completions must not tap it again
        return resp, None
    except httpx.RequestError as e:                                       # request_handler.py:178-182
        await _release()
        return None, f"RequestError connecting to {target_url}: {str(e)}"
    except Exception as e:                                                # request_handler.py:183-187
        await _release()
        return None, f"Unexpected error during request to {target_url}: {str(e)}"
    except BaseException:                                                 # cancelled while priming: the slot must not stay taken
        await asyncio.shield(_release())
        raise


async def log_chat_completions(request, call_next, *, batcher: StreamBatcher):
    """Mirror of the middleware seam chat_logging.py:165-231.  Streaming responses made by `make_llm_request` above were tapped
    inside the engine (usage rows reach the sink at close_stream): they pass through.  Every other response of the
    /chat/completions route -- non-streaming completions, and the 400/503 JSON bodies of the endpoint -- is what the reference
    hands to a ChunkProcessorThread in its non-streaming mode (:188-190, :98-150): the body is collected, the engine reads the
    usage row(s) out of it (lgw_documents_usage) and they go to the usage sink; the client gets the same bytes, re-chunked
    exactly as they came.  When the batcher keeps transcripts (a `TranscriptLog`), the request is read first as the reference
    reads it (:170-178) and every row goes through write_log with the document's text (lgw_documents_text): the log file, then the
    row."""
    if not request.url.path.endswith("/chat/completions"):               # :167-168
        return await call_next(request)
    req = None
    if getattr(batcher, "transcript_log", None) is not None:
        try:                                                              # :170-178 (any failure: the response goes out untapped)
            req_body_bytes = await request.body()
            req_body_str = req_body_bytes.decode("utf-8") if req_body_bytes else ""
            req = (dict(request.headers), req_body_str)
        except Exception:
            return await call_next(request)
    response = await call_next(request)
    try:
        if getattr(response, "lgw_tapped", False):
            return response
        ctype = response.headers.get("content-type") or ""
        if "text/event-stream" in ctype:                                  # a stream that did not come from the engine: not ours to tap
            return response
        if hasattr(response, "body_iterator"):
            original = response.body_iterator

            async def tapping():
                chunks = []
                async for chunk in original:
                    chunks.append(bytes(chunk))
                    yield chunk
                if req is None:
                    await _tap_document(batcher, chunks)
                else:
                    await _tap_document_logged(batcher, chunks, req)

            response.body_iterator = tapping()
        elif getattr(response, "body", None) is not None:
            if req is None:
                await _tap_document(batcher, [bytes(response.body)])
            else:
                await _tap_document_logged(batcher, [bytes(response.body)], req)
    except Exception:                                                     # :228-229 the middleware never breaks the response
        pass
    return response


async def _tap_document(batcher: StreamBatcher, chunks):
    if not chunks:                                                        # no first chunk => no thread => no row (:198-203)
        return
    try:
        text = b"".join(chunks)
        text.decode("utf-8")                                              # (:101 a decode error ends the thread without a row)
    except UnicodeDecodeError:
        return
    rows, _exotic = (await batcher.documents_usage([text]))[0]
    for row in rows:
        batcher._sink(row)


async def _tap_document_logged(batcher: StreamBatcher, chunks, req):
    """_tap_document with transcripts: every write_log call of the tap (:139 for a top-level "error", then :150) writes the log
    file with the document's text and then inserts its row; a text the file cannot hold (a lone surrogate) gives neither."""
    if not chunks:                                                        # no first chunk => no thread => no file, no row
        return
    try:
        text = b"".join(chunks)
        text.decode("utf-8")                                              # (:101)
    except UnicodeDecodeError:
        return
    (rows, _exotic), (accum, _tflags) = (await batcher.documents_tap([text]))[0]
    req_headers, req_body_str = req
    for row in rows:
        batcher.transcript_log.write_log(req_headers, req_body_str, accum, row)


class SqliteUsageSink:
    """Writes GPU-extracted usage records into the reference's `tokens_usage` table (same schema,
    same ISO-text timestamp: tokens_usage_db.py:37-50,135) so the existing stats endpoints keep working.
    One transaction per batch instead of open-insert-commit-close per row (:131-153)."""

    def __init__(self, db_path):
        import sqlite3
        self.conn = sqlite3.connect(db_path, check_same_thread=False)
        self.conn.execute("""CREATE TABLE IF NOT EXISTS tokens_usage (id INTEGER PRIMARY KEY AUTOINCREMENT, timestamp DATETIME NOT NULL,
            prompt_tokens INTEGER DEFAULT 0, completion_tokens INTEGER DEFAULT 0, total_tokens INTEGER DEFAULT 0,
            reasoning_tokens INTEGER DEFAULT 0, cached_tokens INTEGER DEFAULT 0, cost REAL DEFAULT 0.0, model TEXT, provider TEXT)""")
        self.conn.execute("CREATE INDEX IF NOT EXISTS idx_tokens_usage_timestamp ON tokens_usage (timestamp)")
        self.conn.commit()

    def insert_many(self, usages, timestamps=None):
        from datetime import datetime
        rows = []
        for i, u in enumerate(usages):
            ts = (timestamps[i] if timestamps else datetime.now()).isoformat()
            g = u.get
            rows.append((ts, g("prompt_tokens", 0), g("completion_tokens", 0), g("total_tokens", 0), g("reasoning_tokens", 0),
                         g("cached_tokens", 0), g("cost", 0.0), g("model"), g("provider")))
        sql = ("INSERT INTO tokens_usage (timestamp, prompt_tokens, completion_tokens, total_tokens, reasoning_tokens,"
               " cached_tokens, cost, model, provider) VALUES (?,?,?,?,?,?,?,?,?)")
        for row in rows:
            try:                          # the reference swallows insert errors row by row (:155-159): a value SQLite cannot bind
                self.conn.execute(sql, row)       # (an int beyond 64 bits, a dict) loses that row only
            except Exception:
                pass
        try:
            self.conn.commit()
        except Exception:
            pass

    def insert_usage(self, usage: dict):
        self.insert_many([usage])
