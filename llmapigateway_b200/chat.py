"""The `/v1/chat/completions` endpoint body over the engine: the fallback-chain walker (SURVEY 8 config 4).

  chat_completions(request, *, batcher, ...)   <- llm_gateway_core/api/v1/chat.py:20-198  (same request object, same
                                                  responses, same HTTPException status/detail texts)
  ModelRotation                                <- llm_gateway_core/db/model_rotation_db.py:56-110 (same table, same RMW)
  ChainBatch                                   <- the same walk for a whole batch of requests in lock-step rounds
                                                  (what bench.py --config c4 and the full-size parity test drive)

Control stays in Python exactly as SURVEY 8(e) prescribes ("retries stay on the same GPU/stream slot; control stays in
Python"); the byte work of every attempt is the engine's: the request scan (chat.py:31-45 -> lgw_bodies_scan), the per-attempt
body (chat.py:112-119,135-139,160-165 -> lgw_bodies_rewrite with the attempt's compiled plan), the first-event verdict, the
relay and the usage tap (request_handler.py:34-142 -> lgw_sse_step).  There is no CPU JSON parser or serialiser on this path.
"""
from __future__ import annotations

import asyncio
import os
import sqlite3
from dataclasses import dataclass, field

import numpy as np

from . import _abi
from . import rewrite as rw
from .details import attempt_detail
from .gateway import StreamBatcher, make_llm_request, shard_of


class ModelRotation:
    """model_rotation_db.py: one row per (api_key, gateway_model); get_next_model_index is a serial read-modify-write that
    does not shard (SURVEY 8(e): "replicas only / stays on host")."""

    def __init__(self, db_path=":memory:"):
        self.conn = sqlite3.connect(db_path, check_same_thread=False)
        self.conn.execute("CREATE TABLE IF NOT EXISTS model_rotation (api_key TEXT, gateway_model TEXT, last_model_index INTEGER,"
                          " PRIMARY KEY (api_key, gateway_model))")
        self.conn.commit()

    def get_next_model_index(self, api_key: str, gateway_model: str, total_models: int) -> int:
        if total_models <= 0:                                              # :68-70
            return 0
        try:
            cur = self.conn.execute("SELECT last_model_index FROM model_rotation WHERE api_key = ? AND gateway_model = ?", (api_key, gateway_model))
            row = cur.fetchone()
            if row is None:                                                # :84-90 first use starts at 0
                nxt = 0
                self.conn.execute("INSERT INTO model_rotation (api_key, gateway_model, last_model_index) VALUES (?, ?, ?)", (api_key, gateway_model, nxt))
            else:                                                          # :91-98
                nxt = (row[0] + 1) % total_models
                self.conn.execute("UPDATE model_rotation SET last_model_index = ? WHERE api_key = ? AND gateway_model = ?", (nxt, api_key, gateway_model))
            self.conn.commit()
            return nxt
        except Exception:                                                  # :102-107 degrade to the first model
            try:
                self.conn.rollback()
            except Exception:
                pass
            return 0


def _http_exception(status: int, detail: str):
    from fastapi import HTTPException
    return HTTPException(status_code=status, detail=detail)


try:
    from fastapi import HTTPException as _HTTPException
except ImportError:                                                        # (the walker is only ever used under FastAPI)
    _HTTPException = Exception


class RequestNotModelled(_HTTPException):
    """The engine reports the request body but does not model it (duplicate keys, a float that needs 17 significant digits,
    nesting beyond the machine's depth, a value the encoder rejects ...).  Raised BEFORE any upstream attempt, so that the
    integrator can hand the whole request to the reference's own `chat_completions` (INTEGRATION.md 3(g)); uncaught it answers
    501 with the reason.  It must not be walked as a failed attempt: the retry plan of the next attempt drops `messages`
    (chat.py:150's log scrub), the offending value with it, and a scrubbed body would go upstream as the FIRST real attempt."""

    def __init__(self, reason: str):
        self.reason = reason
        if _HTTPException is Exception:
            super().__init__(reason)
        else:
            super().__init__(status_code=501, detail=f"request body not modelled by the engine ({reason})")


def attempt_headers(provider_cfg, rule: dict) -> dict:
    """chat.py:94-123: the headers of every attempt of one rule."""
    key_name = provider_cfg.apikey
    key = os.getenv(key_name) if key_name else None                        # :96
    if not key and key_name:                                               # :99-101 the config may hold the key itself
        key = key_name
    headers = {"Content-Type": "application/json", "HTTP-Referer": "https://github.com/fabiojbg/LLMApiGateway", "X-Title": "LLMGateway",
               **({"Authorization": f"Bearer {key}"} if key else {})}
    for k, v in (rule.get("custom_headers") or {}).items():                # :120-123
        headers[k] = v
    return headers


def rule_sequence(fallback_rules: dict, fallback_provider, requested_model: str, api_key: str, rotation):
    """chat.py:47-78 -> (list of (rule index in the compiled table, rule), gateway model key of the plans or None)."""
    cfg = fallback_rules.get(requested_model)
    if not cfg:                                                            # :49-54
        return [(0, {"provider": fallback_provider, "model": requested_model})], None
    seq = list(enumerate(cfg["fallback_models"]))
    if cfg["rotate_models"] and len(seq) > 1:                              # :63-78
        start = rotation.get_next_model_index(api_key=api_key, gateway_model=requested_model, total_models=len(seq))
        seq = seq[start:] + seq[:start]
    return seq, requested_model


def failure_text(rule: dict, sub_provider, error_detail) -> str:
    """chat.py:154 / :182 `last_error_detail`."""
    if sub_provider is None:
        return f"Model {rule.get('model')} failed with provider '{rule.get('provider')}': {error_detail}"
    return f"Model '{rule.get('model')}' failed from provider '{rule.get('provider')}' and sub-provider {sub_provider} : {error_detail}"


def exhausted_text(requested_model: str, last_error_detail: str) -> str:
    """chat.py:198."""
    return f"All configured providers failed for model '{requested_model}'. Last error: {last_error_detail}"


def attempts_of(rule: dict):
    """The (sub_idx, sub_provider, retry) attempts one pass of the `while retry_count >= 0` loop makes (chat.py:127-185):
    one for a standard provider, one per sub-provider when the provider order is walked as a fallback list."""
    subs = rule.get("providers_order")
    if not subs or rule.get("use_provider_order_as_fallback", False) is False:       # :129
        return [(-1, None)]
    return [(i, sp) for i, sp in enumerate(subs)]


async def chat_completions(request, *, batcher: StreamBatcher, rotation: ModelRotation | None = None, client_factory=None,
                           exotic_fallback=None, sleep=asyncio.sleep):
    """Drop-in body of `@router.post("/completions")` (chat.py:20).  `batcher.load_rules(RulePlans(...))` must have been
    called with the same `fallback_rules` the request's config loader holds (INTEGRATION.md 3)."""
    loader = getattr(request.app.state, "config_loader", None)
    if not loader:                                                         # :22-26
        raise _http_exception(500, "Internal server error: Core configuration not available.")
    providers_config, fallback_rules = loader.providers_config, loader.fallback_rules
    plans: rw.RulePlans = batcher.plans

    try:
        raw = await request.body()
    except Exception as e:                                                 # :37-39
        raise _http_exception(400, f"Error reading request body: {str(e)}")
    scans, models = await batcher.scan_bodies([raw])
    sc = scans[0]
    if sc["status"] == rw.BODY_PARSE_ERROR:                                # :31-39 (decode error, JSON error, non-object root, no "model" key)
        st, _, _, root = (await batcher.rewrite_bodies_matched([raw], [plans.plan_index(None)]))[0]
        raise _http_exception(400, f"Error reading request body: {_request_error_text(raw, (st, root))}")
    if sc["status"] == rw.BODY_NO_MODEL:                                   # :44-45
        raise _http_exception(400, "Missing 'model' in request body")
    if sc["model_kind"] != rw.KIND_STR or sc["model_len"] > len(models[0]):
        raise _http_exception(400, "Error reading request body: 'model' is not a string the engine can route (not modelled)")
    requested_model = models[0].decode("utf-8")
    is_streaming = bool(sc["stream_truthy"])                               # :42 (only its truth value is ever used)

    api_key = request.headers.get("Authorization", "").replace("Bearer ", "")          # :61
    rotation = rotation or _default_rotation()
    seq, gw_key = rule_sequence(fallback_rules, plans.fallback_provider, requested_model, api_key, rotation)

    last_error_detail = "No providers were attempted."                     # :82
    attempted = False
    for rule_idx, rule in seq:                                             # :83
        provider_cfg = providers_config.get(rule.get("provider"))
        target_url = f"{provider_cfg.baseUrl.rstrip('/')}/chat/completions"           # :111
        headers = attempt_headers(provider_cfg, rule)
        retry_delay = rule.get("retry_delay")
        retry_count = rule.get("retry_count") or 0
        tries = attempts_of(rule)
        scrubbed = False
        while retry_count >= 0:                                            # :127
            for sub_idx, sub_provider in tries:
                plan = plans.plan_index(gw_key, rule_idx, sub_idx, retry=scrubbed and sub_idx < 0, stream=is_streaming)
                status, payload = (await batcher.rewrite_bodies([raw], [plan]))[0]
                if status != rw.BODY_OK and not attempted:                 # nothing went upstream yet: hand the request back whole
                    raise RequestNotModelled(rw.STATUS_NAMES[status])
                attempted = True
                if status != rw.BODY_OK:
                    response_data, error_detail = None, f"Unexpected error during request to {target_url}: request body not modelled by the engine ({rw.STATUS_NAMES[status]})"
                else:
                    response_data, error_detail = await make_llm_request(target_url, headers, payload, is_streaming, batcher=batcher,
                                                                         client_factory=client_factory, exotic_fallback=exotic_fallback)
                if response_data and error_detail is None:                 # :146-148 / :173-175
                    return response_data
                if sub_idx < 0:
                    scrubbed = True                                        # :150 the log scrub hits the live payload of every later retry
                last_error_detail = failure_text(rule, sub_provider, error_detail)
            if retry_count > 0 and retry_delay and 0 < retry_delay < 120:  # :190-192
                await sleep(retry_delay)
            retry_count -= 1
    raise _http_exception(503, exhausted_text(requested_model, last_error_detail))     # :197-198


_rotation_singleton: ModelRotation | None = None


def _default_rotation() -> ModelRotation:
    global _rotation_singleton
    if _rotation_singleton is None:
        _rotation_singleton = ModelRotation()
    return _rotation_singleton


_ROOT_ERRORS = {1: "'int' object does not support item assignment", 2: "'float' object does not support item assignment",
                10: "'float' object does not support item assignment", 7: "'int' object does not support item assignment",
                3: "'NoneType' object does not support item assignment", 4: "'bool' object does not support item assignment",
                5: "'bool' object does not support item assignment", 6: "'str' object does not support item assignment",
                9: "list indices must be integers or slices, not str", 8: "'model'"}


def _request_error_text(raw: bytes, probe=None) -> str:
    """str(e) of chat.py:37-39, error path only.  A body that is not UTF-8 gives Python's own UnicodeDecodeError text (reproduced
    by decoding here); a well-formed document that is not an object with a "model" key gives the TypeError/KeyError text of
    chat.py:35-36, chosen by the kind of the root value the engine reports (`probe` = (status, root_kind) of lgw_bodies_rewrite);
    the text of a JSON syntax error is json5's own (json5 is absent from this image: unpinned)."""
    try:
        bytes(raw).decode("utf-8")
    except UnicodeDecodeError as e:
        return str(e)
    # (EXOTIC / ENCODE_ERROR: the document parsed -- it holds a value the engine does not re-render, which does not matter here)
    if probe is not None and probe[0] in (rw.BODY_OK, rw.BODY_EXOTIC, rw.BODY_ENCODE_ERROR) and probe[1] in _ROOT_ERRORS:
        return _ROOT_ERRORS[probe[1]]
    return "request body is not valid JSON"


# ------------------------------------------------------------------------------------------------------------------------
# The same walk for a batch of streaming requests, in lock-step rounds (one round = one attempt of every unserved request).
# ------------------------------------------------------------------------------------------------------------------------
@dataclass
class Answers:
    """What the upstreams answered in one round, in request order: `http_status[k]` (>= 400: `error_bodies` holds the text body,
    request_handler.py:25-30), else the response stream of request k is the next segment of the packed (data, chunk_off, seg_chunk)."""
    http_status: np.ndarray
    error_bodies: list
    data: np.ndarray
    chunk_off: np.ndarray
    seg_chunk: np.ndarray

    @staticmethod
    def from_lists(items) -> "Answers":
        """items[k] = (status, body bytes) or a list of network chunks."""
        st = np.array([it[0] if isinstance(it, tuple) else 200 for it in items], dtype=np.int32)
        streams = [it for it in items if not isinstance(it, tuple)]
        lens = np.fromiter((len(c) for ch in streams for c in ch), dtype=np.int64, count=sum(len(ch) for ch in streams))
        chunk_off = np.zeros(lens.size + 1, np.uint32); np.cumsum(lens, out=chunk_off[1:])
        seg_chunk = np.zeros(len(streams) + 1, np.uint32); np.cumsum([len(ch) for ch in streams], out=seg_chunk[1:])
        data = np.frombuffer(b"".join(c for ch in streams for c in ch), dtype=np.uint8)
        return Answers(st, [it[1] for it in items if isinstance(it, tuple)], data, chunk_off, seg_chunk)


@dataclass
class ChainOutcome:
    served_round: np.ndarray         # int32 per request: round (attempt number) that served it; -1 = all attempts failed (503); -2 = 400;
                                     #   -3 = handed back before any attempt (RequestNotModelled: detail holds the reason)
    detail: list                     # per request: None, or the HTTPException detail (503 / 400)
    spans: np.ndarray                # int64 [n, 2]: the relayed bytes of request i are round_out[served_round[i]][lo:hi]
    round_out: list                  # per round: the step's re-emitted byte buffer
    states: list                     # per round: (request indices, final lgw_stream_state list) of the served streams (usage rows)
    attempts: int = 0
    chunks_relayed: int = 0
    steps: int = 0
    timings: dict = field(default_factory=dict)     # seconds per phase of the walk (host clock)

    def emitted(self, i: int) -> bytes:
        r = int(self.served_round[i])
        return b"" if r < 0 else self.round_out[r][int(self.spans[i, 0]):int(self.spans[i, 1])].tobytes()

    def usage_rows(self):
        """(request index, usage dict) of every served request: the last DB row of chat_logging.py:150."""
        for idx, sts, ok in self.states:
            for i, k in zip(idx, ok):
                st = sts[int(k)]
                if st.flags & _abi.SF_EMITTED_ANY:
                    yield int(i), _abi.usage_rec_to_dict(st.rec)


def _group_rows(rows: np.ndarray, lens: np.ndarray):
    """Group equal (length, bytes) rows: (index of a first member per group, group of every row).  A 64-bit hash of every row
    does the grouping (one pass, no 256-byte key sort); the groups are then verified byte for byte, and in the never-expected
    case of a collision the exact structured sort is used instead."""
    cap = rows.shape[1]
    words = rows.view(np.uint64) if cap % 8 == 0 else rows.astype(np.uint64)
    mult = (np.arange(words.shape[1], dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(0xD6E8FEB86659FD93)) | np.uint64(1)
    h = (words * mult).sum(axis=1, dtype=np.uint64) ^ (lens.astype(np.uint64) * np.uint64(0xFF51AFD7ED558CCD))
    _, first, inverse = np.unique(h, return_index=True, return_inverse=True)
    if ((rows == rows[first[inverse]]).all(axis=1) & (lens == lens[first[inverse]])).all():
        return first, inverse
    key = np.zeros(rows.shape[0], dtype=[("len", "<u8"), ("text", f"S{cap}")])
    key["len"] = lens
    key["text"] = rows.view(f"S{cap}").ravel()
    _, first, inverse = np.unique(key, return_index=True, return_inverse=True)
    return first, inverse


class _NameView:
    """request index -> requested model name, without a per-request Python list"""

    def __init__(self, names, index):
        self.names, self.index = names, index

    def __getitem__(self, i):
        k = int(self.index[i])
        return self.names[k] if k >= 0 else None


class ChainBatch:
    """Lock-step walker over `n` streaming requests that share one engine (one GPU).  `upstream(round, ids, urls, payload
    buffer, payload offsets) -> Answers` is the provider side (in the bench: the local synthetic SSE generator of the north star).

    Every request walks its own chain (its own rules, rotation, retries and sub-providers); a round makes the next attempt of
    every request that has not been served yet: ONE lgw_bodies_rewrite over their bodies with their attempts' plans, ONE
    lgw_sse_step over everything the upstreams answered, ONE lgw_streams_details for the failed first events.  A request whose
    first event fails (request_handler.py:86-88) moves on to its next attempt, one that commits is relayed to its end in the
    same step.  The per-request control (which plan next, which error text last) is array arithmetic over the batch."""

    def __init__(self, engine, plans: rw.RulePlans, providers_config: dict, fallback_rules: dict, rotation: ModelRotation | None = None,
                 relay_from_host: bool = False):
        self.eng, self.plans, self.providers, self.rules = engine, plans, providers_config, fallback_rules
        # True: "verdicts only" steps (lgw_sse_step with out_bytes = NULL): the served bytes are slices of the upstream answers the
        # host already holds, the step downloads the per-segment results only (see StreamBatcher relay_from="host")
        self.relay_from_host = relay_from_host
        self.rotation = rotation or ModelRotation()
        self._sched_cache: dict = {}
        self._arenas: dict = {}                 # round -> pinned egress buffer (lgw_alloc_pinned), grown on demand, reused across runs

    def _arena(self, rnd: int, nbytes: int):
        alloc = getattr(self.eng, "alloc_pinned", None)
        if alloc is None or nbytes == 0:
            return None
        a = self._arenas.get(rnd)
        if a is None or a.size < nbytes:
            a = self._arenas[rnd] = alloc(nbytes)
        return a[:nbytes]

    def _schedule(self, requested_model: str, start: int):
        """The full attempt list of one request: [(plan index, url, rule, sub_provider)] in chat.py's order."""
        key = (requested_model, start)
        if key in self._sched_cache:
            return self._sched_cache[key]
        cfg = self.rules.get(requested_model)
        if not cfg:
            seq, gw_key = [(0, {"provider": self.plans.fallback_provider, "model": requested_model})], None
        else:
            seq, gw_key = list(enumerate(cfg["fallback_models"])), requested_model
            seq = seq[start:] + seq[:start]
        out = []
        for rule_idx, rule in seq:
            cfgp = self.providers.get(rule.get("provider"))
            url = f"{cfgp.baseUrl.rstrip('/')}/chat/completions"
            scrubbed = False
            for _ in range((rule.get("retry_count") or 0) + 1):
                for sub_idx, sp in attempts_of(rule):
                    out.append((self.plans.plan_index(gw_key, rule_idx, sub_idx, retry=scrubbed and sub_idx < 0, stream=True), url, rule, sp))
                    if sub_idx < 0:
                        scrubbed = True
        self._sched_cache[key] = out
        return out

    def run(self, bodies: list, api_keys: list | None, upstream, stream_ids=None) -> ChainOutcome:
        import time
        eng = self.eng
        n = len(bodies)
        ids = np.arange(n) if stream_ids is None else np.asarray(stream_ids)
        tm = {"scan": 0.0, "schedule": 0.0, "rewrite": 0.0, "upstream": 0.0, "open": 0.0, "step": 0.0, "details": 0.0, "close": 0.0, "control": 0.0}
        t_all = t0 = time.perf_counter()

        def lap(key):
            nonlocal t0
            t1 = time.perf_counter(); tm[key] += t1 - t0; t0 = t1

        buf, off = rw.pack_bodies(bodies)
        scans, model_rows = eng.scan_packed(buf, off)
        lap("scan")
        out = ChainOutcome(np.full(n, -1, np.int32), [None] * n, np.zeros((n, 2), np.int64), [], [])
        # ---- schedules: one per distinct (model, rotation start); requests are grouped by their model bytes, not visited one by one ----
        status = scans["status"]
        sched_list = []
        sid = np.full(n, -1, np.int32)
        req_name_of = np.full(n, -1, np.int32)                                     # request -> index into `names`
        names = []
        for i in np.nonzero(status == rw.BODY_PARSE_ERROR)[0]:
            i = int(i)
            pst, _, _, root = eng.rewrite_bodies([bodies[i]], [self.plans.plan_index(None)], with_matched=True)[0]
            out.detail[i] = f"Error reading request body: {_request_error_text(bodies[i], (pst, root))}"; out.served_round[i] = -2
        for i in np.nonzero(status == rw.BODY_NO_MODEL)[0]:
            out.detail[int(i)] = "Missing 'model' in request body"; out.served_round[int(i)] = -2
        okreq = np.nonzero(status == rw.BODY_OK)[0]
        if okreq.size:
            cap = model_rows.shape[1]
            mlen = np.minimum(scans["model_len"][okreq], cap).astype(np.uint64)
            rows = np.ascontiguousarray(model_rows[okreq])
            first, inverse = _group_rows(rows, mlen)
            for u in range(len(first)):
                members = okreq[inverse == u]
                i0 = int(okreq[first[u]])
                name = bytes(model_rows[i0, :int(mlen[first[u]])]).decode("utf-8")
                names.append(name)
                req_name_of[members] = len(names) - 1
                cfg = self.rules.get(name)
                if cfg and cfg["rotate_models"] and len(cfg["fallback_models"]) > 1:   # chat.py:65-78: a serial read-modify-write per request, in request order
                    by_start = {}
                    for i in members:
                        start = self.rotation.get_next_model_index(api_key=(api_keys[int(i)] if api_keys else ""), gateway_model=name,
                                                                   total_models=len(cfg["fallback_models"]))
                        k = by_start.get(start)
                        if k is None:
                            k = by_start[start] = len(sched_list)
                            sched_list.append(self._schedule(name, start))
                        sid[int(i)] = k
                else:
                    sid[members] = len(sched_list)
                    sched_list.append(self._schedule(name, 0))
        req_model = _NameView(names, req_name_of)
        depth = max((len(s) for s in sched_list), default=0)
        plan_tab = np.zeros((max(len(sched_list), 1), max(depth, 1)), np.uint32)
        sched_len = np.zeros(max(len(sched_list), 1), np.int32)
        for k, sc in enumerate(sched_list):
            sched_len[k] = len(sc)
            plan_tab[k, :len(sc)] = [a[0] for a in sc]
        fail_round = np.full(n, -1, np.int32)                                      # request -> round of its last failed attempt ...
        fail_text = [None] * n                                                     # ... and that attempt's error detail (bytes or str; decoded only for the 503s)
        longest = max((len(b) for b in bodies), default=0)
        slot_cap = (6 * longest + self.plans.max_growth() + 64 + 15) & ~15
        active = np.nonzero(sid >= 0)[0]
        rnd = 0
        lap("schedule")
        while active.size:
            going = active[sched_len[sid[active]] > rnd]
            if not going.size:
                break
            # ---- this round's attempt of every unserved request: one rewrite launch set ----------------------------------------
            if going.size == n:
                sub_buf, sub_off = buf, off
            else:
                lens = (off[going + 1] - off[going]).astype(np.int64)
                sub_off = np.zeros(going.size + 1, np.uint64); np.cumsum(lens, out=sub_off[1:])
                gather = np.repeat(off[going].astype(np.int64) - sub_off[:-1].astype(np.int64), lens) + np.arange(int(sub_off[-1]), dtype=np.int64)
                sub_buf = buf[gather]
            plan_idx = plan_tab[sid[going], rnd]
            lap("control")
            pay, pay_off, res = eng.rewrite_packed(sub_buf, sub_off, plan_idx, slot_cap)
            lap("rewrite")
            late_bad = []
            bad_body = res["status"] != rw.BODY_OK
            if bad_body.any():
                # bodies the engine reports but does not model never reach an upstream.  Before any attempt (round 0) the request is
                # handed back whole (RequestNotModelled: a failed attempt would be followed by the retry plan, which drops
                # `messages` and the offending value with it); later it is a failed attempt with that text.
                for k in np.nonzero(bad_body)[0]:
                    i = int(going[k]); reason = rw.STATUS_NAMES[int(res["status"][k])]
                    if rnd == 0:
                        out.served_round[i] = -3
                        out.detail[i] = f"request body not modelled by the engine ({reason})"
                    else:
                        fail_text[i] = f"Unexpected error during request to {sched_list[sid[i]][rnd][1]}: request body not modelled by the engine ({reason})"
                        fail_round[i] = rnd
                        late_bad.append(i)
                keep = ~bad_body
                lens = (pay_off[1:] - pay_off[:-1]).astype(np.int64)
                if int(lens[bad_body].sum()):                                      # (their slots hold bytes: close the gaps)
                    starts = pay_off[:-1].astype(np.int64)[keep]
                    kl = lens[keep]
                    idx = np.repeat(starts - np.concatenate([[0], np.cumsum(kl)[:-1]]), kl) + np.arange(int(kl.sum()), dtype=np.int64)
                    pay = pay[idx]
                new_off = np.zeros(int(keep.sum()) + 1, np.uint64); np.cumsum(lens[keep], out=new_off[1:])
                pay_off, going = new_off, going[keep]
                if not going.size:
                    out.round_out.append(None)
                    active = np.array(sorted(late_bad), dtype=np.int64)
                    rnd += 1
                    continue
            urls = [sched_list[k][rnd][1] for k in sid[going]] if getattr(upstream, "wants_urls", True) else None
            ans: Answers = upstream(rnd, ids[going], urls, pay, pay_off)
            lap("upstream")
            out.attempts += int(going.size)
            http_fail = ans.http_status >= 400
            streaming = ~http_fail                                                 # these sent a response stream, in order
            failed_now = [going[http_fail]] + ([np.array(late_bad, dtype=going.dtype)] if late_bad else [])
            for k, body in zip(np.nonzero(http_fail)[0], ans.error_bodies):
                fail_text[int(going[k])] = ("http", body)                          # (decoded at the end, for the requests that end in a 503)
            fail_round[going[http_fail]] = rnd
            # ---- everything the upstreams streamed back: one step --------------------------------------------------------------
            sreq = going[streaming]
            m = int(sreq.size)
            out.round_out.append(None)
            if m:
                slots = np.arange(m, dtype=np.uint32)
                lap("control")
                eng.open(slots, np.full(m, 200, np.int32))
                arena = None if self.relay_from_host else self._arena(rnd, int(ans.data.size))
                lap("open")
                r = eng.step(ans.data, ans.chunk_off, ans.seg_chunk, slots,
                             **({"relay_from_host": True} if self.relay_from_host else ({"out": arena} if arena is not None else {})))
                lap("step")
                out.steps += 1
                out.round_out[-1] = r.out
                phase, verdict, eb = r.segs["phase"], r.segs["verdict"], r.segs["emit_chunk_begin"].astype(np.int64)
                sflags = r.segs["flags"]
                is_failed = phase == _abi.PHASE_FAILED
                fidx = np.nonzero(is_failed)[0]
                dets = eng.details(slots[fidx])
                lap("details")
                for d, k in zip(dets, fidx):
                    i = int(sreq[k])
                    if verdict[k] == _abi.VERDICT_FAIL_PARSE:
                        d = f"Unexpected error during request to {sched_list[sid[i]][rnd][1]}: first event is not valid JSON: {d.decode('utf-8', errors='replace')[:200]}"
                    elif sflags[k] & _abi.SF_DETAIL_TRUNC:                       # longer than detail_cap: the whole event from the answer
                        co = ans.chunk_off
                        d = attempt_detail(d, int(verdict[k]), int(sflags[k]),
                                           [ans.data[int(co[c]):int(co[c + 1])] for c in range(int(ans.seg_chunk[k]), int(ans.seg_chunk[k + 1]))])
                    fail_text[i] = d
                fail_round[sreq[fidx]] = rnd
                failed_now.append(sreq[fidx])
                ok = np.nonzero(~is_failed)[0]
                seg_end = ans.seg_chunk[1:].astype(np.int64)
                first = np.minimum(eb, seg_end)
                out.spans[sreq[ok], 0] = ans.chunk_off[first[ok]]                   # (indexing the offsets, not converting all of them)
                out.spans[sreq[ok], 1] = ans.chunk_off[seg_end[ok]]
                out.served_round[sreq[ok]] = rnd
                out.chunks_relayed += int((seg_end[ok] - first[ok]).sum())
                lap("control")
                states = eng.close(slots)
                lap("close")
                out.states.append((sreq[ok], states, ok))
            active = np.sort(np.concatenate(failed_now)).astype(np.int64) if failed_now else np.zeros(0, np.int64)
            rnd += 1
        for i in np.nonzero(out.served_round == -1)[0]:                            # chat.py:197-198
            i = int(i)
            if fail_round[i] >= 0:
                text = fail_text[i]
                _, url, rule, sp = sched_list[sid[i]][int(fail_round[i])]
                if isinstance(text, tuple):                                        # request_handler.py:27-30: body.decode("utf-8"); a decode error lands in :183-187
                    try:
                        text = bytes(text[1]).decode("utf-8")
                    except UnicodeDecodeError as e:
                        text = f"Unexpected error during request to {url}: {str(e)}"
                elif not isinstance(text, str):
                    text = bytes(text).decode("utf-8", errors="replace")
                out.detail[i] = exhausted_text(req_model[i], failure_text(rule, sp, text))
            else:
                out.detail[i] = exhausted_text(req_model[i], "No providers were attempted.")
        lap("control")
        tm["total"] = time.perf_counter() - t_all
        out.timings = tm
        return out
