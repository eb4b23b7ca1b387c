"""Non-streaming chat logging cases: documents and requests sent through a FastAPI app whose `/v1/chat/completions` route
answers with the document (or with the endpoint's own HTTPException body), with a chat-logging middleware registered the way the
reference registers it (`app.middleware("http")`).  The same driver records the reference middleware (make_nonstream_log_golden.py)
and runs this package's `gateway.log_chat_completions` (test_documents_text_*.py), so both see the same requests and headers.

What is recorded per case: the write_log events in order -- ("file", name, bytes) when a log file appears, ("row", dict) when a
usage row is inserted -- and the response the client got."""
from __future__ import annotations

import base64
import json
from datetime import datetime, timedelta
from pathlib import Path

GOLDEN = Path(__file__).resolve().parent / "golden"
CLOCK_START = datetime(2026, 10, 16, 12, 0, 0)
CLOCK_STEP = timedelta(seconds=1, milliseconds=7)      # distinct file names for the two write_log calls of one document

REQ = b'{"model":"m","messages":[{"role":"user","content":"line1\\nline2\\n\\nline3"}]}'
U = '"usage":{"prompt_tokens":11,"completion_tokens":7,"total_tokens":18,"completion_tokens_details":{"reasoning_tokens":2},"prompt_tokens_details":{"cached_tokens":3},"cost":0.00042}'


class Clock:
    """datetime.now stand-in: CLOCK_START, then one CLOCK_STEP later at every call."""

    def __init__(self):
        self.t = CLOCK_START

    def now(self, tz=None):
        t = self.t
        self.t = t + CLOCK_STEP
        return t

    __call__ = now


def _doc(name, text, req=REQ):
    return dict(name=name, kind="doc", doc=text if isinstance(text, bytes) else text.encode("utf-8", "surrogatepass"), request=req)


def _http(name, status, detail, req=REQ):
    return dict(name=name, kind="http", status=status, detail=detail, request=req)


def cases() -> list[dict]:
    out = []
    resp = json.loads((GOLDEN / "response_cases.json").read_text())
    seen = set()
    for k, c in enumerate(resp["cases"]):
        body = base64.b64decode(c["body"]) if c["body"] else b""
        if body and body not in seen:
            seen.add(body)
            out.append(_doc(f"response_case_{k}", body))
    for k, c in enumerate(resp["tap_cases"]):
        out.append(_doc(f"tap_case_{k}", base64.b64decode(c["text"])))
    c1 = json.loads((GOLDEN / "c1_case.json").read_text())
    out.append(_doc("c1_response", base64.b64decode(c1["response_body"]), base64.b64decode(c1["request_body"])))
    out += [
        _doc("choices_mixed", '{"choices":[{"delta":{"content":"a"}},{"message":{"content":"b"}},{"delta":{"content":""},"message":{"content":"x"}},'
                              '{"delta":{"role":"assistant"},"message":{"content":"m"}},{"index":4}],' + U + ',"model":"m1","provider":"p1"}'),
        _doc("content_null_empty_absent", '{"choices":[{"message":{"content":null}},{"message":{"content":""}},{"message":{}},{"delta":{"content":null}},'
                                          '{"delta":{"content":"z"}}]}'),
        _doc("every_escape", r'{"choices":[{"message":{"content":"q\" b\\ s\/ \b\f\n\r\t é中 😀 \u0000 \\n\\n end"}}],' + U + '}'),
        _doc("lone_high_surrogate", r'{"choices":[{"message":{"content":"bad \ud83d tail"}}],' + U + '}'),
        _doc("lone_low_surrogate", r'{"choices":[{"message":{"content":"\ude00"}}]}'),
        _doc("high_then_not_low", r'{"choices":[{"message":{"content":"\ud83dA"}}]}'),
        _doc("choices_string", '{"choices":"delta message",' + U + '}'),
        _doc("choice_number_after_text", '{"choices":[{"message":{"content":"kept"}},7,{"message":{"content":"lost"}}],' + U + ',"error":"e"}'),
        _doc("choice_null", '{"choices":[null],' + U + '}'),
        _doc("error_without_usage", '{"error":{"message":"boom \\n x","code":500}}'),
        _doc("error_with_usage", '{"choices":[{"message":{"content":"partial "}}],' + U + ',"error":"upstream failed","model":"m2"}'),
        _doc("data_prefix_trailing_ws", 'data: {"choices":[{"delta":{"content":"d"}}],' + U + '}  \n\t\r\x0b\x0c \n'),
        _doc("data_prefix_error", 'data: {"error":{"message":"x"},"choices":[{"delta":{"content":"y"}}]} \n\n'),
        _doc("invalid_json", '{"choices":[{"message":{"content":"x"}}],'),
        _doc("not_json_prefix", ' {"choices":[{"message":{"content":"x"}}]}'),
        _doc("empty_body", b""),
        _doc("non_utf8_response", b'{"choices":[{"message":{"content":"\xff"}}]}'),
        _doc("non_utf8_request", '{"choices":[{"message":{"content":"fine"}}],' + U + '}', req=b'{"messages":"\xfe\xff"}'),
        _doc("empty_request", '{"choices":[{"message":{"content":"fine"}}]}', req=b""),
        _http("endpoint_400", 400, "Invalid JSON in request body"),
        _http("endpoint_503", 503, "All providers failed. Last error: upstream \"x\"\nline"),
        _doc("pretty_printed_lf_lf", '{\n  "choices": [\n    {\n      "message": {\n        "content": "pretty\\n\\ntext"\n      }\n    }\n  ],\n\n  '
                                     + U + '\n}\n\n'),
        _doc("pretty_error_lf_lf", '{\n  "error": {\n    "message": "e"\n  },\n\n  "choices": [{"delta": {"content": "c"}}]\n}'),
    ]
    return out


def encode_events(events) -> list:
    return [["file", e[1], base64.b64encode(e[2]).decode()] if e[0] == "file" else ["row", e[1]] for e in events]


class Recorder:
    """Usage-row insert that also notes every log file written before it: the order of files and rows."""

    def __init__(self, logs: Path):
        self.logs = logs
        self.events = []
        self._seen = set()

    def _files(self):
        if not self.logs.exists():
            return
        for p in sorted(self.logs.glob("*.txt")):
            if p.name not in self._seen:
                self._seen.add(p.name)
                self.events.append(("file", p.name, p.read_bytes()))

    def __call__(self, usage: dict):
        self._files()
        self.events.append(("row", dict(usage)))

    insert_usage = __call__

    def finish(self):
        self._files()
        return self.events


def post(case: dict, middleware) -> tuple[int, bytes]:
    """The case's request through an app with `middleware` registered like chat_logging's; -> (status, response body)."""
    from fastapi import FastAPI, HTTPException
    from fastapi.responses import Response
    from starlette.testclient import TestClient
    app = FastAPI()
    app.middleware("http")(middleware)

    @app.post("/v1/chat/completions")
    async def chat_completions():
        if case["kind"] == "http":
            raise HTTPException(status_code=case["status"], detail=case["detail"])
        return Response(content=case["doc"], media_type="application/json")

    with TestClient(app) as client:
        r = client.post("/v1/chat/completions", content=case["request"], headers={"content-type": "application/json"})
    return r.status_code, r.content


def load_golden() -> list[dict]:
    doc = json.loads((GOLDEN / "nonstream_log_cases.json").read_text())
    out = []
    for g in doc["cases"]:
        g = dict(g)
        g["request"] = base64.b64decode(g["request"])
        if g["kind"] == "doc":
            g["doc"] = base64.b64decode(g["doc"])
        g["response"] = base64.b64decode(g["response"])
        g["events"] = [("file", e[1], base64.b64decode(e[2])) if e[0] == "file" else ("row", e[1]) for e in g["events"]]
        out.append(g)
    return out


def run_ours(case: dict, engine, tmp: Path) -> tuple[int, bytes, list]:
    """gateway.log_chat_completions with a TranscriptLog over `engine`: (status, response, events)."""
    import functools
    from llmapigateway_b200.gateway import StreamBatcher, log_chat_completions
    from llmapigateway_b200.transcripts import TranscriptLog
    logs = tmp / "logs"
    rec = Recorder(logs)
    log = TranscriptLog(log_dir=str(logs), usage_sink=rec, clock=Clock())
    b = StreamBatcher(engine, transcript_log=log, arena_bytes=0)
    try:
        status, body = post(case, functools.partial(log_chat_completions, batcher=b))
    finally:
        b._worker.shutdown(wait=True)
    return status, body, rec.finish()
