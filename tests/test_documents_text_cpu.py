"""Text of the non-streaming tap (transcript.cuh doc_text, the walk of k_docs_text) and the chat-logging middleware with transcripts,
on the CPU: the host build of the walk against the oracle's tap_nonstream on the golden and on seeded random documents, its
write_log mark against the usage tap's error row, and gateway.log_chat_completions over the fake engine against the log files
and rows the unmodified reference middleware left (tests/golden/nonstream_log_cases.json)."""
from __future__ import annotations

import asyncio
import json
import random
import types

import host_doc_text as hd
import host_machine as hm
import nonstream_log_cases as nc
from fake_engine import FakeEngine
from llmapigateway_b200 import _abi
from oracle.sse_oracle import tap_nonstream

GOLDEN = nc.load_golden()


def random_documents(seed: int, n: int) -> list[bytes]:
    """OpenAI-shaped completion documents with every content shape the walk distinguishes, some wrapped as `data: {...}`."""
    rng = random.Random(seed)
    pieces = ["hi", "", "é中😀", "a\nb", "\\n\\n", "q\"b\\s/", "\t\r\b\f", "\x00\x1f", "\ud83d", "\ude00", "😀", "x" * 300]

    def content():
        r = rng.random()
        if r < 0.1:
            return None
        if r < 0.15:
            return rng.choice([0, False, [], {}, 1.5])
        return "".join(rng.choice(pieces) for _ in range(rng.randint(0, 4)))

    def choice():
        r = rng.random()
        if r < 0.03:
            return rng.choice([None, 3, "s"])
        c = {"index": rng.randint(0, 3)}
        if r < 0.5:
            c["delta"] = {"content": content()} if rng.random() < 0.8 else {"role": "assistant"}
        if r > 0.3:
            c["message"] = {"role": "assistant", "content": content()} if rng.random() < 0.85 else {}
        return c

    out = []
    for _ in range(n):
        d = {"id": "chatcmpl-%d" % rng.randint(0, 999), "object": "chat.completion"}
        if rng.random() < 0.95:
            d["choices"] = [choice() for _ in range(rng.randint(0, 4))] if rng.random() < 0.97 else "choices"
        if rng.random() < 0.6:
            d["usage"] = {"prompt_tokens": rng.randint(0, 9999), "completion_tokens": rng.randint(0, 999), "total_tokens": rng.randint(0, 99999)}
        if rng.random() < 0.15:
            d["error"] = rng.choice(["boom", {"message": "bad\nthing", "code": 500}, None])
        if rng.random() < 0.5:
            d["model"] = "m-%d" % rng.randint(0, 9)
        keys = list(d)
        rng.shuffle(keys)
        d = {k: d[k] for k in keys}
        indent = rng.choice([None, None, 2])
        text = json.dumps(d, ensure_ascii=rng.random() < 0.5, indent=indent)
        if any(0xD800 <= ord(ch) <= 0xDFFF for ch in text):    # a raw lone surrogate is no UTF-8: spell it as its escape
            text = json.dumps(d, ensure_ascii=True, indent=indent)
        if rng.random() < 0.2:
            text = "data: " + text + rng.choice(["", "\n\n", "  \t\n"])
        out.append(text.encode("utf-8"))
    return out


def _check_against_oracle(doc: bytes):
    """-> True when compared (False: the oracle's tap writes nothing for this document, or the walk reports TF_EXOTIC)"""
    tap = tap_nonstream([doc])
    text, flags = hd.doc_text(doc)
    if not tap.rows:
        return False
    assert len(set(tap.transcripts)) == 1                      # both write_log calls of one document write the same text
    if flags & _abi.TF_EXOTIC:
        return False
    assert bool(flags & _abi.TF_DOC_ERROR_LOG) == (len(tap.rows) == 2), doc
    want = tap.transcripts[-1].encode("utf-8", "surrogatepass")
    assert text == want, (doc, text, want)
    lone = any(0xD800 <= ord(ch) <= 0xDFFF for ch in tap.transcripts[-1])
    assert bool(flags & _abi.TF_LONE_SURROGATE) == lone, doc
    return True


def test_host_walk_matches_the_oracle_on_every_golden_document():
    docs = [g["doc"] for g in GOLDEN if g["kind"] == "doc"]
    compared = sum(_check_against_oracle(d) for d in docs)
    assert compared >= len(docs) - 6


def test_host_walk_matches_the_oracle_on_random_documents():
    docs = random_documents(2026, 3000)
    compared = sum(_check_against_oracle(d) for d in docs)
    assert compared > 2700


def test_mark_bit_is_the_usage_taps_error_row():
    docs = [g["doc"] for g in GOLDEN if g["kind"] == "doc"] + random_documents(7, 1000)
    for d in docs:
        _text, flags = hd.doc_text(d)
        assert bool(flags & _abi.TF_DOC_ERROR_LOG) == bool(hm.doc_usage(d).error_row), d


def test_middleware_with_transcripts_writes_the_reference_files_and_rows(tmp_path):
    for k, g in enumerate(GOLDEN):
        d = tmp_path / str(k)
        d.mkdir()
        status, body, events = nc.run_ours(g, hd.text_fake_engine(), d)
        assert (status, body) == (g["response_status"], g["response"]), g["name"]
        assert [e[:2] for e in events] == [e[:2] for e in g["events"]], g["name"]
        for got, want in zip(events, g["events"]):
            assert got == want, (g["name"], got, want)


def test_middleware_without_transcripts_writes_rows_only_and_never_reads_the_request():
    from llmapigateway_b200.gateway import StreamBatcher, log_chat_completions

    class Sink:
        def __init__(self):
            self.rows = []

        def insert_usage(self, u):
            self.rows.append(dict(u))

    async def go(g):
        sink = Sink()
        b = StreamBatcher(FakeEngine(max_streams=2), usage_sink=sink, arena_bytes=0)
        doc = g["doc"] if g["kind"] == "doc" else g["response"]

        async def chunks():
            if doc:
                yield doc

        async def body():
            raise AssertionError("the rows-only path reads no request body")

        req = types.SimpleNamespace(url=types.SimpleNamespace(path="/v1/chat/completions"), body=body, headers={})
        resp = types.SimpleNamespace(headers={"content-type": "application/json"}, body_iterator=chunks())

        async def call_next(_):
            return resp

        out = await log_chat_completions(req, call_next, batcher=b)
        got = b"".join([c async for c in out.body_iterator])
        b._worker.shutdown(wait=True)
        return got, sink.rows

    for g in GOLDEN:
        if g["name"] == "non_utf8_request":        # the reference reads the request first; the rows-only path never does
            continue
        got, rows = asyncio.run(go(g))
        assert got == g["response"]
        assert rows == [e[1] for e in g["events"] if e[0] == "row"] or any(e[0] == "file" and not e[2] for e in g["events"]), g["name"]
