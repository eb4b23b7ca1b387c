"""Text of the non-streaming tap on the H100 (lgw_documents_text: k_docs_text -> k_text_scan -> k_docs_text_pack).  Every text is
compared with the oracle's tap_nonstream (encoded 'surrogatepass') and every text and flag with the host build of the same walk
(transcript.cuh doc_text); the chat-logging middleware over a real engine writes the reference's files and rows."""
import ctypes as C
import random

import numpy as np
import pytest

import host_doc_text as hd
import nonstream_log_cases as nc
from golden_io import load_sse_cases
from llmapigateway_b200 import _abi, rewrite as rw
from llmapigateway_b200.synth import pack_streams
from oracle.sse_oracle import tap_nonstream
from test_documents_text_cpu import random_documents

pytestmark = pytest.mark.gpu

GOLDEN = nc.load_golden()
STAGE = 6144                                   # LGW_DOC_STAGE


def _engine(**kw):
    import llmapigateway_b200 as L
    args = dict(max_streams=64, carry_cap=4096, max_step_chunks=1 << 16, max_step_bytes=1 << 22)
    args.update(kw)
    return L.Engine(**args)


@pytest.fixture(scope="module")
def engine():
    e = _engine()
    yield e
    e.close_engine()


def check(docs, got):
    """device results against the host build (text and flags) and the oracle (text, when it writes one and the walk models it)"""
    assert len(got) == len(docs)
    for d, (text, flags) in zip(docs, got):
        h_text, h_flags = hd.doc_text(d)
        assert (text, flags) == (h_text, h_flags), d[:200]
        tap = tap_nonstream([d])
        if tap.rows and not flags & _abi.TF_EXOTIC:
            assert text == tap.transcripts[-1].encode("utf-8", "surrogatepass"), d[:200]
            assert bool(flags & _abi.TF_DOC_ERROR_LOG) == (len(tap.rows) == 2)


def test_golden_documents_through_the_c_abi(engine):
    docs = [g["doc"] for g in GOLDEN if g["kind"] == "doc"] + [g["response"] for g in GOLDEN if g["kind"] == "http"]
    check(docs, engine.documents_text(docs))


def test_golden_through_the_middleware_on_a_real_engine(tmp_path):
    e = _engine(max_streams=4, max_step_chunks=1 << 10, max_step_bytes=1 << 16)
    try:
        for k, g in enumerate(GOLDEN):
            d = tmp_path / str(k)
            d.mkdir()
            status, body, events = nc.run_ours(g, e, d)
            assert (status, body) == (g["response_status"], g["response"]), g["name"]
            assert events == g["events"], g["name"]
    finally:
        e.close_engine()


def _irregular():
    """documents of every shape the kernels tell apart: empty, not JSON, non-UTF-8, staged, unstaged, error, data: prefix"""
    big = b'{"choices":[{"message":{"content":"' + b"y" * (STAGE + 100) + b'"}}]}'
    return [b"", b"plain text", b'{"choices":[{"message":{"content":"\xff"}}]}', b'{"error":"e","choices":[{"delta":{"content":"\\u00e9"}}]}',
            b'data: {"choices":[{"delta":{"content":"d"}}]} \n', big, b"{", b'{"choices":[{"message":{"content":"\\ud83d"}}]}']


@pytest.mark.parametrize("n", [1, 4, 5, 16384])
def test_batch_sizes_with_irregular_documents_first_last_interleaved_and_absent(engine, n):
    regular = random_documents(n, n)
    irr = _irregular()
    layouts = {"absent": list(regular), "first": irr[:1] + regular[1:], "last": regular[:-1] + irr[-1:]}
    inter = list(regular)
    for k in range(0, n, 3):
        inter[k] = irr[k % len(irr)]
    layouts["interleaved"] = inter
    for name, docs in layouts.items():
        check(docs, engine.documents_text(docs))


def _content_doc(total: int, tail: bytes, error: bool = False) -> bytes:
    """a document of exactly `total` bytes whose content string ends with `tail` (or with the error key right at the end)"""
    head, end = b'{"choices":[{"message":{"content":"', (b'"}}],"error":1}' if error else b'"}}]}')
    fill = total - len(head) - len(tail) - len(end)
    assert fill >= 0
    return head + b"a" * fill + tail + end


@pytest.mark.parametrize("size", [STAGE - 1, STAGE, STAGE + 1])
def test_documents_on_both_sides_of_the_stage(engine, size):
    docs = [_content_doc(size, b"\\n"), _content_doc(size, b"\\ud83d\\ude00"), _content_doc(size, b"\\u00e9", error=True),
            _content_doc(size, b"\\ud83d"), _content_doc(size, b"")]
    assert all(len(d) == size for d in docs)
    check(docs, engine.documents_text(docs))


@pytest.mark.parametrize("mib", [1, 8])
def test_long_documents_walked_from_global_memory(mib):
    e = _engine(max_streams=4)
    try:
        rng = random.Random(mib)
        body = "".join(rng.choice(["abc ", "é", "\\n", "\\u4e2d", "\\ud83d\\ude00", "\\\"", "xyz"]) for _ in range((mib << 20) // 4))
        doc = ('{"id":"x","choices":[{"message":{"content":"%s"}}],"usage":{"prompt_tokens":1}}' % body).encode()
        docs = [doc, b'{"choices":[{"delta":{"content":"s"}}]}', doc[: len(doc) // 2]]
        check(docs, e.documents_text(docs))
    finally:
        e.close_engine()


def test_error_document_at_the_two_times_bound(engine):
    doc = _content_doc(200_000, b"", error=True)
    (text, flags), = engine.documents_text([doc])
    assert flags & _abi.TF_DOC_ERROR_LOG
    assert len(text) == 2 * len(doc) - len(b'{"choices":[{"message":{"content":"') - len(b'"}}],"error":1}')
    check([doc], [(text, flags)])
    # the cap the header promises (2 x the batch) also holds for a batch of nothing but such documents
    docs = [_content_doc(n, b"", error=True) for n in (60, 61, 6144, 6145, 70_000)]
    got = engine.documents_text(docs)
    assert sum(len(t) for t, _ in got) <= 2 * sum(len(d) for d in docs)
    check(docs, got)


def _raw_call(e, docs, cap):
    buf, off = rw.pack_bodies(docs)
    n = len(docs)
    text = np.full(max(cap, 1), 0xAB, dtype=np.uint8)
    text_off = np.full(n + 1, 7, dtype=np.uint64)
    flags = np.full(n, 9, dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = e._lib.lgw_documents_text(e._h, p(buf), p(off), n, p(text), cap, p(text_off), p(flags))
    return rc, text, text_off, flags


def test_text_cap_exactly_enough_and_one_byte_short(engine):
    docs = random_documents(99, 300)
    want = engine.documents_text(docs)
    total = sum(len(t) for t, _ in want)
    rc, text, text_off, flags = _raw_call(engine, docs, total)
    assert rc == 0
    assert [(text[int(text_off[i]):int(text_off[i + 1])].tobytes(), int(flags[i])) for i in range(len(docs))] == want
    rc, text, text_off, flags = _raw_call(engine, docs, total - 1)
    assert rc == -3                                                          # LGW_ERR_CAPACITY
    assert (text == 0xAB).all() and (text_off == 7).all() and (flags == 9).all()


def test_a_warm_engine_equals_fresh_engines():
    big = random_documents(5, 16384) + [_content_doc(1 << 20, b"\\ud83d\\ude00")]
    smaller = [random_documents(6, 5), [_content_doc(STAGE + 1, b"\\n", error=True)], random_documents(8, 1000)]
    warm = _engine(max_streams=4)
    try:
        warm.documents_text(big)
        for docs in smaller:
            fresh = _engine(max_streams=4)
            try:
                assert warm.documents_text(docs) == fresh.documents_text(docs)
            finally:
                fresh.close_engine()
    finally:
        warm.close_engine()


def _run_streams(e, streams, docs):
    """the SSE cases as three steps of one batch, with transcripts; between the steps and their transcript passes documents go
    through lgw_documents_text and lgw_documents_usage when `docs` is given.  -> everything the streams' taps produced"""
    n = len(streams)
    slots = np.arange(n, dtype=np.uint32)
    e.open(slots)
    out = []
    for k in range(3):
        part = [c[k * len(c) // 3:(k + 1) * len(c) // 3] for c in streams]
        pb = pack_streams(part, slots=list(range(n)))
        r = e.step(pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot)
        if docs:
            check(docs, e.documents_text(docs))
            e.documents_usage(docs)
        st = e.step_transcript()
        if docs:
            check(docs[::-1], e.documents_text(docs[::-1]))
        rows = [(x.slot, x.seq, _abi.usage_rec_to_dict(x.rec)) for x in r.rows]
        out.append((r.out.tobytes(), r.segs.tobytes(), rows, st.text.tobytes(), st.seg_off.tolist(), st.flags.tolist(), sorted(st.marks)))
    # (the 64-byte header and the usage record as the host reads it: the string buffers behind model_len / provider_len are not state)
    out.append([(bytes(s)[:64], _abi.usage_rec_to_dict(s.rec)) for s in e.close(slots)])
    return out


def test_document_calls_leave_the_stream_tap_alone():
    streams = [c["chunks"] for c in load_sse_cases() if c["http_status"] < 400][:48]
    docs = random_documents(11, 64) + _irregular()
    results = []
    for with_docs in (False, True):
        e = _engine()
        try:
            e.enable_transcripts()
            results.append(_run_streams(e, streams, docs if with_docs else None))
        finally:
            e.close_engine()
    assert results[0] == results[1]
