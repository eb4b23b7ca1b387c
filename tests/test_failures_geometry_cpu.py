"""CPU: failed streaming attempts (tests/failure_geometry_cases.py) against the oracle and the host build of the stream machine,
the host rebuild of a truncated detail (llmapigateway_b200/details.py) against the oracle on every fuzz generator, and the 503
text of make_llm_request and ChainBatch when the failing first event is longer than detail_cap."""
import asyncio

import httpx
import numpy as np
import pytest

import failure_geometry_cases as F
import host_machine as hm
from fake_engine import FakeEngine
from llmapigateway_b200 import _abi
from llmapigateway_b200.details import attempt_detail, first_event

CARRY_CAP = 65536                                  # the engine's default: every case's event fits its carry


def test_every_attempt_does_what_it_was_built_to_do():
    """the oracle confirms every attempt's verdict and failing event"""
    attempts = F.all_attempts() + F.multi_step_attempts()
    assert len(attempts) > 600
    for a in attempts:
        F.check_against_oracle(a)
    lens = {len(a.event) for a in attempts if a.event is not None}
    for size in (F.DETAIL_CAP - 1, F.DETAIL_CAP, F.DETAIL_CAP + 1, 3 * F.DETAIL_CAP, 60 * F.KiB):
        assert size in lens
    kinds = {a.verdict for a in attempts}
    assert kinds == {_abi.VERDICT_OK, _abi.VERDICT_FAIL_EVENT, _abi.VERDICT_FAIL_PARSE}


@pytest.mark.parametrize("cap", [64, 100, F.DETAIL_CAP])
def test_host_build_keeps_the_event_and_flags_truncation(cap):
    """the host build of the device machine: verdict, kept prefix, SF_DETAIL_TRUNC exactly when the event is longer than
    detail_cap, and the chunks it counted -- over one, two and three steps"""
    for a in F.all_attempts() + F.multi_step_attempts():
        r = hm.run_stream(a.chunks, a.steps, carry_cap=CARRY_CAP, detail_cap=cap)
        st = r["state"]
        assert st.verdict == a.verdict, a.name
        assert not st.flags & _abi.SF_CARRY_OVERFLOW, a.name
        if a.event is None:
            assert st.phase == _abi.PHASE_COMMITTED, a.name
            continue
        assert st.phase == _abi.PHASE_FAILED and st.n_chunks_emitted == 0, a.name
        assert r["detail"] == a.detail(cap) and st.detail_len == len(a.detail(cap)), a.name
        assert bool(st.flags & _abi.SF_DETAIL_TRUNC) == a.truncated(cap), a.name
        assert (st.n_chunks_in, st.bytes_in) == a.counted(), a.name


def test_first_event_matches_the_oracle_on_the_fuzz_generators():
    """details.first_event == the oracle's failing piece on every failing stream of the fuzz campaign's generators and of the SSE
    cases, cut at random bytes as well"""
    import random
    import sse_cases as sc
    from oracle.sse_oracle import run_stream
    from sse_generators import GENERATORS, make_streams
    rng = random.Random(7)
    streams = [s for k, g in enumerate(GENERATORS) for s in make_streams(g, 60, 900 + k)]
    streams += [c for _, c, st in sc.all_cases() if st < 400]
    streams += [a.chunks for a in F.all_attempts() + F.multi_step_attempts()]
    n_event = n_parse = 0
    for chunks in streams:
        for cut in (chunks, sc.rechunk(b"".join(chunks), [rng.randrange(1, 400) for _ in range(3)])):
            relay, _ = run_stream(list(cut))
            if not relay.failed:
                continue
            ev = first_event(cut)
            if relay.error_detail.startswith("Unexpected error during request to "):     # the first event does not parse
                assert ev is not None and ev.startswith("data: {")
                n_parse += 1
            else:
                assert ev == relay.error_detail
                n_event += 1
    assert n_event > 400 and n_parse > 50, (n_event, n_parse)


def test_attempt_detail_gives_the_whole_event_only_when_it_was_cut():
    for a in F.all_attempts():
        if a.event is None:
            continue
        for cap in (100, F.DETAIL_CAP):
            flags = _abi.SF_DETAIL_TRUNC if a.truncated(cap) else 0
            got = attempt_detail(a.detail(cap), a.verdict, flags, a.chunks)
            if a.verdict == _abi.VERDICT_FAIL_EVENT:
                assert got == a.event.decode("utf-8"), a.name
            else:                                          # a parse failure's text is cut to 200 characters by its callers
                assert got == a.detail(cap).decode("utf-8", errors="replace"), a.name


# ---- the 503 text end to end, over the host build ------------------------------------------------------------------------------

class WideFakeEngine(FakeEngine):
    """FakeEngine with the engine's default carry_cap (64 KiB): events split over chunks up to 60 KiB stay whole"""

    def _run(self, h):
        return hm.run_stream(h["chunks"], h["steps"] or [0], h["status"], carry_cap=CARRY_CAP)


def _client(chunks):
    class _Body(httpx.AsyncByteStream):
        async def __aiter__(self):
            for c in chunks:
                yield c

    def handler(request):
        return httpx.Response(200, headers={"content-type": "text/event-stream"}, stream=_Body())

    return lambda **kw: httpx.AsyncClient(transport=httpx.MockTransport(handler), **kw)


def gateway_long_failures():
    """attempts whose first event is longer than detail_cap, split, UTF-8 across byte detail_cap, among dropped chunks"""
    return [a for a in F.all_attempts() + F.multi_step_attempts()
            if a.verdict == _abi.VERDICT_FAIL_EVENT and a.truncated() and ("cut" in a.name or "wide" in a.name or "steps" in a.name
                                                                           or "bad" in a.name or "split" in a.name)]


def run_gateway(engine, attempts):
    """make_llm_request over `engine` for every attempt, in turn: the error details"""
    from llmapigateway_b200.gateway import StreamBatcher, make_llm_request

    async def go():
        batcher = StreamBatcher(engine, window_s=0.0005)
        out = []
        for a in attempts:
            resp, err = await make_llm_request("http://upstream.test/v1/chat/completions", {}, b'{"model":"m"}', True,
                                               batcher=batcher, client_factory=_client(a.chunks))
            assert resp is None, a.name
            out.append(err)
        return out
    return asyncio.run(go())


def test_make_llm_request_returns_the_whole_first_event():
    """the reference's detail is the whole failing event (request_handler.py:51,87): longer than detail_cap, cut at any byte,
    a character across byte detail_cap -- never the engine's first 4 096 bytes, never U+FFFD"""
    attempts = gateway_long_failures()
    assert len(attempts) > 40
    from oracle.sse_oracle import run_stream
    for a, err in zip(attempts, run_gateway(WideFakeEngine(max_streams=8), attempts)):
        assert err == run_stream(a.chunks)[0].error_detail == a.event.decode("utf-8"), a.name


def test_make_llm_request_short_and_parse_failures_are_unchanged():
    from oracle.sse_oracle import run_stream
    short = [a for a in F.all_attempts() if a.event is not None and not a.truncated()][:60]
    for a, err in zip(short, run_gateway(WideFakeEngine(max_streams=8), short)):
        if a.verdict == _abi.VERDICT_FAIL_EVENT:
            assert err == run_stream(a.chunks)[0].error_detail, a.name
        else:
            assert err.startswith("Unexpected error during request to http://upstream.test/v1/chat/completions: first event is not valid JSON: ")


@pytest.mark.parametrize("relay_from_host", [False, True])
def test_chain_batch_503_carries_the_whole_event(relay_from_host):
    """ChainBatch over the host build with long failing events: every request's 503 detail equals the oracle walk's"""
    from llmapigateway_b200 import chat, rewrite, synth
    from oracle import chain_oracle
    import chain_cases as cc
    n = 160
    providers, rules, fallback_provider = synth.chain_world()
    up = F.chain_upstream(n, 4, seed=6, p_fail=0.8)
    bodies = synth.chain_request_bodies(n, seed=6)
    eng = WideFakeEngine(max_streams=n)
    plans = rewrite.RulePlans(rules, fallback_provider=fallback_provider, stream_mode=cc.stream_mode())
    eng.load_rules(plans)
    out = chat.ChainBatch(eng, plans, providers, rules, relay_from_host=relay_from_host).run(bodies, None, up)
    rot = chain_oracle.Rotation()
    n_long = 0
    for i in range(n):
        want = chain_oracle.walk(bodies[i], {}, providers, rules, fallback_provider, lambda a: up.stream_chunks(i, a), rot, cc.stream_mode())
        if want["kind"] == "stream":
            assert out.emitted(i) == want["emitted"], i
        else:
            assert out.detail[i] == want["detail"], (i, out.detail[i][:300], want["detail"][:300])
            n_long += len(want["detail"].encode()) > 4096 + 200
    assert n_long > 5, n_long
