"""GPU: failed streaming attempts at production geometry (tests/failure_geometry_cases.py).  Thousands of failing streams of every
shape among C3 ballast in one 8 192-slot step, through the device entry point and the host-buffer one cut into 1, 8 and 14
slices, with cold and warm template caches; events held in the carry over two and three steps; batched detail reads
(lgw_streams_details) at every stride around the capacities, against lgw_stream_detail; slots reused round after round;
streams that have already failed; and the 503 text of ChainBatch and make_llm_request when the event is longer than
detail_cap.  Every case runs in mode 0 and mode 1 and both must agree."""
import ctypes as C
import random

import numpy as np
import pytest

import failure_geometry_cases as F
import slice_cases as SC
from llmapigateway_b200 import _abi
from llmapigateway_b200.synth import pack_streams, sse_batch
from test_sse_geometry_gpu import device_step

pytestmark = pytest.mark.gpu

N_SLOTS = 8192
N_FAIL = 6000


def _engine(**kw):
    import llmapigateway_b200 as L
    args = dict(max_streams=N_SLOTS, max_step_chunks=1 << 20, max_step_bytes=64 << 20)
    args.update(kw)
    return L.Engine(**args)


def _mix(seed: int):
    """N_FAIL failing (and near-miss) attempts of one step -- every case once, then the short cut-at-every-byte cases again -- and
    C3 ballast in the other slots, shuffled: (streams, attempt or None per slot, ballast truths per slot)"""
    cases = F.single_step(F.all_attempts())
    short = F.short_event_cuts()
    atts = cases + [short[k % len(short)] for k in range(N_FAIL - len(cases))]
    b = sse_batch(n_streams=N_SLOTS - N_FAIL, n_events=64, seed=seed, events_per_chunk=8)
    items = [(a.chunks, a, None) for a in atts] + [(b.stream_chunks(s), None, b.truths[s]) for s in range(N_SLOTS - N_FAIL)]
    random.Random(seed).shuffle(items)
    return [x[0] for x in items], [x[1] for x in items], [x[2] for x in items]


def run_steps(eng, steps, slots, mode, step_fn=SC.host_step):
    """open `slots`, run `steps` ([(slot, chunks)] per step), read every slot's detail (batched, full capacity) and state, close:
    (segment bytes per step, emitted chunks per slot, details, states, closed states)"""
    eng.set_mode(mode)
    slots = np.asarray(slots, dtype=np.uint32)
    eng.open(slots)
    segs, emitted = [], {int(s): [] for s in slots}
    for parts in steps:
        pb = pack_streams([c for _, c in parts], slots=[s for s, _ in parts])
        r = step_fn(eng, pb)
        segs.append(r.segs.copy())
        for k, (slot, _) in enumerate(parts):
            for ch in range(int(r.segs["emit_chunk_begin"][k]), int(pb.seg_chunk[k + 1])):
                emitted[slot].append(r.out[int(pb.chunk_off[ch]):int(pb.chunk_off[ch + 1])].tobytes())
    dets = eng.details(slots, eng.limits.detail_cap)
    states = [bytes(s) for s in eng.state(slots)]
    closed = [bytes(s) for s in eng.close(slots)]
    return segs, emitted, dets, states, closed


def _hdr(raw: bytes):
    return _abi.StreamState.from_buffer_copy(raw)


def check_attempt(a, st, seg, det, emitted, where, cap=F.DETAIL_CAP):
    """one stream against what it was built to do"""
    assert st.verdict == a.verdict, (where, a.name, st.verdict)
    if a.event is None:
        assert st.phase == _abi.PHASE_COMMITTED and emitted, (where, a.name)
        return
    assert st.phase == _abi.PHASE_FAILED and seg["phase"] == _abi.PHASE_FAILED and seg["verdict"] == a.verdict, (where, a.name)
    assert seg["detail_len"] == st.detail_len == len(a.detail(cap)), (where, a.name, int(seg["detail_len"]))
    assert bool(seg["flags"] & _abi.SF_DETAIL_TRUNC) == bool(st.flags & _abi.SF_DETAIL_TRUNC) == a.truncated(cap), (where, a.name)
    assert det == a.detail(cap), (where, a.name)
    assert not [c for c in emitted if c] and st.n_chunks_emitted == 0 and st.bytes_emitted == 0, (where, a.name)
    assert (st.n_chunks_in, st.bytes_in) == a.counted(), (where, a.name, st.n_chunks_in, st.bytes_in, a.counted())


ENTRIES = {"device": (device_step, None), "slices1": (SC.host_step, 1), "slices8": (SC.host_step, 8), "slices14": (SC.host_step, 14)}
CASES = [(e, "warm") for e in ENTRIES] + [("device", "cold"), ("slices8", "cold")]


@pytest.mark.parametrize("entry,templates", CASES, ids=[f"{e}-{t}" for e, t in CASES])
def test_many_failures_in_one_step(entry, templates, monkeypatch):
    step_fn, n_slices = ENTRIES[entry]
    if n_slices:
        monkeypatch.setenv("LGW_SLICES", str(n_slices))
    streams, atts, truths = _mix(seed=11)
    steps = [list(enumerate(streams))]
    eng = _engine()
    try:
        if templates == "warm":                                       # C3 deltas and usage events become templates first
            b = sse_batch(n_streams=512, n_events=64, seed=3, events_per_chunk=8)
            run_steps(eng, [[(s, b.stream_chunks(s)) for s in range(512)]], range(512), 0)
        assert (eng.launch_count() > 0) == (templates == "warm")
        fast = run_steps(eng, steps, range(N_SLOTS), 0, step_fn)
        seq = run_steps(eng, steps, range(N_SLOTS), 1)
    finally:
        eng.close_engine()
    where = f"{entry} {templates}"
    assert fast[0][0].tobytes() == seq[0][0].tobytes(), where + ": segment results: mode 0 != mode 1"
    assert fast[2] == seq[2], where + ": details: mode 0 != mode 1"
    assert [x[:64] for x in fast[4]] == [x[:64] for x in seq[4]], where + ": state headers: mode 0 != mode 1"
    n_trunc = 0
    for i, a in enumerate(atts):
        st = _hdr(fast[4][i])
        assert fast[3][i][:64] == fast[4][i][:64], (where, i)             # state() == close()
        if a is None:
            assert st.phase == _abi.PHASE_COMMITTED and _abi.usage_rec_to_dict(st.rec) == truths[i].expected_row(), (where, i)
            assert b"".join(fast[1][i]) == b"".join(streams[i]), (where, i)
            continue
        check_attempt(a, st, fast[0][0][i], fast[2][i], fast[1][i], where)
        if a.event is None:
            from oracle.sse_oracle import run_stream
            assert [c for c in fast[1][i] if c] == [c for c in run_stream(a.chunks)[0].emitted if c], (where, a.name)
        n_trunc += a.truncated()
    assert n_trunc > 100


def test_events_held_in_the_carry_over_steps():
    """events cut over two and three steps (the head waits in carry_a between launches), a separator cut across steps; mode 0
    (device and sliced) == mode 1 == what the attempts were built to do"""
    atts = F.multi_step_attempts() * 20
    n_steps = 3
    steps = [[] for _ in range(n_steps)]
    for slot, a in enumerate(atts):
        for k, ch in enumerate(a.step_chunks()):
            steps[k].append((slot, ch))
        for k in range(len(a.steps), n_steps):                            # the rest of the stream, or nothing
            steps[k].append((slot, []))
    eng = _engine()
    try:
        got = {"device": run_steps(eng, steps, range(len(atts)), 0, device_step),
               "host": run_steps(eng, steps, range(len(atts)), 0),
               "seq": run_steps(eng, steps, range(len(atts)), 1)}
    finally:
        eng.close_engine()
    for name in ("device", "host"):
        assert [s.tobytes() for s in got[name][0]] == [s.tobytes() for s in got["seq"][0]], name
        assert got[name][2] == got["seq"][2] and [x[:64] for x in got[name][4]] == [x[:64] for x in got["seq"][4]], name
    for i, a in enumerate(atts):
        check_attempt(a, _hdr(got["device"][4][i]), got["device"][0][len(a.steps) - 1][i], got["device"][2][i], got["device"][1][i], a.name)


# ---- batched detail reads -----------------------------------------------------------------------------------------------------

def _raw_details(eng, slots, stride):
    slots = np.ascontiguousarray(slots, dtype=np.uint32)
    buf = np.full(len(slots) * stride, 0xAB, dtype=np.uint8)
    lens = np.zeros(len(slots), dtype=np.uint32)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    eng._ck(eng._lib.lgw_streams_details(eng._h, p(slots), len(slots), p(buf), stride, p(lens)), "streams_details")
    return [buf[i * stride:i * stride + int(lens[i])].tobytes() for i in range(len(slots))], lens


@pytest.mark.parametrize("cap", [64, 100, 4096])
def test_batched_detail_reads(cap):
    """lgw_streams_details at strides 1 .. cap + 1 over 1 .. 8 192 slots (ordered, shuffled, with duplicates) == lgw_stream_detail
    == the kept prefix; Engine.details fetches again at full capacity when a detail reaches its default stride"""
    streams, atts, _ = _mix(seed=5)
    eng = _engine(detail_cap=cap)
    try:
        eng.open(np.arange(N_SLOTS))
        eng.step(*(lambda pb: (pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot))(pack_streams(streams)))
        want = [b"" if a is None else a.detail(cap) for a in atts]
        single = [eng.detail(s) for s in range(N_SLOTS)]
        assert single == want
        for a, st in zip(atts, eng.state(np.arange(N_SLOTS))):
            if a is not None and a.event is not None:
                assert bool(st.flags & _abi.SF_DETAIL_TRUNC) == a.truncated(cap), a.name
        rng = np.random.default_rng(cap)
        lists = {}
        for n in (1, 31, 32, 33, N_SLOTS):
            lists[f"ordered{n}"] = np.arange(n)
            lists[f"shuffled{n}"] = rng.permutation(N_SLOTS)[:n]
            lists[f"dups{n}"] = rng.integers(0, N_SLOTS, n)
        for stride in sorted({1, 63, 64, 1024, cap - 1, cap, cap + 1}):
            for name, sl in lists.items():
                got, lens = _raw_details(eng, sl, stride)
                assert got == [want[int(s)][:stride] for s in sl], (cap, stride, name)
                assert all(int(lens[i]) == min(len(want[int(s)]), stride) for i, s in enumerate(sl)), (cap, stride, name)
        full = eng.details(np.arange(N_SLOTS))
        assert full == want
        assert max(len(d) for d in full) == min(cap, max(len(a.event) for a in atts if a is not None and a.event is not None))
    finally:
        eng.close_engine()


# ---- slots reused, state without closing, streams that already failed ----------------------------------------------------------

def test_slot_reuse_as_chain_batch_does_it():
    """the same slots for three rounds -- long failures, short failures, committed streams -- each round's details, states and
    records are that round's; Engine.state returns what close later returns and leaves the slot open"""
    atts = F.single_step(F.all_attempts())
    long_ = [a for a in atts if a.truncated()]
    short = [a for a in atts if a.event is not None and not a.truncated()]
    n = 2048
    slots = np.arange(n, dtype=np.uint32)
    eng = _engine()
    try:
        for rnd, pool in enumerate((long_, short)):
            mine = [pool[(k * 7 + rnd) % len(pool)] for k in range(n)]
            eng.open(slots)
            r = eng.step(*(lambda pb: (pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot))(pack_streams([a.chunks for a in mine])))
            dets = eng.details(slots)
            sts = [bytes(s) for s in eng.state(slots)]
            closed = [bytes(s) for s in eng.close(slots)]
            assert sts == closed, rnd
            for k, a in enumerate(mine):
                check_attempt(a, _hdr(closed[k]), r.segs[k], dets[k], [], f"round {rnd}")
        b = sse_batch(n_streams=n, n_events=64, seed=8, events_per_chunk=8)
        halves = [b.stream_chunks(s) for s in range(n)]
        cut = [len(c) // 2 for c in halves]
        eng.open(slots)
        eng.step(*(lambda pb: (pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot))(pack_streams([c[:h] for c, h in zip(halves, cut)])))
        mid = eng.state(slots)
        assert all(s.phase == _abi.PHASE_COMMITTED and s.detail_len == 0 and not s.flags & _abi.SF_DETAIL_TRUNC for s in mid)
        assert eng.details(slots) == [b""] * n
        r = eng.step(*(lambda pb: (pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot))(pack_streams([c[h:] for c, h in zip(halves, cut)])))
        assert (r.segs["phase"] == _abi.PHASE_COMMITTED).all()
        end_state = [bytes(s) for s in eng.state(slots)]
        closed = eng.close(slots)
        assert end_state == [bytes(s) for s in closed]
        for s in range(n):
            st = closed[s]
            assert st.n_chunks_in == len(halves[s]) and st.flags & _abi.SF_A_USAGE_BOUND, s
            assert _abi.usage_rec_to_dict(st.rec) == b.truths[s].expected_row(), s
    finally:
        eng.close_engine()


@pytest.mark.parametrize("mode", [0, 1])
def test_streams_that_already_failed_take_no_more_chunks(mode):
    """opened with HTTP >= 400: FAILED / VERDICT_FAIL_HTTP, its chunks neither counted nor relayed; failed in step k: the chunks
    of step k + 1 change nothing"""
    atts = [a for a in F.single_step(F.all_attempts()) if a.event is not None][:600]
    n = len(atts)
    eng = _engine()
    try:
        eng.set_mode(mode)
        eng.open(np.arange(n), np.full(n, 200, np.int32))
        eng.open(np.arange(n, 2 * n), np.array([400, 429, 500, 503] * (n // 4) + [502] * (n % 4), np.int32))
        after = [F.delta("late"), F.DONE]
        pb = pack_streams([a.chunks for a in atts] + [a.chunks for a in atts], slots=list(range(2 * n)))
        r = eng.step(pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot)
        assert (r.segs["emit_chunk_begin"] == pb.seg_chunk[1:]).all()
        before = [bytes(s) for s in eng.state(np.arange(2 * n))]
        dets = eng.details(np.arange(2 * n))
        for k in range(n):
            st = _hdr(before[n + k])
            assert st.phase == _abi.PHASE_FAILED and st.verdict == _abi.VERDICT_FAIL_HTTP, k
            assert st.n_chunks_in == st.bytes_in == st.n_chunks_emitted == 0 and dets[n + k] == b"", k
        pb = pack_streams([after] * (2 * n), slots=list(range(2 * n)))
        r = eng.step(pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot)
        assert (r.segs["emit_chunk_begin"] == pb.seg_chunk[1:]).all() and (r.segs["phase"] == _abi.PHASE_FAILED).all()
        assert [bytes(s) for s in eng.close(np.arange(2 * n))] == before
        assert eng.details(np.arange(2 * n)) == dets
    finally:
        eng.close_engine()


def test_event_longer_than_carry_cap_raises_the_flag():
    """the existing reported limit: an unterminated first event that outgrows carry_cap sets SF_CARRY_OVERFLOW"""
    eng = _engine(max_streams=64, carry_cap=8192)
    try:
        ev = F.event("error_obj", 20000, 3)
        chunks = [ev[:6000], ev[6000:12000], ev[12000:] + F.SEP]
        for mode in (0, 1):
            eng.set_mode(mode)
            eng.open([0])
            pb = pack_streams([chunks], slots=[0])
            r = eng.step(pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot)
            assert r.segs["flags"][0] & _abi.SF_CARRY_OVERFLOW, mode
            assert eng.close([0])[0].flags & _abi.SF_CARRY_OVERFLOW, mode
    finally:
        eng.close_engine()


# ---- the 503 text end to end ------------------------------------------------------------------------------------------------------

def test_chain_batch_503_details_are_the_whole_events():
    """2 048 requests over three rounds, the failing attempts long, split and UTF-8-straddling: every request's 503 detail (not a
    sample) and every served request's bytes equal the oracle walk's"""
    import chain_cases as cc
    from llmapigateway_b200 import chat, rewrite, synth
    from oracle import chain_oracle
    n, n_events = 2048, 16
    providers, rules, fallback_provider = synth.chain_world()
    up = F.chain_upstream(n, n_events, seed=9, p_fail=0.6)
    bodies = synth.chain_request_bodies(n, seed=9)
    eng = _engine(max_streams=n, max_step_chunks=1 << 18, max_step_bytes=64 << 20)
    plans = rewrite.RulePlans(rules, fallback_provider=fallback_provider, stream_mode=cc.stream_mode())
    eng.load_rules(plans)
    try:
        out = chat.ChainBatch(eng, plans, providers, rules).run(bodies, None, up)
    finally:
        eng.close_engine()
    rot = chain_oracle.Rotation()
    n_503 = n_long = 0
    for i in range(n):
        want = chain_oracle.walk(bodies[i], {}, providers, rules, fallback_provider, lambda a: up.stream_chunks(i, a), rot, cc.stream_mode())
        if want["kind"] == "stream":
            assert out.emitted(i) == want["emitted"], i
        else:
            assert out.detail[i] == want["detail"], (i, out.detail[i][:200], want["detail"][:200], len(out.detail[i]), len(want["detail"]))
            n_503 += 1
            n_long += len(want["detail"].encode()) > F.DETAIL_CAP + 200
    assert n_503 > 300 and n_long > 50, (n_503, n_long)


def test_make_llm_request_on_the_engine_returns_the_whole_event():
    from test_failures_geometry_cpu import gateway_long_failures, run_gateway
    from oracle.sse_oracle import run_stream
    attempts = gateway_long_failures()[:12]
    eng = _engine(max_streams=16)
    try:
        for a, err in zip(attempts, run_gateway(eng, attempts)):
            assert err == run_stream(a.chunks)[0].error_detail == a.event.decode("utf-8"), a.name
    finally:
        eng.close_engine()
