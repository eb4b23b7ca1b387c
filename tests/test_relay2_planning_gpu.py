"""k_relay2's own segment planning at production geometry: the layouts of tests/planning_cases.py (skewed stream lengths, dense
runs of tiny segments, runs of segments without bytes, continuation steps, a handful of long segments, adversarial streams among
them) at 2, 20 and 60 MiB, through the device entry point and host steps cut into 3 and 8 slices, warm and cold, in one step
and in three.  A planning mistake does not corrupt bytes -- the kernel notices and hands the segment to the exact sequential
path -- so besides bulk == sequential, the truths and the oracle, every case checks the path counters exactly; the geometry
model shows that the case set reaches every way first_segment can take and window reloads by the dozen.  Then the findings
scratch across steps of very different segment counts, and stream opening, which no longer waits for the device: callers reuse
their arrays at once, opens follow each other and steps without a sync, slots are reopened behind a running step."""
import functools

import numpy as np
import pytest

import planning_cases as P
import slice_cases as SC
from llmapigateway_b200 import _abi
from llmapigateway_b200.synth import pack_streams, sse_batch
from sse_generators import GENERATORS, make_streams
from test_relay2_planning_cpu import check_layout, model_coverage
from test_sse_geometry_gpu import device_step

pytestmark = pytest.mark.gpu

MiB = 1 << 20
MAX_STREAMS = 8192


def _new_engine():
    import llmapigateway_b200 as L
    return L.Engine(max_streams=MAX_STREAMS, max_step_chunks=1 << 21, max_step_bytes=96 * MiB)


@pytest.fixture(scope="module")
def engine():
    e = _new_engine()
    yield e
    e.close_engine()


@functools.lru_cache(maxsize=None)
def sm_count() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@functools.lru_cache(maxsize=None)
def adversarial():
    return tuple(tuple(s) for k, g in enumerate(GENERATORS) for s in make_streams(g, 16, 1300 + k))


_ADV_INDEX = {}


@functools.lru_cache(maxsize=None)
def _oracle(i: int):
    from oracle.sse_oracle import run_stream
    return run_stream(list(adversarial()[i]))


def oracle_of(chunks):
    if not _ADV_INDEX:
        _ADV_INDEX.update({s: i for i, s in enumerate(adversarial())})
    return _oracle(_ADV_INDEX[tuple(chunks)])


@functools.lru_cache(maxsize=4)
def layout(name: str, size: int, n_steps: int = 1) -> P.Layout:
    total = size * MiB
    if name == "zero_byte_runs":
        lay = P.zero_byte_runs_fitted(total, lambda n: P.launch(0, n, sm_count=sm_count())[2])
    elif name == "adversarial_in_runs":
        lay = P.adversarial_in_runs(total, [list(s) for s in adversarial()], run=60)
    else:
        lay = getattr(P, name)(total)
    return P.split_steps(lay, n_steps)


ENTRIES = {"device": (device_step, 1), "slices3": (SC.host_step, 3), "slices8": (SC.host_step, 8)}
LAYOUTS = ["tiny_then_huge", "huge_then_tiny", "alternating_runs", "zero_byte_runs", "continuation_step", "adversarial_in_runs"]
CASES = [(name, size, entry, "warm", 1) for name in LAYOUTS for size in (2, 20, 60) for entry in ENTRIES] + [
    ("few_segments", size, entry, "warm", 1) for size in (2, 20) for entry in ENTRIES] + [
    ("tiny_then_huge", 20, "device", "cold", 1), ("zero_byte_runs", 20, "slices8", "cold", 1),
    ("tiny_then_huge", 20, "device", "warm", 3), ("zero_byte_runs", 60, "slices3", "warm", 3),
    ("adversarial_in_runs", 20, "device", "cold", 3), ("alternating_runs", 60, "device", "warm", 3)]


def case_coverage(name, size, entry, n_steps) -> P.Coverage:
    return model_coverage(layout(name, size, n_steps), ENTRIES[entry][1], sm_count=sm_count())


@pytest.mark.parametrize("name,size,entry,templates,n_steps", CASES, ids=[f"{n}-{s}MiB-{e}-{t}-{k}step" for n, s, e, t, k in CASES])
def test_planning_at_production_geometry(engine, name, size, entry, templates, n_steps, monkeypatch, capsys):
    step_fn, n_slices = ENTRIES[entry]
    if entry != "device":
        monkeypatch.setenv("LGW_SLICES", str(n_slices))
    lay = layout(name, size, n_steps)
    cov = case_coverage(name, size, entry, n_steps)
    where = f"{lay.name} {size}MiB {entry} {templates}"
    with capsys.disabled():
        print(f"\n  {where}: {cov.line()}")
    if n_slices == 1:
        for want in sorted(lay.wants):
            assert P.reaches(cov, want), (where, want, cov.line())
    eng = _new_engine() if templates == "cold" else engine
    try:
        if templates == "cold":
            assert eng.launch_count() == 0
        check_layout(eng, lay, step_fn, where, eng.debug_counters, oracle_of)
    finally:
        if eng is not engine:
            eng.close_engine()


def test_case_set_reaches_every_planning_path(capsys):
    """across the cases above (the geometry model at this device's SM count): every way first_segment can take, its clamp, a
    warp that reloads its window 8 times or more, a warp whose range_lo sits on a run of 33 or more segments without bytes, and
    window reloads that land on a fresh stream's kept chunk and on a committed stream"""
    total = P.Coverage()
    for name, size, entry, _, n_steps in CASES:
        total.add(case_coverage(name, size, entry, n_steps))
    with capsys.disabled():
        print(f"\n  all cases at {sm_count()} SMs: {total.line()}")
    for b in (P.SMALL, P.BRACKETED, P.FIRST, P.BELOW_W0, P.BELOW, P.ABOVE):   # (PAST_END needs a launch whose bytes end before x)
        assert total.branches[b] > 0, (b, total.line())
    assert total.clamped > 0
    assert total.max_reloads >= 8, total.line()
    assert total.zero_run_at_range_lo >= 33, total.line()
    assert total.fresh_after_reload > 0 and total.committed_after_reload > 0, total.line()


# ---- the findings scratch across steps ----------------------------------------------------------------------------------------

def _c3_step(n: int, seed: int, n_events: int = 8, slots=None):
    b = sse_batch(n_streams=n, n_events=n_events, seed=seed, events_per_chunk=2)
    chunks = [b.stream_chunks(s) for s in range(n)]
    slots = list(range(n)) if slots is None else list(slots)
    return [list(zip(slots, chunks))], b.truths


def test_findings_scratch_across_steps(engine, monkeypatch):
    """one engine: 6 000 segments, 40 segments, 6 000 segments with the slots permuted, then the same sliced and unsliced.  A
    finding left in the scratch by a step would show up in the next step that reuses its segment index: every step must equal
    mode 1 and a fresh engine given the same steps, with the same exact path counters (all bulk)."""
    rng = np.random.default_rng(5)
    perm = rng.permutation(6000)
    permuted = _c3_step(6000, 3, slots=perm)
    seqs = [_c3_step(6000, 1), _c3_step(40, 2, n_events=512), permuted, permuted, permuted]
    slicing = [None, None, None, "8", None]
    fresh = _new_engine()
    try:
        for k, ((steps, truths), sl) in enumerate(zip(seqs, slicing)):
            if sl:
                monkeypatch.setenv("LGW_SLICES", sl)
            else:
                monkeypatch.delenv("LGW_SLICES", raising=False)
            slots = [s for s, _ in steps[0]]
            where = f"findings sequence step {k}"
            c0 = engine.debug_counters()
            got = SC.run(engine, steps, slots, 0)
            c1 = engine.debug_counters()
            assert (c1["sequential"] - c0["sequential"], c1["bulk"] - c0["bulk"]) == (0, len(slots)), (where, c0, c1)
            ref = SC.run(engine, steps, slots, 1)
            SC.compare_bulk_sequential(got, ref, where)
            f0 = fresh.debug_counters()
            new = SC.run(fresh, steps, slots, 0)
            f1 = fresh.debug_counters()
            SC.compare_bulk_sequential(got, new, where + " vs a fresh engine")
            assert [f1[k_] - f0[k_] for k_ in ("sequential", "bulk")] == [c1[k_] - c0[k_] for k_ in ("sequential", "bulk")], where
            # (from_template / stashed differ: a fresh engine has not learnt the usage template yet)
            fresh.close_engine()
            fresh = _new_engine()
            for i, s in enumerate(slots):
                assert _abi.usage_rec_to_dict(got.states[i].rec) == truths[i].expected_row(), (where, s)   # (slots[i] ran stream i)
    finally:
        fresh.close_engine()


# ---- stream-ordered opens -----------------------------------------------------------------------------------------------------

STATUSES = np.array([200, 400, 429, 500, 502, 503, 200, 200], dtype=np.int32)


def _headers(states):
    return [bytes(s)[:64] for s in states]


def _busy_step(eng, n=2048, seed=9):
    """a 20 MiB device step left running (no sync): what follows on the engine's stream queues behind it"""
    import torch
    b = sse_batch(n_streams=n, n_events=80, seed=seed, events_per_chunk=1, slot_base=MAX_STREAMS - n)
    d = [torch.from_numpy(x).cuda() for x in (b.data, b.chunk_off, b.seg_chunk, b.seg_slot)]
    out = torch.empty_like(d[0])
    segs = torch.zeros(n * 12, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.open(b.seg_slot)
    eng.step_device(d[0].data_ptr(), int(b.data.size), d[1].data_ptr(), b.n_chunks, d[2].data_ptr(), d[3].data_ptr(), n,
                    out.data_ptr(), segs.data_ptr())
    return (d, out, segs)                                        # (kept alive until the caller syncs)


@pytest.mark.parametrize("kind", ["numpy", "pinned"])
def test_open_copies_the_callers_arrays(kind):
    """open returns before the device has read the slot and status lists; overwriting them right away must not change what is
    opened: every slot shows its own status (200 / 400 / 429 / 5xx), and the slots written over them are untouched"""
    eng = _new_engine()
    try:
        n = 4000
        if kind == "pinned":
            slots = eng.alloc_pinned(4 * n).view(np.uint32)
            status = eng.alloc_pinned(4 * n).view(np.int32)
        else:
            slots, status = np.empty(n, np.uint32), np.empty(n, np.int32)
        slots[:] = np.arange(n, dtype=np.uint32)
        status[:] = np.resize(STATUSES, n)
        keep = _busy_step(eng)
        eng.open(slots, status)
        slots[:] = n + np.arange(n, dtype=np.uint32) % 100           # other slots, all 200
        status[:] = 200
        states = eng.state(np.arange(n + 100, dtype=np.uint32))
        del keep
        want = np.resize(STATUSES, n)
        for i in range(n):
            failed = want[i] >= 400
            assert (states[i].phase == _abi.PHASE_FAILED) == failed, (i, want[i], states[i].phase)
        ref = _new_engine()
        try:
            ref.open(np.arange(n, dtype=np.uint32), want)
            ref.sync()
            assert _headers(states)[:n] == _headers(ref.state(np.arange(n, dtype=np.uint32))), "opened states"
            assert _headers(states)[n:] == _headers(ref.state(np.arange(n, n + 100, dtype=np.uint32))), "slots written after open"
        finally:
            ref.close_engine()
    finally:
        eng.close_engine()


def _run_device(eng, parts, sync_each: bool):
    """one device step of `parts` (slot, chunks); returns (out bytes, seg results) once the caller syncs"""
    import torch
    pb = pack_streams([c for _, c in parts], slots=[s for s, _ in parts])
    d = [torch.from_numpy(x).cuda() for x in (pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot)]
    out = torch.empty_like(d[0])
    segs = torch.zeros(len(parts) * 12, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.step_device(d[0].data_ptr(), int(pb.data.size), d[1].data_ptr(), pb.n_chunks, d[2].data_ptr(), d[3].data_ptr(), len(parts),
                    out.data_ptr(), segs.data_ptr())
    if sync_each:
        eng.sync()
    return d, out, segs


def _opens_and_steps(eng, sync_each: bool):
    """two opens of max_streams slots with other statuses, a step, a reopen of half the slots behind that step, another step,
    open -> close -> open of a quarter, a last step; no host sync between the calls unless sync_each"""
    def sync():
        if sync_each:
            eng.sync()
    all_slots = np.arange(MAX_STREAMS, dtype=np.uint32)
    eng.open(all_slots, np.full(MAX_STREAMS, 503, np.int32)); sync()
    eng.open(all_slots, np.resize(STATUSES, MAX_STREAMS)); sync()
    b1 = sse_batch(n_streams=MAX_STREAMS, n_events=16, seed=21, events_per_chunk=2)
    kept = [_run_device(eng, [(s, b1.stream_chunks(s)) for s in range(MAX_STREAMS)], sync_each)]
    half = all_slots[::2]
    eng.open(half, np.full(len(half), 200, np.int32)); sync()                   # reopened while the step may still run
    b2 = sse_batch(n_streams=len(half), n_events=24, seed=22, events_per_chunk=3)
    kept.append(_run_device(eng, [(int(s), b2.stream_chunks(i)) for i, s in enumerate(half)], sync_each))
    quarter = all_slots[::4]
    eng.open(quarter, np.full(len(quarter), 429, np.int32)); sync()
    closed = eng.close(quarter)
    eng.open(quarter, np.full(len(quarter), 200, np.int32)); sync()
    b3 = sse_batch(n_streams=len(quarter), n_events=8, seed=23, events_per_chunk=1)
    kept.append(_run_device(eng, [(int(s), b3.stream_chunks(i)) for i, s in enumerate(quarter)], sync_each))
    eng.sync()
    res = [(out.cpu().numpy().tobytes(), segs.cpu().numpy().tobytes()) for _, out, segs in kept]
    return res, _headers(closed), eng.close(all_slots), (b2.truths, b3.truths)


def test_opens_and_steps_without_a_sync():
    """back-to-back opens of every slot, a step, reopening slots behind a step that may still run, open -> close -> open: the
    same results, states and usage records as a run that synchronises after every call"""
    eng, ref = _new_engine(), _new_engine()
    try:
        got, got_closed, got_states, (t2, t3) = _opens_and_steps(eng, False)
        want, want_closed, want_states, _ = _opens_and_steps(ref, True)
        assert got == want, "step outputs / segment results"
        assert got_closed == want_closed, "states at close"
        assert _headers(got_states) == _headers(want_states), "final states"
        half, quarter = set(range(0, MAX_STREAMS, 2)), set(range(0, MAX_STREAMS, 4))
        for s in range(MAX_STREAMS):
            st = got_states[s]
            if s in quarter:
                assert _abi.usage_rec_to_dict(st.rec) == t3[s // 4].expected_row(), s
            elif s in half:
                assert _abi.usage_rec_to_dict(st.rec) == t2[s // 2].expected_row(), s
            else:
                assert _abi.usage_rec_to_dict(st.rec) == _abi.usage_rec_to_dict(want_states[s].rec), s
    finally:
        eng.close_engine()
        ref.close_engine()


def test_reopen_clears_the_transcript():
    """with transcripts on, a slot reopened (no sync) after a step holds only the text of its new stream: the same transcript
    as a fresh engine that only ever saw the new stream"""
    def run(eng, old: bool):
        eng.enable_transcripts()
        slots = np.arange(64, dtype=np.uint32)
        if old:
            a = sse_batch(n_streams=64, n_events=40, seed=31, events_per_chunk=4)
            pa = pack_streams([a.stream_chunks(s)[:6] for s in range(64)])     # every stream stays open (no usage event, no [DONE])
            eng.open(slots)
            eng.step(pa.data, pa.chunk_off, pa.seg_chunk, pa.seg_slot)
            eng.step_transcript()
        eng.open(slots)
        b = sse_batch(n_streams=64, n_events=24, seed=32, events_per_chunk=2)
        eng.step(b.data, b.chunk_off, b.seg_chunk, b.seg_slot)
        t = eng.step_transcript()
        return [t.segment(s) for s in range(64)], t.flags.tobytes(), _headers(eng.close(slots))
    eng, ref = _new_engine(), _new_engine()
    try:
        assert run(eng, True) == run(ref, False)
    finally:
        eng.close_engine()
        ref.close_engine()
