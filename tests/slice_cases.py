"""Steps cut into slices: the cut rule of lgw_sse_step restated, a runner that feeds streams over several steps and keeps
everything a step returns, the bulk == sequential == oracle comparison, and hand-built steps whose slices start where the bulk
kernels are easiest to get wrong.  Shared by the emulator tests (tests/test_relay2_slices_cpu.py) and the GPU tests
(tests/test_sse_geometry_gpu.py); the slice count comes from LGW_SLICES, which both engines read on every host-buffer step."""
from __future__ import annotations

import json
import random
from dataclasses import dataclass, field

import numpy as np

import sse_cases as sc
from golden_io import canon_rows
from llmapigateway_b200 import _abi
from llmapigateway_b200.synth import pack_streams


def slice_cuts(chunk_off, seg_chunk, n_slices: int) -> list[int]:
    """csrc/step_types.cuh step_slice_cuts: cut j = the first segment whose start byte is >= n_bytes * j / n_slices"""
    n_segs = len(seg_chunk) - 1
    if n_segs < n_slices:
        n_slices = 1
    n_bytes = int(chunk_off[-1])
    starts = np.asarray(chunk_off, dtype=np.int64)[np.asarray(seg_chunk[:-1], dtype=np.int64)]
    return [0] + [int(np.searchsorted(starts, n_bytes * j // n_slices, side="left")) for j in range(1, n_slices)] + [n_segs]


def slice_starts(chunk_off, seg_chunk, n_slices: int):
    """(first byte, first segment, that segment has no bytes) of every non-empty slice after the first"""
    cuts = slice_cuts(chunk_off, seg_chunk, n_slices)
    out = []
    for j in range(1, len(cuts) - 1):
        s0, s1 = cuts[j], cuts[j + 1]
        if s1 > s0:
            b0 = int(chunk_off[seg_chunk[s0]])
            out.append((b0, s0, int(chunk_off[seg_chunk[s0 + 1]]) == b0))
    return out


@dataclass
class Run:
    states: list                   # final StreamState of every slot (close)
    rows: list                     # sorted (slot, seq, canonical row | "exotic") of the mid-stream row events of all steps
    emitted: dict                  # slot -> the chunks the step relayed, in order
    segs: list                     # SEG_DTYPE bytes of every step
    packed: list = field(default_factory=list)     # the PackedBatch of every step


def host_step(engine, pb, relay_from_host=False):
    return engine.step(pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot, relay_from_host=relay_from_host)


def run(engine, steps, slots, mode: int, step_fn=host_step, keep_packed=False) -> Run:
    """steps: one list of (slot, chunks) per step, in segment order (a slot may get no chunks, or only empty ones)"""
    engine.set_mode(mode)
    slots = np.asarray(slots, dtype=np.uint32)
    engine.open(slots)
    emitted = {int(s): [] for s in slots}
    rows, segs, packed = [], [], []
    for parts in steps:
        pb = pack_streams([c for _, c in parts], slots=[s for s, _ in parts])
        res = step_fn(engine, pb)
        rows += [(r.slot, r.seq, canon_rows([_abi.usage_rec_to_dict(r.rec)]) if not r.rec.exotic else "exotic") for r in res.rows]
        segs.append(res.segs.tobytes())
        for s, (slot, _) in enumerate(parts):
            for ch in range(int(res.segs["emit_chunk_begin"][s]), int(pb.seg_chunk[s + 1])):
                emitted[slot].append(res.out[int(pb.chunk_off[ch]):int(pb.chunk_off[ch + 1])].tobytes())
        if keep_packed:
            packed.append(pb)
    return Run(list(engine.close(slots)), sorted(rows), emitted, segs, packed)


def compare_bulk_sequential(a: Run, b: Run, where=""):
    """everything a step returns and every stream's end state: bulk path (a) == sequential path (b)"""
    assert a.segs == b.segs, where + " segment results: bulk != sequential"
    assert a.rows == b.rows, where + " row events: bulk != sequential"
    for slot in a.emitted:
        assert a.emitted[slot] == b.emitted[slot], f"{where} slot {slot}: relayed bytes: bulk != sequential"
    for i, (x, y) in enumerate(zip(a.states, b.states)):
        assert bytes(x)[:64] == bytes(y)[:64], f"{where} stream {i}: state header: bulk != sequential"
        if x.flags & _abi.SF_REC_VALID:
            assert x.rec.exotic == y.rec.exotic, f"{where} stream {i}: exotic flag"
            if not x.rec.exotic:
                assert canon_rows([_abi.usage_rec_to_dict(x.rec)]) == canon_rows([_abi.usage_rec_to_dict(y.rec)]), f"{where} stream {i}: usage record"


def compare_oracle(r: Run, slots, streams, oracle, where="") -> int:
    """the rules of tools/fuzz_relay2_cpu.one_round: streams whose carry overflowed are left to bulk == sequential, exotic
    records are not compared.  streams[i] = all chunks of slots[i]; oracle(i) -> (relay, tap).  Returns how many were compared."""
    n = 0
    for i, slot in enumerate(slots):
        st = r.states[i]
        if st.flags & _abi.SF_CARRY_OVERFLOW:
            continue
        relay, tap = oracle(i)
        got = [c for c in r.emitted[int(slot)] if c]
        assert got == [c for c in relay.emitted if c], f"{where} slot {slot}: relayed bytes != oracle"
        assert (st.phase == _abi.PHASE_FAILED) == relay.failed, f"{where} slot {slot}: verdict != oracle"
        if not relay.failed and not st.n_exotic:
            rows = [json.loads(x[2])[0] for x in r.rows if x[0] == slot]
            if st.flags & _abi.SF_EMITTED_ANY:
                rows.append(json.loads(canon_rows([_abi.usage_rec_to_dict(st.rec)]))[0])
            assert canon_rows(rows) == canon_rows(tap.rows), f"{where} slot {slot}: usage rows != oracle"
            assert (not (st.flags & _abi.SF_A_USAGE_BOUND)) == relay.end_raises, f"{where} slot {slot}: end_raises != oracle"
        n += 1
    return n


# ---- hand-built steps ------------------------------------------------------------------------------------------------------------

def filler(n: int, seed: int) -> list[bytes]:
    """delta events of exactly n bytes in all (n >= the size of an empty delta)"""
    base = len(sc.delta(""))
    rng = random.Random(seed)
    out, left = [], n
    while left >= base + 400:
        k = rng.randrange(40, 300)
        out.append(sc.delta("x" * k)); left -= base + k
    assert left >= base, n
    out.append(sc.delta("y" * (left - base)))
    return out


def unaligned(n: int) -> int:
    """n rounded up to 3 mod 16 (a slice start at the end of n bytes is then not 16-aligned)"""
    return n + (3 - n) % 16


ERROR_EV = sc.ev({"error": {"message": "upstream overloaded", "code": 502}})


@dataclass
class SliceCase:
    name: str
    n_slices: int
    slots: list
    steps: list                    # [[(slot, chunks)]] as `run` takes them
    streams: list                  # all chunks of every slot (the oracle's input)
    check_step: int                # the step whose slicing the case is about
    expect: callable               # (cuts, starts) -> None: asserts the slicing the case is built for


def _case(name, n_slices, steps, check_step, expect):
    slots = sorted({s for parts in steps for s, _ in parts})
    streams = [[c for parts in steps for s, ch in parts if s == slot for c in ch] for slot in slots]
    return SliceCase(name, n_slices, slots, steps, streams, check_step, expect)


def zero_byte_segment_at_slice_start(zero: str, n_empty: int = 6) -> SliceCase:
    """Slice 1 of step 2 starts at an unaligned byte with a segment that has no bytes (`zero` = "no_chunks" | "empty_chunks"),
    followed by a committed stream whose next 10 KiB (more than one warp range) hold a usage event and an error event in their
    first 3 KiB.  Both steps begin with `n_empty` segments without chunks: the first segment with bytes of slice 0 (and of step 1)
    then sits at index n_empty, which k_prime2 writes into the tile table as tile 0's segment."""
    E = list(range(20, 20 + n_empty))           # slots that get no chunks
    P, Z, L, T = 1, 2, 3, [4, 5, 6, 7]
    first = {s: [sc.delta("first %d" % s)] for s in [P, Z, L] + T}
    step1 = [(e, []) for e in E] + [(s, first[s]) for s in [P, Z, L] + T]
    head = [sc.delta("a"), sc.USAGE_EV, sc.delta("b" * 100), ERROR_EV]
    l_rest = head + filler(10240 - sum(map(len, head)), 1) + [sc.DONE]
    t_rest = [filler(600 + 37 * k, 10 + k) + [sc.USAGE_EV, sc.DONE] for k in range(4)]
    tail = sum(map(len, l_rest)) + sum(len(c) for x in t_rest for c in x)
    p_rest = filler(unaligned(tail + 4003), 2)   # more than half of the step's bytes; its end (slice 1's start) is not 16-aligned
    z_rest = [] if zero == "no_chunks" else [b"", b""]
    step2 = [(e, []) for e in E] + [(P, p_rest), (Z, z_rest), (L, l_rest)] + [(t, r) for t, r in zip(T, t_rest)]

    def expect(cuts, starts):
        assert cuts[1] == n_empty + 1, cuts                        # slice 1 starts at Z
        b0, _, zero_len = starts[0]
        assert zero_len and b0 % 16 != 0, starts
    return _case("zero_byte_segment_at_slice_start_" + zero, 2, [step1, step2], 1, expect)


def fresh_stream_at_slice_start(after_zero: bool) -> SliceCase:
    """A fresh stream whose kept chunk (its first non-empty chunk) is the first chunk of slice 1, right at its start or behind a
    segment without bytes; slice 0 begins with segments without chunks."""
    P, Z, F, T = 1, 2, 3, [4, 5, 6]
    f_chunks = [sc.delta("kept")] + filler(5000, 3) + [sc.USAGE_EV, ERROR_EV, sc.DONE]
    t = [filler(500 + 50 * k, 20 + k) + [sc.USAGE_EV, sc.DONE] for k in range(3)]
    rest = sum(map(len, f_chunks)) + sum(len(c) for x in t for c in x)
    p = filler(unaligned(rest + 1001), 4)
    step = [(e, []) for e in range(20, 24)] + [(P, p)] + ([(Z, [])] if after_zero else []) + [(F, f_chunks)] + list(zip(T, t))

    def expect(cuts, starts):
        b0, s0, zero_len = starts[0]
        assert b0 % 16 != 0 and zero_len == after_zero, starts
    return _case("fresh_stream_at_slice_start" + ("_after_zero" if after_zero else ""), 2, [step], 0, expect)


def segment_larger_than_its_share() -> SliceCase:
    """One segment holds 60 % of the step's bytes: with 8 slices, several cuts fall behind it and their slices are empty."""
    B, S = 1, [2, 3, 4, 5, 6, 7, 8, 9, 10, 11]
    first = {s: [sc.delta("hi %d" % s)] for s in [B] + S}
    small = [filler(700 + 61 * k, 30 + k) + [sc.USAGE_EV, sc.DONE] for k in range(len(S))]
    n_small = sum(len(c) for x in small for c in x)
    big = [sc.USAGE_EV] + filler(int(n_small * 1.5), 5) + [ERROR_EV, sc.DONE]
    step2 = [(S[0], small[0]), (B, big)] + [(s, x) for s, x in zip(S[1:], small[1:])]

    def expect(cuts, starts):
        assert len(set(cuts)) < len(cuts), cuts                   # empty slices
    return _case("segment_larger_than_its_share", 8, [[(s, first[s]) for s in [B] + S], step2], 1, expect)


def usage_event_behind_slice_start(lead: bytes) -> SliceCase:
    """Slice 1 starts (unaligned) with a committed stream whose bytes begin with `lead` (at most 15 bytes of whole events) and a
    usage event, then more than a warp range of deltas."""
    P, U, T = 1, 2, [3, 4]
    first = {s: [sc.delta("x%d" % s)] for s in [P, U] + T}
    u = [lead + sc.USAGE_EV] + filler(7000, 6) + [sc.DONE]
    t = [filler(900, 40 + k) + [sc.DONE] for k in range(2)]
    rest = sum(map(len, u)) + sum(len(c) for x in t for c in x)
    p = filler(unaligned(rest + 2005), 7)
    step2 = [(P, p), (U, u)] + list(zip(T, t))

    def expect(cuts, starts):
        b0, s0, _ = starts[0]
        assert s0 == 1 and b0 % 16 != 0, starts
    return _case("usage_event_%d_bytes_behind_slice_start" % len(lead), 2, [[(s, first[s]) for s in [P, U] + T], step2], 1, expect)


def one_segment_per_slice(n_segs: int = 12, size: int = 1501) -> SliceCase:
    """n_segs segments of exactly `size` bytes and LGW_SLICES = n_segs: every slice is one segment, starting at an unaligned
    byte; fresh and committed streams, usage and error events at the segments' first bytes."""
    slots = list(range(1, n_segs + 1))
    first = [(s, [sc.delta("go")]) for s in slots[: n_segs // 2]]        # half of them are committed in step 2, half are fresh

    def seg(k):
        lead = [sc.USAGE_EV] if k % 3 == 0 else ([ERROR_EV] if k % 3 == 1 else [sc.delta("z")])
        body = lead + filler(size - len(lead[0]) - len(sc.DONE), 50 + k) + [sc.DONE]
        assert sum(map(len, body)) == size
        return body
    step2 = [(s, seg(k)) for k, s in enumerate(slots)]

    def expect(cuts, starts):
        assert cuts == list(range(n_segs + 1)), cuts
        assert all(b0 % 16 != 0 for b0, _, _ in starts), starts
    return _case("one_segment_per_slice", n_segs, [first, step2], 1, expect)


def directed_cases() -> list[SliceCase]:
    return [zero_byte_segment_at_slice_start("no_chunks"), zero_byte_segment_at_slice_start("empty_chunks"),
            fresh_stream_at_slice_start(False), fresh_stream_at_slice_start(True), segment_larger_than_its_share(),
            usage_event_behind_slice_start(b""), usage_event_behind_slice_start(b": ping\n\n"),
            usage_event_behind_slice_start(b": keepalive\n\n"), one_segment_per_slice()]


def check_directed(engine, case: SliceCase, step_fn=host_step):
    """case.steps sliced (mode 0, LGW_SLICES set by the caller) against the same steps in mode 1, and every stream against the
    oracle; the slicing the case is built for is asserted first"""
    from oracle.sse_oracle import run_stream
    pb = pack_streams([c for _, c in case.steps[case.check_step]], slots=[s for s, _ in case.steps[case.check_step]])
    case.expect(slice_cuts(pb.chunk_off, pb.seg_chunk, case.n_slices), slice_starts(pb.chunk_off, pb.seg_chunk, case.n_slices))
    a = run(engine, case.steps, case.slots, 0, step_fn)
    b = run(engine, case.steps, case.slots, 1, step_fn)
    compare_bulk_sequential(a, b, case.name)
    compare_oracle(a, case.slots, case.streams, lambda i: run_stream([c for c in case.streams[i] if c]), case.name)
