"""The transcript tap (csrc/transcript.cuh: k_text_extract -> k_text_scan -> k_text_pack) at production geometry.

Steps of 2, 20 and 60 MiB hold thousands of segments: adversarial streams of every fuzz generator (tests/sse_generators.py)
and of tests/test_transcript_gpu.py, C3 ballast, and "rich" ballast -- long streams of whole events whose content pieces have
every length from 0 to 200 bytes, escapes, surrogate pairs and multi-byte UTF-8, and of which about one in five has one
irregular chunk (a cut event, invalid UTF-8 or an "error" event) beyond its 32nd chunk.  One-chunk streams pad every step to
more than 1 024 segments (k_text_scan's block loop), one case to more than 4 096.  The steps go through the device entry point,
through the host-buffer one cut into 1, 3, 8 or 14 slices, and verdicts-only; in one step or three (cuts inside events: some
segments start with a tap carry).  Every stream's text at every mark and at close is compared with the oracle (C3 ballast: with
the content bytes of its delta events), and every step's marks are paired with the relay's row events.  Hand-built steps put
the segment count at the scan's block edges, fill the sparse buffer's twofold room, put an unterminated tail of carry_cap and
carry_cap + 1 bytes at a step end, relay one 200 KiB event, and overflow the mark queue.  The direct (pinned host buffer) modes
run with transcripts on.  The bodies take the engine as an argument: tests/test_transcript_geometry_cpu.py runs the hand-built
cases on the SIMT emulator."""
from __future__ import annotations

import json
import os
import random
import subprocess
import sys
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np
import pytest

import sse_cases as sc
import test_transcript_gpu as TG
from llmapigateway_b200 import _abi
from llmapigateway_b200.synth import DELTA_EVENT_BYTES, DELTA_HEAD, DELTA_CONTENT, pack_streams, sse_batch
from llmapigateway_b200.transcripts import TranscriptBook, decode_text
from sse_generators import GENERATORS, make_streams

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
MiB = 1 << 20
MAX_BYTES = 96 * MiB
CARRY_CAP = 16384
EXOTIC_SHARE = 0.1                     # adversarial streams whose text the device reports as not authoritative, at most


def new_engine(rowq_cap: int = 4096):
    import llmapigateway_b200 as L
    e = L.Engine(max_streams=8192, carry_cap=CARRY_CAP, max_step_chunks=1 << 21, max_step_bytes=MAX_BYTES, rowq_cap=rowq_cap)
    e.enable_transcripts()
    return e


@pytest.fixture(scope="module")
def engine():
    e = new_engine()
    yield e
    e.close_engine()


# ---- entry points: a step and its transcript pass ------------------------------------------------------------------------------

def host_tap(engine, pb, relay_from_host=False):
    res = engine.step(pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot, relay_from_host=relay_from_host)
    return res, engine.step_transcript()


def device_tap(engine, pb):
    """lgw_sse_step_device on torch CUDA tensors; the tap reads the caller's device arrays, so it runs while they are alive"""
    import torch
    from llmapigateway_b200.engine import SEG_DTYPE, StepResult
    n_segs = len(pb.seg_slot)
    d = [torch.from_numpy(x).cuda() for x in (pb.data if pb.data.size else np.zeros(16, np.uint8), pb.chunk_off, pb.seg_chunk, pb.seg_slot)]
    out = torch.empty_like(d[0])
    segs = torch.zeros(max(n_segs, 1) * SEG_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    engine.step_device(d[0].data_ptr(), int(pb.data.size), d[1].data_ptr(), pb.n_chunks, d[2].data_ptr(), d[3].data_ptr(), n_segs,
                       out.data_ptr(), segs.data_ptr())
    engine.sync()
    rows = engine.fetch_rows()
    st = engine.step_transcript()
    res = StepResult(out.cpu().numpy()[:pb.data.size], segs.cpu().numpy().view(SEG_DTYPE)[:n_segs], rows)
    del d
    return res, st


ENTRIES = {   # name: (step function, LGW_SLICES)
    "device": (device_tap, None),
    "slices1": (host_tap, 1),
    "slices3": (host_tap, 3),
    "slices8": (host_tap, 8),
    "slices14": (host_tap, 14),
    "host_relay8": (lambda e, pb: host_tap(e, pb, relay_from_host=True), 8),
}


# ---- the runner ---------------------------------------------------------------------------------------------------------------

@dataclass
class TapRun:
    snaps: dict                    # slot -> {seq: text at that mark}
    final: dict                    # slot -> text at close (only streams that relayed something)
    flags: dict                    # slot -> TF_* bits of all steps (TF_SEQUENTIAL left out)
    states: dict                   # slot -> StreamState at close
    step_flags: list               # per step: {slot: TF_* bits of its segment}
    step_marks: list               # per step: set of (slot, seq) of the tap's marks
    step_rows: list                # per step: set of (slot, seq) of the relay's row events
    step_sflags: list              # per step: {slot: SegResult flags}
    n_segs: list                   # per step


def run_tapped(engine, steps, slots, step_fn=host_tap) -> TapRun:
    """steps: one list of (slot, chunks) per step, in segment order.  After every step the transcript pass runs and feeds a
    TranscriptBook, as StreamBatcher does."""
    engine.set_mode(0)
    slots = [int(s) for s in slots]
    engine.open(np.asarray(slots, dtype=np.uint32))
    book = TranscriptBook()
    for s in slots:
        book.open(s)
    snaps = {s: {} for s in slots}
    r = TapRun(snaps, {}, {}, {}, [], [], [], [], [])
    for parts in steps:
        pb = pack_streams([c for _, c in parts], slots=[s for s, _ in parts])
        res, st = step_fn(engine, pb)
        n = len(parts)
        assert len(st.seg_off) == n + 1 and int(st.seg_off[-1]) == len(st.text)
        assert np.all(np.diff(st.seg_off.astype(np.int64)) >= 0)
        for slot, seq, text in book.apply(pb.seg_slot, st):
            assert seq not in snaps[slot], (slot, seq)
            snaps[slot][seq] = text
        r.step_flags.append({s: int(st.flags[k]) for k, (s, _) in enumerate(parts)})
        r.step_sflags.append({s: int(res.segs["flags"][k]) for k, (s, _) in enumerate(parts)})
        r.step_marks.append({(int(a), int(b)) for a, b, _ in st.marks})
        assert len(r.step_marks[-1]) == len(st.marks)
        r.step_rows.append({(int(x.slot), int(x.seq)) for x in res.rows})
        r.n_segs.append(n)
    states = engine.close(np.asarray(slots, dtype=np.uint32))
    for i, s in enumerate(slots):
        text, flags = book.close(s)
        r.states[s] = states[i]
        r.flags[s] = flags
        if states[i].flags & _abi.SF_EMITTED_ANY:
            r.final[s] = text
    return r


def texts_of(r: TapRun, slot: int) -> list:
    """the stream's text at every mark, then at close, as the reference's write_log calls see them"""
    out = [r.snaps[slot][k] for k in sorted(r.snaps[slot])]
    if slot in r.final:
        out.append(r.final[slot])
    return out


def check_stream(r: TapRun, slot: int, transcripts: list, where="") -> bool:
    """False when the device reports the stream's text as not authoritative (TF_EXOTIC)"""
    flags = r.flags[slot]
    if flags & _abi.TF_EXOTIC:
        return False
    assert not flags & (_abi.TF_CARRY_OVERFLOW | _abi.TF_MARKQ_OVERFLOW), (where, slot, flags)
    got = [decode_text(t) for t in texts_of(r, slot)]
    assert sorted(r.snaps[slot]) == list(range(1, len(r.snaps[slot]) + 1)), (where, slot, sorted(r.snaps[slot]))
    assert got == transcripts, f"{where} slot {slot}: text != reference"
    has_surr = any(0xD800 <= ord(ch) <= 0xDFFF for t in transcripts[-1:] for ch in t)
    assert bool(flags & _abi.TF_LONE_SURROGATE) == has_surr, (where, slot)
    return True


def check_pairing(r: TapRun, where=""):
    """each step's row events (relay, push_row) and marks (tap, text_push_mark) name the same (slot, seq), for streams that are
    not exotic and whose queues did not overflow"""
    for k, (marks, rows) in enumerate(zip(r.step_marks, r.step_rows)):
        bad = {s for s, f in r.step_flags[k].items() if f & (_abi.TF_EXOTIC | _abi.TF_MARKQ_OVERFLOW | _abi.TF_CARRY_OVERFLOW)}
        bad |= {s for s, f in r.step_sflags[k].items() if f & (_abi.SF_ROWQ_OVERFLOW | _abi.SF_CARRY_OVERFLOW)}
        bad |= {s for s, st in r.states.items() if st.n_exotic}
        a = {m for m in marks if m[0] not in bad}
        b = {m for m in rows if m[0] not in bad}
        assert a == b, f"{where} step {k}: marks without rows {sorted(a - b)[:8]}, rows without marks {sorted(b - a)[:8]}"


# ---- content -------------------------------------------------------------------------------------------------------------------

_FRAGS = ["a", "bc", "hello ", "x" * 17, "y" * 40, '\\"', "\\\\", "\\/", "\\n", "\\t", "\\r\\b\\f", "\\u00e9", "\\u4e2d", "\\u0041",
          "\\ud83d\\ude00", "\\uD83C\\uDF89", "é", "中文", "😀", "ü", "—", " ", "{", "}", "data: ", "\\\\n\\\\n"]


def rich_piece(rng) -> str:
    """a JSON string body of `n` bytes or a little less, n in 0..200"""
    n = rng.randrange(0, 201)
    out, k = [], 0
    while True:
        f = rng.choice(_FRAGS)
        b = len(f.encode())
        if k + b > n:
            break
        out.append(f); k += b
    return "".join(out)


def rich_event(rng, i: int) -> bytes:
    return ('data: {"id":"r%d","object":"chat.completion.chunk","choices":[{"index":0,"delta":{"content":"%s"},"finish_reason":null}]}\n\n'
            % (i, rich_piece(rng))).encode("utf-8")


@dataclass
class Rich:
    chunks: list
    irregular: set = field(default_factory=set)     # chunk indices the one-chunk-per-lane path cannot take (or that start with a tap carry)
    kind: str = ""
    transcripts: list = field(default_factory=list)  # the plain json.loads reading of the events


def rich_stream(rng, force: str | None = None) -> Rich:
    """40..300 chunks of 1..3 whole events; about one stream in five gets one irregular chunk at index >= 33"""
    n = rng.randrange(40, 301)
    chunks = [b"".join(rich_event(rng, 100 * c + j) for j in range(rng.randrange(1, 4))) for c in range(n)]
    r = Rich(chunks)
    kind = force or (rng.choice(["cut", "utf8", "error"]) if rng.random() < 0.2 else "")
    at = rng.randrange(33, n - 1)
    if kind == "cut":                        # an event cut across two chunks: the split crosses a chunk
        blob = chunks[at] + chunks[at + 1]
        k = len(chunks[at]) + rng.randrange(3, 40)
        chunks[at:at + 2] = [blob[:k], blob[k:]]
        r.irregular = {at, at + 1}
    elif kind == "utf8":                     # decode raises: the tap skips the chunk
        chunks.insert(at, b'data: {"choices":[{"delta":{"content":"\xff\xfe lost"}}]}\n\n')
        r.irregular = {at}
    elif kind == "error":                    # a mark; the event's own text is appended
        chunks.insert(at, ('data: {"error":{"message":"upstream %s","code":502}}\n\n' % rich_piece(rng)).encode())
        r.irregular = {at}
    r.kind = kind
    # the plain reading: json.loads of every event of every decodable chunk
    text, marks = "", []
    for c in chunks if kind != "cut" else [b"".join(chunks)]:
        try:
            s = c.decode("utf-8")
        except UnicodeDecodeError:
            continue
        for ev in s.split("\n\n")[:-1]:
            doc = json.loads(ev[len("data: "):])
            if "choices" in doc:
                text += doc["choices"][0]["delta"]["content"]
            if "error" in doc:
                text += ev[len("data: "):].strip()
                marks.append(text)
    r.transcripts = marks + [text]
    return r


def c3_text(chunks) -> bytes:
    """the content bytes of every delta event of a C3 stream (synth.sse_batch), sliced from its bytes"""
    blob = np.frombuffer(b"".join(chunks), dtype=np.uint8)
    n = len(blob) // DELTA_EVENT_BYTES
    while n and bytes(blob[(n - 1) * DELTA_EVENT_BYTES:(n - 1) * DELTA_EVENT_BYTES + len(DELTA_HEAD)]) != DELTA_HEAD:
        n -= 1
    ev = blob[:n * DELTA_EVENT_BYTES].reshape(n, DELTA_EVENT_BYTES)
    assert all(bytes(h) == DELTA_HEAD for h in ev[:, :len(DELTA_HEAD)])
    return ev[:, len(DELTA_HEAD):len(DELTA_HEAD) + DELTA_CONTENT].tobytes()


def pad_stream(i: int) -> list:
    return [sc.delta("p%d" % i)]


_ADV, _ADV_ORACLE = [], {}


def adversarial():
    if not _ADV:
        _ADV.extend(s for k, g in enumerate(GENERATORS) for s in make_streams(g, 24, 3100 + k))
        rng = random.Random(3177)
        _ADV.extend(TG._stream(rng) for _ in range(150))
    return _ADV


def adv_oracle(i: int):
    from oracle.sse_oracle import run_stream
    if i not in _ADV_ORACLE:
        _ADV_ORACLE[i] = run_stream(adversarial()[i])
    return _ADV_ORACLE[i]


_RICH = {}


def rich_set(size: int):
    """about a quarter of a `size` MiB step of rich ballast (12 streams at least); the first three streams have one irregular
    chunk of each kind"""
    if size not in _RICH:
        rng = random.Random(4400 + size)
        out, n = [], 0
        while n < size * MiB // 4 or len(out) < 12:
            st = rich_stream(rng, ["cut", "utf8", "error"][len(out)] if len(out) < 3 else None)
            out.append(st); n += sum(map(len, st.chunks))
        _RICH[size] = out
    return _RICH[size]


def build(size: int, n_steps: int, n_slices: int, seed: int, min_segs: int = 1100):
    """adversarial + rich + C3 streams, shuffled, each cut into n_steps parts at random chunks; every step padded with one-chunk
    streams to min_segs segments; for a sliced entry, segments without bytes at every other slice start (as in
    test_sse_geometry_gpu.build_steps).  -> steps, slots, kinds (slot -> (kind, index)), C3 streams, step of every chunk cut"""
    rng = random.Random(seed)
    adv, rich = adversarial(), rich_set(size)
    used = sum(len(c) for s in adv for c in s) + sum(len(c) for s in rich for c in s.chunks)
    target = size * MiB * n_steps + (size * MiB * n_steps) // 10
    n_events = 256 if size > 4 else 64
    n_c3 = max(1, (target - used) // (n_events * DELTA_EVENT_BYTES + 400))
    b = sse_batch(n_streams=n_c3, n_events=n_events, seed=size * 10 + n_steps, events_per_chunk=8)
    c3 = [b.stream_chunks(s) for s in range(n_c3)]
    kinds = [("adv", i) for i in range(len(adv))] + [("rich", i) for i in range(len(rich))] + [("c3", i) for i in range(n_c3)]
    rng.shuffle(kinds)
    streams = [adv[i] if k == "adv" else (rich[i].chunks if k == "rich" else c3[i]) for k, i in kinds]
    bounds = []
    for st in streams:
        cuts = sorted(set(rng.randrange(0, len(st) + 1) for _ in range(n_steps - 1)))
        bounds.append([0] + cuts + [len(st)])
    steps, nxt = [], len(streams)
    for k in range(n_steps):
        parts = [(i, streams[i][b_[k]:b_[k + 1]]) for i, b_ in enumerate(bounds) if k < len(b_) - 1 and b_[k + 1] > b_[k]]
        while len(parts) < min_segs:
            parts.insert(rng.randrange(len(parts) + 1), (nxt, pad_stream(nxt)))
            kinds.append(("pad", nxt)); nxt += 1
        if n_slices > 1:
            starts = np.cumsum([0] + [sum(map(len, c)) for _, c in parts])
            for j in range(n_slices - 1, 0, -2):
                at = int(np.searchsorted(starts[:-1], int(starts[-1]) * j // n_slices, side="left"))
                parts.insert(at, (nxt, [] if j % 4 == 1 else [b"", b""]))
                kinds.append(("idle", nxt)); nxt += 1
        steps.append(parts)
    assert nxt <= 8192
    return steps, list(range(nxt)), kinds, c3, bounds


# ---- production geometry -------------------------------------------------------------------------------------------------------

CASES = [(size, entry, 1, 1100) for size in (2, 20) for entry in ENTRIES] + [(60, "device", 1, 1100), (60, "slices8", 1, 1100)] + [
    (2, "device", 1, 4200), (20, "device", 3, 1100), (20, "slices8", 3, 1100), (2, "slices3", 3, 1100), (2, "host_relay8", 3, 1100)]


@pytest.mark.parametrize("size,entry,n_steps,min_segs", CASES, ids=[f"{s}MiB-{e}-{n}step-{m}segs" for s, e, n, m in CASES])
def test_tap_at_production_geometry(engine, size, entry, n_steps, min_segs, monkeypatch):
    step_fn, n_slices = ENTRIES[entry]
    if n_slices:
        monkeypatch.setenv("LGW_SLICES", str(n_slices))
    steps, slots, kinds, c3, bounds = build(size, n_steps, n_slices or 1, seed=size * 13 + n_steps, min_segs=min_segs)
    where = f"{size}MiB {entry} {n_steps} step(s)"
    r = run_tapped(engine, steps, slots, step_fn)
    n_bytes = [sum(len(c) for _, ch in parts for c in ch) for parts in steps]
    assert all(n > min_segs - 1 for n in r.n_segs) and all(b <= MAX_BYTES for b in n_bytes), (where, r.n_segs, n_bytes)
    assert max(n_bytes) >= size * MiB, (where, n_bytes)
    if min_segs > 4096:
        assert max(r.n_segs) > 4096

    rich = rich_set(size)
    n_adv = n_cmp = n_seq_ok = n_rich_segs = n_rich_regular = 0
    for slot, (kind, i) in enumerate(kinds):
        if kind == "adv":
            relay, tap = adv_oracle(i)
            n_adv += 1
            if relay.failed:
                assert not r.snaps[slot] and not r.final.get(slot), (where, slot)
                continue
            n_cmp += check_stream(r, slot, tap.transcripts, where)
        elif kind == "rich":
            relay, tap = run_stream_cached(size, i)
            assert tap.transcripts == rich[i].transcripts, (size, i)        # the generator's own reading agrees with the oracle
            assert check_stream(r, slot, tap.transcripts, where)
        elif kind == "c3":
            assert r.flags[slot] == 0 and not r.snaps[slot], (where, slot)
            assert r.final[slot] == c3_text(c3[i]), f"{where} slot {slot}: C3 text"
        elif kind == "pad":
            assert r.final[slot] == b"p%d" % i and r.flags[slot] == 0, (where, slot)
    assert n_adv - n_cmp <= EXOTIC_SHARE * n_adv + sum(adv_oracle(i)[0].failed for k, i in kinds if k == "adv"), (where, n_adv, n_cmp)

    # which path each segment took
    for k, parts in enumerate(steps):
        for slot, chunks in parts:
            kind, i = kinds[slot]
            f = r.step_flags[k][slot]
            if kind in ("c3", "pad"):
                assert not f & _abi.TF_SEQUENTIAL, (where, k, slot)
            elif kind == "rich":
                c0, c1 = bounds[slot][k], bounds[slot][k + 1]
                late = any(c0 <= c < c1 for c in rich[i].irregular)
                assert bool(f & _abi.TF_SEQUENTIAL) == late, (where, k, slot, rich[i].kind, sorted(rich[i].irregular), c0, c1)
                n_rich_segs += 1
                n_rich_regular += not late
    assert n_rich_regular > n_rich_segs / 2, (where, n_rich_regular, n_rich_segs)
    check_pairing(r, where)


_RICH_ORACLE = {}


def run_stream_cached(size: int, i: int):
    from oracle.sse_oracle import run_stream
    if (size, i) not in _RICH_ORACLE:
        _RICH_ORACLE[(size, i)] = run_stream(rich_set(size)[i].chunks)
    return _RICH_ORACLE[(size, i)]


# ---- hand-built steps ----------------------------------------------------------------------------------------------------------

def check_case_vs_oracle(r: TapRun, streams: dict, where=""):
    from oracle.sse_oracle import run_stream
    for slot, chunks in streams.items():
        relay, tap = run_stream([c for c in chunks if c])
        assert not relay.failed, (where, slot)
        assert check_stream(r, slot, tap.transcripts, where), (where, slot)


def _all_chunks(steps):
    out = {}
    for parts in steps:
        for s, ch in parts:
            out.setdefault(s, []).extend(ch)
    return out


SEG_COUNTS = [1023, 1024, 1025, 2048, 2049, 8192]


def many_segments(engine, n_segs: int, step_fn=host_tap):
    """n_segs one-chunk streams whose texts all have different lengths (a permutation of 1..n_segs): k_text_scan's block loop,
    its carry and its reuse of warp_sum between blocks of 1 024 segments"""
    rng = random.Random(n_segs)
    lens = list(range(1, n_segs + 1))
    rng.shuffle(lens)
    steps = [[(s, [sc.delta(chr(0x61 + s % 26) * n)]) for s, n in enumerate(lens)]]
    r = run_tapped(engine, steps, range(n_segs), step_fn)
    assert r.n_segs == [n_segs]
    for s, n in enumerate(lens):
        assert r.final[s] == chr(0x61 + s % 26).encode() * n and r.flags[s] == 0, (n_segs, s)
        assert not r.step_flags[0][s] & _abi.TF_SEQUENTIAL


def error_event(content: str, msg: str = "overloaded") -> bytes:
    return ('data: {"choices":[{"index":0,"delta":{"content":"%s"}}],"error":{"message":"%s"}}\n\n' % (content, msg)).encode()


def adjacent_error_segments(engine, step_fn=host_tap, n_big: int = 3):
    """Adjacent segments that each take the sequential walk with a ~40 KiB "error" event whose bulk is delta.content: each appends
    the content, then the event's own text -- close to twice its bytes, the sparse buffer's whole room; the next segment's region
    starts right behind it.  Regular segments before and after."""
    rng = random.Random(8)
    steps = [[(0, [sc.delta("before")])] + [
        (1 + k, [sc.delta("s%d" % k), error_event("".join(rng.choice("abcdefgh") for _ in range(40960 + 97 * k)), "m%d" % k)])
        for k in range(n_big)] + [(1 + n_big, [sc.delta("after"), sc.delta("!")])]]
    r = run_tapped(engine, steps, range(n_big + 2), step_fn)
    for k in range(n_big):
        assert r.step_flags[0][1 + k] & _abi.TF_SEQUENTIAL
        seg = steps[0][1 + k][1]
        assert len(r.final[1 + k]) > 1.9 * sum(map(len, seg)) - 200, len(r.final[1 + k])
    check_case_vs_oracle(r, _all_chunks(steps), "adjacent error segments")
    check_pairing(r, "adjacent error segments")


def carry_cap_tail(engine, carry_cap: int, step_fn=host_tap):
    """An unterminated event tail of exactly carry_cap bytes at a step end is carried exactly; one of carry_cap + 1 bytes sets
    TF_CARRY_OVERFLOW and the relay's SF_CARRY_OVERFLOW"""
    head = b'data: {"choices":[{"delta":{"content":"'
    rest = b'"}}]}\n\n'
    steps, streams = [[], []], {}
    for slot, extra in ((0, 0), (1, 1), (2, -1)):
        n = carry_cap + extra
        tail = head + b"z" * (n - len(head))
        first = [sc.delta("go %d" % slot), sc.delta("on") + tail]
        steps[0].append((slot, first))
        steps[1].append((slot, [rest + sc.delta("end"), sc.USAGE_EV]))
    steps[0].append((3, [sc.delta("bystander")]))
    steps[1].append((3, [sc.delta("still here")]))
    r = run_tapped(engine, steps, range(4), step_fn)
    all_chunks = _all_chunks(steps)
    check_case_vs_oracle(r, {s: all_chunks[s] for s in (0, 2, 3)}, "carry_cap tail")
    assert not r.step_sflags[0][0] & _abi.SF_CARRY_OVERFLOW and not r.step_flags[0][0] & _abi.TF_CARRY_OVERFLOW
    assert r.flags[1] & _abi.TF_CARRY_OVERFLOW, r.flags[1]
    assert r.step_flags[0][1] & _abi.TF_CARRY_OVERFLOW
    assert r.states[1].flags & _abi.SF_CARRY_OVERFLOW, r.states[1].flags


def one_big_event(engine, step_fn=host_tap, n: int = 200 * 1024):
    """a single 200 KiB event in a chunk that ends on LF LF takes the one-chunk-per-lane path"""
    rng = random.Random(2)
    head, tail = b'data: {"choices":[{"index":0,"delta":{"content":"', b'"}}]}\n\n'
    body, k = [], len(head) + len(tail)
    while k < n:
        f = rng.choice(["q", "\\u00e9", "\\n", "中", '\\"', "\\ud83d\\ude00", "z" * 50])
        f = f if k + len(f.encode()) <= n else "x" * (n - k)
        body.append(f); k += len(f.encode())
    big = head + "".join(body).encode() + tail
    assert len(big) == n
    steps = [[(0, [sc.delta("a")]), (1, [big, sc.USAGE_EV]), (2, [sc.delta("b")])]]
    r = run_tapped(engine, steps, range(3), step_fn)
    assert not r.step_flags[0][1] & _abi.TF_SEQUENTIAL
    check_case_vs_oracle(r, _all_chunks(steps), "one big event")


def mark_queue_overflow(engine, step_fn=host_tap, n_streams: int = 200, n_again: int = 40):
    """rowq_cap (the mark queue's capacity too) below the marks of one step: the first step's 2 * n_streams marks overflow it,
    the second step's n_again fit.  The marks returned carry the oracle's text; a stream without TF_MARKQ_OVERFLOW has all of
    its marks; the flag stays; the second step's seq continues the count past the dropped marks, as the relay's rows do."""
    from oracle.sse_oracle import run_stream
    cap = engine.limits.rowq_cap
    assert 2 * n_streams > cap >= n_again
    again = list(range(0, n_streams, n_streams // n_again))[:n_again]
    steps = [[(s, [sc.delta("s%d" % s), error_event("e1-%d" % s), sc.delta("mid"), error_event("e2-%d" % s)]) for s in range(n_streams)],
             [(s, [error_event("e3-%d" % s), sc.delta("tail")]) for s in again]]
    r = run_tapped(engine, steps, range(n_streams), step_fn)
    streams = _all_chunks(steps)
    tap = {s: run_stream(streams[s])[1].transcripts for s in range(n_streams)}
    assert len(r.step_marks[0]) == cap, len(r.step_marks[0])
    for slot, seq in r.step_marks[0]:
        assert decode_text(r.snaps[slot][seq]) == tap[slot][seq - 1], (slot, seq)
    flagged = set()
    for s in range(n_streams):
        f = r.step_flags[0][s]
        if f & _abi.TF_MARKQ_OVERFLOW:
            flagged.add(s)
            assert r.flags[s] & _abi.TF_MARKQ_OVERFLOW
        else:
            assert {1, 2} <= set(r.snaps[s]), (s, sorted(r.snaps[s]))
    assert len(flagged) >= n_streams - cap // 2
    for s in again:
        if s in flagged:
            assert r.step_flags[1][s] & _abi.TF_MARKQ_OVERFLOW, s
        assert decode_text(r.snaps[s][3]) == tap[s][2], s
        assert decode_text(r.final[s]) == tap[s][3], s
    for s in range(n_streams):
        assert decode_text(r.final[s]) == tap[s][-1], s                  # the text itself does not depend on the queue
    assert len(r.step_marks[1]) == n_again and r.step_marks[1] == r.step_rows[1] == {(s, 3) for s in again}
    assert any(s in flagged for s in again)


@pytest.mark.parametrize("entry", ["device", "slices8"])
@pytest.mark.parametrize("n_segs", SEG_COUNTS)
def test_segment_counts_at_scan_block_edges(engine, n_segs, entry, monkeypatch):
    step_fn, n_slices = ENTRIES[entry]
    if n_slices:
        monkeypatch.setenv("LGW_SLICES", str(n_slices))
    many_segments(engine, n_segs, step_fn)


def late_irregular_chunks(engine, step_fn=host_tap):
    """rich streams whose one irregular chunk (cut event, invalid UTF-8, "error" event) lies in the second or a later batch of
    32 chunks: the regular attempt has already written pieces for the earlier batches, must drop them and leave the segment to
    the sequential walk; and rich streams without one, which stay on the lane path"""
    rng = random.Random(12)
    rich = [rich_stream(rng, kind) for kind in ["cut", "utf8", "error"] * 3 + [""] * 3]
    assert all(min(s.irregular) >= 33 for s in rich[:9])
    steps = [[(k, s.chunks) for k, s in enumerate(rich)]]
    r = run_tapped(engine, steps, range(len(rich)), step_fn)
    for k, s in enumerate(rich):
        assert bool(r.step_flags[0][k] & _abi.TF_SEQUENTIAL) == bool(s.kind), (k, s.kind)
    check_case_vs_oracle(r, _all_chunks(steps), "late irregular chunks")
    for k, s in enumerate(rich):
        assert [decode_text(t) for t in texts_of(r, k)] == s.transcripts, k
    check_pairing(r, "late irregular chunks")


HAND_BUILT = {"adjacent_error_segments": adjacent_error_segments, "one_big_event": one_big_event,
              "late_irregular_chunks": late_irregular_chunks,
              "carry_cap_tail": lambda e, f: carry_cap_tail(e, e.limits.carry_cap, f)}


@pytest.mark.parametrize("entry", ["device", "slices1", "slices8"])
@pytest.mark.parametrize("case", list(HAND_BUILT))
def test_hand_built(engine, case, entry, monkeypatch):
    step_fn, n_slices = ENTRIES[entry]
    if n_slices:
        monkeypatch.setenv("LGW_SLICES", str(n_slices))
    HAND_BUILT[case](engine, step_fn)


@pytest.mark.parametrize("entry", ["device", "slices8"])
def test_mark_queue_overflow(entry, monkeypatch):
    step_fn, n_slices = ENTRIES[entry]
    if n_slices:
        monkeypatch.setenv("LGW_SLICES", str(n_slices))
    e = new_engine(rowq_cap=64)
    try:
        mark_queue_overflow(e, step_fn)
    finally:
        e.close_engine()


# ---- direct modes --------------------------------------------------------------------------------------------------------------

_DIRECT = r'''
import sys
sys.path[:0] = ["tests", "."]
import numpy as np
import test_transcript_geometry_gpu as T

steps, slots, kinds, c3, bounds = T.build(2, 2, 1, seed=41, min_segs=1100)
assert all(sum(len(c) for _, ch in p for c in ch) >= 1 << 20 for p in steps)
eng = T.new_engine()
pins = {}
def pinned_tap(e, pb):
    n = int(pb.data.size)
    if n not in pins:
        pins[n] = (e.alloc_pinned(n), e.alloc_pinned(n))
    pin_in, pin_out = pins[n]
    pin_in[:] = pb.data
    res = e.step(pin_in, pb.chunk_off, pb.seg_chunk, pb.seg_slot, out=pin_out)
    assert e.last_step_direct()
    st = e.step_transcript()
    got.append((st.text.tobytes(), st.seg_off.tobytes(), st.flags.tobytes(), sorted(st.marks)))
    return res, st
def staged_tap(e, pb):
    res, st = T.host_tap(e, pb)
    assert not e.last_step_direct()
    ref.append((st.text.tobytes(), st.seg_off.tobytes(), st.flags.tobytes(), sorted(st.marks)))
    return res, st
got, ref = [], []
a = T.run_tapped(eng, steps, slots, pinned_tap)
b = T.run_tapped(eng, steps, slots, staged_tap)
assert len(got) == len(ref) == 2
for k, (x, y) in enumerate(zip(got, ref)):
    assert x == y, ("step", k, [i for i in range(4) if x[i] != y[i]])
assert sum(len(x[3]) for x in got) > 0 and sum(len(x[0]) for x in got) > 1 << 18
print("DIRECT_OK")
'''


@pytest.mark.parametrize("direct", ["in", "out", "both"])
def test_direct_modes_with_transcripts(direct):
    """LGW_DIRECT is read once per process: a process per value.  With `in` the tap reads the caller's mapped host buffer."""
    env = dict(os.environ, LGW_DIRECT=direct)
    env.pop("LGW_SLICES", None)
    r = subprocess.run([sys.executable, "-c", _DIRECT], capture_output=True, text=True, timeout=600, env=env, cwd=str(ROOT))
    assert r.returncode == 0 and "DIRECT_OK" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
