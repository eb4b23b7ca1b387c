"""The bulk SSE step (k_prime2 -> k_relay2 -> k_commit2) at production geometry: adversarial streams of every fuzz generator
(tests/sse_generators.py) interleaved with C3 ballast, so that a step is 2 MiB (one 3 KiB tile per warp), 20 MiB (>= 4) or
60 MiB (>= 10); through the device entry point (never sliced) and the host-buffer one cut into 1, 3, 8 or 14 slices, with
segments without bytes placed at slice starts; with cold and warm template caches; in one step or three.  Every case runs
the same steps on the exact sequential path (mode 1) and requires the same bytes, segment results, row events, stream states
and usage records; the adversarial streams are checked against the oracle, the ballast against its known usage values.
Counters show that the bulk path did the work.  Hand-built steps (tests/slice_cases.py) put the slice edges where the
kernels are easiest to get wrong, and the direct (pinned host buffer) modes run on adversarial content."""
import os
import random
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import slice_cases as SC
from llmapigateway_b200 import _abi
from llmapigateway_b200.engine import SEG_DTYPE, StepResult
from llmapigateway_b200.synth import sse_batch
from sse_generators import GENERATORS, make_streams

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
_R2 = (ROOT / "llmapigateway_b200" / "csrc" / "relay2.cuh").read_text()
R2_WARPS = int(re.search(r"#define R2_WARPS (\d+)u", _R2).group(1))          # the bulk kernel's block geometry, as compiled
R2_TILE = int(re.search(r"#define R2_TILE (\d+)u", _R2).group(1))
MiB = 1 << 20
MAX_BYTES = 96 * MiB
N_PER_GEN = 36                                   # adversarial streams per generator and step set
BULK_SHARE = 0.3                                 # adversarial segments the bulk path must settle, at least (about half do)


def _new_engine():
    import llmapigateway_b200 as L
    return L.Engine(max_streams=8192, max_step_chunks=1 << 21, max_step_bytes=MAX_BYTES)


@pytest.fixture(scope="module")
def engine():
    e = _new_engine()
    yield e
    e.close_engine()


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles_per_warp(b0: int, b1: int, sm_count: int) -> int:
    """launch_step_fast: tiles of the launch over sm_count * R2_WARPS warps"""
    base0 = b0 & ~15
    n_tiles = (b1 - base0 + R2_TILE - 1) // R2_TILE if b1 > base0 else 0
    max_warps = sm_count * R2_WARPS
    return (n_tiles + max_warps - 1) // max_warps


# ---- content -----------------------------------------------------------------------------------------------------------------------

_ADV, _ORACLE = {}, {}


def adversarial(seed: int):
    if seed not in _ADV:
        _ADV[seed] = [s for k, g in enumerate(GENERATORS) for s in make_streams(g, N_PER_GEN, seed * 100 + k)]
    return _ADV[seed]


def oracle(seed: int, i: int):
    """the oracle's result for stream i of adversarial(seed), computed once per module"""
    from oracle.sse_oracle import run_stream
    key = (seed, i)
    if key not in _ORACLE:
        _ORACLE[key] = run_stream(adversarial(seed)[i])
    return _ORACLE[key]


def ballast(total: int, seed: int):
    """C3 streams (64-byte deltas, 8 per chunk, usage event, [DONE]) of about `total` bytes in all, with their usage truths"""
    n_events = 256 if total > 4 * MiB else 64
    per = n_events * 64 + 400
    b = sse_batch(n_streams=max(1, total // per), n_events=n_events, seed=seed, events_per_chunk=8)
    return [b.stream_chunks(s) for s in range(len(b.truths))], b.truths


def build_steps(size: int, n_steps: int, seed: int, n_slices: int):
    """the adversarial set interleaved with ballast, each stream cut into n_steps parts at random chunks (as in _run_all); for
    a sliced entry, a segment without bytes (no chunks, or empty chunks) of an idle stream is put at every other slice's cut"""
    rng = random.Random(seed)
    adv = adversarial(1)
    adv_bytes = sum(len(c) for s in adv for c in s)
    target = size * MiB * n_steps + (size * MiB * n_steps) // 10
    bal, truths = ballast(max(0, target - adv_bytes), seed=size * 10 + n_steps)
    kinds = [("adv", i) for i in range(len(adv))] + [("bal", i) for i in range(len(bal))]
    rng.shuffle(kinds)
    streams = [adv[i] if k == "adv" else bal[i] for k, i in kinds]
    bounds = []
    for st in streams:
        cuts = sorted(set(rng.randrange(0, len(st) + 1) for _ in range(n_steps - 1)))
        bounds.append([0] + cuts + [len(st)])
    n = len(streams)
    steps, idle = [], n
    for k in range(n_steps):
        parts = [(i, streams[i][b[k]:b[k + 1]]) for i, b in enumerate(bounds) if k < len(b) - 1 and b[k + 1] > b[k]]
        if n_slices > 1:
            starts = np.cumsum([0] + [sum(map(len, c)) for _, c in parts])
            for j in range(n_slices - 1, 0, -2):                     # (from the back: an insertion moves no byte)
                at = int(np.searchsorted(starts[:-1], int(starts[-1]) * j // n_slices, side="left"))
                parts.insert(at, (idle, [] if j % 4 == 1 else [b"", b""]))
                idle += 1
        steps.append(parts)
    return steps, list(range(idle)), kinds, truths


# ---- entry points ----------------------------------------------------------------------------------------------------------------

def device_step(engine, pb):
    """lgw_sse_step_device on torch CUDA tensors"""
    import torch
    n_segs = len(pb.seg_slot)
    d = [torch.from_numpy(x).cuda() for x in (pb.data if pb.data.size else np.zeros(16, np.uint8), pb.chunk_off, pb.seg_chunk, pb.seg_slot)]
    out = torch.empty_like(d[0])
    segs = torch.zeros(max(n_segs, 1) * SEG_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    engine.step_device(d[0].data_ptr(), int(pb.data.size), d[1].data_ptr(), pb.n_chunks, d[2].data_ptr(), d[3].data_ptr(), n_segs,
                       out.data_ptr(), segs.data_ptr())
    engine.sync()
    rows = engine.fetch_rows()
    return StepResult(out.cpu().numpy()[:pb.data.size], segs.cpu().numpy().view(SEG_DTYPE)[:n_segs], rows)


ENTRIES = {   # name: (step function, LGW_SLICES)
    "device": (device_step, None),
    "slices1": (SC.host_step, 1),
    "slices3": (SC.host_step, 3),
    "slices8": (SC.host_step, 8),
    "slices14": (SC.host_step, 14),
    "host_relay8": (lambda e, pb: SC.host_step(e, pb, relay_from_host=True), 8),
}
MIN_TPW = {2: 1, 20: 4, 60: 10}                  # tiles per warp of an unsliced step of that size
MIN_TPW_SLICED = {(20, 3): 2, (60, 3): 4, (60, 8): 2}   # ... of every slice of a sliced one (1 where not listed)

# every size with every entry point (warm, one step); cold / warm and one / three steps crossed on 20 MiB
CASES = [(size, entry, "warm", 1) for size in (2, 20, 60) for entry in ENTRIES] + [
    (20, "slices8", "cold", 1), (20, "slices8", "cold", 3), (20, "slices8", "warm", 3), (20, "device", "cold", 3), (20, "slices1", "warm", 3)]


@pytest.mark.parametrize("size,entry,templates,n_steps", CASES, ids=[f"{s}MiB-{e}-{t}-{n}step" for s, e, t, n in CASES])
def test_bulk_step_at_production_geometry(engine, size, entry, templates, n_steps, monkeypatch):
    step_fn, n_slices = ENTRIES[entry]
    if n_slices:
        monkeypatch.setenv("LGW_SLICES", str(n_slices))
    steps, slots, kinds, truths = build_steps(size, n_steps, seed=size * 7 + n_steps, n_slices=n_slices or 1)
    if templates == "cold":
        eng = _new_engine()
        assert eng.launch_count() == 0                                    # a fresh engine: no step has taught it a template
    else:
        eng = engine
        warm = adversarial(2)                                             # the same generators, another seed
        SC.run(eng, [list(enumerate(warm))], list(range(len(warm))), 0)
    try:
        c0 = eng.debug_counters()
        fast = SC.run(eng, steps, slots, 0, step_fn, keep_packed=True)
        c1 = eng.debug_counters()
        seq = SC.run(eng, steps, slots, 1)
    finally:
        if eng is not engine:
            eng.close_engine()
    where = f"{size}MiB {entry} {templates} {n_steps} step(s)"
    SC.compare_bulk_sequential(fast, seq, where)

    # geometry: tiles per warp of every launch, where the slices start
    sm = _sm_count()
    for pb in fast.packed:
        n_bytes = int(pb.data.size)
        assert n_bytes <= MAX_BYTES
        if n_slices and n_slices > 1:
            cuts = SC.slice_cuts(pb.chunk_off, pb.seg_chunk, n_slices)
            starts = SC.slice_starts(pb.chunk_off, pb.seg_chunk, n_slices)
            assert sum(b0 % 16 != 0 for b0, _, _ in starts) * 2 > len(starts), (where, starts)      # most slices start unaligned
            assert any(zero for _, _, zero in starts), (where, starts)                             # ... and one on a segment without bytes
            bounds = [(int(pb.chunk_off[pb.seg_chunk[cuts[j]]]), int(pb.chunk_off[pb.seg_chunk[cuts[j + 1]]])) for j in range(n_slices) if cuts[j + 1] > cuts[j]]
            tpw = min(tiles_per_warp(b0, b1, sm) for b0, b1 in bounds)
            assert tpw >= MIN_TPW_SLICED.get((size, n_slices), 1), (where, tpw)
        else:
            assert tiles_per_warp(0, n_bytes, sm) >= MIN_TPW[size], (where, n_bytes, tiles_per_warp(0, n_bytes, sm))
            if size == 2:
                assert tiles_per_warp(0, n_bytes, sm) == 1

    # the bulk path did the work: every ballast segment and a share of the adversarial ones
    n_bal = sum(1 for parts in steps for i, c in parts if i < len(kinds) and kinds[i][0] == "bal")
    n_adv = sum(1 for parts in steps for i, c in parts if i < len(kinds) and kinds[i][0] == "adv")
    bulk = c1["bulk"] - c0["bulk"]
    assert bulk >= n_bal + BULK_SHARE * n_adv, (where, c0, c1, n_bal, n_adv)

    # ballast against its usage truths and its own bytes; adversarial streams against the oracle
    for i, (k, j) in enumerate(kinds):
        if k != "bal":
            continue
        st = fast.states[i]
        assert st.phase == _abi.PHASE_COMMITTED and st.flags & _abi.SF_A_USAGE_BOUND, (where, i)
        assert b"".join(fast.emitted[i]) == b"".join(c for parts in steps for s, ch in parts if s == i for c in ch), (where, i)
        assert _abi.usage_rec_to_dict(st.rec) == truths[j].expected_row(), (where, i)
    adv_slots = [i for i, (k, _) in enumerate(kinds) if k == "adv"]
    n_cmp = SC.compare_oracle(SC.Run([fast.states[i] for i in adv_slots], fast.rows, fast.emitted, fast.segs), adv_slots,
                              None, lambda n: oracle(1, kinds[adv_slots[n]][1]), where)
    assert n_cmp > 0.9 * len(adv_slots)


# ---- hand-built slice edges ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", SC.directed_cases(), ids=lambda c: c.name)
def test_directed_slice_edges(engine, case, monkeypatch):
    monkeypatch.setenv("LGW_SLICES", str(case.n_slices))
    SC.check_directed(engine, case)


# ---- direct modes on adversarial content -----------------------------------------------------------------------------------------

_DIRECT = r'''
import sys
sys.path[:0] = ["tests", "."]
import numpy as np
import llmapigateway_b200 as L
import slice_cases as SC
from sse_generators import GENERATORS, make_streams
from llmapigateway_b200.synth import pack_streams, sse_batch

cold = sys.argv[1] == "cold"
adv = [s for k, g in enumerate(GENERATORS) for s in make_streams(g, 24, 500 + k)]
b = sse_batch(n_streams=96, n_events=512, seed=19, events_per_chunk=8)
streams = [s for pair in zip(adv, [b.stream_chunks(s) for s in range(96)]) for s in pair] + adv[96:]
rng = __import__("random").Random(4)
half = [rng.randrange(0, len(s) + 1) for s in streams]
steps = [[(i, s[:h]) for i, (s, h) in enumerate(zip(streams, half)) if h], [(i, s[h:]) for i, (s, h) in enumerate(zip(streams, half)) if h < len(s)]]
assert all(sum(len(c) for _, ch in p for c in ch) >= 1 << 20 for p in steps)
eng = L.Engine(max_streams=1024, max_step_chunks=1 << 18, max_step_bytes=32 << 20)
slots = list(range(len(streams)))
if not cold:
    SC.run(eng, [list(enumerate(adv[:100]))], list(range(100)), 0)
pins = {}
def pinned_step(e, pb):
    n = int(pb.data.size)
    if n not in pins:
        pins[n] = (e.alloc_pinned(n), e.alloc_pinned(n))
    pin_in, pin_out = pins[n]
    pin_in[:] = pb.data
    r = e.step(pin_in, pb.chunk_off, pb.seg_chunk, pb.seg_slot, out=pin_out)
    assert e.last_step_direct()
    return r
got = SC.run(eng, steps, slots, 0, pinned_step)
ref = SC.run(eng, steps, slots, 0)
assert not eng.last_step_direct()
SC.compare_bulk_sequential(got, ref, "direct vs staged")
seq = SC.run(eng, steps, slots, 1)
SC.compare_bulk_sequential(got, seq, "direct vs sequential")
print("DIRECT_OK")
'''


@pytest.mark.parametrize("templates", ["cold", "warm"])
@pytest.mark.parametrize("direct", ["in", "out", "both"])
def test_direct_modes_on_adversarial_content(direct, templates):
    """LGW_DIRECT is read once per process: a process per value.  Two steps of >= 1 MiB of adversarial streams and C3 ballast
    from page-locked buffers (the bulk kernel's TMA reads and / or writes host memory) equal the staged step and mode 1."""
    env = dict(os.environ, LGW_DIRECT=direct)
    env.pop("LGW_SLICES", None)
    r = subprocess.run([sys.executable, "-c", _DIRECT, templates], capture_output=True, text=True, timeout=600, env=env, cwd=str(ROOT))
    assert r.returncode == 0 and "DIRECT_OK" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
