"""k_relay2's own segment planning (csrc/relay2.cuh): a plain restatement of how a launch set is split among warps and of how
each warp finds its first segment (`first_segment`) and walks its plan window (`load_plans`), plus step layouts built to drive
those paths -- skewed stream lengths, dense runs of tiny segments, runs of segments without bytes, continuation steps of one
delta per stream, a handful of very long segments -- with the bulk / sequential path counts each layout must produce.

The model only says which planning paths a case reaches; whether a case passes is decided by its results.  Shared by the
emulator tests (tests/test_relay2_planning_cpu.py) and the GPU tests (tests/test_relay2_planning_gpu.py)."""
from __future__ import annotations

import bisect
import random
import re
from collections import Counter
from dataclasses import dataclass, field
from pathlib import Path

import slice_cases as SC
from llmapigateway_b200.synth import sse_batch

_R2 = (Path(__file__).resolve().parent.parent / "llmapigateway_b200" / "csrc" / "relay2.cuh").read_text()
R2_WARPS = int(re.search(r"#define R2_WARPS (\d+)u", _R2).group(1))          # the bulk kernel's block geometry, as compiled
R2_TILE = int(re.search(r"#define R2_TILE (\d+)u", _R2).group(1))
WINDOW = 32                                                                  # segments in a warp's plan window (one per lane)
MiB = 1 << 20

# first_segment's ways to its answer
SMALL = "n<=32"                  # the launch has at most 32 segments: one window holds them all
BRACKETED = "bracketed"          # the first round's 32 candidates bracket the answer (k > 0)
FIRST = "bracketed_at_0"         # ... at w0 == 0: the first candidate is the answer
BELOW_W0 = "below_w0"            # the first candidate already ends past x, the strided search below finds w0 itself
BELOW = "below"                  # ... and finds an earlier segment
ABOVE = "above"                  # no candidate ends past x: strided search above the window
PAST_END = "past_end"            # every segment ends at or before x (segments without bytes at the launch's end)
BRANCHES = (SMALL, BRACKETED, FIRST, BELOW_W0, BELOW, ABOVE, PAST_END)


# ---- geometry -------------------------------------------------------------------------------------------------------------------

def launch(b0: int, b1: int, sm_count: int | None = None, n_blocks: int | None = None, tiles_per_warp: int = 0):
    """(base0, n_tiles, tiles per warp, warps) of the bulk kernel over bytes [b0, b1).  sm_count: launch_step_fast (the engine);
    n_blocks (+ tiles_per_warp, 0 = spread): the emulator's step driver (tests/support/host_relay2*.cpp)."""
    base0 = b0 & ~15
    n_tiles = (b1 - base0 + R2_TILE - 1) // R2_TILE if b1 > base0 else 0
    if not n_tiles:
        return base0, 0, 0, 0
    if sm_count is not None:
        max_warps = sm_count * R2_WARPS
        tpw = (n_tiles + max_warps - 1) // max_warps
    else:
        max_warps = n_blocks * R2_WARPS
        tpw = tiles_per_warp or (n_tiles + max_warps - 1) // max_warps
        if (n_tiles + tpw - 1) // tpw > max_warps:
            tpw = (n_tiles + max_warps - 1) // max_warps
    return base0, n_tiles, tpw, (n_tiles + tpw - 1) // tpw


def warp_ranges(b0: int, b1: int, **geo):
    """[range_lo, range_hi) of every warp that has tiles (k_relay2: range_lo clamped to tile_base, range_hi to n_bytes)"""
    base0, n_tiles, tpw, warps = launch(b0, b1, **geo)
    out = []
    for gw in range(warps):
        base = base0 + gw * tpw * R2_TILE
        nt = min(tpw, n_tiles - gw * tpw)
        out.append((max(base, b0), min(base + nt * R2_TILE, b1)))
    return out


def first_segment(ends, tile_base: int, n_bytes: int, x: int):
    """relay2.cuh first_segment over segment ends `ends` (launch-relative indices): (segment, window's first segment, w0,
    branch, clamped).  clamped: the guess was moved down to n - 32."""
    n = len(ends)
    nb = n_bytes - tile_base
    g = n * (x - tile_base) // nb if nb else 0
    lo_guess = g - 16 if g > 16 else 0
    clamped = n > WINDOW and lo_guess > n - WINDOW
    w0 = 0 if n <= WINDOW else min(lo_guess, n - WINDOW)
    past = [i for i in range(WINDOW) if w0 + i < n and ends[w0 + i] > x]
    if past:
        k = past[0]
        if k or w0 == 0:
            return w0 + k, w0, w0, SMALL if n <= WINDOW else (BRACKETED if k else FIRST), clamped
        s = bisect.bisect_right(ends, x, 0, w0)                # the first segment in [0, w0) that ends past x, else w0
        return s, s, w0, BELOW_W0 if s == w0 else BELOW, clamped
    if w0 + WINDOW >= n:
        return n, w0, w0, SMALL if n <= WINDOW else PAST_END, clamped
    s = bisect.bisect_right(ends, x, w0 + WINDOW, n)
    return s, s, w0, ABOVE, clamped


@dataclass
class WarpPlan:
    slice: int
    range_lo: int
    range_hi: int
    w0: int
    branch: str
    clamped: bool
    seg0: int                    # first segment (step index)
    visited: int                 # segments the walk enters
    reloads: list                # step indices of the segments at which the window is reloaded


def walk(starts, ends, seg0: int, win_lo: int, range_lo: int, range_hi: int):
    """k_relay2's segment loop: (segments entered, segments at which the plan window is reloaded).  A warp leaves its loop at the
    first segment that starts at or past range_hi (a segment whose walk ends the warp's work reaches past range_hi itself)."""
    n = len(ends)
    seg, seg_first, visited, reloads = seg0, range_lo, 0, []
    while seg < n and seg_first < range_hi:
        if seg - win_lo >= WINDOW:
            win_lo = seg
            reloads.append(seg)
        visited += 1
        seg_first = ends[seg]
        seg += 1
    return visited, reloads


def model_step(chunk_off, seg_chunk, n_slices: int = 1, **geo) -> list[WarpPlan]:
    """every warp of every launch set of a step: unsliced (n_slices = 1, the device entry point) or cut as lgw_sse_step cuts a
    host-buffer step.  A slice is modelled as step_device launches it: tile_base = its first byte, segments counted from its
    first segment."""
    cuts = SC.slice_cuts(chunk_off, seg_chunk, n_slices) if n_slices > 1 else [0, len(seg_chunk) - 1]
    plans = []
    for j in range(len(cuts) - 1):
        s0, s1 = cuts[j], cuts[j + 1]
        if s1 <= s0:
            continue
        b0, b1 = int(chunk_off[seg_chunk[s0]]), int(chunk_off[seg_chunk[s1]])
        ends = [int(chunk_off[seg_chunk[s + 1]]) for s in range(s0, s1)]
        starts = [int(chunk_off[seg_chunk[s]]) for s in range(s0, s1)]
        for lo, hi in warp_ranges(b0, b1, **geo):
            seg, win_lo, w0, branch, clamped = first_segment(ends, b0, b1, lo)
            visited, reloads = walk(starts, ends, seg, win_lo, lo, hi)
            plans.append(WarpPlan(j, lo, hi, w0 + s0, branch, clamped, seg + s0, visited, [r + s0 for r in reloads]))
    return plans


@dataclass
class Coverage:
    branches: Counter = field(default_factory=Counter)
    clamped: int = 0
    max_visited: int = 0
    max_reloads: int = 0
    reloads: int = 0
    fresh_after_reload: int = 0          # reloads whose first segment is a fresh stream's segment with its kept chunk
    committed_after_reload: int = 0
    zero_run_at_range_lo: int = 0        # longest run of segments without bytes that sits at some warp's range_lo

    def add(self, o: "Coverage"):
        self.branches.update(o.branches)
        self.clamped += o.clamped
        self.max_visited = max(self.max_visited, o.max_visited)
        self.max_reloads = max(self.max_reloads, o.max_reloads)
        self.reloads += o.reloads
        self.fresh_after_reload += o.fresh_after_reload
        self.committed_after_reload += o.committed_after_reload
        self.zero_run_at_range_lo = max(self.zero_run_at_range_lo, o.zero_run_at_range_lo)

    def line(self) -> str:
        b = " ".join(f"{k}={self.branches[k]}" for k in BRANCHES if self.branches[k])
        return (f"branches[{b}] clamp={self.clamped} max_segs_per_warp={self.max_visited} max_reloads={self.max_reloads} "
                f"reloads={self.reloads} fresh_after_reload={self.fresh_after_reload} committed_after_reload={self.committed_after_reload} "
                f"zero_run_at_range_lo={self.zero_run_at_range_lo}")


def coverage(chunk_off, seg_chunk, fresh, plans: list[WarpPlan]) -> Coverage:
    """fresh[s]: segment s belongs to a stream that has had no bytes before this step"""
    c = Coverage()
    n = len(seg_chunk) - 1
    starts = [int(chunk_off[seg_chunk[s]]) for s in range(n)]
    ends = [int(chunk_off[seg_chunk[s + 1]]) for s in range(n)]
    for p in plans:
        c.branches[p.branch] += 1
        c.clamped += p.clamped
        c.max_visited = max(c.max_visited, p.visited)
        c.max_reloads = max(c.max_reloads, len(p.reloads))
        c.reloads += len(p.reloads)
        for r in p.reloads:
            if ends[r] > starts[r]:
                if fresh[r]:
                    c.fresh_after_reload += 1
                else:
                    c.committed_after_reload += 1
        s = bisect.bisect_left(starts, p.range_lo)
        k = s
        while k < n and starts[k] == ends[k] == p.range_lo:
            k += 1
        c.zero_run_at_range_lo = max(c.zero_run_at_range_lo, k - s)
    return c


# ---- layouts ----------------------------------------------------------------------------------------------------------------------

@dataclass
class Layout:
    name: str
    steps: list                  # one [(slot, chunks)] per step, as slice_cases.run takes them
    slots: list
    truths: dict                 # regular stream slot -> its synth.UsageTruth (None: deltas only, no usage event)
    adversarial: dict = field(default_factory=dict)    # adversarial stream slot -> its chunks (all steps)
    wants: set = field(default_factory=set)             # model coverage the layout is built for (see `reaches`)

    def chunks_of(self, slot: int) -> list[bytes]:
        return [c for parts in self.steps for s, ch in parts if s == slot for c in ch]

    def fresh(self, k: int) -> list[bool]:
        """per segment of step k: its stream has had no bytes in an earlier step"""
        seen = {s for parts in self.steps[:k] for s, ch in parts if any(ch)}
        return [s not in seen for s, _ in self.steps[k]]


class _Slots:
    def __init__(self):
        self.n = 0

    def take(self, k: int = 1) -> list[int]:
        self.n += k
        return list(range(self.n - k, self.n))


def _regular(n: int, n_events: int, seed: int, epc: int = 1):
    """n C3 streams (64-byte deltas, usage event, [DONE]) with their usage truths"""
    b = sse_batch(n_streams=n, n_events=n_events, seed=seed, events_per_chunk=epc)
    return [b.stream_chunks(s) for s in range(n)], b.truths


def _huge(total: int, n: int, seed: int):
    """n regular streams of about total / n bytes each, 8 deltas per chunk"""
    ev = max(8, (total // max(n, 1) - 400) // 64 // 8 * 8)
    return _regular(n, ev, seed, epc=8)


def _one_step(name, order, truths, wants) -> Layout:
    return Layout(name, [order], [s for s, _ in order], truths, wants=set(wants))


def tiny_then_huge(total: int, seed: int = 1, tiny_share: float = 0.35, n_huge: int = 0, flip: bool = False) -> Layout:
    """thousands of one-event streams (~370 B: a delta, the usage event, [DONE]) and then a few streams of total / n_huge bytes
    (flip: huge first).  The byte position misguesses the segment by hundreds: the search goes above (tiny first) or below
    (huge first)."""
    sl = _Slots()
    n_tiny = min(6000, max(40, int(total * tiny_share) // 370))
    n_huge = n_huge or max(3, total // (4 * MiB))                   # (at most ~4 MiB each: the sequential reference walks a segment on one thread)
    tiny, t_truth = _regular(n_tiny, 1, seed)
    big, b_truth = _huge(total - n_tiny * 370, n_huge, seed + 1)
    ts, bs = sl.take(n_tiny), sl.take(n_huge)
    truths = dict(zip(ts, t_truth)) | dict(zip(bs, b_truth))
    a, b = list(zip(ts, tiny)), list(zip(bs, big))
    return _one_step("huge_then_tiny" if flip else "tiny_then_huge", b + a if flip else a + b, truths,
                     {BELOW} if flip else {ABOVE})


def huge_then_tiny(total: int, seed: int = 2, **kw) -> Layout:
    return tiny_then_huge(total, seed, flip=True, **kw)


RUNS = (31, 32, 33, 64, 97)


def alternating_runs(total: int, seed: int = 3, cycles: int = 3) -> Layout:
    """runs of 31, 32, 33, 64 and 97 one-event streams between long streams of random lengths, so that the window's edges fall
    at every offset of a warp's range; every other run is of streams continued from an earlier step (committed), the others are
    fresh"""
    rng = random.Random(seed)
    sl = _Slots()
    n_tiny = cycles * sum(RUNS)
    n_long = cycles * len(RUNS) + 1
    long_total = max(total - n_tiny * 370, n_long * 4096)
    lengths = [rng.uniform(0.5, 1.5) for _ in range(n_long)]
    truths, order, first = {}, [], []
    for i in range(n_long):
        ch, tr = _huge(int(long_total * lengths[i] / sum(lengths)), 1, seed * 1000 + i)
        s = sl.take()[0]
        truths[s] = tr[0]
        order.append((s, ch[0]))
        if i < n_long - 1:
            run = RUNS[i % len(RUNS)]
            ch, tr = _regular(run, 2, seed * 1000 + 500 + i)
            ss = sl.take(run)
            truths.update(zip(ss, tr))
            if i % 2:                                           # committed: their first delta came in the step before
                first += [(s_, c[:1]) for s_, c in zip(ss, ch)]
                order += [(s_, c[1:]) for s_, c in zip(ss, ch)]
            else:
                order += list(zip(ss, ch))
    steps = [first, order] if first else [order]
    return Layout("alternating_runs", steps, [s for s in range(sl.n)], truths, wants={BRACKETED, "reload"})


ZERO_RUNS = (31, 32, 33, 65)


def zero_byte_runs(total: int, align: int, seed: int = 4) -> Layout:
    """runs of 31, 32, 33 and 65 segments without bytes (idle streams: no chunks, or only empty ones) at the step's start, at a
    warp's range_lo (a byte position that is a multiple of `align`: tiles per warp x R2_TILE) and inside warp ranges, between
    one-event streams and long streams"""
    rng = random.Random(seed)
    sl = _Slots()
    truths, order = {}, []
    pos = 0

    def zero_run(n, kind):
        for s in sl.take(n):
            order.append((s, [] if kind == "none" or (kind == "mixed" and s % 2) else [b""] * (1 + s % 3)))

    def tiny(n, sd):
        nonlocal pos
        ch, tr = _regular(n, 1, sd)
        ss = sl.take(n)
        truths.update(zip(ss, tr))
        order.extend(zip(ss, ch))
        pos += sum(len(c) for x in ch for c in x)

    def long(nbytes, sd):
        nonlocal pos
        ch, tr = _huge(nbytes, 1, sd)
        s = sl.take()[0]
        truths[s] = tr[0]
        order.append((s, ch[0]))
        pos += sum(map(len, ch[0]))

    def pad_to(p):                                              # deltas of exactly p - pos bytes (no usage event)
        nonlocal pos
        s = sl.take()[0]
        truths[s] = None
        order.append((s, SC.filler(p - pos, seed + s)))
        pos = p

    n_tiny = min(2000, max(20, total // 370 // 12))
    zero_run(31, "none")                                        # the step's start
    tiny(n_tiny, seed)
    zero_run(33, "empty")                                       # inside a warp's range
    tiny(n_tiny, seed + 1)
    at = (pos + 4096 + align - 1) // align * align
    pad_to(at)
    zero_run(65, "mixed")                                       # at a warp's range_lo
    tiny(n_tiny, seed + 2)
    zero_run(32, "none")
    long(max(4096, total - pos - 2 * 4096), seed + 3)
    at = (pos + 4096 + align - 1) // align * align
    pad_to(at)
    zero_run(33, "empty")                                       # at a warp's range_lo, behind a long stream
    tiny(rng.randrange(40, 80), seed + 4)
    return Layout("zero_byte_runs", [order], [s for s in range(sl.n)], truths, wants={"zero_run_at_range_lo"})


def zero_byte_runs_fitted(total: int, tiles_per_warp) -> Layout:
    """zero_byte_runs aligned to the warp ranges of its own launch: tiles_per_warp(n_bytes) of the geometry it runs on"""
    align = tiles_per_warp(total) * R2_TILE
    for _ in range(4):
        lay = zero_byte_runs(total, align)
        n_bytes = sum(len(c) for _, ch in lay.steps[0] for c in ch)
        if tiles_per_warp(n_bytes) * R2_TILE == align:
            break
        align = tiles_per_warp(n_bytes) * R2_TILE
    return lay


def continuation_step(total: int, seed: int = 5, n_small: int = 6000, n_long: int = 0, split_every: int = 5) -> Layout:
    """three steps of n_small streams and n_long long ones.  Step 1: the first deltas of every stream (fresh); step 2: ONE delta
    (64 B) per small stream, in runs between the long streams' continuations -- dozens of segments per tile -- with every
    split_every-th small stream's delta cut in two, so that its event is still open at the step's end; step 3: the rest, the usage
    events and [DONE]."""
    sl = _Slots()
    small, s_truth = _regular(n_small, 4, seed)
    ss = sl.take(n_small)
    n_long = n_long or max(4, total // (8 * MiB))                  # (about 8 MiB a step each at most: see tiny_then_huge)
    per_long = max(8192, (total - n_small * 64) // n_long)
    long, l_truth = _huge(2 * per_long * n_long, n_long, seed + 1)
    ls = sl.take(n_long)
    truths = dict(zip(ss, s_truth)) | dict(zip(ls, l_truth))
    step1 = [(s, c[:2]) for s, c in zip(ss, small)] + [(s, c[: len(c) // 2 - 1]) for s, c in zip(ls, long)]
    step2, step3 = [], []
    runs = [list(range(k, n_small, n_long)) for k in range(n_long)]   # (streams of a run are spread: slots out of order)
    for r, run in enumerate(runs):
        for i in run:
            d = small[i][2]
            if i % split_every == 0:
                step2.append((ss[i], [d[:30]]))
                step3.append((ss[i], [d[30:]] + small[i][3:]))
            else:
                step2.append((ss[i], [d]))
                step3.append((ss[i], small[i][3:]))
        c = long[r]
        step2.append((ls[r], c[len(c) // 2 - 1: -2]))
        step3.append((ls[r], c[-2:]))
    return Layout("continuation_step", [step1, step2, step3], ss + ls, truths, wants={"reload", "committed_after_reload"})


def few_segments(total: int, seed: int = 6, counts=(1, 31, 32, 33)) -> Layout:
    """one step per count: that many streams of total / count bytes (the n <= 32 path, the clamp w0 = n - 32, segments longer than
    many warp ranges)"""
    sl = _Slots()
    steps, truths = [], {}
    for k, n in enumerate(counts):
        ch, tr = _huge(total, n, seed * 10 + k)
        ss = sl.take(n)
        truths.update(zip(ss, tr))
        steps.append(list(zip(ss, ch)))
    wants = {SMALL} | ({"clamp"} if max(counts) > WINDOW else set())
    return Layout("few_segments", steps, [s for s in range(sl.n)], truths, wants=wants)


def adversarial_in_runs(total: int, adv: list, seed: int = 7, run: int = 40) -> Layout:
    """the fuzz generators' streams (`adv`: lists of chunks) placed inside runs of one-event regular streams and next to long
    regular streams"""
    rng = random.Random(seed)
    sl = _Slots()
    truths, adversarial, order = {}, {}, []
    n_groups = max(1, len(adv) // 4)
    adv_bytes = sum(len(c) for s in adv for c in s)
    long_each = max(8192, (total - adv_bytes - n_groups * run * 370) // n_groups)
    a = iter(adv)
    for g in range(n_groups):
        ch, tr = _regular(run, 1, seed * 100 + g)
        ss = sl.take(run)
        truths.update(zip(ss, tr))
        group = list(zip(ss, ch))
        for _ in range(4):
            x = next(a, None)
            if x is not None:
                s = sl.take()[0]
                adversarial[s] = x
                group.insert(rng.randrange(len(group) + 1), (s, x))
        order += group
        lc, lt = _huge(long_each, 1, seed * 100 + 50 + g)
        s = sl.take()[0]
        truths[s] = lt[0]
        order.append((s, lc[0]))
    return Layout("adversarial_in_runs", [order], [s for s in range(sl.n)], truths, adversarial,
                  wants={BRACKETED} | ({"reload"} if run >= 60 else set()))


def split_steps(lay: Layout, n_steps: int, seed: int = 11) -> Layout:
    """the same streams over n_steps steps, each regular stream cut at whole chunks (events never open across a cut), adversarial
    ones at random chunks; a step keeps the layout's segment order"""
    if n_steps == 1 or len(lay.steps) != 1:
        return lay
    rng = random.Random(seed)
    steps = [[] for _ in range(n_steps)]
    for s, ch in lay.steps[0]:
        if not ch:
            for k in range(n_steps):
                steps[k].append((s, ch))
            continue
        cuts = sorted(rng.randrange(0, len(ch) + 1) for _ in range(n_steps - 1))
        b = [0] + cuts + [len(ch)]
        for k in range(n_steps):
            if b[k + 1] > b[k]:
                steps[k].append((s, ch[b[k]:b[k + 1]]))
    return Layout(f"{lay.name}_{n_steps}steps", steps, lay.slots, lay.truths, lay.adversarial,
                  lay.wants - {"zero_run_at_range_lo"})           # (the cuts move the runs off their byte positions)


# ---- expected path counts -------------------------------------------------------------------------------------------------------

def expected_paths(lay: Layout):
    """per step: (sequential, bulk) segment counts k_commit2 must report, derived from the layout alone.  A segment with chunks
    goes sequential when one of them is empty (request_handler.py never yields an empty chunk: the concatenation argument does not
    cover it) or when an event of its stream is still open from an earlier step; every other segment of a regular stream takes the
    bulk path.  Segments without chunks are not counted.  Adversarial streams are counted apart: (sequential + bulk, None)."""
    out = []
    text = {s: b"" for s in lay.slots}
    for parts in lay.steps:
        seq = bulk = adv = 0
        for s, ch in parts:
            if ch:
                if s in lay.adversarial:
                    adv += 1
                elif any(not c for c in ch) or (text[s] and not text[s].endswith(b"\n\n")):
                    seq += 1
                else:
                    bulk += 1
            text[s] += b"".join(ch)
        out.append((seq, bulk, adv))
    return out


def reaches(cov: Coverage, want: str) -> bool:
    """the model coverage a layout is built for"""
    if want in BRANCHES:
        return cov.branches[want] > 0
    return {"clamp": cov.clamped > 0, "reload": cov.reloads > 0, "fresh_after_reload": cov.fresh_after_reload > 0,
            "committed_after_reload": cov.committed_after_reload > 0, "zero_run_at_range_lo": cov.zero_run_at_range_lo >= 33}[want]
