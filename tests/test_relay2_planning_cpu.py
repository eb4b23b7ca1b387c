"""k_relay2's own segment planning on the CPU box, through the SIMT emulator: skewed stream lengths, dense runs of tiny segments,
runs of segments without bytes, continuation steps and a handful of long segments (tests/planning_cases.py), at 1, 4 and 16 tiles
per warp, unsliced and cut into slices.  A planning mistake does not corrupt bytes -- the kernel notices and hands the segment
to the exact sequential path -- so besides bulk == sequential, the truths and the oracle, every case checks the path counters
exactly against what its layout implies, that the model reaches the planning paths the case is built for, and that the findings
scratch is zero after every step."""
import functools

import pytest

import planning_cases as P
import slice_cases as SC
from llmapigateway_b200 import _abi
from llmapigateway_b200.synth import pack_streams
from sse_generators import GENERATORS, make_streams
from test_relay2_findings_cpu import FindingsEngine, _nonzero

# name: (blocks, tiles per warp, step size): each size fills the geometry's warps without raising its tiles per warp
GEOMETRIES = {"tpw1": (1, 1, 44_000), "tpw4": (1, 4, 180_000), "tpw16": (2, 16, 360_000)}


@functools.lru_cache(maxsize=None)
def adversarial():
    return tuple(tuple(s) for k, g in enumerate(GENERATORS) for s in make_streams(g, 3, 700 + k))


@functools.lru_cache(maxsize=None)
def oracle(i: int):
    from oracle.sse_oracle import run_stream
    return run_stream(list(adversarial()[i]))


@functools.lru_cache(maxsize=None)
def layout(name: str, geo: str, n_steps: int = 1) -> P.Layout:
    n_blocks, tpw, total = GEOMETRIES[geo]
    if name == "zero_byte_runs":
        lay = P.zero_byte_runs_fitted(total, lambda n: P.launch(0, n, n_blocks=n_blocks, tiles_per_warp=tpw)[2])
    elif name == "continuation_step":
        lay = P.continuation_step(total, n_small=max(60, total // 300), n_long=3)
    elif name == "alternating_runs":
        lay = P.alternating_runs(total, cycles=1)
    elif name == "few_segments":
        lay = P.few_segments(total)
    elif name == "adversarial_in_runs":
        lay = P.adversarial_in_runs(total, [list(s) for s in adversarial()], run=60 if tpw > 1 else 8)
    else:
        lay = getattr(P, name)(total, tiny_share=0.5)
    return P.split_steps(lay, n_steps)


LAYOUTS = ["tiny_then_huge", "huge_then_tiny", "alternating_runs", "zero_byte_runs", "continuation_step", "few_segments",
           "adversarial_in_runs"]
CASES = [(name, geo, n_slices, 1) for name in LAYOUTS for geo in GEOMETRIES for n_slices in (1, 3)] + [
    (name, "tpw4", 1, 3) for name in ("tiny_then_huge", "zero_byte_runs", "adversarial_in_runs")]


@pytest.fixture(scope="module")
def engines():
    made = {}

    def get(geo):
        if geo not in made:
            n_blocks, tpw, _ = GEOMETRIES[geo]
            made[geo] = FindingsEngine(max_streams=8192, n_blocks=n_blocks, tiles_per_warp=tpw, n_slices=1)
        return made[geo]
    yield get
    for e in made.values():
        e.close_engine()


def model_coverage(lay: P.Layout, n_slices: int, **geo) -> P.Coverage:
    cov = P.Coverage()
    for k, parts in enumerate(lay.steps):
        pb = pack_streams([c for _, c in parts], slots=[s for s, _ in parts])
        cov.add(P.coverage(pb.chunk_off, pb.seg_chunk, lay.fresh(k), P.model_step(pb.chunk_off, pb.seg_chunk, n_slices, **geo)))
    return cov


def check_layout(eng, lay: P.Layout, step_fn, where: str, counters, oracle_of):
    """mode 0 through step_fn against mode 1, the exact path counts, the regular streams' truths and the adversarial ones'
    oracle; returns the counter deltas"""
    c0 = counters()
    fast = SC.run(eng, lay.steps, lay.slots, 0, step_fn)
    c1 = counters()
    seq = SC.run(eng, lay.steps, lay.slots, 1)
    SC.compare_bulk_sequential(fast, seq, where)
    d_seq, d_bulk = c1["sequential"] - c0["sequential"], c1["bulk"] - c0["bulk"]
    exp = P.expected_paths(lay)
    e_seq, e_bulk, n_adv = (sum(x[i] for x in exp) for i in range(3))
    if not lay.adversarial:
        assert (d_seq, d_bulk) == (e_seq, e_bulk), (where, "path counts", (d_seq, d_bulk), exp)
    else:
        assert d_bulk >= e_bulk and d_seq >= e_seq, (where, "path counts", (d_seq, d_bulk), exp)
        if len(lay.steps) == 1:                         # every adversarial stream is fresh: each segment with chunks is counted
            assert d_seq + d_bulk == e_seq + e_bulk + n_adv, (where, (d_seq, d_bulk), exp)
    slot_at = {s: i for i, s in enumerate(lay.slots)}
    for s, truth in lay.truths.items():
        st = fast.states[slot_at[s]]
        assert b"".join(fast.emitted[s]) == b"".join(lay.chunks_of(s)), (where, s, "relayed bytes")
        assert st.phase == _abi.PHASE_COMMITTED, (where, s, st.phase)
        if truth is not None:
            assert st.flags & _abi.SF_A_USAGE_BOUND and _abi.usage_rec_to_dict(st.rec) == truth.expected_row(), (where, s)
    if lay.adversarial:
        adv_slots = sorted(lay.adversarial)
        run = SC.Run([fast.states[slot_at[s]] for s in adv_slots], fast.rows, fast.emitted, fast.segs)
        n = SC.compare_oracle(run, adv_slots, None, lambda i: oracle_of(lay.adversarial[adv_slots[i]]), where)
        assert n > 0.8 * len(adv_slots), where
    return d_seq, d_bulk


_ADV_INDEX = None


def _oracle_of(chunks):
    global _ADV_INDEX
    if _ADV_INDEX is None:
        _ADV_INDEX = {tuple(s): i for i, s in enumerate(adversarial())}
    return oracle(_ADV_INDEX[tuple(chunks)])


@pytest.mark.parametrize("name,geo,n_slices,n_steps", CASES, ids=[f"{n}-{g}-slices{s}-{k}step" for n, g, s, k in CASES])
def test_planning_on_the_emulator(engines, name, geo, n_slices, n_steps, capsys):
    eng = engines(geo)
    eng.n_slices = n_slices
    n_blocks, tpw, _ = GEOMETRIES[geo]
    lay = layout(name, geo, n_steps)
    cov = model_coverage(lay, n_slices, n_blocks=n_blocks, tiles_per_warp=tpw)
    where = f"{lay.name} {geo} slices={n_slices}"
    with capsys.disabled():
        print(f"\n  {where}: {cov.line()}")
    if n_slices == 1:
        for want in sorted(lay.wants):
            assert P.reaches(cov, want), (where, want, cov.line())

    def step_fn(e, pb):
        r = SC.host_step(e, pb)
        assert _nonzero(e) == 0, (where, "findings left behind")
        return r
    check_layout(eng, lay, step_fn, where, eng.counters, _oracle_of)


# ---- the model itself, on hand-made launches --------------------------------------------------------------------------------------

def _ends(sizes, base=0):
    out, p = [], base
    for n in sizes:
        p += n
        out.append(p)
    return out


def test_first_segment_branches():
    """each of first_segment's ways to its answer on segment ends worked out by hand"""
    # 10 segments of 100 B: n <= 32, one window
    e = _ends([100] * 10)
    assert P.first_segment(e, 0, 1000, 0) == (0, 0, 0, P.SMALL, False)
    assert P.first_segment(e, 0, 1000, 350) == (3, 0, 0, P.SMALL, False)
    # 100 segments of 100 B: g = 100 * x / 10000; x = 5000 -> g = 50, w0 = 34, answer 50 = w0 + 16: bracketed
    e = _ends([100] * 100)
    assert P.first_segment(e, 0, 10000, 5000) == (50, 34, 34, P.BRACKETED, False)
    # x = 0: w0 = 0, k = 0
    assert P.first_segment(e, 0, 10000, 0) == (0, 0, 0, P.FIRST, False)
    # x = 9990: g = 99, w0 = min(83, 68) = 68 (clamped), answer 99
    assert P.first_segment(e, 0, 10000, 9990) == (99, 68, 68, P.BRACKETED, True)
    # 40 one-byte segments, then one of 9960 B, then 59 of 0 B (100 segments, 10000 B): x = 3000 -> g = 30, w0 = 14
    # candidates 14..45: segments 14..39 end at 15..40 <= 3000, segment 40 ends at 10000 > 3000 -> k = 26
    e = _ends([1] * 40 + [9960] + [0] * 59)
    assert P.first_segment(e, 0, 10000, 3000) == (40, 14, 14, P.BRACKETED, False)
    # x = 9000: g = 90, w0 = 68 (clamped); segments 68.. end at 10000 > 9000 -> k = 0, w0 > 0: search below finds 40
    assert P.first_segment(e, 0, 10000, 9000) == (40, 40, 68, P.BELOW, True)
    # one long segment first: 1 of 9000 B, then 99 of ~10 B; x = 2000 -> g = 20, w0 = 4: k = 0, search below finds 0
    e = _ends([9000] + [10] * 99 + [10])[:100]
    assert P.first_segment(e, 0, e[-1], 2000) == (0, 0, 4, P.BELOW, False)
    # search below whose answer is w0: segments of 100 B but segment 20 holds [2000, 6000); x = 3600 -> g = 100*3600/13600 = 26,
    # w0 = 10 ... make the guess land exactly: x such that g - 16 == 20
    e = _ends([100] * 20 + [4000] + [100] * 79)
    n_bytes = e[-1]                                             # 13900
    x = next(x for x in range(2000, 6000) if 100 * x // n_bytes - 16 == 20)
    assert P.first_segment(e, 0, n_bytes, x) == (20, 20, 20, P.BELOW_W0, False)
    # search above: 90 tiny segments then 10 long ones; x in the long part guesses far too low
    e = _ends([10] * 90 + [1000] * 10)
    assert P.first_segment(e, 0, e[-1], 5000) == (94, 94, 29, P.ABOVE, False)


def test_model_of_a_slice_with_an_unaligned_start():
    """a slice whose first byte is not 16-aligned: its first warp's range starts at tile_base, tiles are counted from
    tile_base & ~15, segment indices from the slice's first segment"""
    import numpy as np
    sizes = [20003] + [150] * 140                               # 41 003 bytes; cut 1 = the first segment starting at >= 20 501
    off = np.array([0] + _ends(sizes), dtype=np.uint32)
    seg_chunk = np.arange(len(sizes) + 1, dtype=np.uint32)
    assert SC.slice_cuts(off, seg_chunk, 2) == [0, 5, 141]        # segment 5 starts at 20 003 + 4 * 150 = 20 603 (11 mod 16)
    assert P.launch(20603, 41003, n_blocks=1, tiles_per_warp=1) == (20592, 7, 1, 7)
    s1 = [p for p in P.model_step(off, seg_chunk, 2, n_blocks=1, tiles_per_warp=1) if p.slice == 1]
    assert [(p.range_lo, p.range_hi) for p in s1][:2] == [(20603, 23664), (23664, 26736)]
    assert s1[-1].range_hi == 41003
    # warp 0 starts at the slice's first byte: guess 0, the first candidate holds it
    assert (s1[0].w0, s1[0].seg0, s1[0].branch) == (5, 5, P.FIRST)
    # warp 1: g = 136 * (23664 - 20603) // 20400 = 20, w0 = 4 (+ 5); slice segment j ends at 20753 + 150 j, the first past 23664
    # is j = 20 (k = 16); it walks j = 20..40 (starts below 26736) and reloads its window (from j = 4) at j = 36
    assert (s1[1].w0, s1[1].seg0, s1[1].branch, s1[1].visited, s1[1].reloads) == (9, 25, P.BRACKETED, 21, [41])


def test_window_reloads():
    """a warp whose range holds 100 segments reloads its window at the 32nd, 64th and 96th segment after its first"""
    starts = list(range(0, 1000, 10))
    ends = [s + 10 for s in starts]
    assert P.walk(starts, ends, 0, 0, 0, 1000) == (100, [32, 64, 96])
    assert P.walk(starts, ends, 5, 0, 55, 1000) == (95, [32, 64, 96])      # the window was loaded from segment 0 (the bracketing round)
    assert P.walk(starts, ends, 5, 5, 55, 400) == (35, [37])
    # segments without bytes count like any other
    starts, ends = [0] * 40 + [0], [0] * 40 + [500]
    assert P.walk(starts, ends, 0, 0, 0, 500) == (41, [32])


def test_expected_paths():
    lay = P.Layout("x", [[(0, [b"a\n\n"]), (1, []), (2, [b"", b""]), (3, [b"b\n\n", b""]), (4, [b"c"])],
                         [(4, [b"\n\n"]), (0, [b"d\n\n"]), (2, [b"e\n\n"])]], [0, 1, 2, 3, 4], {})
    assert P.expected_paths(lay) == [(2, 2, 0), (1, 2, 0)]
