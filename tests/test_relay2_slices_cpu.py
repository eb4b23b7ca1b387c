"""Host-buffer steps cut into slices, on the CPU box: the bulk kernels of csrc/relay2.cuh run once per slice through the SIMT
emulator (tests/support/host_relay2_sliced.cpp), cut by the engine's own rule (step_slice_cuts) and with the engine's launch arguments.
Hand-built steps (tests/slice_cases.py) put segments without bytes, fresh streams, usage and error events and oversized segments
at the slices' first bytes; each is compared with the same steps on the exact sequential path and with the oracle."""
import pytest

import slice_cases as SC
import test_sse_gpu as G
from host_relay_sliced import SlicedHostBulkEngine


@pytest.fixture(scope="module", params=[(2, 1), (3, 0)], ids=["one_tile_per_warp", "spread"])
def engine(request):
    n_blocks, tpw = request.param
    e = SlicedHostBulkEngine(max_streams=256, n_blocks=n_blocks, tiles_per_warp=tpw)
    yield e
    e.close_engine()


@pytest.mark.parametrize("case", SC.directed_cases(), ids=lambda c: c.name)
def test_directed_slice_edges(engine, case, monkeypatch):
    monkeypatch.setenv("LGW_SLICES", str(case.n_slices))
    SC.check_directed(engine, case)


def test_cut_rule_matches_the_engine():
    """slice_cuts (the tests' restatement) against hand-computed cuts: equal segments, a zero-byte segment at the cut, one
    oversized segment, fewer segments than slices"""
    import numpy as np
    off = np.array([0, 10, 20, 30, 40], dtype=np.uint32)
    assert SC.slice_cuts(off, np.array([0, 1, 2, 3, 4]), 4) == [0, 1, 2, 3, 4]
    assert SC.slice_cuts(off, np.array([0, 2, 2, 4]), 2) == [0, 1, 3]           # segment 1 has no chunks and starts at byte 20
    assert SC.slice_cuts(off, np.array([0, 3, 4]), 2) == [0, 1, 2]
    assert SC.slice_cuts(off, np.array([0, 1, 4]), 2) == [0, 2, 2]
    assert SC.slice_cuts(off, np.array([0, 2, 4]), 3) == [0, 2]


@pytest.mark.parametrize("n_slices", [3, 8, 14])
def test_random_streams_sliced(engine, n_slices, monkeypatch):
    """the fuzz campaign's check on the generators of test_sse_gpu.py, every bulk step cut into n_slices"""
    from oracle.sse_oracle import run_stream
    monkeypatch.setenv("LGW_SLICES", str(n_slices))
    streams = G._random_streams(120, seed=900 + n_slices) + G._template_variant_streams(60, seed=950 + n_slices)
    fast = G._run_all(engine, streams, 0, 2, seed=n_slices)
    seq = G._run_all(engine, streams, 1, 2, seed=n_slices)
    assert fast[1] == seq[1] and fast[2] == seq[2]
    for i, (a, b) in enumerate(zip(fast[0], seq[0])):
        assert bytes(a)[:64] == bytes(b)[:64], i
        relay, _ = run_stream(streams[i])
        assert fast[2][i] == relay.emitted, i
