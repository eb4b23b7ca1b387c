"""The hand-built transcript cases of tests/test_transcript_geometry_gpu.py on the CPU box: the transcript kernels compiled with g++
over the SIMT emulator, after steps cut into 1 or 8 slices (tests/host_relay_sliced.py).  Segment counts at k_text_scan's block
edges (up to 2 049; the 8 192-segment step runs on the GPU only), adjacent segments that fill the sparse buffer's twofold room,
unterminated tails of carry_cap and carry_cap + 1 bytes, one 200 KiB event, and a mark queue that overflows."""
import pytest

import test_transcript_geometry_gpu as G
from host_relay_sliced import SlicedHostBulkEngine

CARRY_CAP = 4096


def _engine(rowq_cap=4096):
    e = SlicedHostBulkEngine(max_streams=2304, carry_cap=CARRY_CAP, rowq_cap=rowq_cap, n_blocks=2)
    e.enable_transcripts()
    return e


@pytest.fixture(scope="module", params=[1, 8], ids=["slices1", "slices8"])
def engine(request):
    e = _engine()
    e.n_slices = request.param
    yield e
    e.close_engine()


@pytest.mark.parametrize("n_segs", [n for n in G.SEG_COUNTS if n <= 2049])
def test_segment_counts_at_scan_block_edges(engine, n_segs):
    G.many_segments(engine, n_segs)


@pytest.mark.parametrize("case", list(G.HAND_BUILT))
def test_hand_built(engine, case):
    G.HAND_BUILT[case](engine, G.host_tap)


@pytest.mark.parametrize("n_slices", [1, 8])
def test_mark_queue_overflow(n_slices):
    e = _engine(rowq_cap=64)
    e.n_slices = n_slices
    try:
        G.mark_queue_overflow(e)
    finally:
        e.close_engine()
