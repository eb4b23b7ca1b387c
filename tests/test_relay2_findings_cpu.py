"""The bulk kernel's findings scratch (SegPlan) is all zero between launch sets: k_relay2 only adds to it, and k_commit2 zeroes
every segment's record once it has read it -- bulk, sequential and segments without bytes alike.  Run on the CPU box through the
SIMT emulator (tests/support/host_relay2_findings.cpp): the same step twice in a row, then a step cut into slices."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import host_relay as H
import host_relay_sliced as HS
import slice_cases as SC
from llmapigateway_b200 import _abi
from llmapigateway_b200.synth import pack_streams, sse_batch

SRC = H.SUP / "host_relay2_findings.cpp"
LIB = H.SUP / "_host_relay2_findings.so"


def _lib():
    """the sliced emulator library with lgwt_bulk_findings_nonzero; the other functions declared as in host_relay_sliced.lib()"""
    base = HS.lib()
    deps = [SRC, HS.SRC, H.SRC, H.SUP / "simt_emu.h"] + list(H.CSRC.glob("*.cuh")) + list(H.CSRC.glob("*.inc"))
    if not LIB.exists() or any(d.stat().st_mtime > LIB.stat().st_mtime for d in deps):
        tmp = LIB.with_suffix(".%d.tmp" % os.getpid())
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-g", "-shared", "-fPIC", "-o", str(tmp), str(SRC)])
        os.replace(tmp, LIB)
    lb = C.CDLL(str(LIB))
    for name in dir(base):
        if name.startswith("lgwt_"):
            f, g = getattr(base, name), getattr(lb, name)
            g.argtypes, g.restype = f.argtypes, f.restype
    lb.lgwt_bulk_findings_nonzero.argtypes = [C.c_void_p]
    lb.lgwt_bulk_findings_nonzero.restype = C.c_uint64
    return lb


class FindingsEngine(HS.SlicedHostBulkEngine):
    """SlicedHostBulkEngine on the library that can look at its findings scratch"""

    def __init__(self, max_streams: int, n_blocks: int, tiles_per_warp: int, n_slices: int):
        self._lib = _lib()
        self.limits = _abi.Limits(max_streams, 4096, 4096, 4096, 1 << 22, 1 << 28)
        self._h = C.c_void_p(self._lib.lgwt_bulk_new(max_streams, 4096, 4096, 4096, n_blocks))
        self.tiles_per_warp = tiles_per_warp
        self.n_slices = n_slices


@pytest.fixture(scope="module")
def engine():
    e = FindingsEngine(max_streams=256, n_blocks=2, tiles_per_warp=1, n_slices=1)
    yield e
    e.close_engine()


def _nonzero(engine) -> int:
    return int(engine._lib.lgwt_bulk_findings_nonzero(engine._h))


def test_findings_are_zero_after_every_launch_set(engine, monkeypatch):
    engine.set_mode(0)
    engine.reset_templates()
    assert _nonzero(engine) == 0
    b = sse_batch(n_streams=48, n_events=24, seed=31)
    engine.open(b.seg_slot)
    c0 = engine.counters()
    for _ in range(2):                  # the same step twice: fresh streams (speculated), then committed ones
        engine.step(b.data, b.chunk_off, b.seg_chunk, b.seg_slot)
        assert _nonzero(engine) == 0
    c1 = engine.counters()
    assert c1["bulk"] - c0["bulk"] > 0      # the bulk kernel did report findings for these steps
    engine.close(b.seg_slot)

    # a sliced step whose slice 1 starts at a segment without bytes, behind segments without chunks
    case = SC.zero_byte_segment_at_slice_start("empty_chunks")
    monkeypatch.setenv("LGW_SLICES", str(case.n_slices))
    engine.n_slices = case.n_slices
    slots = np.asarray(case.slots, dtype=np.uint32)
    engine.open(slots)
    for parts in case.steps:
        pb = pack_streams([c for _, c in parts], slots=[s for s, _ in parts])
        engine.step(pb.data, pb.chunk_off, pb.seg_chunk, pb.seg_slot)
        assert _nonzero(engine) == 0
    engine.close(slots)
