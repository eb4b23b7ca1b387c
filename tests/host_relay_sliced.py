"""TEST AID: `HostBulkEngine` (tests/host_relay.py) whose steps are cut into slices the way lgw_sse_step cuts a host-buffer step
(tests/support/host_relay2_sliced.cpp).  Not a product path."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import host_relay as H
from llmapigateway_b200 import _abi
from llmapigateway_b200.engine import SEG_DTYPE, StepResult

SRC = H.SUP / "host_relay2_sliced.cpp"
LIB = H.SUP / "_host_relay2_sliced.so"

_lib = None


def _stale() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = [SRC, H.SRC, H.SUP / "simt_emu.h"] + list(H.CSRC.glob("*.cuh")) + list(H.CSRC.glob("*.inc")) + [H.CSRC.parent.parent / "include" / "llmgw_b200.h"]
    return any(d.stat().st_mtime > t for d in deps)


def lib():
    """the emulator library with lgwt_bulk_step_sliced; every other function is declared as in host_relay.lib()"""
    global _lib
    if _lib is None:
        base = H.lib()
        if _stale():
            tmp = LIB.with_suffix(".%d.tmp" % os.getpid())
            subprocess.check_call(["g++", "-std=c++17", "-O2", "-g", "-shared", "-fPIC", "-o", str(tmp), str(SRC)])
            os.replace(tmp, LIB)
        lb = C.CDLL(str(LIB))
        for name in dir(base):
            if name.startswith("lgwt_"):
                f, g = getattr(base, name), getattr(lb, name)
                g.argtypes, g.restype = f.argtypes, f.restype
        lb.lgwt_bulk_step_sliced.argtypes = list(base.lgwt_bulk_step.argtypes) + [C.c_uint32]
        _lib = lb
    return _lib


class SlicedHostBulkEngine(H.HostBulkEngine):
    """n_slices: every step is cut into that many slices; None: LGW_SLICES, read on every step as the engine reads it (else 1)"""

    def __init__(self, max_streams: int = 2048, carry_cap: int = 4096, detail_cap: int = 4096, rowq_cap: int = 4096,
                 n_blocks: int = 2, tiles_per_warp: int = 0, n_slices: int | None = None):
        self._lib = lib()
        self.limits = _abi.Limits(max_streams, carry_cap, detail_cap, rowq_cap, 1 << 22, 1 << 28)
        self._h = C.c_void_p(self._lib.lgwt_bulk_new(max_streams, carry_cap, detail_cap, rowq_cap, n_blocks))
        self.tiles_per_warp = tiles_per_warp
        self.n_slices = n_slices

    def step(self, data, chunk_off, seg_chunk, seg_slot, out=None, relay_from_host=False) -> StepResult:
        data = np.ascontiguousarray(data, dtype=np.uint8)
        chunk_off = np.ascontiguousarray(chunk_off, dtype=np.uint32)
        seg_chunk = np.ascontiguousarray(seg_chunk, dtype=np.uint32)
        seg_slot = np.ascontiguousarray(seg_slot, dtype=np.uint32)
        n_bytes, n_chunks, n_segs = data.size, chunk_off.size - 1, seg_slot.size
        out = np.zeros(max(n_bytes, 1), dtype=np.uint8) if out is None else out
        segs = np.zeros(max(n_segs, 1), dtype=SEG_DTYPE)
        cap = self.limits.rowq_cap
        rows = (_abi.RowEvent * max(cap, 1))()
        n_rows = C.c_uint32(0)
        n_slices = self.n_slices or int(os.environ.get("LGW_SLICES", "1") or 1)
        p = H._ptr
        self._lib.lgwt_bulk_step_sliced(self._h, p(data), n_bytes, p(chunk_off), n_chunks, p(seg_chunk), p(seg_slot), n_segs,
                                        p(out), p(segs), rows, cap, C.byref(n_rows), self.tiles_per_warp, n_slices)
        self._last = (data, chunk_off, seg_chunk, seg_slot, segs)
        return StepResult((data if relay_from_host else out)[:n_bytes], segs[:n_segs], [rows[i] for i in range(n_rows.value)])
