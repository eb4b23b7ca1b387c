"""Loader for the TEST-AID host build of the usage-table writer (tests/support/host_save.cpp over csrc/save.cuh), a CPU stand-in
UsageTable that saves through it, and the same source built as a program under -fsanitize=address.
CPU-only helper: lets the CPU suite run the device writer's own code without a GPU."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

from llmapigateway_b200 import usage as U
from test_usage_append_cpu import AppendStandIn

SUP = Path(__file__).resolve().parent / "support"
SRC = SUP / "host_save.cpp"
LIB = SUP / "_host_save.so"
ASAN = SUP / "_host_save_asan"
CSRC = Path(__file__).resolve().parent.parent / "llmapigateway_b200" / "csrc"


def _build(out: Path, flags: list[str]):
    deps = [SRC] + [CSRC / f for f in ("save.cuh", "load.cuh", "rollup.cuh")]
    if out.exists() and all(d.stat().st_mtime <= out.stat().st_mtime for d in deps):
        return
    tmp = out.with_suffix(".%d.tmp" % os.getpid())     # (built aside and moved into place: other processes may be using it)
    subprocess.check_call(["g++", "-std=c++17", *flags, "-o", str(tmp), str(SRC)])
    os.replace(tmp, out)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _build(LIB, ["-O2", "-shared", "-fPIC"])
        _lib = C.CDLL(str(LIB))
        _lib.lgwt_save_plan.argtypes = [C.POINTER(C.c_void_p), C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        _lib.lgwt_save_write.argtypes = [C.c_void_p, C.c_void_p]
        _lib.lgwt_save_release.argtypes = []
    return _lib


class HostSaveTable(AppendStandIn):
    """the append test's numpy stand-in for the device columns, saving through the host build (the calls in the kernels'
    order) into numpy buffers.  `fail_at`: a step whose call raises instead (failure injection through the seam)."""
    fail_at = None

    def _save_call(self, step, *args):
        if step == self.fail_at:
            raise RuntimeError(f"injected failure at {step}")
        rc = getattr(lib(), "lgwt_save_" + step)(*args)
        assert rc == 0, (step, rc)

    def _save_cols(self):
        return (C.c_void_p * 8)(*[self._dev_ptrs[c].ctypes.data for c in self.COLS])

    def _save_alloc(self, nbytes):
        return np.zeros(nbytes, np.uint8)

    def _save_free(self, buf):
        pass


def asan_run(t: U.UsageTable, page_size: int, tmp: Path) -> tuple[list[int], bytes]:
    """the writer over t's columns (every array in a buffer of exactly its size) under AddressSanitizer: ([pages, table root,
    index root, kept, refused], pages 3 .. of the file); AssertionError with the sanitizer's report on any bad access"""
    _build(ASAN, ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-DLGWT_MAIN"])
    t._upload()
    n = int(t._host["ts_us"].size)
    codes: dict = {None: 0}
    prov = np.array([codes.setdefault(p, len(codes)) for p in t._providers], np.int32)
    parts = [np.uint64(n).tobytes()] + [t._dev_ptrs[c][:n].tobytes() for c in t.COLS]
    parts += [t._ids[:n].astype(np.int64).tobytes(), prov.tobytes()]
    for texts in (t._names, list(codes)):
        _, (blob, off, lens) = U._save_text_table(texts)
        parts += [np.uint64(len(texts)).tobytes(), off.tobytes(), lens.tobytes(), blob[:int(off[-1])].tobytes()]
    cols, out = tmp / "cols.bin", tmp / "pages.bin"
    cols.write_bytes(b"".join(parts))
    r = subprocess.run([str(ASAN), str(cols), str(page_size), str(out)], capture_output=True, text=True,
                       env={**os.environ, "ASAN_OPTIONS": "detect_leaks=1"})
    assert r.returncode == 0, r.stderr[-3000:]
    return [int(x) for x in r.stdout.split()], out.read_bytes()
