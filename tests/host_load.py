"""Loader for the TEST-AID host build of the usage-table loader (tests/support/host_load.cpp over csrc/load.cuh), a CPU stand-in
UsageTable that loads through it, and the same source built as a program under -fsanitize=address for damaged files.
CPU-only helper: lets the CPU suite run the device decoder's own code without a GPU."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

from llmapigateway_b200.usage import UsageTable

SUP = Path(__file__).resolve().parent / "support"
SRC = SUP / "host_load.cpp"
LIB = SUP / "_host_load.so"
ASAN = SUP / "_host_load_asan"
CSRC = Path(__file__).resolve().parent.parent / "llmapigateway_b200" / "csrc"


def _build(out: Path, flags: list[str]):
    deps = [SRC, CSRC / "load.cuh"]
    if out.exists() and all(d.stat().st_mtime <= out.stat().st_mtime for d in deps):
        return
    tmp = out.with_suffix(".%d.tmp" % os.getpid())     # (built aside and moved into place: other processes may be using it)
    subprocess.check_call(["g++", "-std=c++17", *flags, "-o", str(tmp), str(SRC)])
    os.replace(tmp, out)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _build(LIB, ["-O1", "-shared", "-fPIC"])
        _lib = C.CDLL(str(LIB))
        _lib.lgwt_load_decode.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        _lib.lgwt_load_names.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib.lgwt_load_mark.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        _lib.lgwt_load_release.argtypes = []
        _lib.lgwt_load_finish.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def asan_run(path, page_size: int, n_pages: int, root: int) -> list[int]:
    """the decoder over the file's bytes (a buffer of exactly its size) under AddressSanitizer: [error, records, kept, models,
    providers]; AssertionError with the sanitizer's report on any bad access"""
    _build(ASAN, ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-DLGWT_MAIN"])
    r = subprocess.run([str(ASAN), str(path), str(page_size), str(n_pages), str(root)], capture_output=True, text=True,
                       env={**os.environ, "ASAN_OPTIONS": "detect_leaks=0"})
    assert r.returncode == 0, r.stderr[-3000:]
    return [int(x) for x in r.stdout.split()]


class HostLoadTable(UsageTable):
    """UsageTable whose load runs the host build (the four calls in the kernels' order), with numpy buffers for the file and
    numpy copies of the host columns standing for the device columns.  Without an engine otherwise: only the load and the
    host paths work (see test_usage_append_cpu.py for a stand-in of the other device calls)."""

    def __init__(self):
        super().__init__(engine=object())
        self.loads = 0

    def _load_call(self, step, *args):
        if step == "finish":
            self._finish_args = args
        rc = getattr(lib(), "lgwt_load_" + step)(*args)
        assert rc == 0, (step, rc)

    def _load_alloc(self, nbytes):
        return np.zeros(nbytes, np.uint8)

    def _load_free(self, buf):
        pass

    def _load_cols_alloc(self, n):
        self.loads += 1
        return None

    def load_tokens_usage_db(self, db_path):
        n = super().load_tokens_usage_db(db_path)
        self._dev_ptrs = {c: self._host[c].copy() for c in self.COLS}
        self._dev = (n, self._dev_ptrs)
        return n

    def _free_ptrs(self, ptrs):
        pass
