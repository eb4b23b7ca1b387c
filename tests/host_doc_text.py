"""Loader for the TEST-AID host build of the non-streaming tap's text walk (tests/support/host_doc_text.cpp: transcript.cuh
doc_text, what k_docs_text runs for one document), and a CPU stand-in engine that serves Engine.documents_text from it.
CPU-only helper: lets the CPU suite run the exact device code path without a GPU."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

SUP = Path(__file__).resolve().parent / "support"
SRC = SUP / "host_doc_text.cpp"
LIB = SUP / "_host_doc_text.so"
CSRC = Path(__file__).resolve().parent.parent / "llmapigateway_b200" / "csrc"


def _stale() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = [SRC, SUP / "simt_emu.h"] + list(CSRC.glob("*.cuh")) + [CSRC.parent.parent / "include" / "llmgw_b200.h"]
    return any(d.stat().st_mtime > t for d in deps)


_lib = None


def lib():
    global _lib
    if _lib is None:
        if _stale():
            tmp = LIB.with_suffix(".%d.tmp" % os.getpid())      # (built aside and moved into place: other processes may be loading the library)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", str(tmp), str(SRC)])
            os.replace(tmp, LIB)
        _lib = C.CDLL(str(LIB))
        _lib.lgwt_doc_text.restype = C.c_uint32
    return _lib


def doc_text(raw: bytes):
    """(text bytes, flags) of one document: flags are _abi.TF_* bits, TF_DOC_ERROR_LOG when write_log also ran at
    chat_logging.py:139"""
    text = np.zeros(2 * len(raw) + 1, dtype=np.uint8)
    n = C.c_uint32(0)
    buf = np.frombuffer(raw, dtype=np.uint8) if raw else np.zeros(1, np.uint8)
    flags = lib().lgwt_doc_text(buf.ctypes.data_as(C.c_void_p), C.c_uint32(len(raw)), text.ctypes.data_as(C.c_void_p), C.byref(n))
    return bytes(text[:n.value]), int(flags)


def text_fake_engine(max_streams: int = 2):
    """fake_engine.FakeEngine plus documents_text from the host build above, for a StreamBatcher that keeps transcripts (the
    stream tap itself is not used by non-streaming requests, so enabling it does nothing here)"""
    from fake_engine import FakeEngine

    class TextFakeEngine(FakeEngine):
        def enable_transcripts(self):
            pass

        def documents_text(self, docs):
            return [doc_text(bytes(d)) for d in docs]

    return TextFakeEngine(max_streams=max_streams)
