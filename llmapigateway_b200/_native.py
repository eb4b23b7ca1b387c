"""Loads the C-ABI shared library (include/llmgw_b200.h).  There is deliberately no fallback:
if the CUDA library is missing or no device is usable, importing/creating raises."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

from . import _abi

LIB_PATH = Path(__file__).resolve().parent / "_native" / "libllmgw_b200.so"
if os.environ.get("LGW_NATIVE_LIB"):          # kernel-geometry experiments (tools/run_geometry_variants.sh): another build of the same library
    LIB_PATH = Path(os.environ["LGW_NATIVE_LIB"]).resolve()

EXPORTS = [
    "lgw_abi_version", "lgw_engine_create", "lgw_engine_destroy", "lgw_last_error", "lgw_engine_set_stream",
    "lgw_streams_open", "lgw_streams_state", "lgw_stream_detail", "lgw_streams_close",
    "lgw_sse_step", "lgw_sse_step_device", "lgw_fetch_rows", "lgw_sync", "lgw_last_step_ms", "lgw_last_step_kernel_ms", "lgw_engine_set_kernel_timing",
    "lgw_launch_count", "lgw_documents_error_detail", "lgw_last_step_direct", "lgw_rollup_set_path", "lgw_streams_details", "lgw_alloc_pinned", "lgw_free_pinned",
    "lgw_usage_rollup_accum", "lgw_usage_rollup_emit", "lgw_rollup_bucket_of", "lgw_rollup_buckets_of", "lgw_rollup_last_ms",
    "lgw_usage_latest", "lgw_usage_latest_last_ms", "lgw_usage_retain", "lgw_usage_retain_last_ms",
    "lgw_usage_append", "lgw_usage_append_last_ms", "lgw_usage_load_decode", "lgw_usage_load_names", "lgw_usage_load_mark",
    "lgw_usage_load_finish", "lgw_usage_load_release", "lgw_usage_load_last_ms",
    "lgw_usage_save_plan", "lgw_usage_save_write", "lgw_usage_save_release", "lgw_usage_save_last_ms", "lgw_device_alloc", "lgw_device_free", "lgw_device_upload", "lgw_device_download", "lgw_device_zero",
    "lgw_transcripts_enable", "lgw_step_transcript_run", "lgw_step_transcript_fetch", "lgw_transcript_last_ms",
    "lgw_documents_usage", "lgw_rules_load", "lgw_bodies_scan", "lgw_bodies_rewrite", "lgw_bodies_rewrite_device", "lgw_bodies_last_ms",
    "lgw_documents_text", "lgw_documents_text_last_ms",
]

_lib = None


class NativeLibraryMissing(RuntimeError):
    pass


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise NativeLibraryMissing(
            f"{LIB_PATH} not built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). This package has no CPU implementation.")
    lib = C.CDLL(str(LIB_PATH))
    missing = [n for n in EXPORTS if not hasattr(lib, n)]
    if missing:
        raise NativeLibraryMissing(f"{LIB_PATH} lacks symbols {missing}")
    lib.lgw_last_error.restype = C.c_char_p
    lib.lgw_last_error.argtypes = [C.c_void_p]
    lib.lgw_engine_create.argtypes = [C.c_int, C.POINTER(_abi.Limits), C.POINTER(C.c_void_p)]
    lib.lgw_engine_destroy.argtypes = [C.c_void_p]
    lib.lgw_engine_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    lib.lgw_streams_open.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.lgw_streams_state.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    lib.lgw_streams_close.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    lib.lgw_stream_detail.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    step_args = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.lgw_sse_step.argtypes = step_args + [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    lib.lgw_sse_step_device.argtypes = step_args
    lib.lgw_fetch_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    lib.lgw_sync.argtypes = [C.c_void_p]
    lib.lgw_last_step_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
    lib.lgw_last_step_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
    lib.lgw_engine_set_kernel_timing.argtypes = [C.c_void_p, C.c_int]
    lib.lgw_launch_count.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.lgw_streams_details.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    lib.lgw_rollup_set_path.argtypes = [C.c_void_p, C.c_int]
    lib.lgw_last_step_direct.argtypes = [C.c_void_p]
    lib.lgw_documents_error_detail.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.lgw_alloc_pinned.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
    lib.lgw_free_pinned.argtypes = [C.c_void_p, C.c_void_p]
    lib.lgw_usage_rollup_accum.argtypes = [C.c_void_p] + [C.c_void_p] * 8 + [C.c_uint64, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int64,
                                           C.c_int64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lgw_usage_rollup_emit.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.lgw_rollup_bucket_of.argtypes = [C.c_int64, C.c_int]
    lib.lgw_rollup_bucket_of.restype = C.c_int64
    lib.lgw_rollup_buckets_of.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    lib.lgw_rollup_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 2)]
    lib.lgw_usage_latest.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p]
    lib.lgw_usage_latest_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    lib.lgw_usage_retain.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_uint64, C.c_int64, C.c_uint64]
    lib.lgw_usage_retain_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    lib.lgw_usage_append.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_uint64, C.POINTER(C.c_void_p), C.c_uint64,
                                     C.c_void_p, C.c_uint32]
    lib.lgw_usage_append_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    lib.lgw_usage_load_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.lgw_usage_load_names.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.lgw_usage_load_mark.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.lgw_usage_load_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                          C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lgw_usage_load_release.argtypes = [C.c_void_p]
    lib.lgw_usage_load_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
    lib.lgw_usage_save_plan.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_uint32, C.c_void_p]
    lib.lgw_usage_save_write.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lgw_usage_save_release.argtypes = [C.c_void_p]
    lib.lgw_usage_save_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 6)]
    lib.lgw_device_alloc.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
    lib.lgw_device_free.argtypes = [C.c_void_p, C.c_void_p]
    lib.lgw_device_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    lib.lgw_device_download.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    lib.lgw_device_zero.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.lgw_rules_load.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    lib.lgw_bodies_scan.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.lgw_bodies_rewrite.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                       C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.lgw_bodies_rewrite_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint32,
                                              C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.lgw_bodies_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 3)]
    lib.lgw_documents_usage.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    lib.lgw_transcripts_enable.argtypes = [C.c_void_p]
    lib.lgw_step_transcript_run.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    lib.lgw_step_transcript_fetch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.lgw_transcript_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    lib.lgw_documents_text.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.lgw_documents_text_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    if hasattr(lib, "lgw_engine_set_mode"):
        lib.lgw_engine_set_mode.argtypes = [C.c_void_p, C.c_int]
    if lib.lgw_abi_version() != 1:
        raise NativeLibraryMissing("ABI version mismatch")
    _lib = lib
    return lib
