"""Times UsageTable.load_tokens_usage_db on a 10 M-record `tokens_usage` file written from synth_usage_columns (SURVEY 8(d)
C5), phase by phase, against the row path (sqlite3 rows into load_columns, then the first upload) on the same box, and prints
one JSON line with the GPU's name and power limit read in the same run.  HBM bytes per record are computed from the file and
column sizes.  Writes only into a temporary directory.

    python tools/bench_load.py [--records 10000000] [--repeat 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sqlite3
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import llmapigateway_b200 as LG  # noqa: E402
import load_cases as L  # noqa: E402
from llmapigateway_b200 import usage as U  # noqa: E402


def note(msg: str):
    print(msg, file=sys.stderr, flush=True)


def gpu_info() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, limit = (out.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if out.returncode == 0 else ("?", "?")
    return {"gpu": name, "power_limit": limit}


def write_file(path: str, n: int):
    ts, models, tok, cost = U.synth_usage_columns(n)
    conn = L.create(path, 4096)
    stamps = np.datetime_as_string(ts.astype("datetime64[us]"), unit="us")
    text = np.where(ts % 10**6 == 0, stamps.astype("U19"), stamps).tolist()
    conn.executemany(L.INSERT, zip(text, *[a.tolist() for a in tok], cost.tolist(), models.tolist(), ["provider-%d" % (k % 7) for k in range(n)]))
    conn.commit()
    conn.close()


def row_path(eng, path: str) -> float:
    t0 = time.perf_counter()
    conn = sqlite3.connect(path)
    rows = conn.execute("SELECT timestamp, prompt_tokens, completion_tokens, total_tokens, reasoning_tokens, cached_tokens, cost,"
                        " model FROM tokens_usage ORDER BY id").fetchall()
    conn.close()
    cols = list(zip(*rows))
    ts = (np.array(cols[0], dtype="datetime64[us]").astype(np.int64))
    t = U.UsageTable(eng)
    t.load_columns(ts, cols[7], *[np.array(c, np.int32) for c in cols[1:6]], np.array([np.nan if c is None else c for c in cols[6]], np.float64))
    t._upload()
    dt = time.perf_counter() - t0
    t.close()
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=10_000_000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--no-row-path", action="store_true")
    a = ap.parse_args()
    info = gpu_info()
    eng = LG.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tokens_usage.db")
        note(f"writing {a.records} records")
        write_file(path, a.records)
        note("loading")
        size = os.path.getsize(path)
        t = U.UsageTable(eng)
        walls, phases, reads, lists = [], [], [], []
        for _ in range(a.repeat + 1):                       # the first load also pays the process's first CUDA allocations
            t0 = time.perf_counter()
            n = t.load_tokens_usage_db(path)
            walls.append(time.perf_counter() - t0)
            phases.append(t.load_last_ms())
            # the two host phases of a load, timed on their own right after it: the snapshot (pinned allocation and the
            # read of the file) and the per-record model and provider lists
            t0 = time.perf_counter()
            snap = U.read_tokens_usage_snapshot(path, t._load_alloc, t._load_free)
            reads.append(time.perf_counter() - t0)
            t._load_free(snap["buf"])
            t0 = time.perf_counter()
            U._object_array(t._names).take(t._host["model_rank"]).tolist()
            U._object_array([None, "provider"]).take(np.ones(n, np.int32)).tolist()      # (the provider list: the same take)
            lists.append(time.perf_counter() - t0)
            note(f"load {len(walls)}: {walls[-1]:.3f} s")
        t.close()
        note("row path")
        rows_s = None if a.no_row_path else row_path(eng, path)
    warm = walls[1:] or walls
    med = int(np.argsort(warm)[len(warm) // 2]) + (1 if len(walls) > 1 else 0)
    hbm = size + 88 * n * 2 + 40 * n * 2 + 12 * n             # file read once; per-record scratch written and read; columns written and read back; ids and codes
    print(json.dumps({"records": n, "file_bytes": size, "load_wall_s": [round(w, 4) for w in walls], "median_load": med,
                      "device_ms": [{k: round(v, 3) for k, v in p.items()} for p in phases],
                      "snapshot_s": [round(r, 4) for r in reads], "host_lists_s": [round(x, 4) for x in lists],
                      "row_path_s": None if rows_s is None else round(rows_s, 3),
                      "hbm_bytes_per_record": round(hbm / max(n, 1), 1), **info}))
    eng.close_engine()


if __name__ == "__main__":
    main()
