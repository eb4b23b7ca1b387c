"""Times UsageTable.save_tokens_usage_db on the 10 M-record C5 table (synth_usage_columns, SURVEY 8(d)) with 4 KiB pages: the wall
time split into the host's text tables and codes, the device phases (CUDA events: ids and codes up, keep, sort, pack, page
writes, download into page-locked memory), the page-locked allocation and the disk write; then the startup sequence load ->
cleanup_old_records(180) -> save; then the sqlite3 path for the same cleanup (DELETE + VACUUM on a copy of the file).  Prints
one JSON line with the GPU's name and power limit read in the same run.  Writes only into a temporary directory.

    python tools/bench_save.py [--records 10000000] [--repeat 3]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sqlite3
import subprocess
import sys
import tempfile
import time
from datetime import timedelta
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import llmapigateway_b200 as LG  # noqa: E402
from llmapigateway_b200 import usage as U  # noqa: E402


def note(msg: str):
    print(msg, file=sys.stderr, flush=True)


def gpu_info() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, limit = (out.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if out.returncode == 0 else ("?", "?")
    return {"gpu": name, "power_limit": limit}


class Timed:
    """wall time of the calls of one function of usage.py, summed"""

    def __init__(self, name):
        self.name, self.ms = name, 0.0
        self.real = getattr(U, name)

        def run(*a, **k):
            t0 = time.perf_counter()
            try:
                return self.real(*a, **k)
            finally:
                self.ms += (time.perf_counter() - t0) * 1e3
        setattr(U, name, run)


def timed_save(t, path) -> dict:
    write, texts = Timed("_write_replace"), Timed("_save_text_table")
    alloc_ms = [0.0]
    real_alloc = t._save_alloc

    def alloc(nbytes):
        t0 = time.perf_counter()
        try:
            return real_alloc(nbytes)
        finally:
            alloc_ms[0] += (time.perf_counter() - t0) * 1e3
    t._save_alloc = alloc
    t0 = time.perf_counter()
    try:
        n = t.save_tokens_usage_db(path, 4096)
    finally:
        wall = (time.perf_counter() - t0) * 1e3
        U._write_replace, U._save_text_table = write.real, texts.real
        del t._save_alloc
    return {"records": n, "bytes": os.path.getsize(path), "wall_ms": round(wall, 1), "device_ms": {k: round(v, 3) for k, v in t.save_last_ms().items()},
            "text_tables_ms": round(texts.ms, 1), "pinned_alloc_ms": round(alloc_ms[0], 1), "disk_write_ms": round(write.ms, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=10_000_000)
    ap.add_argument("--repeat", type=int, default=3)
    args = ap.parse_args()
    eng = LG.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    ts, models, tok, cost = U.synth_usage_columns(args.records)
    now = U._EPOCH + timedelta(microseconds=int(ts.max()))
    res = {"records": args.records, **gpu_info()}
    with tempfile.TemporaryDirectory() as d:
        d = Path(d)
        t = U.UsageTable(eng)
        t.load_columns(ts, models, *tok, cost)
        t._upload()
        runs = []
        for k in range(args.repeat):
            runs.append(timed_save(t, d / "c5.db"))
            note(f"save {k}: {runs[-1]}")
        res["save"] = runs
        t.close()
        seq = []
        for k in range(args.repeat):
            shutil.copy(d / "c5.db", d / "start.db")
            u = U.UsageTable(eng)
            t0 = time.perf_counter()
            u.load_tokens_usage_db(d / "start.db")
            t1 = time.perf_counter()
            u.cleanup_old_records(180, now=now)
            t2 = time.perf_counter()
            s = timed_save(u, d / "start.db")
            seq.append({"load_ms": round((t1 - t0) * 1e3, 1), "cleanup_ms": round((t2 - t1) * 1e3, 1), "save": s})
            note(f"load -> cleanup -> save {k}: {seq[-1]}")
            u.close()
        res["load_cleanup_save"] = seq
        shutil.copy(d / "c5.db", d / "sql.db")
        conn = sqlite3.connect(d / "sql.db")
        t0 = time.perf_counter()
        conn.execute("DELETE FROM tokens_usage WHERE timestamp < ?", ((now - timedelta(days=180)).isoformat(),))
        conn.commit()
        t1 = time.perf_counter()
        note(f"sqlite3 DELETE: {(t1 - t0) * 1e3:.0f} ms; VACUUM next")
        conn.execute("VACUUM")
        t2 = time.perf_counter()
        conn.close()
        res["sqlite3"] = {"delete_ms": round((t1 - t0) * 1e3, 1), "vacuum_ms": round((t2 - t1) * 1e3, 1), "bytes": os.path.getsize(d / "sql.db")}
        note(f"sqlite3: {res['sqlite3']}")
    eng.close_engine()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
