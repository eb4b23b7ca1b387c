"""Inserted usage records reaching the device (UsageTable._upload appending with lgw_usage_append) on BASELINE config 5's table
(10 M records over 400 days), against the full re-rank and upload that a table without a device copy still pays.  JSON lines:
  - the GPU's name, power limit and SM clock limit;
  - the full re-rank and upload of the table (load_columns, then _upload), wall ms per repetition;
  - the first append after that upload, which grows the columns (a copy of every record into room for twice as many);
  - per case (1 / 100 / 10 000 / 65 537 inserted rows, with and without a new model name that sorts before every other, so
    that every rank moves), per repetition: wall ms of get_aggregated_usage("day", *stats_window("day")) right after the
    inserts (the append happens inside it), the append's device ms (lgw_usage_append_last_ms: the copy of the new rows and
    k_usage_append), wall ms of the next listing page (25, 0) and of a second stats call;
  - medians per case.
The inserts themselves (insert_usage, a Python call per row) are not timed.
    python tools/bench_append.py [--records 10000000] [--reps 5]
"""
import argparse
import json
import subprocess
import sys
import time
from datetime import datetime, timedelta
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

NOW = datetime(2026, 9, 21, 6, 57, 17, 47518)


def _gpu():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _ms(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import llmapigateway_b200 as L
    from llmapigateway_b200.usage import UsageTable, synth_usage_columns, stats_window, _EPOCH
    print(json.dumps(_gpu()), flush=True)
    ts, models, tok, cost = synth_usage_columns(args.records, seed=5, end=NOW)
    eng = L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    window = stats_window("day", NOW)
    rng = np.random.default_rng(7)
    names = sorted({m for m in models[:100_000] if m is not None})

    def insert(t, m, new_name):
        stamps = ts[-1] + rng.integers(0, 10**9, m)
        picks = rng.integers(0, len(names), m)
        for k in range(m):
            model = new_name if (new_name and k == m // 2) else names[picks[k]]
            t.insert_usage({"prompt_tokens": k, "completion_tokens": 2 * k, "total_tokens": 3 * k, "cost": k * 1e-6, "model": model,
                            "provider": "P"}, timestamp=_EPOCH + timedelta(microseconds=int(stamps[k])))

    full = []
    for rep in range(args.reps + 1):                                   # (rep 0 warms every kernel and allocation up)
        u = UsageTable(eng)
        u.load_columns(ts, models, *tok, cost)
        ms = _ms(u._upload)
        u.close()
        if rep:
            full.append(ms)
    print(json.dumps({"records": int(ts.size), "full_rerank_upload_wall_ms": [round(x, 3) for x in full]}), flush=True)

    t = UsageTable(eng)
    t.load_columns(ts, models, *tok, cost)
    t.get_aggregated_usage("day", *window)                              # resident and ranked, as a running gateway has it
    insert(t, 1, None)
    first = {"first_append_wall_ms": _ms(lambda: t.get_aggregated_usage("day", *window)), "device_ms": t.append_last_ms(),
             "capacity": t._dev_cap}
    print(json.dumps({"first_append_after_upload": first}), flush=True)
    out = {}
    for m in (1, 100, 10_000, 65_537):
        for new in (False, True):
            rows = []
            for rep in range(args.reps + 1):
                insert(t, m, "0-new-%d-%d" % (m, rep) if new else None)
                r = {"stats_wall_ms": _ms(lambda: t.get_aggregated_usage("day", *window)), "device_ms": t.append_last_ms()}
                r["page_wall_ms"] = _ms(lambda: t.get_latest_usage_records(25, 0))
                r["stats_again_wall_ms"] = _ms(lambda: t.get_aggregated_usage("day", *window))
                if rep:
                    rows.append(r)
            key = "%d%s" % (m, "_new_name" if new else "")
            out[key] = {f: round(float(np.median([x[f] for x in rows])), 3) for f in rows[0]}
            print(json.dumps({"inserted": m, "new_name": new, "records": len(t), "reps": rows}), flush=True)
    print(json.dumps({"records": int(ts.size), "full_rerank_upload_median_ms": round(float(np.median(full)), 3), "median": out}), flush=True)
    t.close()
    eng.close_engine()


if __name__ == "__main__":
    main()
