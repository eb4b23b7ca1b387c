"""Deleting old usage records (UsageTable.cleanup_old_records) on BASELINE config 5's table (10 M records over 400 days) at
180 days' retention, against the alternative of reloading the survivors with load_columns.  JSON lines:
  - the GPU's name and power limit;
  - per repetition, on a fresh upload of the table: device ms of the compaction (lgw_usage_retain_last_ms, CUDA events), wall
    ms of cleanup_old_records, of the first rollup after it (the stats endpoint's `day` window) and of the first listing page;
  - the same three wall times for load_columns of the survivors (the rollup then re-ranks the models and uploads the table);
  - medians of both.
    python tools/bench_retention.py [--records 10000000] [--reps 7]
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
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--days", type=float, default=180)
    args = ap.parse_args()
    import llmapigateway_b200 as L
    from llmapigateway_b200.usage import UsageTable, synth_usage_columns, stats_window, to_us
    print(json.dumps(_gpu()), flush=True)
    ts, models, tok, cost = synth_usage_columns(args.records, seed=5, end=NOW)
    eng = L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    start, end = stats_window("day", NOW)
    keep = ts >= to_us(NOW - timedelta(days=args.days))
    rows = {"cleanup": [], "reload": []}
    for rep in range(args.reps + 1):                                   # (rep 0 warms every kernel and allocation up)
        t = UsageTable(eng)
        t.load_columns(ts, models, *tok, cost)
        t.get_aggregated_usage("day", start, end)                       # resident and ranked, as a running gateway has it
        r = {"cleanup_wall_ms": _ms(lambda: t.cleanup_old_records(args.days, now=NOW))}
        r["device_ms"] = t.retain_last_ms()
        r["first_rollup_wall_ms"] = _ms(lambda: t.get_aggregated_usage("day", start, end))
        r["first_page_wall_ms"] = _ms(lambda: t.get_latest_usage_records(25, 0))
        kept = len(t)
        t.close()
        u = UsageTable(eng)
        u.load_columns(ts, models, *tok, cost)
        u.get_aggregated_usage("day", start, end)
        s = {"reload_wall_ms": _ms(lambda: u.load_columns(ts[keep], models[keep], *[c[keep] for c in tok], cost[keep]))}
        s["first_rollup_wall_ms"] = _ms(lambda: u.get_aggregated_usage("day", start, end))
        s["first_page_wall_ms"] = _ms(lambda: u.get_latest_usage_records(25, 0))
        assert len(u) == kept
        u.close()
        if rep:
            rows["cleanup"].append(r)
            rows["reload"].append(s)
            print(json.dumps({"rep": rep, "records": int(ts.size), "kept": kept, "cleanup": r, "reload": s}), flush=True)
    med = {k: {f: round(float(np.median([x[f] for x in v])), 3) for f in v[0]} for k, v in rows.items()}
    print(json.dumps({"records": int(ts.size), "retention_days": args.days, "median": med}), flush=True)
    eng.close_engine()


if __name__ == "__main__":
    main()
