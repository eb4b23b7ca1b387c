"""The record listing (/v1/api/usage-records, UsageTable.get_latest_usage_records) on BASELINE config 5's table (10 M records):
pages (25, 0), (25, n/2), (25, n-25), a 65 536-row page and the full listing, selected on the device (csrc/listing.cuh) and
by the host path (engine=None).  One JSON line per page: device ms from lgw_usage_latest_last_ms (CUDA events), host wall ms
per call including the row dicts, the same for the host path; first a line with the GPU's name and power limit.
    python tools/bench_listing.py [--records 10000000] [--reps 20]
"""
import argparse
import json
import subprocess
import sys
import time
from datetime import datetime
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def _gpu():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _wall(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=2)
    args = ap.parse_args()
    import llmapigateway_b200 as L
    from llmapigateway_b200.usage import UsageTable, synth_usage_columns
    print(json.dumps(_gpu()), flush=True)
    n = args.records
    ts, models, tok, cost = synth_usage_columns(n, seed=5, end=datetime(2026, 9, 21, 6, 57, 17, 47518))
    eng = L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    dev, host = UsageTable(eng), UsageTable(None)
    for t in (dev, host):
        t.load_columns(ts, models, *tok, cost)
    t0 = time.perf_counter()
    dev.get_latest_usage_records(25, 0)
    print(json.dumps({"first_listing_with_upload_ms": round((time.perf_counter() - t0) * 1e3, 1)}), flush=True)
    want = np.argsort(-ts, kind="stable")
    for name, limit, offset in (("page_25_at_0", 25, 0), ("page_25_at_half", 25, n // 2), ("page_25_at_end", 25, n - 25),
                                ("page_65536", 65536, n // 3), ("full", -1, 0)):
        big = limit < 0 or limit > 1000
        reps = max(1, args.reps // (10 if big else 1)) if limit > 0 else 1
        got = dev.get_latest_usage_records(limit, offset)              # warm-up, and the result check
        count = n - offset if limit < 0 else min(limit, n - offset)
        assert [r["id"] - 1 for r in got[:100]] == want[offset:offset + min(count, 100)].tolist() and len(got) == count, name
        del got
        dev_ms, wall = [], []
        for _ in range(reps):
            wall += _wall(lambda: dev.get_latest_usage_records(limit, offset), 1)
            dev_ms.append(dev.listing_last_ms())
        # the selection alone (indices, no dicts): what the device work costs a caller
        sel = _wall(lambda: dev._latest_on_device(n, offset, count), reps)
        host_wall = _wall(lambda: host.get_latest_usage_records(limit, offset), args.host_reps if not big else 1)
        print(json.dumps({"page": name, "limit": limit, "offset": offset, "rows": count, "reps": reps,
                          "device_ms_median": round(float(np.median(dev_ms)), 4), "device_ms_min": round(float(min(dev_ms)), 4),
                          "select_call_wall_ms_median": round(float(np.median(sel)), 3),
                          "wall_ms_median_with_dicts": round(float(np.median(wall)), 3),
                          "host_path_wall_ms_median": round(float(np.median(host_wall)), 1)}), flush=True)
    dev.close()
    eng.close_engine()


if __name__ == "__main__":
    main()
