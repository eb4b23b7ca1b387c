"""Seeded usage tables for the save tests (test_usage_save_cpu.py, test_usage_save_gpu.py) and what sqlite3 must read back from a
saved file: every row, sqlite_sequence, sqlite_schema, the index order and the density against VACUUM INTO."""
from __future__ import annotations

import math
import os
import sqlite3
import struct
from datetime import datetime, timedelta

import numpy as np

from llmapigateway_b200.usage import _EPOCH, _sink_schema, synth_usage_columns

T0 = datetime(2026, 9, 21, 6, 57, 17, 47518)
PAGE_SIZES = (1024, 2048, 4096, 8192, 16384, 32768, 65536)
SPILL_LENS = (1100, 2100, 5000, 70_000, 140_000, 700_000)       # one, two and many overflow pages at every page size


def _row(rng, k, models=("m-a", "m-b", "zz/m", None), providers=("p1", "p2", None)):
    tok = [int(x) for x in rng.integers(0, 2**17, 5)]
    return ({"prompt_tokens": tok[0], "completion_tokens": tok[1], "total_tokens": tok[2], "reasoning_tokens": tok[3],
             "cached_tokens": tok[4], "cost": int(rng.integers(0, 10**6)) * 1e-6, "model": models[k % len(models)],
             "provider": providers[k % len(providers)]},
            T0 - timedelta(microseconds=int(rng.integers(0, 400 * 86400 * 10**6))))


def fill(t, name: str, seed: int = 7):
    """table t (a fresh UsageTable or stand-in) filled as family `name`"""
    rng = np.random.default_rng([seed, len(name)])
    ins = t.insert_usage
    if name == "c5like":
        ts, models, tok, cost = synth_usage_columns(3000, seed=seed)
        for k in range(3000):
            ins({"prompt_tokens": int(tok[0][k]), "completion_tokens": int(tok[1][k]), "total_tokens": int(tok[2][k]),
                 "reasoning_tokens": int(tok[3][k]), "cached_tokens": int(tok[4][k]), "cost": float(cost[k]), "model": models[k],
                 "provider": "provider-%d" % (k % 5)}, _EPOCH + timedelta(microseconds=int(ts[k])))
    elif name == "gaps":                          # a cleanup leaves gaps; the newest ids are old records, so _seq > max(id)
        for k in range(2600):
            u, when = _row(rng, k)
            ins(u, when if k % 3 and k < 2500 else T0 - timedelta(days=300 + k % 50))
        t._upload()
        t.cleanup_old_records(200, now=T0)
        t._upload()
        assert t._seq > int(t._ids.max()) + 50
    elif name == "empty":
        pass
    elif name == "one":
        ins({"prompt_tokens": 3, "model": "only", "provider": "p", "cost": 0.25}, T0)
    elif name.startswith("n"):                    # record counts at the tile edges
        for k in range(int(name[1:])):
            ins(*_row(rng, k))
    elif name == "ties":                          # long runs of equal timestamps
        for k in range(6000):
            u, _ = _row(rng, k)
            ins(u, T0 - timedelta(seconds=(k * 7919 % 6000) // 1500))
    elif name == "calendar":                      # zero microseconds, years 0001 and 9999
        stamps = [datetime(1, 1, 1), datetime(1, 1, 1, 0, 0, 0, 1), datetime(9999, 12, 31, 23, 59, 59),
                  datetime(9999, 12, 31, 23, 59, 59, 999999), datetime(2000, 2, 29, 12), datetime(1969, 12, 31, 23, 59, 59, 999999),
                  datetime(1970, 1, 1), datetime(2026, 1, 1, 0, 0, 0, 100000)]
        for k in range(400):
            ins({"prompt_tokens": k, "model": "m%d" % (k % 3)}, stamps[k % len(stamps)])
    elif name == "tokens":
        vals = [2**31 - 1, -(2**31 - 1), -2**31, 0, 1, -1, 127, 128, -128, -129, 32767, 32768, -32768, 8388607, 8388608]
        for k in range(300):
            ins({c: vals[(k + j) % len(vals)] for j, c in enumerate(("prompt_tokens", "completion_tokens", "total_tokens",
                                                                      "reasoning_tokens", "cached_tokens"))}, T0 - timedelta(minutes=k))
    elif name == "costs":
        vals = [math.nan, math.inf, -math.inf, -0.0, 0.0, 5e-324, -2.2250738585072014e-308 / 3, 3.0, -7.0, 1e15, 1.5, 1e308, None]
        for k in range(260):
            ins({"prompt_tokens": k, "cost": vals[k % len(vals)]}, T0 - timedelta(seconds=k))
    elif name == "spill":                         # texts onto one, two and many overflow pages
        for k in range(60):
            n = SPILL_LENS[k % len(SPILL_LENS)]
            ins({"prompt_tokens": k, "model": "M%03d" % k + "x" * n if k % 4 else None,
                 "provider": "P" + "é" * (n // 3) if k % 3 else "p"}, T0 - timedelta(hours=k))
    elif name == "texts":                         # NUL bytes, NULL models and providers, non-ASCII
        names = ["a\x00b", "\x00", "", "ünï\x00cødé", "\U0001F600", None]
        for k in range(500):
            ins({"prompt_tokens": k, "model": names[k % 6], "provider": names[(k // 6) % 6]}, T0 - timedelta(seconds=k * 13))
    else:
        raise KeyError(name)
    return t


FAMILIES = ("c5like", "gaps", "empty", "one", "n2047", "n2048", "n2049", "n4097", "ties", "calendar", "tokens", "costs", "spill", "texts")


def expect_rows(t) -> list[tuple]:
    """the rows SELECT * FROM tokens_usage ORDER BY id must give: NaN costs as NULL, costs as their bit patterns"""
    t._materialise()
    h = t._host
    rows = []
    for i in range(int(h["ts_us"].size)):
        cost = float(h["cost"][i])
        rows.append((int(t._ids[i]), (_EPOCH + timedelta(microseconds=int(h["ts_us"][i]))).isoformat(),
                     *[int(h[c][i]) for c in t.COLS[2:7]], None if math.isnan(cost) else struct.pack("<d", cost),
                     t._models[i], t._providers[i]))
    return rows


def check_file(path, t, vacuum_dir=None):
    """the file at path against table t, as sqlite3 reads it"""
    conn = sqlite3.connect(path)
    try:
        assert conn.execute("PRAGMA integrity_check").fetchall() == [("ok",)]
        got = conn.execute("SELECT * FROM tokens_usage ORDER BY id").fetchall()
        got = [(*r[:7], None if r[7] is None else struct.pack("<d", r[7]), *r[8:]) for r in got]
        want = expect_rows(t)
        assert got == want
        for r in conn.execute("SELECT typeof(cost) FROM tokens_usage WHERE cost IS NOT NULL LIMIT 5"):
            assert r[0] == "real"
        seq = conn.execute("SELECT name, seq FROM sqlite_sequence").fetchall()
        assert seq == ([("tokens_usage", t._seq)] if t._seq > 0 else [])
        schema = conn.execute("SELECT type, name, tbl_name, sql FROM sqlite_schema ORDER BY rowid").fetchall()
        assert schema == _sink_schema()
        idx = conn.execute("SELECT timestamp, id FROM tokens_usage INDEXED BY idx_tokens_usage_timestamp WHERE timestamp >= ''").fetchall()
        assert idx == sorted((r[1], r[0]) for r in want)
        if vacuum_dir is not None:
            vac = os.path.join(vacuum_dir, "vacuum.db")
            if os.path.exists(vac):
                os.remove(vac)
            conn.execute("VACUUM INTO ?", (vac,))            # (at the source's page size)
            assert os.path.getsize(path) <= 1.10 * os.path.getsize(vac), (os.path.getsize(path), os.path.getsize(vac))
    finally:
        conn.close()
