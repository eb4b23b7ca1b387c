"""GPU: UsageTable.load_tokens_usage_db decodes a `tokens_usage` file on the device (csrc/load.cuh).  The seeded file families
of test_usage_load_cpu.py go through the device and are compared with sqlite3 reading the same file: the eight device columns
byte for byte, ids, models, providers and refused ids.  Every query after a load is compared with SQLite on the same file:
rollups (the repo's restatement of the reference SQL, oracle/rollup_oracle.py), listing pages (ORDER BY timestamp DESC, id ASC),
cleanup_old_records (the SQL DELETE on a copy) and the next id.  C5's 10 M records load as the row path does, with no
upload at the first query; 65 536-byte pages, 100 000 distinct names, two loads on one engine and a load over a table with
pending rows and a device copy.  Damaged files fail with UsageDbCorrupt and leave the table and its device copy as they were."""
import shutil
import sqlite3
from datetime import datetime, timedelta

import numpy as np
import pytest

import load_cases as L
from llmapigateway_b200.usage import UsageTable, stats_window, synth_usage_columns
from oracle import rollup_oracle as ro
from test_rollup_gpu import _ulps
from test_usage_retention_gpu import CountingLib, _download, _new_engine

pytestmark = pytest.mark.gpu
FAMILIES = L.families()
PERIODS = ("hour", "day", "week", "month")


@pytest.fixture(scope="module")
def engine():
    e = _new_engine()
    yield e
    e.close_engine()


@pytest.fixture(scope="module")
def dbs(tmp_path_factory):
    d = tmp_path_factory.mktemp("load")
    out = {}
    for name, write in FAMILIES:
        out[name] = d / f"{name}.db"
        write(str(out[name]), 11)
    return out


def _device_matches_host(t):
    got = _download(t)
    for c in UsageTable.COLS:
        assert got[c].tobytes() == t._host[c].tobytes(), c


@pytest.mark.parametrize("name", [f[0] for f in FAMILIES])
def test_family_on_device(engine, dbs, name):
    t = UsageTable(engine)
    n = t.load_tokens_usage_db(dbs[name])
    expect = L.sqlite_expect(dbs[name])
    assert n == len(expect["kept"])
    L.assert_loaded(t, expect)
    _device_matches_host(t)
    t.close()


@pytest.mark.parametrize("kind,family", [("child_past_end", "pages1024"), ("interior_cycle", "pages512"),
                                         ("cell_pointer_outside", "pages1024"), ("payload_beyond_file", "pages1024"),
                                         ("overflow_cycle", "spill512"), ("cells_misordered", "pages4096")])
def test_damaged_file_on_device(engine, dbs, tmp_path, kind, family):
    """a damaged file fails with UsageDbCorrupt after the device decode, and the table keeps its records and device copy"""
    from test_usage_load_cpu import _damage
    from llmapigateway_b200.usage import UsageDbCorrupt
    path = tmp_path / "bad.db"
    _damage(kind, dbs[family], path)
    t = UsageTable(engine)
    t.load_tokens_usage_db(dbs["root_leaf"])
    before, ptrs = _download(t), t._dev_ptrs
    with pytest.raises(UsageDbCorrupt):
        t.load_tokens_usage_db(path)
    assert t._dev_ptrs is ptrs and len(t) == 3
    after = _download(t)
    assert all(before[c].tobytes() == after[c].tobytes() for c in UsageTable.COLS)
    t.load_tokens_usage_db(dbs["deleted"])                   # the engine loads the next file
    L.assert_loaded(t, L.sqlite_expect(dbs["deleted"]))
    t.close()


def _sql_listing(path, limit, offset):
    conn = sqlite3.connect(path)
    rows = conn.execute("SELECT id FROM tokens_usage ORDER BY timestamp DESC, id ASC LIMIT ? OFFSET ?", (limit, offset)).fetchall()
    conn.close()
    return [r[0] for r in rows]


@pytest.mark.parametrize("name", ["pages4096", "deleted", "pages65536"])
def test_queries_against_sqlite(engine, dbs, tmp_path, name):
    path = dbs[name]
    t = UsageTable(engine)
    t.load_tokens_usage_db(path)
    lib = CountingLib(t._lib)
    t._lib = lib
    conn = sqlite3.connect(path)
    now = L.T0
    for period in PERIODS:
        for window in (None, stats_window(period, now)):
            got = t.get_aggregated_usage(period, *(window or (None, None)))
            want = ro.aggregated_usage(conn, period, *(window or (None, None)))
            assert len(got) == len(want) and got, (period, window)
            for g, w in zip(got, want):
                assert {k: v for k, v in g.items() if k != "cost"} == {k: v for k, v in w.items() if k != "cost"}
                assert (g["cost"] is None) == (w["cost"] is None) and (g["cost"] is None or _ulps(g["cost"], w["cost"]) <= 4), (g, w)
    conn.close()
    assert lib.uploads == 0
    for limit, offset in ((25, 0), (100, 37), (10, len(t) - 3)):
        assert [r["id"] for r in t.get_latest_usage_records(limit, offset)] == _sql_listing(path, limit, offset)
    copy = tmp_path / "copy.db"
    shutil.copy(path, copy)
    cutoff = now - timedelta(days=100)
    t.cleanup_old_records(100, now=now)
    conn = sqlite3.connect(copy)
    conn.execute("DELETE FROM tokens_usage WHERE timestamp < ?", (cutoff.isoformat(),))
    ids = [r[0] for r in conn.execute("SELECT id FROM tokens_usage ORDER BY id")]
    seq = conn.execute("SELECT seq FROM sqlite_sequence WHERE name = 'tokens_usage'").fetchone()[0]
    conn.close()
    assert t._ids.tolist() == ids
    assert t.insert_usage({"prompt_tokens": 1, "model": "new"}, now)
    assert t.get_latest_usage_records(1)[0]["id"] == seq + 1
    t.close()


def test_c5_geometry(engine, tmp_path):
    """10 M records of synth_usage_columns plus refused ones, against the row path (sqlite3 rows into load_columns)"""
    n = 10_000_000
    ts, models, tok, cost = synth_usage_columns(n)
    path = str(tmp_path / "c5.db")
    conn = L.create(path, 4096)
    stamps = np.datetime_as_string(ts.astype("datetime64[us]"), unit="us")
    whole = stamps.astype("U19")
    text = np.where(ts % 10**6 == 0, whole, stamps).tolist()
    conn.executemany(L.INSERT, zip(text, *[a.tolist() for a in tok], cost.tolist(), models.tolist(), ["p"] * n))
    bad = [("2026-01-01 00:00:00", 1, 1, 1, 1, 1, 0.5, "m", None), ("2026-01-01T00:00:00", 2**31, 1, 1, 1, 1, 0.5, "m", None),
           ("2026-01-01T00:00:00", 1, 1, 1, 1, 1, "x", "m", None)]
    conn.executemany(L.INSERT, bad)
    conn.commit()
    conn.close()
    t = UsageTable(engine)
    lib = CountingLib(t._lib)
    t._lib = lib
    got = t.load_tokens_usage_db(path)
    assert got == n and t.rejected_ids.tolist() == [n + 1, n + 2, n + 3] and t._seq == n + 3
    ref = UsageTable(engine)
    ref.load_columns(ts, models, *tok, cost)
    ref._materialise()
    for c in UsageTable.COLS:
        assert t._host[c].tobytes() == ref._host[c].tobytes(), c
    assert t._names == ref._names and t._models == list(models)
    _device_matches_host(t)
    rows = t.rollup_rows("day")
    assert lib.uploads == 0
    assert np.array_equal(rows, ref.rollup_rows("day"))
    t.close()
    ref.close()


def test_many_names_two_loads_and_replace(engine, tmp_path):
    path = str(tmp_path / "names.db")
    names = ["name-%06d-%s" % (k, "é" * (k % 5)) for k in range(100_000)]
    conn = L.fill(path, 150_000, 4, 4096, names=names)
    conn.executemany(L.INSERT, [("2026-05-06T07:08:09", 1, 2, 3, 4, 5, 0.5, m, m[:7]) for m in names])     # every name at least once
    conn.commit()
    conn.close()
    t = UsageTable(engine)
    for k in range(30):                                       # pending rows and a device copy, replaced by the load
        t.insert_usage({"prompt_tokens": k, "model": "old-%d" % (k % 3)}, datetime(2026, 1, 1) + timedelta(seconds=k))
    t.rollup_rows("day")
    assert t._dev_n == 30
    t.insert_usage({"prompt_tokens": 99, "model": "pending"})
    expect = L.sqlite_expect(path)
    for _ in range(2):                                         # two loads on one engine
        t.load_tokens_usage_db(path)
        L.assert_loaded(t, expect)
        _device_matches_host(t)
    assert len(t._names) == 100_001
    small = tmp_path / "small.db"
    L.fill(str(small), 10, 2, 65536).close()
    t.load_tokens_usage_db(small)
    L.assert_loaded(t, L.sqlite_expect(small))
    _device_matches_host(t)
    t.close()
