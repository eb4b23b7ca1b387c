"""UsageTable.save_tokens_usage_db with the device writer's own code (csrc/save.cuh) built with g++ (tests/host_save.py): seeded
tables saved at every page size and read back with sqlite3 (integrity, rows bit for bit, sqlite_sequence, sqlite_schema, index
order, density against VACUUM INTO); the round trip through the loader's host build; the file kept writable by SqliteUsageSink
and answering the rollup and listing SQL as a sink-written file; refused records; atomic replacement and every failure leaving
the old file and the table as they were; the writer under AddressSanitizer."""
import os
import shutil
import sqlite3
from datetime import datetime, timedelta

import numpy as np
import pytest

import save_cases as S
from host_load import HostLoadTable
from host_save import HostSaveTable, asan_run
from llmapigateway_b200.gateway import SqliteUsageSink
from llmapigateway_b200.usage import UsageDbNotModelled, UsageTable, db_geometry
from oracle import rollup_oracle as ro


@pytest.mark.parametrize("page_size", S.PAGE_SIZES)
@pytest.mark.parametrize("name", S.FAMILIES)
def test_family_read_back_by_sqlite(tmp_path, name, page_size):
    t = S.fill(HostSaveTable(), name)
    path = tmp_path / "saved.db"
    assert t.save_tokens_usage_db(path, page_size) == len(t)
    raw = path.read_bytes()
    assert db_geometry(raw[:100], len(raw)) == (page_size, len(raw) // page_size)
    assert raw[18:24] == bytes((1, 1, 0, 64, 32, 32)) and raw[24:28] == raw[92:96] and raw[32:40] == bytes(8)
    assert int.from_bytes(raw[44:48], "big") == 4 and int.from_bytes(raw[52:56], "big") == 0
    assert int.from_bytes(raw[28:32], "big") * page_size == len(raw)
    S.check_file(path, t, vacuum_dir=tmp_path)
    assert t.save_refused_ids.size == 0


def test_family_shapes():
    t = S.fill(HostSaveTable(), "spill")
    t._materialise()
    lens = sorted(len(m.encode()) for m in t._models if m)
    assert lens[0] > 1024 and lens[-1] > 10 * 65536
    t = S.fill(HostSaveTable(), "gaps")
    assert np.any(np.diff(t._ids) > 1) and t._seq > t._ids.max()


class RoundTrip(HostSaveTable):
    """the host builds of both the writer and the loader over the append test's numpy stand-in"""
    _load_call = HostLoadTable._load_call
    _load_alloc = HostLoadTable._load_alloc
    _load_free = HostLoadTable._load_free

    def _load_cols_alloc(self, n):
        return None

    def load_tokens_usage_db(self, db_path):
        n = UsageTable.load_tokens_usage_db(self, db_path)
        self._dev_ptrs = {c: self._host[c].copy() for c in self.COLS}
        self._dev = (n, self._dev_ptrs)
        return n


@pytest.mark.parametrize("page_size", [1024, 4096, 65536])
@pytest.mark.parametrize("name", S.FAMILIES)
def test_round_trip(tmp_path, name, page_size):
    t = S.fill(RoundTrip(), name)
    t._upload()
    a, b = tmp_path / "a.db", tmp_path / "b.db"
    t.save_tokens_usage_db(a, page_size)
    u = RoundTrip()
    assert u.load_tokens_usage_db(a) == len(t) and u.rejected == 0
    for c in t.COLS:
        if c != "model_rank" or u._names == t._names:
            assert u._host[c].tobytes() == t._host[c].tobytes(), c
    assert u._ids.tolist() == t._ids.tolist() and u._seq == t._seq
    assert u._models == t._models and u._providers == t._providers
    u.save_tokens_usage_db(b, page_size)
    assert a.read_bytes() == b.read_bytes()


def _sink_file(path, t):
    """a file SqliteUsageSink writes with t's rows and timestamps (ids 1..n)"""
    sink = SqliteUsageSink(str(path))
    rows = S.expect_rows(t)
    usages = [{"prompt_tokens": r[2], "completion_tokens": r[3], "total_tokens": r[4], "reasoning_tokens": r[5], "cached_tokens": r[6],
               "cost": float(t._host["cost"][i]), "model": r[8], "provider": r[9]} for i, r in enumerate(rows)]
    sink.insert_many(usages, [datetime.fromisoformat(r[1]) for r in rows])
    sink.conn.close()


def _answers(path, now):
    conn = sqlite3.connect(path)
    try:
        out = [ro.aggregated_usage(conn, p, *w) for p in ("hour", "day", "week", "month") for w in ((None, None), (now - timedelta(days=30), now))]
        out.append(conn.execute("SELECT id, timestamp FROM tokens_usage ORDER BY timestamp DESC, id LIMIT 40 OFFSET 7").fetchall())
        out.append(conn.execute("SELECT id FROM tokens_usage ORDER BY timestamp DESC, id").fetchall())
        return out
    finally:
        conn.close()


@pytest.mark.parametrize("page_size", [1024, 4096])
def test_stays_writable_by_sqlite(tmp_path, page_size):
    t = S.fill(HostSaveTable(), "c5like")
    saved, ref = tmp_path / "saved.db", tmp_path / "sink.db"
    t.save_tokens_usage_db(saved, page_size)
    _sink_file(ref, t)
    new = [({"prompt_tokens": k, "cost": 0.5, "model": "m-new-%d" % (k % 3), "provider": "p"}, S.T0 - timedelta(hours=k)) for k in range(50)]
    for path in (saved, ref):
        sink = SqliteUsageSink(str(path))
        sink.insert_many([u for u, _ in new], [w for _, w in new])
        assert sink.conn.execute("SELECT max(id) FROM tokens_usage").fetchone()[0] == t._seq + 50
        sink.conn.close()
    assert _answers(saved, S.T0) == _answers(ref, S.T0)
    cutoff = (S.T0 - timedelta(days=180)).isoformat()
    for path in (saved, ref):
        copy = tmp_path / ("copy-" + path.name)
        shutil.copy(path, copy)
        conn = sqlite3.connect(copy)
        conn.execute("DELETE FROM tokens_usage WHERE timestamp < ?", (cutoff,))
        conn.commit()
        assert conn.execute("PRAGMA integrity_check").fetchall() == [("ok",)]
        conn.close()
    assert _answers(tmp_path / "copy-saved.db", S.T0) == _answers(tmp_path / "copy-sink.db", S.T0)


def test_refusals(tmp_path, caplog):
    """a provider with a lone surrogate (a model with one cannot be ranked, so no table holds one) and timestamps with no
    isoformat text (only load_columns gives those)"""
    t = HostSaveTable()
    n = 300
    ts = np.array([1_790_000_000_000_000 + k * 10**6 for k in range(n)], np.int64)
    ts[7] = np.iinfo(np.int64).min
    ts[8] = 253402300800000000                       # 10000-01-01: no isoformat text
    z = np.zeros(n, np.int32)
    t.load_columns(ts, ["m%d" % (k % 4) for k in range(n)], z + 1, z, z, z, z, np.full(n, 0.5))
    t._providers[3] = "bad\udc80"
    path = tmp_path / "r.db"
    with caplog.at_level("WARNING"):
        assert t.save_tokens_usage_db(path, 4096) == n - 3
    refused = sorted(int(i) for i in t.save_refused_ids)
    assert refused == [4, 8, 9]
    assert "save_refused_ids" in caplog.text
    conn = sqlite3.connect(path)
    ids = [r[0] for r in conn.execute("SELECT id FROM tokens_usage ORDER BY id")]
    conn.close()
    assert ids == [i for i in range(1, n + 1) if i not in refused]


@pytest.mark.parametrize("page_size", [512, 3000, 131072, 0, 4096.0, True])
def test_bad_page_size(tmp_path, page_size):
    t = S.fill(HostSaveTable(), "one")
    with pytest.raises(ValueError):
        t.save_tokens_usage_db(tmp_path / "x.db", page_size)
    assert not os.listdir(tmp_path)


def _state(t):
    t._materialise()
    return ({c: a.copy() for c, a in t._host.items()}, t._ids.copy(), list(t._models), list(t._providers), t._seq, t._dev_ptrs, t._dev_n)


def _same_state(t, before):
    now = _state(t)
    assert all(np.array_equal(now[0][c], before[0][c]) for c in t.COLS)
    assert np.array_equal(now[1], before[1]) and now[2:5] == before[2:5] and now[5] is before[5] and now[6] == before[6]


def test_replaces_atomically(tmp_path):
    path = tmp_path / "usage.db"
    old = S.fill(HostSaveTable(), "ties")
    old.save_tokens_usage_db(path, 4096)
    ino = path.stat().st_ino
    path.chmod(0o640)
    t = S.fill(HostSaveTable(), "c5like")
    t.save_tokens_usage_db(path, 4096)
    assert path.stat().st_ino != ino and (path.stat().st_mode & 0o777) == 0o640
    S.check_file(path, t)
    assert sorted(os.listdir(tmp_path)) == ["usage.db"]


def test_hot_journal_rolled_back_first(tmp_path):
    path = tmp_path / "usage.db"
    _sink_file(path, S.fill(HostSaveTable(), "n2049"))
    script = ("import os, sqlite3, sys\n"
              "c = sqlite3.connect(sys.argv[1]); c.execute('PRAGMA cache_size = 1'); c.execute('BEGIN')\n"
              "c.execute('DELETE FROM tokens_usage'); c.execute(\"INSERT INTO tokens_usage (timestamp) VALUES ('x')\")\n"
              "os._exit(0)\n")
    import subprocess
    import sys
    subprocess.check_call([sys.executable, "-c", script, str(path)])
    journal = tmp_path / "usage.db-journal"
    assert journal.exists() and journal.stat().st_size > 0
    t = S.fill(HostSaveTable(), "one")
    t.save_tokens_usage_db(path, 4096)
    assert not journal.exists() and sorted(os.listdir(tmp_path)) == ["usage.db"]
    S.check_file(path, t)


def _failing_save(tmp_path, t, setup, exc):
    path = tmp_path / "usage.db"
    old = S.fill(HostSaveTable(), "texts")
    old.save_tokens_usage_db(path, 4096)
    t._upload()
    before = _state(t)
    keep = setup(path)
    before_bytes = path.read_bytes()
    with pytest.raises(exc):
        t.save_tokens_usage_db(path, 4096)
    if keep is not None:
        keep.close()
    assert path.read_bytes() == before_bytes
    assert not [f for f in os.listdir(tmp_path) if f.endswith(".saving")]
    _same_state(t, before)


def test_lock_held_elsewhere(tmp_path):
    def hold(path):
        c = sqlite3.connect(path, isolation_level=None)
        c.execute("BEGIN IMMEDIATE")
        return c
    _failing_save(tmp_path, S.fill(HostSaveTable(), "c5like"), hold, sqlite3.OperationalError)


def test_wal_target(tmp_path):
    def wal(path):
        c = sqlite3.connect(path)
        assert c.execute("PRAGMA journal_mode = WAL").fetchone()[0] == "wal"
        c.close()
        return None
    _failing_save(tmp_path, S.fill(HostSaveTable(), "c5like"), wal, UsageDbNotModelled)


@pytest.mark.parametrize("step", ["plan", "write"])
def test_injected_failure(tmp_path, step):
    t = S.fill(HostSaveTable(), "spill")
    t.fail_at = step
    _failing_save(tmp_path, t, lambda p: None, RuntimeError)


def test_failed_replace(tmp_path, monkeypatch):
    def boom(a, b):
        raise OSError("replace failed")
    _failing_save(tmp_path, S.fill(HostSaveTable(), "c5like"), lambda p: monkeypatch.setattr(os, "replace", boom), OSError)


def test_too_large(tmp_path, monkeypatch):
    from llmapigateway_b200 import usage as U
    _failing_save(tmp_path, S.fill(HostSaveTable(), "c5like"), lambda p: monkeypatch.setattr(U, "LOAD_MAX_BYTES", 16 * 4096), UsageDbNotModelled)


def test_pending_rows_saved(tmp_path):
    t = S.fill(HostSaveTable(), "n2049")
    t._upload()
    uploads = t.full_uploads
    for k in range(10):
        t.insert_usage({"prompt_tokens": k, "model": "a-first"}, S.T0 + timedelta(seconds=k))
    path = tmp_path / "p.db"
    assert t.save_tokens_usage_db(path, 4096) == 2059
    assert t.full_uploads == uploads and not t._pending_rows
    S.check_file(path, t)


@pytest.mark.parametrize("name,page_size", [("spill", 1024), ("spill", 4096), ("n2047", 1024), ("n2049", 4096), ("n4097", 1024),
                                            ("empty", 1024), ("texts", 65536)])
def test_under_asan(tmp_path, name, page_size):
    t = S.fill(HostSaveTable(), name)
    res, pages = asan_run(t, page_size, tmp_path)
    path = tmp_path / "s.db"
    t.save_tokens_usage_db(path, page_size)
    raw = path.read_bytes()
    assert res[0] * page_size == len(raw) and res[3] == len(t)
    assert pages[2 * page_size:] == raw[2 * page_size:]


def test_past_the_lock_byte_page(tmp_path):
    """a file past 2^30 bytes: the page holding that offset is never used, here inside an overflow chain"""
    t = HostSaveTable()
    name = "L" * 700_000
    for k in range(1560):
        t.insert_usage({"prompt_tokens": k, "model": name if k % 2 else "s", "provider": name if k % 2 == 0 else None}, S.T0 - timedelta(seconds=k))
    path = tmp_path / "big.db"
    t.save_tokens_usage_db(path, 4096)
    assert path.stat().st_size > (1 << 30) + 4096
    raw = open(path, "rb")
    raw.seek(1 << 30)
    assert raw.read(4096) == bytes(4096)
    raw.close()
    conn = sqlite3.connect(path)
    assert conn.execute("PRAGMA integrity_check").fetchall() == [("ok",)]
    got = conn.execute("SELECT id, length(model), length(provider), prompt_tokens FROM tokens_usage ORDER BY id").fetchall()
    conn.close()
    assert got == [(k + 1, 700_000 if k % 2 else 1, None if k % 2 else 700_000, k) for k in range(1560)]
