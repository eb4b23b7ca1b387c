"""UsageTable.load_tokens_usage_db with the device decoder's own code (csrc/load.cuh) built with g++ (tests/host_load.py), against
sqlite3 reading the same files: every record's id, eight columns, model and provider, the refused ids and the next id, over
files the installed sqlite3 writes from a seed (tests/load_cases.py).  Damaged files run under AddressSanitizer; files the
loader does not model raise UsageDbNotModelled and leave the table as it was; a loaded table answers listings, cleanups and
inserts as the same records inserted one by one do."""
import sqlite3
from datetime import datetime, timedelta

import numpy as np
import pytest

import load_cases as L
from host_load import HostLoadTable, asan_run
from test_usage_append_cpu import AppendStandIn
from llmapigateway_b200.usage import UsageDbCorrupt, UsageDbNotModelled, UsageTable, db_geometry

FAMILIES = L.families()


@pytest.fixture(scope="module")
def dbs(tmp_path_factory):
    d = tmp_path_factory.mktemp("load")
    out = {}
    for name, write in FAMILIES:
        out[name] = d / f"{name}.db"
        write(str(out[name]), 11)
    return out


@pytest.mark.parametrize("name", [f[0] for f in FAMILIES])
def test_family_against_sqlite(dbs, name):
    t = HostLoadTable()
    n = t.load_tokens_usage_db(dbs[name])
    expect = L.sqlite_expect(dbs[name])
    assert n == len(expect["kept"]) and t.rejected == len(expect["refused"])
    L.assert_loaded(t, expect)


def test_family_shapes(dbs):
    assert L.tree_depth(dbs["root_leaf"]) == 1 and L.tree_depth(dbs["pages512"]) >= 4
    assert len(L.sqlite_expect(dbs["values"])["refused"]) > 40
    for ps in (512, 4096):                                  # texts spill into one, two and many overflow pages
        lens = [len(r[4].encode()) for r in L.sqlite_expect(dbs[f"spill{ps}"])["kept"] if r[4] and r[4].startswith("M")]
        assert max(lens) > 8 * ps and min(lens) < 2 * ps


def _pages(path):
    data = bytearray(open(path, "rb").read())
    ps, n_pages = db_geometry(bytes(data[:100]), len(data))
    conn = sqlite3.connect(path)
    root = conn.execute("SELECT rootpage FROM sqlite_schema WHERE name = 'tokens_usage'").fetchone()[0]
    conn.close()
    return data, ps, n_pages, root


def _cell_ptr(data, ps, pg, k):
    o = (pg - 1) * ps + (100 if pg == 1 else 0)
    hl = 12 if data[o] == 5 else 8
    return o + hl + 2 * k, (pg - 1) * ps + int.from_bytes(data[o + hl + 2 * k:o + hl + 2 * k + 2], "big")


def _first_leaf(data, ps, root):
    pg = root
    while data[(pg - 1) * ps] == 5:
        _, c = _cell_ptr(data, ps, pg, 0)
        pg = int.from_bytes(data[c:c + 4], "big")
    return pg


def _damage(kind, src, dst):
    data, ps, n_pages, root = _pages(src)
    if kind == "truncated":
        data = data[:len(data) // 2]
    elif kind == "child_past_end":
        _, c = _cell_ptr(data, ps, root, 0)
        data[c:c + 4] = (n_pages + 7).to_bytes(4, "big")
    elif kind == "interior_cycle":
        _, c = _cell_ptr(data, ps, root, 0)
        data[c:c + 4] = root.to_bytes(4, "big")
    elif kind == "cell_pointer_outside":
        p, _ = _cell_ptr(data, ps, _first_leaf(data, ps, root), 1)
        data[p:p + 2] = (ps - 1).to_bytes(2, "big") if ps < 65536 else b"\x00\x01"
    elif kind in ("cells_misordered", "cell_duplicated"):
        leaf = _first_leaf(data, ps, root)
        p0, _ = _cell_ptr(data, ps, leaf, 0)
        a, b = bytes(data[p0:p0 + 2]), bytes(data[p0 + 2:p0 + 4])
        data[p0:p0 + 4] = (b + a) if kind == "cells_misordered" else (a + a)
    elif kind == "payload_beyond_file":
        _, c = _cell_ptr(data, ps, _first_leaf(data, ps, root), 0)
        data[c:c + 4] = b"\xff\xff\xff\x7f"
    elif kind == "overflow_cycle":
        leaf = _first_leaf(data, ps, root)
        for k in range(int.from_bytes(data[(leaf - 1) * ps + 3:(leaf - 1) * ps + 5], "big")):
            _, c = _cell_ptr(data, ps, leaf, k)
            if data[c] & 0x80:                              # a payload size of two or more bytes: this record spilled
                break
        P = 0
        i = c
        while True:
            P = (P << 7) | (data[i] & 0x7F)
            i += 1
            if not data[i - 1] & 0x80:
                break
        while data[i] & 0x80:
            i += 1
        i += 1
        U = ps
        X, M = U - 35, ((U - 12) * 32 // 255) - 23
        K = M + (P - M) % (U - 4)
        local = K if K <= X else M
        first = int.from_bytes(data[i + local:i + local + 4], "big")
        data[(first - 1) * ps:(first - 1) * ps + 4] = first.to_bytes(4, "big")
    open(dst, "wb").write(bytes(data))


@pytest.mark.parametrize("kind,family,want", [("truncated", "pages1024", 1), ("child_past_end", "pages1024", 1),
                                              ("interior_cycle", "pages512", 6), ("cell_pointer_outside", "pages1024", 3),
                                              ("payload_beyond_file", "pages1024", 4), ("overflow_cycle", "spill512", 4),
                                              ("cells_misordered", "pages4096", 8), ("cell_duplicated", "pages1024", 8)])
def test_damaged_file_under_asan(dbs, tmp_path, kind, family, want):
    path = tmp_path / "bad.db"
    _damage(kind, dbs[family], path)
    data, ps, n_pages, root = _pages(path) if kind != "truncated" else (None, None, None, None)
    if kind == "truncated":
        raw = open(path, "rb").read()
        ps, n_pages = db_geometry(raw[:100], len(raw))
        _, _, _, root = _pages(dbs[family])
    res = asan_run(path, ps, n_pages, root)
    assert res[0] == want, res
    t = HostLoadTable()
    t.insert_usage({"prompt_tokens": 1, "model": "keep"}, datetime(2026, 1, 1))
    with pytest.raises(UsageDbCorrupt):
        t._load_records({"buf": np.frombuffer(open(path, "rb").read(), np.uint8).copy(), "size": path.stat().st_size,
                         "page_size": ps, "n_pages": n_pages, "root": root, "seq": 0})
    assert len(t) == 1 and t._pending_rows


def test_undamaged_under_asan(dbs):
    for name in ("pages512", "values", "spill512", "spill4096", "short", "autovacuum_FULL"):
        _, ps, n_pages, root = _pages(dbs[name])
        res = asan_run(dbs[name], ps, n_pages, root)
        assert res[0] == 0 and res[1] == len(L.sqlite_expect(dbs[name])["kept"]) + len(L.sqlite_expect(dbs[name])["refused"])


def _not_modelled(tmp_path, kind):
    path = str(tmp_path / f"{kind}.db")
    if kind == "wal":
        conn = L.fill(path, 50, 3)
        conn.execute("PRAGMA journal_mode = WAL")
        conn.executemany(L.INSERT, [L._row(np.random.default_rng(1))])
        conn.commit()
        return path, conn                                   # (kept open: the WAL stays)
    if kind == "utf16":
        conn = sqlite3.connect(path)
        conn.execute("PRAGMA encoding = 'UTF-16le'")
        conn.execute(L.SCHEMA)
        conn.executemany(L.INSERT, [L._row(np.random.default_rng(1))])
    else:
        conn = sqlite3.connect(path)
        sql = {"schema": L.SCHEMA.replace("cost REAL DEFAULT 0.0", "cost REAL DEFAULT 1.0"),
               "without_rowid": L.SCHEMA.replace("AUTOINCREMENT", "") + " WITHOUT ROWID",
               "extra_column": L.SCHEMA[:-1] + ", extra TEXT)", "missing": "CREATE TABLE other (x)",
               "view": "CREATE VIEW tokens_usage AS SELECT 1 AS id, '2026-01-01T00:00:00' AS timestamp"}[kind]
        conn.execute(sql)
    conn.commit()
    conn.close()
    return path, None


@pytest.mark.parametrize("kind", ["wal", "utf16", "schema", "without_rowid", "extra_column", "missing", "view"])
def test_not_modelled_leaves_table(tmp_path, dbs, kind):
    t = HostLoadTable()
    t.load_tokens_usage_db(dbs["pages1024"])
    before = (t._ids.copy(), {c: a.copy() for c, a in t._host.items()}, list(t._models), t._dev_ptrs, t._seq, t.rejected)
    path, keep = _not_modelled(tmp_path, kind)
    with pytest.raises(UsageDbNotModelled):
        t.load_tokens_usage_db(path)
    if keep is not None:
        keep.close()
    assert np.array_equal(t._ids, before[0]) and all(np.array_equal(t._host[c], before[1][c]) for c in UsageTable.COLS)
    assert t._models == before[2] and t._dev_ptrs is before[3] and t._seq == before[4] and t.rejected == before[5]


class LoadStandIn(AppendStandIn):
    """the append test's numpy stand-in for every device call, loading through the host build"""
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


@pytest.mark.parametrize("name", ["deleted", "values", "pages4096"])
def test_queries_after_load(dbs, tmp_path, name):
    expect = L.sqlite_expect(dbs[name])
    t = LoadStandIn()
    t.insert_usage({"prompt_tokens": 5, "model": "replaced"})       # pending rows are replaced by the load
    t.load_tokens_usage_db(dbs[name])
    ref = L.inserted_table(expect, AppendStandIn)
    ref._ids = t._ids.copy()
    ref._seq = t._seq
    ref._upload()
    for limit, offset in ((25, 0), (7, 3), (-1, 0), (10, len(t) - 4)):
        assert t.get_latest_usage_records(limit, offset) == ref.get_latest_usage_records(limit, offset)
    assert t.full_uploads == 0
    row = {"prompt_tokens": 1, "completion_tokens": 2, "model": "zzz-new", "provider": "p"}
    for tab in (t, ref):
        assert tab.insert_usage(row, datetime(2026, 9, 22)) and tab.insert_usage(dict(row, model=""), datetime(2026, 9, 23))
    assert t.get_latest_usage_records(5) == ref.get_latest_usage_records(5)
    assert t._seq == expect["seq"] + 2 and t._pending_rows[-1][-1] == t._seq
    now = datetime(2026, 9, 21) if name != "values" else datetime(2026, 3, 4, 5, 6, 8)
    for tab in (t, ref):
        tab.cleanup_old_records(100, now=now)
    assert t._ids.tolist() == ref._ids.tolist()
    assert t.get_latest_usage_records(-1) == ref.get_latest_usage_records(-1)
    assert t.full_uploads == 0


def test_seq_without_sequence_row(tmp_path):
    path = str(tmp_path / "noseq.db")
    L.fill(path, 40, 5).close()
    conn = sqlite3.connect(path)
    conn.execute("DELETE FROM tokens_usage WHERE id > 30")
    conn.execute("DELETE FROM sqlite_sequence")
    conn.commit()
    conn.close()
    t = HostLoadTable()
    t.load_tokens_usage_db(path)
    assert t._seq == 30 and t._ids.tolist() == list(range(1, 31))


def test_file_too_large(dbs, monkeypatch):
    from llmapigateway_b200 import usage as U
    monkeypatch.setattr(U, "LOAD_MAX_BYTES", dbs["pages1024"].stat().st_size)
    with pytest.raises(UsageDbNotModelled):
        HostLoadTable().load_tokens_usage_db(dbs["pages1024"])


def test_read_only_file(dbs, tmp_path):
    path = tmp_path / "ro.db"
    path.write_bytes(dbs["pages4096"].read_bytes())
    path.chmod(0o444)
    t = HostLoadTable()
    t.load_tokens_usage_db(path)
    L.assert_loaded(t, L.sqlite_expect(path))
