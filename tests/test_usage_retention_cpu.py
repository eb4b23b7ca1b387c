"""UsageTable.cleanup_old_records on the host path (engine=None) against the unmodified reference method
(tests/golden/retention_cases.json) and the oracle's restatement of it (tests/retention_oracle.py): surviving ids, the record
count, every listing page, the next id, the log lines, bad inputs, rows pending, an empty table.  A numpy stand-in for the
device columns checks the bookkeeping of the device path (_dev_n, the listing's merge of rows not yet uploaded)."""
import json
import logging
import random
from datetime import datetime, timedelta
from pathlib import Path

import numpy as np
import pytest

import retention_oracle as RO
from llmapigateway_b200 import usage as U
from llmapigateway_b200.usage import UsageTable, to_us, _EPOCH
from oracle import rollup_oracle as ro

GOLDEN = json.loads((Path(__file__).resolve().parent / "golden" / "retention_cases.json").read_text())
ROWS = GOLDEN["rows"]
CASES = GOLDEN["cases"]


def _iso(us: int) -> str:
    return (_EPOCH + timedelta(microseconds=int(us))).isoformat()


def _columns(rows):
    ts = np.array([to_us(datetime.fromisoformat(r[0])) for r in rows], np.int64)
    tok = [np.array([r[k] for r in rows], np.int32) for k in range(1, 6)]
    cost = np.array([r[6] for r in rows], np.float64)
    return ts, [r[7] for r in rows], tok, cost


def _load(t, rows):
    ts, models, tok, cost = _columns(rows)
    t.load_columns(ts, models, *tok, cost)
    return t


def _ids(t) -> list[int]:
    return sorted(r["id"] for r in t.get_latest_usage_records(-1, 0))


def _usage(i):
    return {"prompt_tokens": i, "completion_tokens": 2 * i, "total_tokens": 3 * i, "cost": i * 1e-6, "model": "m-%d" % (i % 3)}


@pytest.mark.parametrize("k", range(len(CASES)), ids=lambda k: "%s-%r" % (CASES[k]["now"][-6:], CASES[k]["retention_days"]))
def test_golden_case(k, caplog):
    c = CASES[k]
    now = datetime.fromisoformat(c["now"])
    t = _load(UsageTable(None), ROWS)
    with caplog.at_level(logging.DEBUG):
        assert t.cleanup_old_records(c["retention_days"], now=now) is None
    assert [[r.levelname, r.getMessage()] for r in caplog.records] == c["log"]
    assert _ids(t) == c["survivors"]
    assert t.get_total_records_count() == len(c["survivors"])
    conn = ro.make_db(ROWS)                                             # the oracle, pinned to the same golden
    RO.cleanup_old_records(conn, c["retention_days"], now)
    assert RO.ids(conn) == c["survivors"]
    t.insert_usage({"prompt_tokens": 1}, timestamp=now)
    assert [r["id"] for r in t.get_latest_usage_records(-1, 0) if r["id"] not in set(c["survivors"])] == [c["next_id"]]
    assert RO.insert_usage(conn, now) == c["next_id"]


def _pages(n):
    out = [(25, 0), (25, n // 2), (25, max(0, n - 25)), (-1, 0), (0, 0), (7, max(0, n - 3)), (50, n + 5), (1, max(0, n - 1)), (25, -4)]
    return out + [(p, q) for p in (1, 3, 64) for q in (0, 1, 17, n // 3)]


@pytest.mark.parametrize("k", [i for i, c in enumerate(CASES) if isinstance(c["retention_days"], (int, float)) and c["retention_days"] < 10**6])
def test_every_page_after_cleanup(k):
    c = CASES[k]
    now = datetime.fromisoformat(c["now"])
    t = _load(UsageTable(None), ROWS)
    t.cleanup_old_records(c["retention_days"], now=now)
    conn = ro.make_db(ROWS)
    RO.cleanup_old_records(conn, c["retention_days"], now)
    by_id = {i + 1: r for i, r in enumerate(ROWS)}
    n = len(c["survivors"])
    for limit, offset in _pages(n):
        got = t.get_latest_usage_records(limit, offset)
        assert [r["id"] for r in got] == RO.latest_ids(conn, limit, max(offset, 0)), (limit, offset)
        for r in got:                                                   # each record is still the row it was inserted as
            src = by_id[r["id"]]
            assert [r["timestamp"], r["prompt_tokens"], r["cached_tokens"], r["cost"], r["model"]] == [src[0], src[1], src[5], src[6], src[7]]


def test_next_id_after_further_inserts():
    now = datetime.fromisoformat(CASES[0]["now"])
    t = _load(UsageTable(None), ROWS)
    conn = ro.make_db(ROWS)
    for step in range(4):
        stamps = [now - timedelta(days=300 - 40 * step, microseconds=k) for k in range(5)] + [now + timedelta(seconds=step)]
        for k, s in enumerate(stamps):
            assert t.insert_usage(_usage(k), timestamp=s)
            RO.insert_usage(conn, s)
        t.cleanup_old_records(200 - 30 * step, now=now)                  # deletes the old rows just inserted: the largest ids
        RO.cleanup_old_records(conn, 200 - 30 * step, now)
        assert _ids(t) == RO.ids(conn), step
    t.cleanup_old_records(-60, now=now)                                 # everything (the latest record is < 30 days ahead)
    RO.cleanup_old_records(conn, -60, now)
    assert len(t) == 0 and RO.ids(conn) == [] and t.get_latest_usage_records() == []
    t.insert_usage(_usage(1), timestamp=now)
    assert _ids(t) == [RO.insert_usage(conn, now)] == [len(ROWS) + 4 * 6 + 1]


@pytest.mark.parametrize("bad", ["x", None, 10**9, -10**9, float("nan"), float("inf"), [], object()])
def test_bad_input_changes_nothing(bad, caplog):
    now = datetime.fromisoformat(CASES[0]["now"])
    t = _load(UsageTable(None), ROWS)
    t.insert_usage(_usage(1), timestamp=now - timedelta(days=1000))    # a pending row a valid cleanup would delete
    before = t.get_latest_usage_records(-1, 0)
    with caplog.at_level(logging.ERROR):
        assert t.cleanup_old_records(bad, now=now) is None
    assert [r.levelname for r in caplog.records] == ["ERROR"]
    assert t.get_latest_usage_records(-1, 0) == before and len(t) == len(ROWS) + 1
    conn = ro.make_db(ROWS)
    assert RO.cleanup_old_records(conn, bad, now) is None and len(RO.ids(conn)) == len(ROWS)


def test_cutoff_overflow_below_datetime_min_changes_nothing():
    t = _load(UsageTable(None), ROWS)
    assert t.cleanup_old_records(10, now=datetime(1, 1, 5)) is None and len(t) == len(ROWS)


def test_pending_rows_then_insert_then_again():
    now = datetime.fromisoformat(CASES[0]["now"])
    rng = random.Random(7)
    t = _load(UsageTable(None), ROWS)
    conn = ro.make_db(ROWS)

    def insert(m):
        for k in range(m):
            s = now - timedelta(days=rng.randrange(0, 400), microseconds=rng.randrange(10**6))
            t.insert_usage(_usage(k), timestamp=s)
            RO.insert_usage(conn, s)

    insert(40)
    t.cleanup_old_records(180, now=now)                                 # pending rows: some deleted
    RO.cleanup_old_records(conn, 180, now)
    assert _ids(t) == RO.ids(conn)
    insert(25)
    t._materialise()                                                    # some rows in the host columns, some pending
    insert(10)
    t.cleanup_old_records(90, now=now)
    RO.cleanup_old_records(conn, 90, now)
    n = len(RO.ids(conn))
    assert t.get_total_records_count() == n
    for limit, offset in _pages(n):
        assert [r["id"] for r in t.get_latest_usage_records(limit, offset)] == RO.latest_ids(conn, limit, max(offset, 0))
    insert(3)
    assert _ids(t) == RO.ids(conn)


def test_empty_table():
    t = UsageTable(None)
    assert t.cleanup_old_records() is None and len(t) == 0
    t.insert_usage(_usage(1), timestamp=datetime(2026, 1, 1))
    t.cleanup_old_records(0, now=datetime(2026, 1, 2))
    assert len(t) == 0 and t.get_latest_usage_records() == []
    t.insert_usage(_usage(2), timestamp=datetime(2026, 1, 3))
    assert _ids(t) == [2]


def test_integer_order_is_the_text_order():
    """ts < cutoff on the integers decides exactly as SQLite's `timestamp < ?` on isoformat() text, whole seconds included"""
    rng = np.random.default_rng(3)
    base = to_us(datetime(2026, 3, 1))
    ts = base + rng.integers(-5 * 10**6, 5 * 10**6, 4000)
    ts[::3] = ts[::3] // 10**6 * 10**6
    ts[1::3] = ts[1::3] // 10**6 * 10**6 + rng.choice([-1, 1], ts[1::3].size)
    text = [_iso(x) for x in ts]
    for cut in list(ts[:300]) + [base, base + 1, base - 1]:
        c = _iso(cut)
        assert [x < c for x in text] == (ts < cut).tolist()


class DeviceStandIn(UsageTable):
    """the device path with numpy in place of the device: columns 'uploaded' as copies, the listing's page selection by a
    stable argsort, lgw_usage_retain by a boolean mask"""

    def __init__(self):
        super().__init__(engine=object())
        self.uploads = self.retains = 0

    def _upload(self):
        if self._dev is not None:
            return
        self._materialise()
        self._dev_ptrs = {c: self._host[c].copy() for c in self.COLS}
        self._dev = (self._host["ts_us"].size, self._dev_ptrs)
        self._dev_n = int(self._host["ts_us"].size)
        self.uploads += 1

    def _latest_on_device(self, n, first, count):
        assert n == self._dev_n == self._dev_ptrs["ts_us"].size
        return np.argsort(~self._dev_ptrs["ts_us"], kind="stable")[first:first + count].astype(np.uint64)

    def _retain_on_device(self, n, cutoff, n_keep):
        assert n == self._dev_ptrs["ts_us"].size
        keep = self._dev_ptrs["ts_us"] >= cutoff
        assert int(keep.sum()) == n_keep < n
        self.retains += 1
        return {c: a[keep] for c, a in self._dev_ptrs.items()}

    def _free_ptrs(self, ptrs):
        pass


@pytest.mark.parametrize("n_pending", [0, 1, 100, U.LISTING_PENDING_MAX // 64])
def test_device_bookkeeping(n_pending, monkeypatch):
    """with nothing pending the cleanup and the following listing never materialise or upload; with rows pending the listing
    merges them as before; nothing uploaded deleted: no device call"""
    monkeypatch.setattr(U, "LISTING_PENDING_MAX", 200)
    now = datetime.fromisoformat(CASES[0]["now"])
    rng = random.Random(n_pending)
    dev, host = _load(DeviceStandIn(), ROWS), _load(UsageTable(None), ROWS)
    conn = ro.make_db(ROWS)
    dev.get_latest_usage_records(25, 0)
    assert dev.uploads == 1
    for k in range(n_pending):
        s = now - timedelta(days=rng.randrange(0, 400), microseconds=rng.randrange(10**6))
        for t in (dev, host):
            t.insert_usage(_usage(k), timestamp=s)
        RO.insert_usage(conn, s)
    dev.cleanup_old_records(1000, now=now)                             # nothing old enough
    assert dev.retains == 0
    if n_pending == 0:
        monkeypatch.setattr(DeviceStandIn, "_materialise", lambda self: pytest.fail("materialised"))
    for t in (dev, host):
        t.cleanup_old_records(180, now=now)
    RO.cleanup_old_records(conn, 180, now)
    assert dev.retains == 1 and dev.uploads == 1
    assert dev._dev_n == dev._dev_ptrs["ts_us"].size == int((_columns(ROWS)[0] >= to_us(now - timedelta(days=180))).sum())
    n = len(RO.ids(conn))
    for limit, offset in _pages(n):
        want = RO.latest_ids(conn, limit, max(offset, 0))
        assert [r["id"] for r in dev.get_latest_usage_records(limit, offset)] == want, (limit, offset)
        assert [r["id"] for r in host.get_latest_usage_records(limit, offset)] == want, (limit, offset)
    assert dev.uploads == 1 + (n_pending > 200)
    if n_pending == 0:
        assert dev._dev is not None and all(np.array_equal(dev._dev_ptrs[c], dev._host[c]) for c in dev.COLS)
