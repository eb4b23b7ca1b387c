"""The record listing's merge of rows inserted since the last upload (UsageTable._latest_records_device), with a numpy stand-in
for the device selection: pages at the edges of the merge must equal the host path's."""
from datetime import datetime, timedelta

import numpy as np
import pytest

from llmapigateway_b200 import usage as U


class HostListingTable(U.UsageTable):
    """the device path of the listing, with the upload and the page selection done by numpy"""

    def __init__(self):
        super().__init__(engine=object())
        self.uploads = 0

    def _upload(self):
        if self._dev is not None:
            return
        self._materialise()
        self._dev_ts = self._host["ts_us"].copy()
        self._dev = (self._dev_ts.size, {})
        self._dev_n = int(self._dev_ts.size)
        self.uploads += 1

    def _latest_on_device(self, n, first, count):
        assert n == self._dev_n and 0 <= first and first + count <= n and count > 0
        return np.argsort(~self._dev_ts[:n], kind="stable")[first:first + count].astype(np.uint64)


def _usage(i):
    return {"prompt_tokens": i, "completion_tokens": 2 * i, "total_tokens": 3 * i, "reasoning_tokens": i % 5, "cached_tokens": i % 3,
            "cost": None if i % 13 == 0 else i * 1e-6, "model": None if i % 17 == 0 else "m-%d" % (i % 4), "provider": "P%d" % (i % 3)}


def _fill(tables, stamps, start):
    for k, ts in enumerate(stamps):
        for t in tables:
            t.insert_usage(_usage(start + k), timestamp=ts)


def _pages(n):
    out = [(25, 0), (25, 25), (-1, 0), (0, 0), (7, n - 3), (50, n + 5), (n + 10, 0), (25, -4), (1, n - 1)]
    for p in (1, 2, 5, 37, 100):
        out += [(p, 0), (3, p - 1), (3, p), (3, p + 1), (p + 3, 0), (11, max(0, p - 5)), (p, n - p)]
    return out


@pytest.mark.parametrize("n_pending", [1, 2, 5, 37, 100])
def test_pending_rows_merge_at_page_edges(n_pending):
    base = datetime(2026, 9, 20, 12, 0, 0)
    uploaded = [base + timedelta(seconds=(i * 7919) % 300, microseconds=(i * 104729) % 1000000 if i % 7 else 0) for i in range(400)]
    dev, host = HostListingTable(), U.UsageTable(engine=None)
    _fill((dev, host), uploaded, 0)
    assert dev.get_latest_usage_records(25, 0) == host.get_latest_usage_records(25, 0) and dev.uploads == 1
    # new rows between, equal to, newer than and older than uploaded ones
    rng = np.random.default_rng(n_pending)
    fresh = [uploaded[int(rng.integers(0, 400))] if k % 3 == 0 else base + timedelta(seconds=int(rng.integers(-20, 320)), microseconds=int(rng.integers(0, 10**6)))
             for k in range(n_pending)]
    _fill((dev, host), fresh, 400)
    n = 400 + n_pending
    for limit, offset in _pages(n):
        assert dev.get_latest_usage_records(limit, offset) == host.get_latest_usage_records(limit, offset), (limit, offset)
    assert dev.uploads == 1 and dev._pending_rows                      # merged on the host: no upload, nothing materialised


def test_pending_rows_beyond_the_limit_upload_again(monkeypatch):
    monkeypatch.setattr(U, "LISTING_PENDING_MAX", 8)
    base = datetime(2026, 9, 20, 12, 0, 0)
    dev, host = HostListingTable(), U.UsageTable(engine=None)
    _fill((dev, host), [base + timedelta(seconds=i % 50) for i in range(100)], 0)
    dev.get_latest_usage_records(10, 0)
    _fill((dev, host), [base + timedelta(seconds=(3 * i) % 50) for i in range(8)], 100)
    assert dev.get_latest_usage_records(-1, 0) == host.get_latest_usage_records(-1, 0) and dev.uploads == 1
    _fill((dev, host), [base + timedelta(seconds=7)], 108)
    assert dev.get_latest_usage_records(-1, 0) == host.get_latest_usage_records(-1, 0) and dev.uploads == 2
    assert dev.get_latest_usage_records(30, 80) == host.get_latest_usage_records(30, 80) and dev.uploads == 2


def test_empty_and_loaded_tables():
    dev = HostListingTable()
    assert dev.get_latest_usage_records() == [] and dev.uploads == 0
    ts = np.array([5, 3, 5, -7, 9], np.int64) * 10**6
    dev.load_columns(ts, ["a", None, "b", "c", "a"], *[np.arange(5, dtype=np.int32)] * 5, np.array([0.5, np.nan, 1, 2, 3.0]))
    got = dev.get_latest_usage_records(-1, 0)
    assert [r["id"] for r in got] == [5, 1, 3, 2, 4] and got[4]["timestamp"] == "1969-12-31T23:59:53" and got[3]["cost"] is None
    dev.insert_usage({"model": "z"}, timestamp=datetime(1970, 1, 1, 0, 0, 5))
    assert [r["id"] for r in dev.get_latest_usage_records(-1, 0)] == [5, 1, 3, 6, 2, 4] and dev.uploads == 1
