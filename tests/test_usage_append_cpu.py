"""UsageTable brings its device copy up to date by appending (_upload -> _append_on_device), with a numpy stand-in for the
device columns.  Inserts (new model names sorting first, between and last, NULL models, tables with a fixed dictionary)
interleave with rollup uploads, listings on both sides of LISTING_PENDING_MAX and cleanups.  After every step: the host
columns, ids, models and providers equal a host-only table's; the stand-in's device columns equal the host columns byte for
byte; the model ranks order like a full re-rank; the append seam ran exactly when rows were new; nothing was uploaded whole
after the first upload."""
import random
from datetime import datetime, timedelta

import numpy as np
import pytest

from llmapigateway_b200 import usage as U
from llmapigateway_b200.usage import UsageTable, to_us

NOW = datetime(2026, 9, 21, 6, 57, 17, 47518)
SENTINEL = {np.dtype(np.int64): -0x5A5A5A5A5A5A5A5A, np.dtype(np.int32): -0x5A5A5A5A, np.dtype(np.float64): -1.5e300}


def _key(s):
    return s.encode("utf-8")


class AppendStandIn(UsageTable):
    """the device path with numpy arrays of _dev_cap records as the device columns: the whole upload and lgw_usage_append by
    slicing (a growth into fresh arrays filled with a sentinel), the page selection by a stable argsort, lgw_usage_retain by
    a mask"""

    def __init__(self):
        super().__init__(engine=object())
        self.full_uploads = self.appends = self.retains = 0
        self.full_ranks = 0

    def _rank_all(self):
        self.full_ranks += 1
        super()._rank_all()

    def _upload_all(self):
        self._free_device()
        self._materialise()
        n = int(self._host["ts_us"].size)
        self._dev_ptrs = {c: self._host[c].copy() for c in self.COLS}
        self._dev = (n, self._dev_ptrs)
        self._dev_n = self._dev_cap = n
        self.full_uploads += 1

    def _append_on_device(self, n, m, rank_map, cap):
        self.appends += 1
        old = self._dev_ptrs
        assert all(a.size == self._dev_cap for a in old.values()) and n == self._dev_n
        if cap is None:
            assert n + m <= self._dev_cap
            dst = dict(old)
        else:
            assert n + m <= cap <= U.APPEND_MAX and cap >= min(2 * self._dev_cap, U.APPEND_MAX)
            dst = {c: np.full(cap, SENTINEL[np.dtype(d)], d) for c, d in zip(self.COLS, self.DTYPES)}
            for c in self.COLS:
                dst[c][:n] = old[c][:n]
        if rank_map is not None:
            mr = dst["model_rank"]
            assert rank_map.dtype == np.int32 and rank_map.size > 0 and np.all((mr[:n] >= 0) & (mr[:n] < rank_map.size))
            mr[:n] = rank_map[mr[:n]]
        for c in self.COLS:
            dst[c][n:n + m] = self._host[c][n:n + m]
        return dst

    def _latest_on_device(self, n, first, count):
        assert n == self._dev_n
        return np.argsort(~self._dev_ptrs["ts_us"][:n], kind="stable")[first:first + count].astype(np.uint64)

    def _retain_on_device(self, n, cutoff, n_keep):
        keep = self._dev_ptrs["ts_us"][:n] >= cutoff
        assert int(keep.sum()) == n_keep < n
        self.retains += 1
        return {c: a[:n][keep] for c, a in self._dev_ptrs.items()}

    def _free_ptrs(self, ptrs):
        pass


def _check(dev, host):
    dev._materialise()
    host._materialise()
    for c in dev.COLS:
        if c != "model_rank":
            assert dev._host[c].tobytes() == host._host[c].tobytes(), c
    assert np.array_equal(dev._ids, host._ids) and dev._models == host._models and dev._providers == host._providers
    for t in (dev, host):                                               # ranks order like a full re-rank
        names, mr = t._names, t._host["model_rank"]
        assert names[0] is None and all(_key(a) < _key(b) for a, b in zip(names[1:], names[2:]))
        assert [names[r] for r in mr.tolist()] == t._models
        assert t._rank == {m: i for i, m in enumerate(names)}
    for c in dev.COLS:
        assert dev._host[c].size == len(dev)


def _check_device(dev):
    """the device columns equal the host columns byte for byte while the device copy is current"""
    assert dev._dev is not None and dev._dev_n == len(dev) and not dev._pending_rows
    for c in dev.COLS:
        assert dev._dev_ptrs[c].size == dev._dev_cap >= dev._dev_n
        assert dev._dev_ptrs[c][:dev._dev_n].tobytes() == dev._host[c].tobytes(), c


def _upload(dev):
    """what a rollup does first: the append runs exactly when there are records the device lacks"""
    before, behind = dev.appends, dev._dev_n is not None and len(dev) > dev._dev_n
    dev._upload()
    assert dev.appends - before == int(behind)
    _check_device(dev)


def _geometry_fresh(dev):
    f = UsageTable(None)
    h = dev._host
    f.load_columns(h["ts_us"], dev._models, *[h[c] for c in dev.COLS[2:7]], h["cost"])
    for p in ("hour", "day"):
        for s, e in ((None, None), U.stats_window(p, NOW)):
            assert dev.geometry(p, s, e)[:2] == f.geometry(p, s, e)[:2], p


class Script:
    """one seeded run of inserts and queries on a stand-in table and a host-only table"""

    def __init__(self, seed, pending_max, monkeypatch):
        monkeypatch.setattr(U, "LISTING_PENDING_MAX", pending_max)
        self.rng = random.Random(seed)
        self.dev, self.host = AppendStandIn(), UsageTable(None)
        self.k = 0

    def insert(self, m, names):
        for _ in range(m):
            self.k += 1
            ts = NOW - timedelta(days=self.rng.randrange(0, 400), microseconds=self.rng.randrange(10**6))
            u = {"prompt_tokens": self.k, "completion_tokens": 2 * self.k, "total_tokens": self.rng.randrange(2**31),
                 "reasoning_tokens": self.k % 5, "cached_tokens": self.k % 3, "cost": None if self.k % 13 == 0 else self.k * 1e-6,
                 "model": self.rng.choice(names), "provider": self.rng.choice([None, "P", "Q"])}
            for t in (self.dev, self.host):
                assert t.insert_usage(u, timestamp=ts)

    def listing(self, limit, offset):
        assert self.dev.get_latest_usage_records(limit, offset) == self.host.get_latest_usage_records(limit, offset), (limit, offset)

    def cleanup(self, days):
        for t in (self.dev, self.host):
            t.cleanup_old_records(days, now=NOW)


NAMES_MID = ["m-%02d" % i for i in range(0, 40, 4)]


def test_interleaved_inserts_queries_and_cleanups(monkeypatch):
    s = Script(1, 40, monkeypatch)
    dev = s.dev
    s.insert(500, NAMES_MID + [None])
    _upload(dev)
    assert dev.full_uploads == 1 and dev.full_ranks == 1
    steps = [
        (3, NAMES_MID),                     # known names: no shift
        (1, ["a-first"]),                   # sorts before every name: every rank moves
        (5, ["m-05", "m-17", None]),        # between
        (2, ["z-last", "zz-last"]),         # after every name: no old rank moves
        (45, NAMES_MID + ["é-accent", "M-upper", "m-"]),  # past the listing's merge limit
        (1, [None]),
        (300, ["%c-%d" % (c, i) for c in "abyz" for i in range(30)]),       # many names at once
    ]
    for i, (m, names) in enumerate(steps):
        s.insert(m, names)
        s.listing(25, 0)                                                 # merges on the host up to the limit, else appends
        s.listing(7, len(dev) - 3)
        assert bool(dev._pending_rows) == (m <= U.LISTING_PENDING_MAX)
        _check(dev, s.host)
        _upload(dev)
        _check(dev, s.host)
        _geometry_fresh(dev)
        if i % 3 == 2:
            s.cleanup(300 - 40 * i)
            _check(dev, s.host)
            s.listing(-1, 0)
    assert dev.full_uploads == 1 and dev.full_ranks == 1 and dev.retains > 0


@pytest.mark.parametrize("seed", range(6))
def test_random_scripts(seed, monkeypatch):
    s = Script(100 + seed, 30, monkeypatch)
    dev, rng = s.dev, s.rng
    pool = ["m-%03d" % i for i in range(0, 1000, 50)]
    s.insert(rng.randrange(0, 80), pool[:5] + [None])
    for _ in range(40):
        op = rng.randrange(6)
        if op <= 1:
            fresh = ["%s-%d" % (rng.choice(["", "a", "m-05", "m-999", "zz", "é"]), rng.randrange(10**6)) for _ in range(rng.randrange(0, 3))]
            s.insert(rng.choice([1, 2, 7, 29, 31, 64, 200]), pool[:rng.randrange(1, len(pool))] + fresh + [None])
        elif op == 2:
            _upload(dev)
        elif op == 3:
            s.listing(rng.choice([1, 25, 100]), rng.randrange(0, len(dev) + 2))
        elif op == 4:
            s.cleanup(rng.choice([380, 300, 200, 60]))
        else:
            dev._materialise()                                           # rows moved to the host columns before the upload
        _check(dev, s.host)
    _upload(dev)
    _check(dev, s.host)
    _geometry_fresh(dev)
    assert dev.full_uploads <= 1 and dev.full_ranks <= 1


def test_growth_doubles_and_in_place_keeps_the_buffers(monkeypatch):
    s = Script(3, 10, monkeypatch)
    dev = s.dev
    s.insert(2000, NAMES_MID)
    _upload(dev)
    assert dev._dev_cap == 2000
    s.insert(1, NAMES_MID)
    _upload(dev)
    assert dev._dev_cap == 4000
    ptrs = dev._dev_ptrs
    hbuf = {c: dev._hbuf[c] for c in dev.COLS}
    for m in (1, 17, 1981):                                              # up to the capacity exactly
        s.insert(m, NAMES_MID)
        _upload(dev)
        assert dev._dev_cap == 4000 and dev._dev_ptrs is not ptrs and all(dev._dev_ptrs[c] is ptrs[c] for c in dev.COLS)
        assert all(dev._host[c].base is hbuf[c] for c in dev.COLS)      # the host columns grew in place too
        assert dev._ts_range[0] is dev._host["ts_us"]                    # and kept their bounds without a pass
        ptrs = dev._dev_ptrs
    assert len(dev) == 4000
    s.insert(1, NAMES_MID)                                               # one more: grows
    _upload(dev)
    assert dev._dev_cap == 8000 and all(dev._dev_ptrs[c] is not ptrs[c] for c in dev.COLS)
    _check(dev, s.host)
    assert dev.full_uploads == 1 and dev.full_ranks == 1


def test_growth_from_empty_and_after_a_cleanup(monkeypatch):
    s = Script(4, 10, monkeypatch)
    dev = s.dev
    _upload(dev)                                                         # an empty table on the device
    assert dev.full_uploads == 1 and dev._dev_cap == 0
    s.insert(3, ["b", None])
    _upload(dev)
    assert dev._dev_cap == 1024 and dev.appends == 1
    s.insert(3000, ["a", "c"])
    _upload(dev)
    assert dev._dev_cap == 3003
    s.cleanup(200)                                                       # compacted: the capacity is the survivors
    assert dev._dev_cap == dev._dev_n == len(dev) < 3003
    s.insert(1, ["0-first"])
    _upload(dev)
    assert dev._dev_cap == 2 * (len(dev) - 1)
    _check(dev, s.host)
    s.cleanup(-1)                                                        # everything
    assert dev._dev_cap == 0 == len(dev)
    s.insert(2, ["zz"])
    _upload(dev)
    _check(dev, s.host)
    assert dev.full_uploads == 1 and dev.full_ranks == 1


def test_rank_map_composes_over_materialisations(monkeypatch):
    """several shifts between two uploads reach the device as one map"""
    s = Script(5, 10**6, monkeypatch)
    dev = s.dev
    s.insert(50, ["m", "p", None])
    _upload(dev)
    for first in ("l", "k", "j", "n"):
        s.insert(2, [first])
        dev._materialise()
    assert dev._dev_rank_map is not None and dev._dev_rank_map.size == 3
    _upload(dev)
    assert dev._dev_rank_map is None
    s.insert(1, ["zzz"])                                                 # after every name: no map
    dev._materialise()
    assert dev._dev_rank_map is None
    _check(dev, s.host)


def test_fixed_dictionary_keeps_its_ranks(monkeypatch):
    monkeypatch.setattr(U, "LISTING_PENDING_MAX", 5)
    names = ["b", "a", "c", "é"]
    rng = np.random.default_rng(9)
    n = 400
    ts = to_us(NOW) - rng.integers(0, 400 * 86400 * 10**6, n)
    models = np.array(names + [None], dtype=object)[rng.integers(0, 5, n)]
    tok = [rng.integers(0, 100, n, dtype=np.int32) for _ in range(5)]
    cost = rng.random(n)
    dev, host = AppendStandIn(), UsageTable(None)
    for t in (dev, host):
        t.load_columns(ts, models, *tok, cost, names=names)
    _upload(dev)
    want = [None, "a", "b", "c", "é"]
    for k in range(20):
        for t in (dev, host):
            t.insert_usage({"prompt_tokens": k, "model": names[k % 4] if k % 5 else None}, timestamp=NOW - timedelta(hours=k))
        if k % 7 == 0:
            _upload(dev)
        assert dev._names == want
    _upload(dev)
    _check(dev, host)
    assert dev._names == want and dev.full_uploads == 1 and dev.full_ranks == 1


def test_a_failed_append_frees_the_device_copy(monkeypatch):
    s = Script(6, 10, monkeypatch)
    dev = s.dev
    s.insert(100, NAMES_MID)
    _upload(dev)
    s.insert(20, ["a-shift"])

    def fail(*a):
        raise RuntimeError("usage_append: failed")
    monkeypatch.setattr(dev, "_append_on_device", fail)
    with pytest.raises(RuntimeError):
        dev._upload()
    assert dev._dev is None and dev._dev_n is None and dev._dev_ptrs is None and dev._dev_rank_map is None
    monkeypatch.undo()
    dev._upload()                                                        # the whole table again, ranks as the host has them
    assert dev.full_uploads == 2
    _check_device(dev)
    _check(dev, s.host)


def test_load_columns_starts_over():
    dev = AppendStandIn()
    dev.insert_usage({"model": "x"}, timestamp=NOW)
    _upload(dev)
    ts = np.array([3, 1, 2], np.int64) * 10**6
    dev.load_columns(ts, ["b", None, "a"], *[np.arange(3, dtype=np.int32)] * 5, np.zeros(3))
    assert dev._dev_n is None and dev._rank is None
    dev._upload()
    assert dev.full_uploads == 2 and dev.full_ranks == 2 and dev._names == [None, "a", "b"]
    _check_device(dev)
