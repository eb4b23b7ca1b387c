"""GPU: UsageTable.cleanup_old_records on device-resident columns (csrc/retain.cuh, lgw_usage_retain).  Every case runs on a
device table and on an identical UsageTable(None), whose host path is the reference: the eight device columns equal the
compacted host columns byte for byte; the rollup's rows equal those of a fresh device table loaded with the survivors, bit for
bit, and SQLite's after the oracle's DELETE; listing pages equal numpy's stable argsort over the survivors, mapped to the
preserved ids, and the host table's pages; the launch counter shows exactly the retain kernels, and with nothing pending
neither the cleanup nor the rollup and listing after it materialise or upload a column again."""
import ctypes as C
from datetime import datetime, timedelta

import numpy as np
import pytest

import retention_oracle as RO
from llmapigateway_b200 import usage as U
from llmapigateway_b200.usage import UsageTable, synth_usage_columns, to_us, stats_window, _EPOCH

pytestmark = pytest.mark.gpu
NOW = datetime(2026, 9, 21, 6, 57, 17, 47518)
DAY = 86400 * 10**6
TILE = 2048                     # csrc/listing.cuh LGW_LIST_CTILE: the compaction tile
RETAIN_LAUNCHES = 3             # k_retain_count, k_list_scan, k_retain_write
PERIODS = ("hour", "day", "week", "month")
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def _new_engine():
    import llmapigateway_b200 as L
    return L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)


@pytest.fixture(scope="module")
def engine():
    e = _new_engine()
    yield e
    e.close_engine()


def _iso(us: int) -> str:
    return (_EPOCH + timedelta(microseconds=int(us))).isoformat()


def _columns(ts, seed=1, n_models=7):
    n = ts.size
    rng = np.random.default_rng([seed, n])
    tok = [rng.integers(0, 2**17, n, dtype=np.int32) for _ in range(5)]
    cost = rng.integers(0, 10**6, n).astype(np.float64) * 1e-6
    cost[::29] = np.nan
    models = np.array(["m-%d" % (i % n_models) if i % 11 else None for i in range(n)], dtype=object)
    return np.ascontiguousarray(ts, np.int64), models, tok, cost


def _pair(engine, ts, models, tok, cost):
    dev, host = UsageTable(engine), UsageTable(None)
    for t in (dev, host):
        t.load_columns(ts, models, *tok, cost)
    dev._upload()
    return dev, host


class CountingLib:
    """the native library with its lgw_device_upload calls counted"""

    def __init__(self, lib):
        self._lib, self.uploads = lib, 0

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name != "lgw_device_upload":
            return f

        def upload(*a):
            self.uploads += 1
            return f(*a)
        return upload


def _download(t) -> dict:
    n = t._dev_n
    out = {}
    for c, d in zip(t.COLS, t.DTYPES):
        a = np.empty(n, d)
        t.eng._ck(t._lib.lgw_device_download(t.eng._h, a.ctypes.data_as(C.c_void_p), t._dev_ptrs[c], a.nbytes), "device_download")
        out[c] = a
    return out


def _check_columns(dev, host):
    """the device columns equal the compacted host columns byte for byte (model ranks too while the upload is current), and
    the host columns, ids and models equal those of the host-only table"""
    hs = host._host
    got = _download(dev)
    n = dev._dev_n
    cols = dev.COLS if dev._dev is not None else ("ts_us",) + dev.COLS[2:]
    for c in cols:
        assert got[c].tobytes() == dev._host[c][:n].tobytes(), c
    for c in dev.COLS[2:]:
        assert dev._host[c].tobytes() == hs[c].tobytes(), c
    assert np.array_equal(dev._ids, host._ids) and dev._models == host._models


def _listing(dev, host, limit_all=True, dicts=True):
    """pages against numpy's stable argsort over the survivors, mapped to the preserved ids, and against the host table"""
    ts = np.concatenate([host._host["ts_us"], np.array([r[0] for r in host._pending_rows], np.int64)])
    ids = np.concatenate([host._ids, np.array([r[-1] for r in host._pending_rows], np.int64)])
    want = ids[np.argsort(~ts, kind="stable")]
    n = want.size
    pages = [(25, 0), (25, n // 2), (25, max(0, n - 25)), (65536, 0)] + ([(-1, 0)] if limit_all else [])
    for limit, offset in pages:
        got = dev.get_latest_usage_records(limit, offset)
        w = want[offset:offset + (n if limit < 0 else limit)]
        assert [r["id"] for r in got] == w.tolist(), (limit, offset)
        if dicts:
            assert got == host.get_latest_usage_records(limit, offset), (limit, offset)


def _listing_ids(dev, host):
    """the whole listing as ids through the device selection (tables whose timestamps have no text form)"""
    n = dev._dev_n
    assert n == len(dev) == len(host)
    want = host._ids[np.argsort(~host._host["ts_us"], kind="stable")]
    got = dev._ids[dev._latest_on_device(n, 0, n).astype(np.int64)] if n else np.zeros(0, np.int64)
    assert np.array_equal(got, want)


def _fresh(engine, dev):
    """a device table loaded with dev's survivors, ranked against dev's model dictionary"""
    f = UsageTable(engine)
    h = dev._host
    f.load_columns(h["ts_us"], dev._models, *[h[c] for c in dev.COLS[2:7]], h["cost"], names=[m for m in dev._names if m is not None])
    return f


def _rollup_same(engine, dev, periods=PERIODS, windows=True):
    dev._upload()                                                       # (rows pending: into the host columns first)
    f = _fresh(engine, dev)
    try:
        for p in periods:
            for s, e in ([(None, None), stats_window(p, NOW)] if windows else [(None, None)]):
                if len(dev) == 0:
                    assert dev.get_aggregated_usage(p, s, e) == [] == f.get_aggregated_usage(p, s, e)
                    continue
                a, b = dev.rollup_rows(p, s, e), f.rollup_rows(p, s, e)
                assert a.tobytes() == b.tobytes(), (p, s, e)
    finally:
        f.close()


def _cleanup(engine, dev, host, days, now=NOW):
    before = engine.launch_count()
    n_dev = dev._dev_n
    deleted_dev = int(np.count_nonzero(dev._host["ts_us"][:n_dev] < to_us(now - timedelta(days=days)))) if n_dev else 0
    for t in (dev, host):
        assert t.cleanup_old_records(days, now=now) is None
    assert engine.launch_count() - before == (RETAIN_LAUNCHES if deleted_dev else 0)
    if deleted_dev:
        assert dev.retain_last_ms() > 0


def test_c5_10m_at_180_days(engine, monkeypatch):
    """C5's 10 M records at 180 days (about 55 % deleted): no materialise, no upload during the cleanup or the rollup and
    listing after it; columns, rollup and pages as the fresh table and the host path give them"""
    ts, models, tok, cost = synth_usage_columns(10_000_000, end=NOW)
    dev, host = _pair(engine, ts, models, tok, cost)
    try:
        dev.get_aggregated_usage("day")
        lib = CountingLib(dev._lib)
        monkeypatch.setattr(dev, "_lib", lib)
        monkeypatch.setattr(dev, "_materialise", lambda: pytest.fail("materialised"))
        _cleanup(engine, dev, host, 180)
        frac = 1 - len(dev) / ts.size
        assert 0.5 < frac < 0.6 and dev._dev_n == len(dev) == len(host)
        _check_columns(dev, host)
        _listing(dev, host, limit_all=False, dicts=False)
        _listing_ids(dev, host)
        for limit, offset in ((25, 0), (25, len(dev) // 2), (65536, 12345)):
            assert dev.get_latest_usage_records(limit, offset) == host.get_latest_usage_records(limit, offset)
        _rollup_same(engine, dev)
        assert lib.uploads == 0
    finally:
        monkeypatch.undo()
        dev.close()


def test_matches_sqlite_300k(engine):
    """the rollup and the listing after the cleanup against SQLite after the oracle's DELETE, with the golden's timestamp
    shapes: whole seconds next to neighbours 1 us away, records at the cutoff, runs of equal timestamps across it"""
    from oracle import rollup_oracle as ro
    from test_rollup_gpu import _ulps
    n = 300_000
    ts, models, tok, cost = synth_usage_columns(n, seed=8, end=NOW)
    cut = to_us(NOW - timedelta(days=180))
    ts[::9] = ts[::9] // 10**6 * 10**6
    ts[1::101] = ts[1::101] // 10**6 * 10**6 + 1
    ts[2::103] = ts[2::103] // 10**6 * 10**6 - 1
    ts[3::997] = cut
    ts[4::991] = cut - 1
    ts[5::13] = ts[7::13][:ts[5::13].size]
    cost[::23] = np.nan
    dev, host = _pair(engine, ts, models, tok, cost)
    conn = ro.make_db([(_iso(ts[i]), int(tok[0][i]), int(tok[1][i]), int(tok[2][i]), int(tok[3][i]), int(tok[4][i]),
                        float(cost[i]), models[i], None) for i in range(n)])
    try:
        _cleanup(engine, dev, host, 180)
        assert RO.cleanup_old_records(conn, 180, NOW) == n - len(dev)
        assert np.array_equal(dev._ids, np.array(RO.ids(conn)))
        for p in PERIODS:
            for s, e in ((None, None), stats_window(p, NOW)):
                got, want = dev.get_aggregated_usage(p, s, e), ro.aggregated_usage(conn, p, s, e)
                assert len(got) == len(want)
                for g, w in zip(got, want):
                    assert {k: v for k, v in g.items() if k != "cost"} == {k: v for k, v in w.items() if k != "cost"}
                    assert (g["cost"] is None) == (w["cost"] is None) and (g["cost"] is None or _ulps(g["cost"], w["cost"]) <= 4), (g, w)
        for limit, offset in ((25, 0), (25, len(dev) // 2), (25, len(dev) - 25), (65536, 0)):
            assert [r["id"] for r in dev.get_latest_usage_records(limit, offset)] == RO.latest_ids(conn, limit, offset)
        _check_columns(dev, host)
    finally:
        dev.close()


def test_nothing_then_everything(engine):
    ts, models, tok, cost = _columns(to_us(NOW) - np.random.default_rng(2).integers(0, 100 * DAY, 5000))
    dev, host = _pair(engine, ts, models, tok, cost)
    try:
        ptrs = {c: p.value for c, p in dev._dev_ptrs.items()}
        _cleanup(engine, dev, host, 180)                                # nothing that old: no launch, pointers unchanged
        assert {c: p.value for c, p in dev._dev_ptrs.items()} == ptrs and len(dev) == 5000 and dev._dev is not None
        _cleanup(engine, dev, host, -1)                                 # everything
        assert len(dev) == dev._dev_n == 0 and dev.get_total_records_count() == 0
        _check_columns(dev, host)
        assert dev.get_latest_usage_records() == [] and all(dev.get_aggregated_usage(p) == [] for p in PERIODS)
        dev.insert_usage({"prompt_tokens": 1}, timestamp=NOW)
        assert [r["id"] for r in dev.get_latest_usage_records()] == [5001]
        assert dev.get_aggregated_usage("day")[0]["count"] == 1
    finally:
        dev.close()


def test_cutoff_at_a_record_and_inside_ties(engine):
    rng = np.random.default_rng(4)
    ts = to_us(NOW) - rng.integers(0, 400 * DAY, 50_000)
    ts[1000:1400] = ts[77]                                              # a run of 401 equal timestamps
    ts[rng.integers(0, ts.size, 300)] = ts[77]
    for at in (int(ts[123]), int(ts[77])):
        now = _EPOCH + timedelta(microseconds=at) + timedelta(days=30)  # cutoff == that record's timestamp: it stays
        dev, host = _pair(engine, *_columns(ts))
        try:
            _cleanup(engine, dev, host, 30, now=now)
            assert int(dev._host["ts_us"].min()) == at and np.count_nonzero(dev._host["ts_us"] == at) == np.count_nonzero(ts == at)
            _check_columns(dev, host)
            _listing(dev, host)
            _rollup_same(engine, dev, periods=("day", "hour"))
        finally:
            dev.close()


def test_extreme_keys(engine):
    rng = np.random.default_rng(6)
    ts = to_us(NOW) - rng.integers(0, 400 * DAY, 20_000)
    ts[::7] = I64_MIN
    ts[3::11] = I64_MAX
    ts[-1] = I64_MIN
    ts[0] = I64_MAX
    dev, host = _pair(engine, *_columns(ts))
    try:
        for cutoff in (I64_MIN + 1, to_us(NOW - timedelta(days=180)), I64_MAX):
            before = engine.launch_count()
            for t in (dev, host):
                assert t._retain(cutoff) > 0
            assert engine.launch_count() - before == RETAIN_LAUNCHES
            _check_columns(dev, host)
            _listing_ids(dev, host)
        assert np.all(dev._host["ts_us"] == I64_MAX) and len(dev) == np.count_nonzero(ts == I64_MAX)
    finally:
        dev.close()


def _shape(n, pattern):
    i = np.arange(n)
    if pattern == "alternate":
        keep = i % 2 == 0
    elif pattern == "alternate_odd":
        keep = i % 2 == 1
    elif pattern == "tile_ends":
        keep = (i % TILE == 0) | (i % TILE == TILE - 1) | (i == n - 1)
    elif pattern == "first_only":
        keep = i == 0
    elif pattern == "last_only":
        keep = i == n - 1
    else:
        keep = np.random.default_rng(n).random(n) < 0.5
    return to_us(NOW) - np.where(keep, np.arange(n) % DAY, 300 * DAY + np.arange(n))


SIZES = list(range(1, 34)) + [TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE + 1, 32 * TILE + 1]


@pytest.mark.parametrize("pattern", ["alternate", "alternate_odd", "tile_ends", "first_only", "last_only", "random"])
def test_small_and_tile_edge_tables(engine, pattern):
    for n in SIZES:
        ts = _shape(n, pattern)
        if np.all(ts >= to_us(NOW - timedelta(days=180))):
            continue
        dev, host = _pair(engine, *_columns(ts))
        try:
            _cleanup(engine, dev, host, 180)
            _check_columns(dev, host)
            _listing(dev, host)
            _rollup_same(engine, dev, periods=("day",), windows=False)
        finally:
            dev.close()


def test_past_2_24_records(engine):
    n = (1 << 24) + (1 << 20) + 3
    rng = np.random.default_rng(24)
    ts = to_us(NOW) - rng.integers(0, 400 * DAY, n)
    tok = [rng.integers(0, 2**17, n, dtype=np.int32) for _ in range(5)]
    cost = rng.integers(0, 10**6, n).astype(np.float64) * 1e-6
    models = np.array(["m-%d" % k for k in range(9)], dtype=object)[rng.integers(0, 9, n)]
    dev, host = _pair(engine, ts, models, tok, cost)
    try:
        _cleanup(engine, dev, host, 180)
        _check_columns(dev, host)
        _listing(dev, host, limit_all=False, dicts=False)
        _listing_ids(dev, host)
        _rollup_same(engine, dev, periods=("month",), windows=False)
    finally:
        dev.close()


@pytest.mark.parametrize("n_pending", [1, 100, U.LISTING_PENDING_MAX - 1, U.LISTING_PENDING_MAX + 1])
def test_pending_rows(engine, n_pending):
    rng = np.random.default_rng(n_pending)
    ts = to_us(NOW) - rng.integers(0, 400 * DAY, 30_000)
    dev, host = _pair(engine, *_columns(ts))
    try:
        dev.get_latest_usage_records(25, 0)
        pend = to_us(NOW) - rng.integers(0, 400 * DAY, n_pending)
        for k, p in enumerate(pend):
            for t in (dev, host):
                t.insert_usage({"prompt_tokens": k, "model": "p-%d" % (k % 3), "provider": "P"}, timestamp=_EPOCH + timedelta(microseconds=int(p)))
        _cleanup(engine, dev, host, 180)
        assert dev._dev_n == np.count_nonzero(ts >= to_us(NOW - timedelta(days=180)))
        assert len(dev._pending_rows) == np.count_nonzero(pend >= to_us(NOW - timedelta(days=180)))
        _check_columns(dev, host)
        _listing(dev, host, limit_all=n_pending < 1000)
        dev.insert_usage({"prompt_tokens": 1}, timestamp=NOW)
        host.insert_usage({"prompt_tokens": 1}, timestamp=NOW)
        _cleanup(engine, dev, host, 90)
        _listing(dev, host, limit_all=False)
        assert dev.get_latest_usage_records(1, 0)[0]["id"] == 30_000 + n_pending + 1
        _rollup_same(engine, dev, periods=("day", "week"))
    finally:
        dev.close()


SEQUENCE = ((40_000, 180), (3_000_000, 200), (5_000, 100), (TILE + 1, 150), (3_000_000, 30), (1, -1))


def test_repeated_cleanups_on_one_engine(engine):
    """one engine's tile scratch grown, then reused with fewer tiles; each result equal to a fresh engine's"""
    for step, (n, days) in enumerate(SEQUENCE):
        ts, models, tok, cost = _columns(to_us(NOW) - np.random.default_rng([step, n]).integers(0, 400 * DAY, n), seed=step)
        dev, host = _pair(engine, ts, models, tok, cost)
        fresh_eng = _new_engine()
        try:
            other = UsageTable(fresh_eng)
            other.load_columns(ts, models, *tok, cost)
            other._upload()
            _cleanup(engine, dev, host, days)
            other.cleanup_old_records(days, now=NOW)
            a, b = _download(dev), _download(other)
            assert all(a[c].tobytes() == b[c].tobytes() for c in dev.COLS), step
            _check_columns(dev, host)
            _listing(dev, host, limit_all=n < 100_000, dicts=n < 100_000)
            other.close()
        finally:
            dev.close()
            fresh_eng.close_engine()


def test_between_rollups_on_a_side_stream(engine):
    import torch
    ts, models, tok, cost = synth_usage_columns(400_000, seed=3, end=NOW)
    dev, host = _pair(engine, ts, models, tok, cost)
    stream = torch.cuda.Stream()
    try:
        engine.set_stream(stream.cuda_stream)
        before = dev.rollup_rows("day")
        for days in (300, 180, 30):
            _cleanup(engine, dev, host, days)
            _rollup_same(engine, dev, periods=("day", "hour"))
            _listing(dev, host, limit_all=False)
        _check_columns(dev, host)
        assert dev.rollup_rows("day")["count"].sum() < before["count"].sum()
    finally:
        engine.set_stream(None)
        dev.close()


def _alloc(engine, nbytes):
    p = C.c_void_p()
    engine._ck(engine._lib.lgw_device_alloc(engine._h, nbytes, C.byref(p)), "device_alloc")
    return p


def test_abi_guards(engine):
    """n_keep one too small: the mismatch error, nothing written past the output, and the engine serves the next valid call;
    LGW_ERR_ARG for n >= 2^32, n_keep > n, null pointers and a timestamp column that is not 16-byte aligned"""
    lib, h = engine._lib, engine._h
    n = 3 * TILE + 5
    ts, models, tok, cost = _columns(_shape(n, "random"))
    dev = UsageTable(engine)
    dev.load_columns(ts, models, *tok, cost)
    dev._upload()
    cutoff = to_us(NOW - timedelta(days=180))
    keep = int(np.count_nonzero(ts >= cutoff))
    guard = 4096
    outs = []
    try:
        for d in dev.DTYPES:
            size = np.dtype(d).itemsize
            p = _alloc(engine, keep * size + guard)
            pattern = np.full(keep * size + guard, 0xAB, np.uint8)
            engine._ck(lib.lgw_device_upload(h, p, pattern.ctypes.data_as(C.c_void_p), pattern.nbytes), "device_upload")
            outs.append((p, size))
        src = (C.c_void_p * 8)(*[dev._dev_ptrs[c].value for c in dev.COLS])
        dst = (C.c_void_p * 8)(*[p.value for p, _ in outs])
        rc = lib.lgw_usage_retain(h, src, dst, n, cutoff, keep - 1)
        assert rc == -2 and b"expected %d" % (keep - 1) in lib.lgw_last_error(h)
        for p, size in outs:                                            # nothing past the n_keep - 1 records asked for
            tail = np.empty(size + guard, np.uint8)
            engine._ck(lib.lgw_device_download(h, tail.ctypes.data_as(C.c_void_p), C.c_void_p(p.value + (keep - 1) * size), tail.nbytes), "device_download")
            assert np.all(tail == 0xAB)
        engine._ck(lib.lgw_usage_retain(h, src, dst, n, cutoff, keep), "usage_retain")     # the next valid call
        sel = ts >= cutoff
        for (p, size), c in zip(outs, dev.COLS):
            got = np.empty(keep * size + guard, np.uint8)
            engine._ck(lib.lgw_device_download(h, got.ctypes.data_as(C.c_void_p), p, got.nbytes), "device_download")
            want = dev._host[c][sel]
            assert got[:keep * size].tobytes() == want.tobytes() and np.all(got[keep * size:] == 0xAB), c
        null = (C.c_void_p * 8)(*([None] + [p.value for p, _ in outs[1:]]))
        odd = (C.c_void_p * 8)(*([dev._dev_ptrs["ts_us"].value + 8] + [dev._dev_ptrs[c].value for c in dev.COLS[1:]]))
        before = engine.launch_count()
        assert lib.lgw_usage_retain(h, src, dst, 1 << 32, cutoff, keep) == -1
        assert lib.lgw_usage_retain(h, src, dst, n, cutoff, n + 1) == -1
        assert lib.lgw_usage_retain(h, null, dst, n, cutoff, keep) == -1
        assert lib.lgw_usage_retain(h, src, null, n, cutoff, keep) == -1
        assert lib.lgw_usage_retain(h, None, dst, n, cutoff, keep) == -1
        assert lib.lgw_usage_retain(h, odd, dst, n - 1, cutoff, keep) == -1
        assert lib.lgw_usage_retain(h, None, None, 0, cutoff, 0) == 0
        assert engine.launch_count() == before
    finally:
        for p, _ in outs:
            lib.lgw_device_free(h, p)
        dev.close()


def test_failed_device_call_changes_nothing(engine, monkeypatch):
    """a device call that fails leaves host and device as they were, and the cleanup logs it and returns None"""
    ts, models, tok, cost = _columns(_shape(10_000, "random"))
    dev, host = _pair(engine, ts, models, tok, cost)
    try:
        ptrs = {c: p.value for c, p in dev._dev_ptrs.items()}
        real = dev._lib

        class Failing(CountingLib):
            def __getattr__(self, name):
                return (lambda *a: -2) if name == "lgw_usage_retain" else getattr(self._lib, name)
        monkeypatch.setattr(dev, "_lib", Failing(real))
        assert dev.cleanup_old_records(180, now=NOW) is None
        monkeypatch.setattr(dev, "_lib", real)
        assert {c: p.value for c, p in dev._dev_ptrs.items()} == ptrs and len(dev) == 10_000 and dev._dev_n == 10_000
        _check_columns(dev, host)
        _cleanup(engine, dev, host, 180)
        _check_columns(dev, host)
    finally:
        dev.close()
