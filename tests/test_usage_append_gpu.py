"""GPU: rows inserted into a device-resident UsageTable are appended to its columns (csrc/append.cuh, lgw_usage_append) instead
of uploading and re-ranking the table again.  Each case checks the eight device columns, downloaded, against the host columns;
rollup_rows bit for bit against a fresh table loaded with the same records and the same model dictionary, for all four periods
with and without the stats window; listing pages against numpy's stable argsort, with the ids preserved.  The launch counter
shows one launch per append, and lgw_device_upload is not called after the first upload."""
import ctypes as C
from datetime import datetime, timedelta

import numpy as np
import pytest

from llmapigateway_b200 import usage as U
from llmapigateway_b200.usage import UsageTable, synth_usage_columns, to_us, stats_window, _EPOCH
from test_usage_retention_gpu import CountingLib, _alloc, _download, _new_engine

pytestmark = pytest.mark.gpu
NOW = datetime(2026, 9, 21, 6, 57, 17, 47518)
DAY = 86400 * 10**6
PERIODS = ("hour", "day", "week", "month")
LPM = U.LISTING_PENDING_MAX


@pytest.fixture(scope="module")
def engine():
    e = _new_engine()
    yield e
    e.close_engine()


def _usage(k, model):
    return {"prompt_tokens": k, "completion_tokens": 2 * k, "total_tokens": 3 * k, "reasoning_tokens": k % 5, "cached_tokens": k % 3,
            "cost": None if k % 29 == 0 else (k % 10**6) * 1e-6, "model": model, "provider": "P"}


def _insert(tables, ts, models, k0=0):
    for k, (s, m) in enumerate(zip(ts.tolist(), models)):
        stamp = _EPOCH + timedelta(microseconds=s)
        for t in tables:
            assert t.insert_usage(_usage(k0 + k, m), timestamp=stamp)


def _upload(engine, dev):
    """bring the device copy up to date, counting the launches: exactly one when the device lacks records"""
    behind = dev._dev_n is not None and len(dev) > dev._dev_n
    before = engine.launch_count()
    dev._upload()
    assert engine.launch_count() - before == int(behind)
    if behind:
        assert dev.append_last_ms() > 0


def _check_columns(engine, dev):
    _upload(engine, dev)
    got = _download(dev)
    assert dev._dev_n == len(dev) <= dev._dev_cap
    for c in dev.COLS:
        assert got[c].tobytes() == dev._host[c].tobytes(), c
    names, mr = dev._names, dev._host["model_rank"]
    assert all(a.encode() < b.encode() for a, b in zip(names[1:], names[2:]))
    assert [names[r] for r in np.unique(mr)] == sorted(set(dev._models), key=lambda s: b"" if s is None else b"\1" + s.encode())


def _fresh(engine, dev):
    f = UsageTable(engine)
    h = dev._host
    f.load_columns(h["ts_us"], dev._models, *[h[c] for c in dev.COLS[2:7]], h["cost"], names=[m for m in dev._names if m is not None])
    return f


def _rollup_same(engine, dev, periods=PERIODS, windows=True):
    _upload(engine, dev)
    f = _fresh(engine, dev)
    try:
        for p in periods:
            for s, e in ([(None, None), stats_window(p, NOW)] if windows else [(None, None)]):
                a, b = dev.rollup_rows(p, s, e), f.rollup_rows(p, s, e)
                assert a.tobytes() == b.tobytes(), (p, s, e)
    finally:
        f.close()


def _listing(dev, ts, ids, pages=None):
    """pages against numpy's stable argsort of every record's timestamp (pending rows included), mapped to the ids"""
    want = ids[np.argsort(~ts, kind="stable")]
    n = want.size
    for limit, offset in pages or ((25, 0), (25, n // 2), (25, max(0, n - 25)), (65536, 0)):
        got = dev.get_latest_usage_records(limit, offset)
        assert [r["id"] for r in got] == want[offset:offset + (n if limit < 0 else limit)].tolist(), (limit, offset)


def _state(t):
    """(ts, ids) of every record of t, host columns and pending rows"""
    ts = np.concatenate([t._host["ts_us"], np.array([r[0] for r in t._pending_rows], np.int64)])
    ids = np.concatenate([t._ids, np.array([r[-1] for r in t._pending_rows], np.int64)])
    return ts, ids


def _names_for(rng, m, pool):
    return [pool[i] for i in rng.integers(0, len(pool), m)]


def test_c5_10m_inserts_without_upload_or_rerank(engine, monkeypatch):
    """C5's 10 M records, then 1, 100, LISTING_PENDING_MAX - 1, LISTING_PENDING_MAX + 1 and 10^6 inserted rows, some with new
    names: no lgw_device_upload and no full re-rank after the first upload"""
    n = 10_000_000
    ts, models, tok, cost = synth_usage_columns(n, end=NOW)
    dev = UsageTable(engine)
    dev.load_columns(ts, models, *tok, cost)
    dev.get_aggregated_usage("day")
    lib = CountingLib(dev._lib)
    monkeypatch.setattr(dev, "_lib", lib)
    monkeypatch.setattr(dev, "_rank_all", lambda: pytest.fail("ranked every record again"))
    all_ts, all_ids = [ts], [np.arange(1, n + 1, dtype=np.int64)]
    rng = np.random.default_rng(10)
    pool = ["provider-%02d/model-%02d" % (i % 7, i) for i in range(64)] + [None, "a-new/first", "provider-03/model-31b", "zz-new/last"]
    try:
        for m in (1, 100, LPM - 1, LPM + 1, 1_000_000):
            new_ts = to_us(NOW) - rng.integers(0, 400 * DAY, m)
            _insert([dev], new_ts, _names_for(rng, m, pool + ["new-%d-%d" % (m, i) for i in range(3)]), k0=len(dev))
            all_ts.append(new_ts)
            all_ids.append(np.arange(len(dev) - m + 1, len(dev) + 1, dtype=np.int64))
            t, i = np.concatenate(all_ts), np.concatenate(all_ids)
            _listing(dev, t, i, ((25, 0), (25, len(dev) // 2), (25, len(dev) - 25)))      # a host merge up to the limit, else an append
            assert bool(dev._pending_rows) == (m <= LPM)
            _check_columns(engine, dev)
            assert np.array_equal(dev._host["ts_us"], t) and np.array_equal(dev._ids, i)
            _rollup_same(engine, dev, periods=PERIODS if m in (1, 1_000_000) else ("day",))
            _listing(dev, t, i)
        assert lib.uploads == 0
    finally:
        monkeypatch.undo()
        dev.close()


def test_matches_sqlite_300k(engine):
    from oracle import rollup_oracle as ro
    from test_rollup_gpu import _ulps
    import retention_oracle as RO
    n, m = 300_000, 20_000
    ts, models, tok, cost = synth_usage_columns(n, seed=8, end=NOW)
    ts = ts // 10**6 * 10**6                                            # whole seconds: inserts tie with loaded records
    dev = UsageTable(engine)
    dev.load_columns(ts, models, *tok, cost)
    dev._upload()
    rows = [(_EPOCH + timedelta(microseconds=int(ts[i]))).isoformat() for i in range(n)]
    rows = [(rows[i], int(tok[0][i]), int(tok[1][i]), int(tok[2][i]), int(tok[3][i]), int(tok[4][i]), float(cost[i]), models[i], None) for i in range(n)]
    rng = np.random.default_rng(11)
    new_ts = np.where(rng.random(m) < 0.5, ts[rng.integers(0, n, m)], (to_us(NOW) - rng.integers(0, 400 * DAY, m)) // 10**6 * 10**6)
    names = _names_for(rng, m, ["provider-01/model-01", "0-first", "provider-02/model-02x", "zz", None])
    try:
        for part in (slice(0, 10), slice(10, 5000), slice(5000, m)):
            _insert([dev], new_ts[part], names[part], k0=part.start)
            for k in range(part.start, part.stop):
                u = _usage(k, names[k])
                rows.append(((_EPOCH + timedelta(microseconds=int(new_ts[k]))).isoformat(), u["prompt_tokens"], u["completion_tokens"],
                             u["total_tokens"], u["reasoning_tokens"], u["cached_tokens"], u["cost"], u["model"], "P"))
            conn = ro.make_db(rows)
            for p in PERIODS:
                for s, e in ((None, None), stats_window(p, NOW)):
                    got, want = dev.get_aggregated_usage(p, s, e), ro.aggregated_usage(conn, p, s, e)
                    assert len(got) == len(want)
                    for g, w in zip(got, want):
                        assert {k: v for k, v in g.items() if k != "cost"} == {k: v for k, v in w.items() if k != "cost"}
                        assert (g["cost"] is None) == (w["cost"] is None) and (g["cost"] is None or _ulps(g["cost"], w["cost"]) <= 4), (g, w)
            for limit, offset in ((25, 0), (25, len(dev) // 2), (25, len(dev) - 25), (65536, 0)):
                assert [r["id"] for r in dev.get_latest_usage_records(limit, offset)] == RO.latest_ids(conn, limit, offset)
            _check_columns(engine, dev)
    finally:
        dev.close()


def _small(engine, n, seed=1, names=("m-10", "m-20", "m-30", None)):
    rng = np.random.default_rng(seed)
    ts = to_us(NOW) - rng.integers(0, 400 * DAY, n)
    tok = [rng.integers(0, 2**17, n, dtype=np.int32) for _ in range(5)]
    cost = rng.integers(0, 10**6, n).astype(np.float64) * 1e-6
    models = np.array(names, dtype=object)[rng.integers(0, len(names), n)]
    dev = UsageTable(engine)
    dev.load_columns(ts, models, *tok, cost)
    dev._upload()
    return dev, rng


def test_fill_the_capacity_exactly_then_one_more(engine):
    dev, rng = _small(engine, 5000)
    try:
        assert dev._dev_cap == 5000
        pool = ["m-10", "m-25", None]
        _insert([dev], to_us(NOW) - rng.integers(0, 400 * DAY, 1), pool[:1])
        _check_columns(engine, dev)                                     # grows by doubling
        assert dev._dev_cap == 10_000
        ptrs = {c: p.value for c, p in dev._dev_ptrs.items()}
        for m in (1, 2998, 1999, 1):                                    # in place, up to exactly the capacity
            _insert([dev], to_us(NOW) - rng.integers(0, 400 * DAY, m), _names_for(rng, m, pool))
            _check_columns(engine, dev)
            assert {c: p.value for c, p in dev._dev_ptrs.items()} == ptrs and dev._dev_cap == 10_000
        assert len(dev) == 10_000
        _rollup_same(engine, dev, periods=("day",))
        _insert([dev], to_us(NOW) - rng.integers(0, 400 * DAY, 1), ["a-first"])          # one more: grows, and every rank moves
        _check_columns(engine, dev)
        assert dev._dev_cap == 20_000 and all(dev._dev_ptrs[c].value != ptrs[c] for c in dev.COLS)
        _rollup_same(engine, dev)
        _listing(dev, *_state(dev), ((25, 0), (25, 5000), (-1, 0)))
    finally:
        dev.close()


def test_growth_after_a_cleanup_and_from_empty(engine):
    dev, rng = _small(engine, 30_000, seed=2)
    try:
        dev.cleanup_old_records(180, now=NOW)
        keep = len(dev)
        assert dev._dev_cap == dev._dev_n == keep
        _insert([dev], to_us(NOW) - rng.integers(0, 100 * DAY, 7), ["m-15"] * 7)
        _check_columns(engine, dev)
        assert dev._dev_cap == 2 * keep
        _rollup_same(engine, dev)
        dev.cleanup_old_records(-1, now=NOW)                            # everything
        assert len(dev) == dev._dev_cap == 0
        _insert([dev], to_us(NOW) - rng.integers(0, 100 * DAY, 3), ["zz", None, "m-10"])
        _check_columns(engine, dev)
        assert dev._dev_cap == 1024
        _rollup_same(engine, dev, periods=("day", "hour"))
        _listing(dev, *_state(dev), ((25, 0), (-1, 0)))
    finally:
        dev.close()
    empty = UsageTable(engine)
    try:
        empty._upload()
        assert empty._dev_n == empty._dev_cap == 0
        _insert([empty], to_us(NOW) - rng.integers(0, 100 * DAY, 2000), _names_for(rng, 2000, ["b", "a", None]))
        _check_columns(engine, empty)
        assert empty._dev_cap == 2000
        _rollup_same(engine, empty)
        _listing(empty, *_state(empty), ((25, 0), (-1, 0)))
    finally:
        empty.close()


def test_a_table_crossing_2_24_records(engine):
    n = (1 << 24) - 100
    dev, rng = _small(engine, n, seed=24, names=tuple("m-%d" % k for k in range(9)) + (None,))
    try:
        _insert([dev], to_us(NOW) - rng.integers(0, 400 * DAY, 300), _names_for(rng, 300, ["m-4", "m-45", "a"]))
        _check_columns(engine, dev)
        assert len(dev) == n + 300 > 1 << 24
        _listing(dev, *_state(dev), ((25, 0), (25, n), (25, len(dev) - 25)))
        got = dev._latest_on_device(len(dev), 0, len(dev)).astype(np.int64)
        ts, ids = _state(dev)
        assert np.array_equal(ids[got], ids[np.argsort(~ts, kind="stable")])
        _rollup_same(engine, dev, periods=("month",), windows=False)
    finally:
        dev.close()


@pytest.mark.parametrize("shape", ["every", "none", "middle", "many"])
def test_new_names_that_shift_ranks(engine, shape):
    dev, rng = _small(engine, 50_000, seed=3)
    new = {"every": ["0-first", "A-upper"], "none": ["zz", "é"], "middle": ["m-15"],
           "many": ["%s-%04d" % (p, i) for p in ("a", "m-2", "m-9", "z") for i in range(500)]}[shape]
    try:
        before = dev._host["model_rank"].copy()
        _insert([dev], to_us(NOW) - rng.integers(0, 400 * DAY, 4000), _names_for(rng, 4000, new + ["m-20", None]))
        dev._materialise()
        moved = np.count_nonzero(dev._host["model_rank"][:50_000] != before)
        assert (moved > 0) == (shape != "none") and (dev._dev_rank_map is None) == (shape == "none")
        _check_columns(engine, dev)
        assert dev._dev_rank_map is None
        _rollup_same(engine, dev)
        _listing(dev, *_state(dev))
    finally:
        dev.close()


def test_alternating_on_one_engine_against_fresh_engines(engine):
    """inserts, rollups on a torch side stream, listings and cleanups on one engine; each result against a table of the same
    records on a fresh engine"""
    import torch
    dev, rng = _small(engine, 200_000, seed=5)
    stream = torch.cuda.Stream()
    pool = ["m-10", "m-05", "m-31", "m-99", None]
    try:
        engine.set_stream(stream.cuda_stream)
        for step, (m, days) in enumerate(((1, None), (70_000, None), (10, 300), (3, None), (100_000, 120), (1, None))):
            _insert([dev], to_us(NOW) - rng.integers(0, 400 * DAY, m), _names_for(rng, m, pool + ["s%d" % step]))
            if days is not None:
                dev.cleanup_old_records(days, now=NOW)
            _listing(dev, *_state(dev), ((25, 0), (25, len(dev) // 3)))
            rows = {p: dev.rollup_rows(p, *stats_window(p, NOW)).tobytes() for p in ("day", "hour")}
            got = _download(dev)
            fresh_eng = _new_engine()
            try:
                other = _fresh(fresh_eng, dev)
                other._upload()
                want = _download(other)
                assert all(got[c].tobytes() == want[c].tobytes() for c in dev.COLS), step
                assert all(other.rollup_rows(p, *stats_window(p, NOW)).tobytes() == rows[p] for p in rows), step
                other.close()
            finally:
                fresh_eng.close_engine()
        _check_columns(engine, dev)
    finally:
        engine.set_stream(None)
        dev.close()


def _dev_cols(engine, cap, guard, fill=0xAB):
    """eight device columns with room for cap records and a guard region past them, filled with one byte"""
    out = []
    for d in UsageTable.DTYPES:
        nbytes = cap * np.dtype(d).itemsize + guard
        p = _alloc(engine, nbytes)
        pattern = np.full(nbytes, fill, np.uint8)
        engine._ck(engine._lib.lgw_device_upload(engine._h, p, pattern.ctypes.data_as(C.c_void_p), nbytes), "device_upload")
        out.append(p)
    return out


def _read(engine, p, nbytes, off=0):
    a = np.empty(nbytes, np.uint8)
    engine._ck(engine._lib.lgw_device_download(engine._h, a.ctypes.data_as(C.c_void_p), C.c_void_p(p.value + off), nbytes), "device_download")
    return a


def _put(engine, p, a):
    engine._ck(engine._lib.lgw_device_upload(engine._h, p, a.ctypes.data_as(C.c_void_p), a.nbytes), "device_upload")


def test_abi_guards(engine):
    """LGW_ERR_ARG for n + m >= 2^32, null pointers the call needs, a ts_us column that is not 16-byte aligned and a map with
    n_map == 0, with nothing launched; a resident rank past the map fails the call and writes nothing past n + m, in place and
    growing; then a valid call is served"""
    lib, h = engine._lib, engine._h
    n, m, guard, n_map = 3000, 500, 4096, 6
    rng = np.random.default_rng(12)
    old = [rng.integers(-9, 9, n).astype(d) for d in UsageTable.DTYPES]
    old[1] = rng.integers(0, n_map, n).astype(np.int32)
    new = [rng.integers(-9, 9, m).astype(d) for d in UsageTable.DTYPES]
    rank_map = np.array([5, 4, 3, 2, 1, 0], np.int32)
    cols, grow = _dev_cols(engine, n + m, guard), _dev_cols(engine, n + m, guard)
    try:
        for p, a in zip(cols, old):
            _put(engine, p, a)
        P8 = C.c_void_p * 8
        d_cols, d_grow = P8(*[p.value for p in cols]), P8(*[p.value for p in grow])
        h_new = P8(*[a.ctypes.data for a in new])
        rm = rank_map.ctypes.data_as(C.c_void_p)
        before = engine.launch_count()
        assert lib.lgw_usage_append(h, d_cols, None, (1 << 32) - 1, h_new, 1, None, 0) == -1
        assert lib.lgw_usage_append(h, d_cols, None, 1 << 32, h_new, 0, None, 0) == -1
        assert lib.lgw_usage_append(h, None, None, n, h_new, m, None, 0) == -1
        assert lib.lgw_usage_append(h, P8(*([cols[0].value] + [None] + [p.value for p in cols[2:]])), None, n, h_new, m, None, 0) == -1
        assert lib.lgw_usage_append(h, d_cols, P8(*([None] + [p.value for p in grow[1:]])), n, h_new, m, None, 0) == -1
        assert lib.lgw_usage_append(h, d_cols, None, n, None, m, None, 0) == -1
        assert lib.lgw_usage_append(h, d_cols, None, n, P8(*([None] + list(h_new)[1:])), m, None, 0) == -1
        assert lib.lgw_usage_append(h, P8(*([cols[0].value + 8] + [p.value for p in cols[1:]])), None, n - 1, h_new, m, None, 0) == -1
        assert lib.lgw_usage_append(h, d_cols, P8(*([grow[0].value + 8] + [p.value for p in grow[1:]])), n, h_new, m, None, 0) == -1
        assert lib.lgw_usage_append(h, d_cols, None, n, h_new, m, rm, 0) == -1
        assert lib.lgw_usage_append(h, d_cols, None, n, h_new, 0, None, 0) == 0           # nothing to do
        assert lib.lgw_usage_append(h, None, None, 0, None, 0, None, 0) == 0
        assert engine.launch_count() == before
        bad = old[1].copy()
        bad[17], bad[n - 1] = n_map, -1                                  # past the map, and negative
        _put(engine, cols[1], bad)
        for target, g in ((cols, None), (grow, d_grow)):
            rc = lib.lgw_usage_append(h, d_cols, g, n, h_new, m, rm, n_map)
            assert rc == -2 and b"2 resident model ranks" in lib.lgw_last_error(h)
            for p, d in zip(target, UsageTable.DTYPES):                 # nothing past n + m
                size = np.dtype(d).itemsize
                assert np.all(_read(engine, p, guard, (n + m) * size) == 0xAB)
        assert engine.launch_count() == before + 2
        _put(engine, cols[1], old[1])
        for target, g in ((grow, d_grow), (cols, None)):                # valid calls: growing, then in place
            engine._ck(lib.lgw_usage_append(h, d_cols, g, n, h_new, m, rm, n_map), "usage_append")
            for k, (p, d) in enumerate(zip(target, UsageTable.DTYPES)):
                size = np.dtype(d).itemsize
                want = np.concatenate([rank_map[old[1]] if k == 1 else old[k], new[k]])
                got = _read(engine, p, (n + m) * size + guard)
                assert got[:(n + m) * size].tobytes() == want.tobytes() and np.all(got[(n + m) * size:] == 0xAB), k
        assert engine.launch_count() == before + 4
    finally:
        for p in cols + grow:
            lib.lgw_device_free(h, p)


def test_a_failed_append_then_a_full_upload(engine, monkeypatch):
    dev, rng = _small(engine, 20_000, seed=7)
    try:
        real = dev._lib

        class Failing(CountingLib):
            def __getattr__(self, name):
                return (lambda *a: -2) if name == "lgw_usage_append" else getattr(self._lib, name)
        monkeypatch.setattr(dev, "_lib", Failing(real))
        _insert([dev], to_us(NOW) - rng.integers(0, 400 * DAY, 10), ["0-first"] * 10)
        with pytest.raises(Exception):
            dev.get_aggregated_usage("day")
        assert dev._dev is None and dev._dev_n is None and dev._dev_ptrs is None and not dev._pending_rows
        lib = CountingLib(real)
        monkeypatch.setattr(dev, "_lib", lib)
        assert dev.get_aggregated_usage("day")
        assert lib.uploads == 8 and dev._dev_cap == dev._dev_n == 20_010
        monkeypatch.setattr(dev, "_lib", real)
        _check_columns(engine, dev)
        _rollup_same(engine, dev)
        _listing(dev, *_state(dev))
    finally:
        monkeypatch.undo()
        dev.close()
