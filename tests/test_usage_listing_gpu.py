"""GPU: the newest-first record listing (/v1/api/usage-records) selected on the device (csrc/listing.cuh) against SQLite running
the reference statement, against numpy's stable argsort at the table size of BASELINE config 5, and against the host path
(UsageTable(engine=None)) on key shapes that stress the radix select and with rows inserted since the last upload."""
from datetime import datetime, timedelta

import numpy as np
import pytest

from llmapigateway_b200 import usage as U
from llmapigateway_b200.usage import UsageTable, synth_usage_columns, to_us, _EPOCH
from oracle import rollup_oracle as ro

pytestmark = pytest.mark.gpu
NOW = datetime(2026, 9, 21, 6, 57, 17, 47518)
CAND_DIV = 16          # csrc/listing.cuh LGW_LIST_CAND_DIV
SMEM_SORT = 8192       # csrc/listing.cuh LGW_LIST_SMEM_SORT


@pytest.fixture(scope="module")
def engine():
    import llmapigateway_b200 as L
    e = L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    yield e
    e.close_engine()


def _iso(us: int) -> str:
    return (_EPOCH + timedelta(microseconds=int(us))).isoformat()


def _tables(engine, ts, models=None, cost=None):
    n = ts.size
    rng = np.random.default_rng(n)
    tok = [rng.integers(0, 2**17, n, dtype=np.int32) for _ in range(5)]
    cost = rng.integers(0, 10**6, n).astype(np.float64) * 1e-6 if cost is None else cost
    models = ["m-%d" % (i % 5) for i in range(n)] if models is None else models
    dev, host = UsageTable(engine), UsageTable(None)
    for t in (dev, host):
        t.load_columns(ts, models, *tok, cost)
    return dev, host, tok, cost, models


def _against_host(dev, host, pages):
    for limit, offset in pages:
        assert dev.get_latest_usage_records(limit, offset) == host.get_latest_usage_records(limit, offset), (limit, offset)


def test_listing_matches_sqlite(engine):
    n = 300_000
    ts, models, tok, cost = synth_usage_columns(n, seed=8, end=NOW)
    ts[::9] = ts[::9] // 10**6 * 10**6                             # microsecond == 0: isoformat() drops the fraction
    ts[5::13] = ts[7::13][:ts[5::13].size]                          # runs of equal timestamps
    ts[1::101] = ts[1::101] // 10**6 * 10**6 + 1                    # ... and their neighbours one microsecond later
    cost[::23] = np.nan
    dev, host = UsageTable(engine), UsageTable(None)
    for t in (dev, host):
        t.load_columns(ts, models, *tok, cost)
    conn = ro.make_db([(_iso(ts[i]), int(tok[0][i]), int(tok[1][i]), int(tok[2][i]), int(tok[3][i]), int(tok[4][i]),
                        float(cost[i]), models[i], None) for i in range(n)])
    cols = None
    for limit, offset in ((25, 0), (25, 25), (25, n - 10), (7, n - 3), (0, 0), (-1, 0), (50, n + 5), (n + 1000, 0), (25, -7), (300, 12_345)):
        got = dev.get_latest_usage_records(limit, offset)
        assert got == host.get_latest_usage_records(limit, offset), (limit, offset)
        cur = conn.execute("SELECT id, timestamp, prompt_tokens, completion_tokens, total_tokens, reasoning_tokens, cached_tokens, cost, model, provider"
                           " FROM tokens_usage ORDER BY timestamp DESC LIMIT ? OFFSET ?", (limit, offset))
        cols = cols or [d[0] for d in cur.description]
        want = [dict(zip(cols, r)) for r in cur.fetchall()]
        assert [g["timestamp"] for g in got] == [w["timestamp"] for w in want], (limit, offset)
        # rows equal up to order inside runs of equal timestamps; a run cut by the page's edge may hold other members in SQLite
        edge = {got[0]["timestamp"], got[-1]["timestamp"]} if got else set()
        key = lambda r: (r["timestamp"], r["id"])
        assert sorted((r for r in got if r["timestamp"] not in edge), key=key) == sorted((r for r in want if r["timestamp"] not in edge), key=key)
    assert dev._pending_rows == [] and dev._dev_n == n


def test_listing_at_size(engine):
    n = 10_000_000
    ts, models, tok, cost = synth_usage_columns(n, seed=5, end=NOW)
    t = UsageTable(engine)
    t.load_columns(ts, models, *tok, cost)
    want = np.argsort(-ts, kind="stable")
    t.get_latest_usage_records(1, 0)                                  # uploads
    for offset in (0, 1, n // 2, n - 25, n - 1):
        got = t._latest_on_device(n, offset, min(25, n - offset))
        assert np.array_equal(got.astype(np.int64), want[offset:offset + 25]), offset
        assert t.listing_last_ms() > 0
    rows = t.get_latest_usage_records(25, n // 2)
    assert [r["id"] - 1 for r in rows] == want[n // 2:n // 2 + 25].tolist()
    assert rows[3]["timestamp"] == _iso(ts[want[n // 2 + 3]]) and rows[3]["model"] == models[want[n // 2 + 3]]
    t.close()
    m = 1_000_000
    ts, models, tok, cost = synth_usage_columns(m, seed=6, end=NOW)
    t = UsageTable(engine)
    t.load_columns(ts, models, *tok, cost)
    listed = t.get_latest_usage_records(-1, 0)
    assert [r["id"] - 1 for r in listed] == np.argsort(-ts, kind="stable").tolist()
    t.close()


def _key_shapes():
    rng = np.random.default_rng(3)
    base = to_us(datetime(2026, 5, 1, 12))
    n = 40_000
    yield "all_equal", np.full(n, base, np.int64)
    yield "two_values", np.where(rng.random(n) < 0.5, base, base - 3_600_000_000).astype(np.int64)
    yield "bit0", (base & ~1) + rng.integers(0, 2, n, dtype=np.int64)
    old = [to_us(datetime.min), to_us(datetime.max), to_us(datetime(1969, 12, 31, 23, 59, 59, 999999)), 0, -1, 1, to_us(datetime(1900, 3, 1))]
    mixed = rng.integers(to_us(datetime(1940, 1, 1)), to_us(datetime(2000, 1, 1)), n, dtype=np.int64)
    mixed[rng.integers(0, n, 700)] = rng.choice(old, 700)
    yield "pre_1970_and_extremes", mixed


@pytest.mark.parametrize("name,ts", list(_key_shapes()), ids=[s[0] for s in _key_shapes()])
def test_key_shapes(engine, name, ts):
    dev, host, *_ = _tables(engine, ts)
    n = ts.size
    _against_host(dev, host, ((25, 0), (25, 1), (25, n // 2), (25, n - 25), (1, n - 1), (-1, 0), (SMEM_SORT + 1, n // 3), (3, 17_000)))


@pytest.mark.parametrize("size", [SMEM_SORT - 1, SMEM_SORT, SMEM_SORT + 1])
def test_page_sizes_at_the_one_block_sort_bound(engine, size):
    ts, models, tok, cost = synth_usage_columns(100_000, seed=size, end=NOW)
    ts[::5] = ts[1::5][:ts[::5].size]
    dev, host, *_ = _tables(engine, ts)
    _against_host(dev, host, ((size, 0), (size, 31_337), (size, ts.size - size)))


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_candidates_at_the_compaction_threshold(engine, delta):
    """A cluster of the newest records alone under the select's prefix after the digit of bits 40..47: n/16 - 1, n/16 and
    n/16 + 1 of them, so that the candidates are compacted at that pass or (at +1) a later one."""
    n = 16 * 20_000
    a = n // CAND_DIV + delta
    rng = np.random.default_rng(a)
    t0 = 5 << 48 | 7 << 40
    ts = np.empty(n, np.int64)
    ts[:n - a] = (5 << 48) + rng.integers(0, 7 << 40, n - a, dtype=np.int64)
    ts[n - a:] = t0 + rng.integers(0, 1 << 20, a, dtype=np.int64)
    ts[n - a::97] = t0 + 12345                                       # (equal timestamps inside the cluster)
    ts = ts[rng.permutation(n)]
    dev, host, *_ = _tables(engine, ts)
    _against_host(dev, host, ((25, 0), (25, a - 25), (40, a - 20), (25, n - 25), (SMEM_SORT + 1, 100)))


@pytest.mark.parametrize("n_new", [1, 100, U.LISTING_PENDING_MAX - 1, U.LISTING_PENDING_MAX, U.LISTING_PENDING_MAX + 1])
def test_rows_inserted_since_the_upload(engine, n_new):
    from test_rollup_gpu import _compare
    n = 20_000
    ts, models, tok, cost = synth_usage_columns(n, seed=2, end=NOW)
    ts = ts // 10**6 * 10**6                                          # whole seconds: many inserts equal an uploaded timestamp
    dev, host = UsageTable(engine), UsageTable(None)
    for t in (dev, host):
        t.load_columns(ts, models, *tok, cost)
    assert dev.get_latest_usage_records(25, 0) == host.get_latest_usage_records(25, 0)
    ptrs = dev._dev_ptrs
    before = {c: p.value for c, p in ptrs.items()}
    rng = np.random.default_rng(n_new)
    lo, hi = int(ts.min()), int(ts.max())
    new_ts = np.where(rng.random(n_new) < 0.5, ts[rng.integers(0, n, n_new)], rng.integers(lo, hi, n_new) // 10**6 * 10**6)
    new_ts[:3] = [hi, lo, hi + 1][:n_new] if n_new >= 3 else new_ts[:3]
    rows = [(_iso(ts[i]), int(tok[0][i]), int(tok[1][i]), int(tok[2][i]), int(tok[3][i]), int(tok[4][i]), float(cost[i]), models[i], None) for i in range(n)]
    for k, s in enumerate(new_ts.tolist()):
        u = {"prompt_tokens": k, "completion_tokens": 2 * k, "total_tokens": 3 * k, "reasoning_tokens": k % 5, "cached_tokens": k % 3,
             "cost": k * 1e-6, "model": "m-new-%d" % (k % 3), "provider": "P"}
        stamp = _EPOCH + timedelta(microseconds=s)
        for t in (dev, host):
            t.insert_usage(u, timestamp=stamp)
        rows.append((stamp.isoformat(), k, 2 * k, 3 * k, k % 5, k % 3, k * 1e-6, u["model"], "P"))
    total = n + n_new
    pages = [(25, 0), (25, n_new - 1), (25, n_new), (25, n_new + 1), (25, max(0, n_new - 25)), (7, total - 3), (25, total // 2), (1, total - 1)]
    pages += [(-1, 0)] if n_new < 1000 else [(3000, n_new - 1500)]
    _against_host(dev, host, pages)
    if n_new <= U.LISTING_PENDING_MAX:
        assert dev._dev_ptrs is ptrs and {c: p.value for c, p in ptrs.items()} == before and len(dev._pending_rows) == n_new
    else:
        assert dev._dev_ptrs is not ptrs and dev._dev_n == total and not dev._pending_rows
    conn = ro.make_db(rows)
    for period in ("day", "month"):
        _compare(dev.get_aggregated_usage(period), ro.aggregated_usage(conn, period))
    _against_host(dev, host, pages[:3])
    dev.close()
