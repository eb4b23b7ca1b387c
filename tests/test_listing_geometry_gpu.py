"""GPU: the record listing (csrc/listing.cuh, lgw_usage_latest) at production geometry.  Every page of every case of
tests/listing_geometry_cases.py -- tables past 2^24 records, every divergence depth of the two boundary keys, compaction after
every select pass and never, int64 extremes at 10 M records, tables at the kernels' size edges, pages at both sorts' edges --
is listed twice on the device and must equal the stable argsort reference element for element, both times.  Then one engine
runs pages that grow its listing scratch and reuse it with smaller layouts (against fresh engines), and the product path
alternates pages with the rollup over the same uploaded columns, on a side stream and on the engine's own."""
import ctypes as C
from contextlib import ExitStack, contextmanager

import numpy as np
import pytest

import listing_geometry_cases as LG

pytestmark = pytest.mark.gpu


def _new_engine():
    import llmapigateway_b200 as L
    return L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)


@pytest.fixture(scope="module")
def engine():
    e = _new_engine()
    yield e
    e.close_engine()


@pytest.fixture(scope="module")
def tables():
    """name -> Table, built once per module: a table's reference (Table.order) is sorted once, however many pages use it"""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = LG.build(name)
        return cache[name]
    yield get
    cache.clear()


@contextmanager
def on_device(engine, ts):
    """the timestamp column in device memory, as UsageTable uploads it (cudaMalloc: 16-byte aligned), freed on the way out"""
    ts = np.ascontiguousarray(ts, np.int64)
    lib, h = engine._lib, engine._h
    p = C.c_void_p()
    try:
        engine._ck(lib.lgw_device_alloc(h, max(ts.nbytes, 16), C.byref(p)), "device_alloc")
        engine._ck(lib.lgw_device_upload(h, p, ts.ctypes.data_as(C.c_void_p), ts.nbytes), "device_upload")
        yield p
    finally:
        if p.value:
            lib.lgw_device_free(h, p)


def latest(engine, col, n: int, first: int, count: int) -> np.ndarray:
    """lgw_usage_latest as UsageTable._latest_on_device calls it; its check that exactly `count` records lie between the
    boundary keys raises here"""
    out = np.empty(max(count, 1), np.uint64)
    engine._ck(engine._lib.lgw_usage_latest(engine._h, col, n, first, count, out.ctypes.data_as(C.c_void_p)), "usage_latest")
    return out[:count].astype(np.int64)


def last_ms(engine) -> float:
    ms = C.c_float()
    engine._ck(engine._lib.lgw_usage_latest_last_ms(engine._h, C.byref(ms)), "usage_latest_last_ms")
    return ms.value


def _same(got, want, what):
    if np.array_equal(got, want):
        return
    if got.size != want.size:
        pytest.fail(f"{what}: {got.size} records, expected {want.size}")
    bad = np.flatnonzero(got != want)
    pytest.fail(f"{what}: {bad.size} of {got.size} differ, first at {bad[0]}: {got[bad[0]]} expected {want[bad[0]]}")


@pytest.mark.parametrize("name", list(LG.BUILDERS))
def test_every_page(engine, tables, name):
    t = tables(name)
    with on_device(engine, t.ts) as col:
        for p in t.pages:
            got = latest(engine, col, t.n, p.first, p.count)
            assert last_ms(engine) > 0, (name, p)
            _same(got, t.expected(p), (name, p))
            _same(latest(engine, col, t.n, p.first, p.count), got, (name, p, "listed again"))
        assert latest(engine, col, t.n, t.n // 2, 0).size == 0 and last_ms(engine) == 0.0
        assert latest(engine, col, t.n, t.n, 0).size == 0 and last_ms(engine) == 0.0


# (table, first, count): grows the engine's listing scratch, reuses it with smaller layouts, switches between the two sorts
SEQUENCE = (("ties_10m", "mid", 25), ("size_33", 0, 33), ("c5_20m", 0, "all"), ("size_4097", 0, "all"),
            ("ties_10m", 12_345, 65_536), ("size_1", 0, 1), ("ties_10m", "mid", 25))


def test_scratch_reuse_on_one_engine(engine, tables):
    reused = _new_engine()
    try:
        with ExitStack() as stack:
            cols = {name: stack.enter_context(on_device(engine, tables(name).ts)) for name in sorted({s[0] for s in SEQUENCE})}
            for step, (name, first, count) in enumerate(SEQUENCE):
                t = tables(name)
                first = t.n // 2 if first == "mid" else first
                count = t.n - first if count == "all" else count
                got = latest(reused, cols[name], t.n, first, count)
                _same(got, t.expected(LG.Page(first, count)), (step, name, first, count))
                fresh = _new_engine()
                try:
                    _same(latest(fresh, cols[name], t.n, first, count), got, (step, name, first, count, "fresh engine"))
                finally:
                    fresh.close_engine()
    finally:
        reused.close_engine()


def test_product_path_alternating_with_the_rollup(engine):
    """UsageTable pages through the device selection (both sorts, a full listing, the last record) between rollup queries over
    the same uploaded columns: once with the engine on a torch side stream, once on its own stream.  Pages equal the host
    path's, the rollup equals SQLite's, and nothing is uploaded again"""
    import torch
    from test_rollup_gpu import _compare
    from test_usage_listing_gpu import _iso
    from llmapigateway_b200.usage import UsageTable, synth_usage_columns
    from oracle import rollup_oracle as ro
    n = 60_001
    ts, models, tok, cost = synth_usage_columns(n, seed=12, end=LG.NOW)
    ts = ts // LG.SEC * LG.SEC                                        # whole seconds: ties across the table
    ts[1::7] = ts[::7][:ts[1::7].size]                                # and runs of equal timestamps
    dev, host = UsageTable(engine), UsageTable(None)
    for t in (dev, host):
        t.load_columns(ts, models, *tok, cost)
    conn = ro.make_db([(_iso(ts[i]), int(tok[0][i]), int(tok[1][i]), int(tok[2][i]), int(tok[3][i]), int(tok[4][i]),
                        float(cost[i]), models[i], None) for i in range(n)])
    pages = [(25, 0), (25, n // 2), (LG.SMEM_SORT + 1, 1000), (-1, 0), (3 * LG.STILE + 1, n - 3 * LG.STILE - 1), (1, n - 1),
             (LG.SMEM_SORT, 17)]
    periods = ("day", "month", "hour", "week")
    ptrs = None
    stream = torch.cuda.Stream()
    try:
        for side in (True, False):
            engine.set_stream(stream.cuda_stream if side else None)
            for k, (limit, offset) in enumerate(pages):
                assert dev.get_latest_usage_records(limit, offset) == host.get_latest_usage_records(limit, offset), (side, limit, offset)
                ptrs = ptrs or {c: p.value for c, p in dev._dev_ptrs.items()}
                period = periods[k % 4]
                _compare(dev.get_aggregated_usage(period), ro.aggregated_usage(conn, period))
            assert {c: p.value for c, p in dev._dev_ptrs.items()} == ptrs and dev._dev_n == n
    finally:
        engine.set_stream(None)
        dev.close()
