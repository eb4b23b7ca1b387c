"""GPU: the usage rollup at production geometry against the exact reference of tests/rollup_geometry_cases.py.  Every query runs
on both accumulation paths (the default choice, then global reductions only) and its whole row array must equal the reference
bit for bit: order, bucket, model rank, flag, the five token sums, count and cost.  Every query also checks which accumulation
path ran (launch count) and that no record fell outside the table."""
import copy
import ctypes as C
import math

import numpy as np
import pytest

import rollup_geometry_cases as G
from llmapigateway_b200.usage import ROLLUP_CELLS, UsageTable, stats_window
from oracle import rollup_oracle as ro

pytestmark = pytest.mark.gpu
PERIODS = ("hour", "day", "week", "month")


@pytest.fixture(scope="module")
def engine():
    import llmapigateway_b200 as L
    e = L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    yield e
    e.close_engine()


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def c5(engine):
    cols = G.c5()
    t = cols.load(UsageTable(engine))
    yield cols, t
    t.close()


def _query(engine, table, period, start=None, end=None, path=0, geometry=None, pinned=False):
    """accumulate + emit into tables owned here: (rows, privatised).  Checks the launches of the path that must have run
    (2 privatised, 1 global, + 3 for the emit) and that `oob` stayed 0."""
    lib, h = engine._lib, engine._h
    b0, nb, nm = geometry or table.geometry(period, start, end)
    groups = nb * nm
    table._upload()
    bufs = [C.c_void_p() for _ in range(3)]
    try:
        for p, nbytes in zip(bufs, (groups * ROLLUP_CELLS * 8, groups * 4, 8)):
            engine._ck(lib.lgw_device_alloc(h, nbytes, C.byref(p)), "device_alloc")
            engine._ck(lib.lgw_device_zero(h, p, nbytes), "device_zero")
        engine._ck(lib.lgw_rollup_set_path(h, path), "rollup_set_path")
        before = engine.launch_count()
        table.accumulate(period, start, end, b0, nb, nm, *bufs)
        rows = table.emit(b0, nb, nm, bufs[0], bufs[1], pinned=pinned).copy()
        launches = engine.launch_count() - before
        oob = np.zeros(1, np.uint32)
        engine._ck(lib.lgw_device_download(h, oob.ctypes.data_as(C.c_void_p), bufs[2], 4), "device_download")
    finally:
        lib.lgw_rollup_set_path(h, 0)
        for p in bufs:
            if p.value:
                lib.lgw_device_free(h, p)
    priv = G.privatised(groups, len(table), path)
    assert launches == (2 if priv else 1) + 3, (period, start, end, path, groups, len(table), launches)
    assert int(oob[0]) == 0, (period, start, end, path, int(oob[0]))
    return rows, priv


def _same(got, want, what):
    if got.tobytes() == want.tobytes():
        return
    if len(got) != len(want):
        pytest.fail(f"{what}: {len(got)} rows, expected {len(want)}")
    bad = np.flatnonzero((got.view(np.uint8).reshape(len(got), -1) != want.view(np.uint8).reshape(len(want), -1)).any(axis=1))
    pytest.fail(f"{what}: {len(bad)} of {len(got)} rows differ, first {got[bad[0]]} expected {want[bad[0]]}")


def _both_paths(engine, table, cols, period, start=None, end=None, n=None, geometry=None):
    """the query on both paths against the reference: the default path's choice (privatised or not)"""
    want = G.ref_rollup(cols, period, start, end, n=n)
    out = None
    for path in (0, 1):
        rows, priv = _query(engine, table, period, start, end, path, geometry)
        _same(rows, want, (period, start, end, n, path))
        out = priv if path == 0 else out
    return out


# ---- 1. C5 at 10 M records ---------------------------------------------------------------------------------------------
def test_c5_every_group_exact(engine, sm_count, c5):
    """the stats endpoint's four windows and the four unwindowed tables of 10 M records; the windows of `day`, `week` and
    `month` and unwindowed `month` are privatised, many trips deep; the 24-hour `hour` window (3 250 groups) is not"""
    cols, t = c5
    priv = set()
    for period in PERIODS:
        for label, (s, e) in (("window", stats_window(period, G.NOW)), ("all", (None, None))):
            if _both_paths(engine, t, cols, period, s, e):
                priv.add((period, label))
    assert priv == {("day", "window"), ("week", "window"), ("month", "window"), ("month", "all")}
    assert G.warp_trips(len(cols), sm_count).min() >= 16                # (any H100: 132 SMs or fewer)


def test_c5_pinned_emit_and_side_stream(engine, c5):
    """emit into the pinned buffer gives the pageable bytes; the engine on a torch side stream (as bench.py runs C5) too"""
    import torch
    cols, t = c5
    for period in ("day", "hour"):
        s, e = stats_window(period, G.NOW)
        want = G.ref_rollup(cols, period, s, e)
        rows, _ = _query(engine, t, period, s, e, pinned=True)
        _same(rows, want, (period, "pinned"))
        stream = torch.cuda.Stream()
        engine.set_stream(stream.cuda_stream)
        try:
            rows, _ = _query(engine, t, period, s, e)
        finally:
            engine.set_stream(None)
        _same(rows, want, (period, "side stream"))


# ---- 6. flagged groups at volume -------------------------------------------------------------------------------------
def test_c5_flagged_groups_at_volume(engine, c5):
    """NaN, 1e-30 and +-inf costs in day groups at the table's first and last rows, its first dense position and around tile
    edges: exactly those rows are flagged, their host sum is SQLite's over their members, every other row is bit-exact"""
    cols, t0 = c5
    b0, nb, nm = t0.geometry("day", None, None)
    ref = G.ref_rollup(cols, "day")
    key = ref["bucket"] * nm + ref["model_rank"]

    def dense(j):                                                       # output position j of the dense table -> group key
        return (b0 + nb - 1 - j // nm) * nm + j % nm
    targets = {int(key[0]): [1e-30], int(key[-1]): [math.nan], b0 * nm: [math.inf],
               dense(1023): [-math.inf], dense(1024): [math.inf, -math.inf], dense(2047): [math.nan, 1e-30], dense(2048): [1e-30, 2.0 ** 12]}
    assert set(targets) <= set(key.tolist()) and len(targets) == 7
    order, skey, _ = cols.sorted_by_group("day")
    flagged = copy.copy(cols)
    flagged.cost = cols.cost.copy()
    members = {}
    for k, costs in targets.items():
        lo, hi = np.searchsorted(skey, [k, k + 1])
        members[k] = np.sort(order[lo:hi])
        flagged.cost[members[k][:len(costs)]] = costs
    t = flagged.load(UsageTable(engine))
    try:
        want = G.ref_rollup(flagged, "day")
        assert sorted((want["bucket"] * nm + want["model_rank"])[want["inexact"] == 1].tolist()) == sorted(targets)
        idx = np.concatenate([members[k] for k in sorted(targets)])
        conn = ro.make_db([((G.us_datetime(int(cols.ts[i]))).isoformat(), *[int(x[i]) for x in cols.tok],
                            None if math.isnan(flagged.cost[i]) else float(flagged.cost[i]), cols.models[i], "P") for i in idx.tolist()])
        sql = ro.aggregated_usage(conn, "day")
        for path in (0, 1):
            engine._lib.lgw_rollup_set_path(engine._h, path)
            try:
                rows = t.rollup_rows("day")
            finally:
                engine._lib.lgw_rollup_set_path(engine._h, 0)
            fl = rows["inexact"] == 1
            assert (fl == (want["inexact"] == 1)).all(), path
            _same(rows[~fl], want[~fl], ("day flagged", path))
            got, exp = rows[fl].copy(), want[fl].copy()
            got["cost"] = exp["cost"] = 0
            _same(got, exp, ("day flagged rows", path))
            assert len(sql) == int(fl.sum())
            for r, w in zip(rows[fl], sql):
                c, wc = float(r["cost"]), w["cost"]
                if wc is None or not math.isfinite(wc):
                    assert (math.isnan(c) and wc is None) or c == wc, (path, w, c)
                else:
                    assert abs(int(np.float64(c).view(np.int64)) - int(np.float64(wc).view(np.int64))) <= 4, (path, w, c)
        # month (privatised): the same records flag their months
        want = G.ref_rollup(flagged, "month")
        for path in (0, 1):
            rows, priv = _query(engine, t, "month", path=path)
            assert priv == (path == 0)
            fl = want["inexact"] == 1
            assert fl.any() and (rows["inexact"] == want["inexact"]).all()
            _same(rows[~fl], want[~fl], ("month flagged", path))
    finally:
        t.close()


# ---- 2. trip ladder --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", G.LADDER_K)
def test_trip_ladder(engine, sm_count, k):
    """n = 4 * S * k + delta (S = one record per thread of the grid) around whole trips of the privatised accumulation, under
    windows that pass everything, about half, about 3 %, one record and none"""
    sizes = [4 * sm_count * 1024 * k + d for d in G.LADDER_DELTA] + ([65_535, 65_536] if k == 1 else [])
    cols = G.trip_ladder(max(sizes))
    for n in sizes:
        t = cols.load(UsageTable(engine), n)
        try:
            for label, s, e in G.ladder_windows(cols.ts[:n]):
                priv = _both_paths(engine, t, cols, "day", s, e, n=n)
                assert priv == (n >= 65_536), (n, label)
                if label == "none":
                    assert t.get_aggregated_usage("day", s, e) == []
        finally:
            t.close()


# ---- 3. table-size ladder --------------------------------------------------------------------------------------------
SHAPES = ((1, 1), (2559, 1), (2560, 1), (2561, 1), (40, 64), (41, 64), (1, 2559), (1, 2560), (1, 2561))


def test_table_size_ladder(engine):
    """caller geometries of G = 1 .. 2 561 groups (one model, many buckets; 64 x 40; thousands of models in one bucket), the
    first and the last group occupied: privatised up to 2 560 groups, global from 2 561"""
    for nb, nm in SHAPES:
        cols, b0 = G.group_table(nb, nm)
        t = cols.load(UsageTable(engine))
        try:
            priv = _both_paths(engine, t, cols, "hour", geometry=(b0, nb, nm))
            assert priv == (nb * nm <= 2560), (nb, nm)
        finally:
            t.close()


def test_partial_scratch_reuse_matches_a_fresh_engine(engine):
    """2 560 groups, then 1, then 2 560 again on one engine (its per-block scratch reused) against a fresh engine"""
    import llmapigateway_b200 as L
    big, b0 = G.group_table(2560, 1)
    one, b1 = G.group_table(1, 1)
    tb, to = big.load(UsageTable(engine)), one.load(UsageTable(engine))
    try:
        first, _ = _query(engine, tb, "hour", geometry=(b0, 2560, 1))
        _same(_query(engine, to, "hour", geometry=(b1, 1, 1))[0], G.ref_rollup(one, "hour"), "one group")
        again, _ = _query(engine, tb, "hour", geometry=(b0, 2560, 1))
    finally:
        tb.close(); to.close()
    fresh = L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    try:
        tf = big.load(UsageTable(fresh))
        other, priv = _query(fresh, tf, "hour", geometry=(b0, 2560, 1))
        tf.close()
    finally:
        fresh.close_engine()
    assert priv
    want = G.ref_rollup(big, "hour")
    for rows, what in ((first, "first"), (again, "again"), (other, "fresh engine")):
        _same(rows, want, what)


# ---- 4. more than 1 024 and 2 048 tiles --------------------------------------------------------------------------------
def test_long_span_hour_table(engine):
    """C5 over 1 500 days: the unwindowed `hour` table has more than 2 048 tiles, so the scan of tile counts takes three passes"""
    cols = G.c5(days=1500)
    t = cols.load(UsageTable(engine))
    try:
        b0, nb, nm = t.geometry("hour", None, None)
        assert nb * nm > 2048 * G.TILE
        assert not _both_paths(engine, t, cols, "hour")
    finally:
        t.close()


@pytest.mark.parametrize("tile", G.SPARSE_TILES + (-1,))
def test_sparse_tile_positions(engine, tile):
    """one occupied group at the last position of a tile (alone, and after a group in tile 0) of a table of 2 050 tiles"""
    for tiles in ((tile,), (0, tile)) if tile != 0 else ((0,),):
        cols, b0, nb = G.sparse_table(tiles)
        t = cols.load(UsageTable(engine))
        try:
            _both_paths(engine, t, cols, "hour", geometry=(b0, nb, 1))
        finally:
            t.close()


# ---- 5. one hot group ------------------------------------------------------------------------------------------------
def test_hot_group_of_10m_records(engine):
    """10 M records in one group: full-range tokens of both signs, costs over every limb whose exact total is a double tie that
    only its lowest bit breaks; against Python-int sums and fsum"""
    cols, target = G.hot_group()
    assert G.exact_units(cols.cost) == target
    t = cols.load(UsageTable(engine))
    try:
        for period in ("hour", "month"):
            want = G.ref_rollup(cols, period)
            assert len(want) == 1 and float(want["cost"][0]) == G.units_to_float(target)
            for name, x in zip(G.TOKENS, cols.tok):
                assert int(want[name][0]) == sum(int(v) for v in np.add.reduceat(x.astype(np.int64), np.arange(0, x.size, 1 << 20)))
            assert _both_paths(engine, t, cols, period)
    finally:
        t.close()


def test_two_alternating_hot_groups(engine):
    cols, _ = G.hot_group(groups=2)
    t = cols.load(UsageTable(engine))
    try:
        assert _both_paths(engine, t, cols, "day")
    finally:
        t.close()


# ---- calendar edges --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ("epoch", "century"))
def test_calendar_edges(engine, which):
    """1969-06 .. 1970-06 (negative buckets, bucket0 < 0) and 2100-02-20 .. 2100-03-10 (a century year that is not a leap year),
    every period, unwindowed and over the middle half"""
    cols = G.epoch_span() if which == "epoch" else G.century_span()
    ts = np.sort(cols.ts)
    mid = (G.us_datetime(ts[ts.size // 4]), G.us_datetime(ts[3 * ts.size // 4]))
    t = cols.load(UsageTable(engine))
    try:
        for period in PERIODS:
            for s, e in ((None, None), mid):
                _both_paths(engine, t, cols, period, s, e)
    finally:
        t.close()
