"""CPU: the exact rollup reference of tests/rollup_geometry_cases.py against SQLite, and the claims its datasets make about the
geometry the GPU tests (tests/test_rollup_geometry_gpu.py) reach: table sizes, accumulation paths and trip counts."""
import math
import random
import sqlite3
from datetime import datetime, timedelta

import numpy as np
import pytest

import rollup_cost_cases as RC
import rollup_geometry_cases as G
from llmapigateway_b200.usage import UsageTable, stats_window, to_us
from oracle import rollup_oracle as ro

EPOCH = datetime(1970, 1, 1)
SMS = (132, 114)                   # H100 SXM and PCIe


def _bucket_samples() -> np.ndarray:
    rng = np.random.default_rng(3)
    out = [rng.integers(to_us(datetime(1900, 1, 1)), to_us(datetime(2100, 12, 31)), 160_000, dtype=np.int64)]
    h = np.arange(to_us(datetime(1969, 12, 1)), to_us(datetime(1970, 2, 1)), G.HOUR_US)
    out += [h, h + rng.integers(0, G.HOUR_US, h.size)]
    for y in range(1968, 2102):
        jan1 = to_us(datetime(y, 1, 1))
        d = jan1 + np.arange(-7, 8) * G.DAY_US
        out += [d, d - 1, d + rng.integers(0, G.DAY_US, d.size)] + [d + rng.integers(0, G.DAY_US, d.size) for _ in range(20)]
    for y in (1900, 2000, 2024, 2100):
        for m, dd in ((2, 28), (2, 29), (3, 1)):
            try:
                day = to_us(datetime(y, m, dd))
            except ValueError:                                      # 1900-02-29, 2100-02-29
                continue
            out += [day + np.arange(24) * G.HOUR_US, day + rng.integers(0, G.DAY_US, 200), np.array([day - 1, day + G.DAY_US - 1001])]
    ts = np.concatenate(out).astype(np.int64)
    return ts[~G.in_roll(ts)]


def _sqlite_labels(conn, fmt: str) -> list:
    return [r[0] for r in conn.execute(f"SELECT strftime('{fmt}', t) FROM x ORDER BY rowid")]


def test_ref_bucket_matches_sqlite_strftime():
    ts = _bucket_samples()
    assert ts.size >= 200_000
    iso = [(EPOCH + timedelta(microseconds=int(u))).isoformat() for u in ts.tolist()]
    conn = sqlite3.connect(":memory:")
    conn.execute("CREATE TABLE x (t TEXT)")
    conn.executemany("INSERT INTO x VALUES (?)", ((s,) for s in iso))
    for period, fmt in ro.PERIOD_FORMATS.items():
        want = _sqlite_labels(conn, fmt)
        got = [G.ref_label(period, b) for b in G.ref_bucket(ts, period).tolist()]
        bad = [(iso[i], got[i], want[i]) for i in range(ts.size) if got[i] != want[i]]
        assert not bad, (period, len(bad), bad[:5])


def test_vectorised_representable_matches_the_cost_cases():
    rng = random.Random(5)
    costs = [c for c, _ in RC.BOUNDARY] + [RC.exact_cost(rng) for _ in range(5000)] + [x for v in RC.FLAGGED.values() for x in v if x is not None]
    costs += [rng.randrange(10 ** 6) * 1e-6 for _ in range(2000)] + [math.ldexp(rng.getrandbits(53), rng.randint(-140, 40)) for _ in range(2000)]
    assert G.representable(costs).tolist() == [RC.representable(c) for c in costs]


def _to_dicts(cols, period, rows):
    names = [None] + cols.names
    return [{"time_period": G.ref_label(period, int(r["bucket"])), "model": names[int(r["model_rank"])],
             **{k: int(r[k]) for k in G.TOKENS}, "cost": float(r["cost"]), "count": int(r["count"])} for r in rows]


def _ulps(a: float, b: float) -> int:
    ia, ib = np.array([a, b], np.float64).view(np.int64).tolist()
    return abs(ia - ib)


def test_ref_rollup_matches_sqlite():
    cols = G.c5(100_000, seed=6)
    rows = [((EPOCH + timedelta(microseconds=int(cols.ts[i]))).isoformat(), *[int(t[i]) for t in cols.tok], float(cols.cost[i]), cols.models[i], "P")
            for i in range(len(cols))]
    conn = ro.make_db(rows)
    for period in ("hour", "day", "week", "month"):
        for s, e in ((None, None), stats_window(period, G.NOW)):
            got = _to_dicts(cols, period, G.ref_rollup(cols, period, s, e))
            want = ro.aggregated_usage(conn, period, s, e)
            assert len(got) == len(want) > 0, period
            for g, w in zip(got, want):
                assert {k: v for k, v in g.items() if k != "cost"} == {k: v for k, v in w.items() if k != "cost"}, (period, g, w)
                assert _ulps(g["cost"], w["cost"]) <= 4, (period, g, w)


def test_ref_rollup_flags_and_sums():
    """the reference's flag and cost on hand-made groups: fsum where every member is representable, flagged (NaN) else"""
    rng = random.Random(8)
    recipes = [v for v, _ in RC.FIXED_EXACT.values()] + [[c for c in v] for v in RC.FLAGGED.values()]
    ts, models, cost = [], [], []
    for k, costs in enumerate(recipes):
        for c in costs:
            ts.append(to_us(datetime(2025, 1, 1)) + k * G.DAY_US + rng.randrange(G.DAY_US - 1000))
            models.append("m"); cost.append(math.nan if c is None else c)
    n = len(ts)
    zero = np.zeros(n, np.int32)
    cols = G.Columns(np.array(ts), np.array(models, dtype=object), [zero] * 5, np.array(cost))
    rows = G.ref_rollup(cols, "day")[::-1]
    assert len(rows) == len(recipes)
    for r, (k, v) in zip(rows, enumerate(RC.FIXED_EXACT.values())):
        assert not r["inexact"] and float(r["cost"]) == v[1] and (v[1] != 0 or math.copysign(1, r["cost"]) == 1), k
    assert rows["inexact"][len(RC.FIXED_EXACT):].all()


def test_exact_units_and_the_hot_group():
    rng = random.Random(9)
    costs = [RC.exact_cost(rng) for _ in range(20_000)]
    want = sum(int(math.ldexp(c, 80)) for c in costs)
    assert G.exact_units(costs) == want
    cols, target = G.hot_group(400_000)
    assert G.exact_units(cols.cost) == target
    fs = math.fsum(cols.cost.tolist())
    assert fs == G.units_to_float(target)
    assert abs(fs) != G.units_to_float(abs(target) - 1)           # without the lowest bit the tie rounds the other way
    assert np.abs(cols.cost).max() > 2 ** 11 and np.abs(cols.cost[cols.cost != 0]).min() < 2 ** -60
    assert (np.sign(cols.cost[:-2:2]) >= 0).all() and (np.sign(cols.cost[1:-2:2]) <= 0).all()
    assert cols.tok[1].min() == -2 ** 31 and cols.tok[0].max() == 2 ** 31 - 1 and (cols.tok[2] < 0).any()


def test_trip_geometry_of_the_ladder_and_c5():
    for sm in SMS:
        for n in G.ladder_sizes(sm):
            k, d = divmod(n, 4 * sm * 1024)
            if d > 4 * sm * 1024 // 2:
                k, d = k + 1, d - 4 * sm * 1024
            trips = G.warp_trips(n, sm)
            assert trips.max() == k + (d > 0) and trips.min() == k, (sm, n)
            assert (trips == k + 1).sum() == (-(-d // 32) if d > 0 else 0), (sm, n)
            assert G.privatised(130, n)
        trips = G.warp_trips(10_000_000, sm)
        assert trips.min() == trips.max() == -(-10_000_000 // (4 * sm * 1024)) >= 16
    assert not G.privatised(130, 65_535) and G.privatised(130, 65_536)
    assert G.privatised(2560, 65_536) and not G.privatised(2561, 65_536) and not G.privatised(2560, 65_536, path=1)


@pytest.fixture(scope="module")
def c5_geometry():
    out = {}
    for days in (400, 1500):
        cols = G.c5(days=days)
        t = UsageTable(engine=None)
        cols.load(t)
        out[days] = (cols, t)
    return out


def test_c5_paths_and_table_sizes(c5_geometry):
    cols, t = c5_geometry[400]
    priv = set()
    for period in ("hour", "day", "week", "month"):
        for label, (s, e) in (("window", stats_window(period, G.NOW)), ("all", (None, None))):
            b0, nb, nm = t.geometry(period, s, e)
            assert nm == 65
            sel = np.ones(len(cols), bool) if s is None else (cols.ts >= to_us(s)) & (cols.ts <= to_us(e))
            b = G.ref_bucket(cols.ts[sel], period)
            assert b0 <= b.min() and b.max() < b0 + nb
            if G.privatised(nb * nm, len(cols)):
                priv.add((period, label))
    assert priv == {("day", "window"), ("week", "window"), ("month", "window"), ("month", "all")}
    assert t.geometry("hour", *stats_window("hour", G.NOW))[1] * 65 == 3250
    cols, t = c5_geometry[1500]
    b0, nb, nm = t.geometry("hour", None, None)
    assert nb * nm > 2048 * G.TILE and -(-nb * nm // G.TILE) > 2048


def test_small_tables_and_sparse_tables():
    for nb, nm in ((1, 1), (2559, 1), (2560, 1), (2561, 1), (40, 64), (41, 64), (1, 2559), (1, 2560), (1, 2561)):
        cols, b0 = G.group_table(nb, nm)
        b = G.ref_bucket(cols.ts, "hour") - b0
        g = b * nm + cols.rank
        assert b.min() >= 0 and b.max() < nb and cols.rank.max() < nm
        assert g.min() == 0 and g.max() == nb * nm - 1 and len(cols) >= G.SMEM_MIN_RECORDS
        assert G.privatised(nb * nm, len(cols)) == (nb * nm <= 2560)
    cols, b0, nb = G.sparse_table(G.SPARSE_TILES + (-1,))
    assert nb > 2048 * G.TILE and -(-nb // G.TILE) == 2050
    j = nb - 1 - (G.ref_bucket(cols.ts, "hour") - b0)
    assert sorted(set((j // G.TILE).tolist())) == sorted(G.SPARSE_TILES + (2049,)) and j.max() == nb - 1
    assert ((j % G.TILE == G.TILE - 1) | (j == nb - 1)).all()


def test_calendar_edge_tables():
    cols = G.epoch_span()
    for period in ("hour", "day"):
        assert G.ref_bucket(cols.ts, period).min() < 0 < G.ref_bucket(cols.ts, period).max()
    month = G.ref_bucket(cols.ts, "month")
    assert month.min() == 1969 * 12 + 5 and month.max() == 1970 * 12 + 4
    cols = G.century_span()
    assert G.ref_label("day", int(G.ref_bucket(np.array([to_us(datetime(2100, 2, 28, 23))]), "day")[0]) + 1) == "2100-03-01"
    assert set(G.ref_bucket(cols.ts, "month").tolist()) == {2100 * 12 + 1, 2100 * 12 + 2}
