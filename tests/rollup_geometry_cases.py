"""The usage rollup at production geometry (csrc/rollup.cuh): an exact reference of the rollup that shares no code with the
kernel, and seeded datasets that drive the kernels through the code paths a 10 M-record table runs on every query -- many trips
of the privatised accumulation, the global path's grid-stride loop, more than 1 024 / 2 048 compaction tiles, one group of
millions of records, and the path switch at its group and record limits.

`ref_bucket` is numpy's calendar (datetime64), not the kernel's date arithmetic, and it does NOT model SQLite's millisecond
roll (23:59:59.9995+ formats as the next day in some fields): every builder moves such a record 1 ms down and checks that none
is left.  The roll itself is pinned on both accumulation paths by tests/test_rollup_gpu.py::test_device_buckets_match_sqlite_at_volume.
"""
from __future__ import annotations

import math
from datetime import datetime, timedelta

import numpy as np

from llmapigateway_b200.usage import ROW_DTYPE, synth_usage_columns, to_us

NOW = datetime(2026, 9, 21, 6, 57, 17, 47518)
DAY_US = 86_400_000_000
HOUR_US = 3_600_000_000
ROLL_US = 500                      # the last 500 us of a day round up to midnight in SQLite's strftime
TOP = 2.0 ** 12                    # |cost| from here up is not taken exactly
SMEM_GROUPS = 2560                 # largest table the privatised accumulation takes
SMEM_MIN_RECORDS = 65536           # fewest records it takes
TILE = 1024                        # compaction: table positions per tile, and tiles per pass of the scan
TOKENS = ("prompt_tokens", "completion_tokens", "total_tokens", "reasoning_tokens", "cached_tokens")


# ---- reference --------------------------------------------------------------------------------------------------------
def ref_bucket(ts_us, period: str) -> np.ndarray:
    """bucket index of every timestamp as the rollup numbers them (hour: day * 24 + hour, day: days since 1970-01-01,
    week: year * 64 + %W (Monday first), month: year * 12 + month - 1); floor division, so right before 1970 too"""
    ts = np.asarray(ts_us, np.int64)
    days = ts // DAY_US
    if period == "hour":
        return days * 24 + (ts - days * DAY_US) // HOUR_US
    if period == "day":
        return days
    d = days.astype("datetime64[D]")
    year = d.astype("datetime64[Y]").astype(np.int64) + 1970
    if period == "month":
        return d.astype("datetime64[M]").astype(np.int64) + 1970 * 12
    assert period == "week", period
    yday = days - d.astype("datetime64[Y]").astype("datetime64[D]").astype(np.int64)
    wd = (days + 3) % 7                                              # Monday = 0: 1970-01-01 was a Thursday
    return year * 64 + (yday + 7 - wd) // 7


def ref_label(period: str, bucket: int) -> str:
    """SQLite's strftime text of a bucket (tokens_usage_db.py's formats)"""
    if period == "hour":
        return "%s %02d:00:00" % (np.datetime64(bucket // 24, "D"), bucket % 24)
    if period == "day":
        return str(np.datetime64(bucket, "D"))
    if period == "week":
        return "%04d-W%02d" % (bucket // 64, bucket % 64)
    return "%04d-%02d" % (bucket // 12, bucket % 12 + 1)


def representable(cost) -> np.ndarray:
    """vectorised tests/rollup_cost_cases.representable: finite, |c| < 2^12 and a multiple of 2^-80"""
    c = np.asarray(cost, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        x = c * 2.0 ** 80
        return np.isfinite(c) & (np.abs(c) < TOP) & (np.floor(x) == x)


def in_roll(ts_us) -> np.ndarray:
    return np.asarray(ts_us, np.int64) % DAY_US >= DAY_US - ROLL_US


def clear_roll(ts: np.ndarray) -> np.ndarray:
    """move every record of the last 500 us of a day 1 ms down (in place), and check that none is left"""
    ts[in_roll(ts)] -= 1000
    assert not in_roll(ts).any()
    return ts


def sorted_names(models) -> list:
    return sorted({m for m in models if m is not None}, key=lambda s: s.encode("utf-8"))


class Columns:
    """one dataset: the columns UsageTable.load_columns takes, its model dictionary, and the reference's per-period order"""

    def __init__(self, ts, models, tok, cost, names=None):
        self.ts = clear_roll(np.ascontiguousarray(ts, np.int64))
        self.models = models
        self.tok = [np.ascontiguousarray(t, np.int32) for t in tok]
        self.cost = np.ascontiguousarray(cost, np.float64)
        self.names = sorted_names(models) if names is None else names
        rank = {m: i + 1 for i, m in enumerate(self.names)}
        rank[None] = 0
        self.rank = np.fromiter((rank[m] for m in models), np.int64, len(models))
        self._by_period = {}

    def __len__(self):
        return int(self.ts.size)

    def load(self, table, n: int | None = None):
        n = len(self) if n is None else n
        table.load_columns(self.ts[:n], self.models[:n], *[t[:n] for t in self.tok], self.cost[:n], names=self.names)
        return table

    def sorted_by_group(self, period: str):
        """records ordered by (bucket, model rank, index): computed once per period"""
        if period not in self._by_period:
            nm = len(self.names) + 1
            key = ref_bucket(self.ts, period) * nm + self.rank
            order = np.argsort(key, kind="stable")
            self._by_period[period] = (order, key[order], self.ts[order])
        return self._by_period[period]


def ref_rollup(cols: Columns, period: str, start=None, end=None, n: int | None = None) -> np.ndarray:
    """GROUP BY bucket, model over records [0, n) with start <= ts <= end (microseconds), in ROW_DTYPE, bucket DESC, rank ASC.
    Token sums and counts are exact int64; cost is math.fsum of the members, bit for bit what an unflagged device row holds;
    `inexact` is 1 where a member is not representable (the device's cost of such a row is not the group's sum: NaN here)."""
    order, key, ts = cols.sorted_by_group(period)
    sel = np.ones(order.size, bool) if n is None else order < n
    if start is not None:
        sel &= ts >= (to_us(start) if isinstance(start, datetime) else start)
    if end is not None:
        sel &= ts <= (to_us(end) if isinstance(end, datetime) else end)
    idx, key = order[sel], key[sel]
    if idx.size == 0:
        return np.zeros(0, ROW_DTYPE)
    first = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    nm = len(cols.names) + 1
    rows = np.zeros(first.size, ROW_DTYPE)
    rows["bucket"] = key[first] // nm
    rows["model_rank"] = key[first] % nm
    for name, t in zip(TOKENS, cols.tok):
        rows[name] = np.add.reduceat(t[idx].astype(np.int64), first)
    rows["count"] = np.diff(np.r_[first, idx.size])
    cost = cols.cost[idx]
    bad = np.add.reduceat((~representable(cost)).astype(np.int64), first) > 0
    rows["inexact"] = bad
    cl = cost.tolist()
    bounds = np.r_[first, idx.size].tolist()
    rows["cost"] = [math.nan if b else math.fsum(cl[a:z]) + 0.0 for a, z, b in zip(bounds[:-1], bounds[1:], bad.tolist())]
    return rows[np.lexsort((rows["model_rank"], -rows["bucket"]))]


def exact_units(cost) -> int:
    """sum of representable costs exactly, in units of 2^-80 (a Python int)"""
    c = np.asarray(cost, np.float64)
    assert representable(c).all() and c.size < 1 << 25       # (per-exponent float64 sums below 2^53 stay exact)
    m, e = np.frexp(c)
    mi = (m * 2.0 ** 53).astype(np.int64)                     # c * 2^80 = mi * 2^k
    k = e.astype(np.int64) - 53 + 80
    low = k < 0
    mi[low] >>= -k[low]                                       # (exact: a representable cost has no bits below 2^-80)
    k[low] = 0
    hi = np.bincount(k, weights=(mi >> 26).astype(np.float64))
    lo = np.bincount(k, weights=(mi & ((1 << 26) - 1)).astype(np.float64))
    return sum(((int(h) << 26) + int(l)) << j for j, (h, l) in enumerate(zip(hi, lo)))


def units_to_float(u: int) -> float:
    """u * 2^-80 rounded to nearest, ties to even"""
    from fractions import Fraction
    return float(Fraction(u, 1 << 80))


# ---- path and trip geometry (restated from lgw_usage_rollup_accum / k_rollup_accum_smem) ----------------------------------
def privatised(groups: int, n: int, path: int = 0) -> bool:
    return path == 0 and groups <= SMEM_GROUPS and SMEM_MIN_RECORDS <= n < 0xFFFFFFFF


def warp_trips(n: int, sm_count: int) -> np.ndarray:
    """trips of every warp of k_rollup_accum_smem (one block of 1 024 threads per SM, 4 records per thread per trip)"""
    stride = sm_count * 1024
    first = np.arange(0, stride, 32, dtype=np.int64)
    return np.where(n > first, (n - first + 4 * stride - 1) // (4 * stride), 0)


LADDER_K = (1, 2, 5)
LADDER_DELTA = (-33, -32, -1, 0, 1, 31, 32, 33)


def ladder_sizes(sm_count: int) -> list:
    """n = 4 * S * k + delta with S = sm_count * 1024: one record short of, at and past a whole number of trips, and one or
    two warps more or fewer on the last trip"""
    return [4 * sm_count * 1024 * k + d for k in LADDER_K for d in LADDER_DELTA]


# ---- datasets ----------------------------------------------------------------------------------------------------------
def c5(n: int = 10_000_000, days: int = 400, seed: int = 5) -> Columns:
    """BASELINE config 5: synth_usage_columns (400 days or `days`, 64 models Zipf 1.1 + 1 % NULL, costs k x 1e-6)"""
    ts, models, tok, cost = synth_usage_columns(n, seed=seed, end=NOW, days=days)
    return Columns(ts, models, tok, cost)


def _costs(rng, n: int) -> np.ndarray:
    """representable costs of alternating sign: leading bit 2^t with t uniform in [-80, 11], 1..53 significant bits"""
    t = rng.integers(-80, 12, n)
    w = 1 + rng.integers(0, 1 << 62, n) % np.minimum(53, t + 81)
    m = rng.integers(1 << 52, 1 << 53, n, dtype=np.int64) >> (53 - w)
    c = np.ldexp(m.astype(np.float64), (t - w + 1).astype(np.int32))
    c[1::2] *= -1.0
    return c


def _sticky_tail(bulk: int) -> tuple:
    """two representable costs that bring an exact sum `bulk` (units of 2^-80, |bulk| >= 2^64) to a total of the form
    +-(K * 2^(top-52) + 2^(top-53) + 1) with K even: a tie at double precision that only the lowest bits break (sticky)"""
    s = -1 if bulk < 0 else 1
    top = abs(bulk).bit_length() - 1
    assert top >= 70
    K = (abs(bulk) >> (top - 52)) & ~1
    target = s * ((K << (top - 52)) + (1 << (top - 53)) + 1)
    tail = target - bulk
    a, b = tail >> 26, tail & ((1 << 26) - 1)
    return target, (math.ldexp(a, 26 - 80), math.ldexp(b, -80))


def hot_group(n: int = 10_000_000, seed: int = 7, groups: int = 1):
    """n records in one hour (2026-03-10 12:00) of one model, or alternating over `groups` models.  Tokens: +-(2^31 - 1),
    -2^31 and small values; costs of alternating sign over every limb of the fixed point.  With one group the exact cost total
    is a double-precision tie broken only by its lowest bit: (Columns, exact total in units of 2^-80 or None)"""
    rng = np.random.default_rng([seed, n, groups])
    base = to_us(datetime(2026, 3, 10, 12))
    ts = base + rng.integers(0, HOUR_US, n, dtype=np.int64)
    big = (1 << 31) - 1
    even = np.arange(n) % 2 == 0
    small = rng.integers(0, 1000, n).astype(np.int32)
    tok = [np.where(even, big, small).astype(np.int32),                                  # + full range, never cancels
           np.where(even, np.int32(-big - 1), small).astype(np.int32),                   # INT32_MIN
           np.where(np.arange(n) % 4 == 0, big, np.where(even, -big, small)).astype(np.int32),   # both signs
           rng.integers(-(1 << 31), 1 << 31, n, dtype=np.int64).astype(np.int32),        # random over the full range
           small]
    cost = _costs(rng, n)
    target = None
    if groups == 1:
        target, tail = _sticky_tail(exact_units(cost[:-2]))
        cost[-2:] = tail
    names = ["hot/model-%d" % g for g in range(groups)]
    models = np.array(names, dtype=object)[np.arange(n) % groups]
    return Columns(ts, models, tok, cost), target


def epoch_span(n: int = 400_000, seed: int = 11) -> Columns:
    """1969-06-01 .. 1970-06-01: bucket0 (and every bucket of the first half) is negative"""
    rng = np.random.default_rng(seed)
    lo, hi = to_us(datetime(1969, 6, 1)), to_us(datetime(1970, 6, 1))
    ts = rng.integers(lo, hi, n, dtype=np.int64)
    ts[:4] = [lo, hi - 1001, -1001, 0]
    return _small_models(ts, rng)


def century_span(n: int = 400_000, seed: int = 12) -> Columns:
    """2100-02-20 .. 2100-03-10: 2100 is not a leap year, 2100-02-28 is followed by 2100-03-01"""
    rng = np.random.default_rng(seed)
    lo = to_us(datetime(2100, 2, 20))
    ts = lo + rng.integers(0, 18 * DAY_US, n, dtype=np.int64)
    ts[:3] = [to_us(datetime(2100, 2, 28, 23, 59, 59)), to_us(datetime(2100, 3, 1)), to_us(datetime(2100, 3, 1, 0, 0, 0, 1))]
    return _small_models(ts, rng)


def _small_models(ts, rng, n_models: int = 5, tok_max: int = 1 << 17) -> Columns:
    n = ts.size
    names = np.array([None] + ["m-%d" % i for i in range(n_models)], dtype=object)
    models = names[rng.integers(0, n_models + 1, n)]
    tok = [rng.integers(0, tok_max, n, dtype=np.int32) for _ in range(5)]
    cost = rng.integers(0, 10 ** 6, n).astype(np.float64) * 1e-6
    return Columns(ts, models, tok, cost)


def trip_ladder(n: int, seed: int = 13) -> Columns:
    """n C5-shaped records over 30 days ending at NOW, 3 models + NULL (a day table of ~130 groups)"""
    rng = np.random.default_rng([seed, n])
    ts = to_us(NOW) - rng.integers(0, 30 * DAY_US, n, dtype=np.int64)
    return _small_models(ts, rng, n_models=3)


def us_datetime(us: int) -> datetime:
    return datetime(1970, 1, 1) + timedelta(microseconds=int(us))


def ladder_windows(ts_us: np.ndarray) -> list:
    """(label, start, end) over these timestamps: everything, about half, about 3 %, exactly one record, none"""
    ts = np.sort(ts_us)
    n = ts.size
    one = int(ts_us[n // 2])
    assert (ts_us == one).sum() == 1
    gap = int(ts[-1]) + 1
    w = [("half", ts[n // 4], ts[3 * n // 4]), ("3%", ts[n // 2], ts[n // 2 + n * 3 // 100]), ("one", one, one), ("none", gap, gap + HOUR_US)]
    return [("all", None, None)] + [(k, us_datetime(a), us_datetime(b)) for k, a, b in w]


def group_table(nb: int, nm: int, n: int = 70_000, seed: int = 17):
    """`n` records over a caller-geometry `hour` table of nb buckets x nm models whose first group (g = 0: oldest bucket, NULL
    model) and last group (g = G - 1: newest bucket, highest rank) are occupied: (Columns, bucket0)"""
    rng = np.random.default_rng([seed, nb, nm])
    b0 = to_us(datetime(2026, 1, 5)) // HOUR_US
    names = ["n%05d" % i for i in range(nm - 1)]
    g = rng.integers(0, nb * nm, n)
    g[:2] = [0, nb * nm - 1]
    b, mr = g // nm, g % nm
    ts = (b0 + b) * HOUR_US + rng.integers(0, HOUR_US - 1000, n)
    models = np.array([None] + names, dtype=object)[mr]
    tok = [rng.integers(-(1 << 31), 1 << 31, n, dtype=np.int64).astype(np.int32) for _ in range(5)]
    cost = _costs(rng, n)
    return Columns(ts, models, tok, cost, names=names), b0


SPARSE_TILES = (0, 1, 1022, 1023, 1024, 1025, 2047, 2048)


def sparse_table(tiles, n_tiles: int = 2050, short: int = 7):
    """a `hour` table of one model (NULL) and n_tiles * 1 024 - short buckets in which only the groups at the last position of
    the given output tiles (and at the table's last position, tile -1) hold records, 3 each: (Columns, bucket0, n_buckets)"""
    nb = n_tiles * TILE - short
    b0 = to_us(datetime(1990, 1, 1)) // HOUR_US
    pos = [nb - 1 if t == -1 else t * TILE + TILE - 1 for t in tiles]              # output position j = nb - 1 - bucket
    ts = np.array([(b0 + nb - 1 - j) * HOUR_US + k * 60_000_000 for j in pos for k in range(3)], np.int64)
    n = ts.size
    tok = [np.arange(1, n + 1, dtype=np.int32) * (k + 1) for k in range(5)]
    cost = np.arange(1, n + 1, dtype=np.float64) * 0.25
    return Columns(ts, np.array([None] * n, dtype=object), tok, cost, names=[]), b0, nb
