"""The record listing at production geometry (csrc/listing.cuh, lgw_usage_latest): timestamp tables built by construction, each
with the pages it is meant to test, the exact reference of a page, and a numpy model of the radix select's pass structure.

The key of a record is (kd, index) with kd = ts ^ 0x7FFF'FFFF'FFFF'FFFF: 96 bits, 12 digits of 8 bits (8 of kd, then 4 of the
index), most significant first.  A page (first, count) is selected by two boundary keys, at ranks `first` and
`first + count - 1`.  The model reports, for a page, how many leading digits the two boundary keys share (the divergence depth,
12 for one key) and after which select pass the kernel compacts the records under the boundaries' prefixes into its candidate
list (or that it never does).  It certifies what a case reaches (tests/test_listing_geometry_cpu.py); the device's pages are
checked only against `reference` (tests/test_listing_geometry_gpu.py), never against the model.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from datetime import datetime
from functools import cached_property

import numpy as np

from llmapigateway_b200.usage import to_us

NOW = datetime(2026, 9, 21, 6, 57, 17, 47518)
SEC = 10 ** 6
DAY_US = 86_400 * SEC
CAND_DIV = 16                      # csrc/listing.cuh LGW_LIST_CAND_DIV: compact once the candidates are at most n / 16
SMEM_SORT = 8192                   # LGW_LIST_SMEM_SORT: pages up to this many records sort in one block (bitonic)
DIGITS = 12                        # LGW_LIST_DIGITS
CTILE = 2048                       # LGW_LIST_CTILE: records per compaction tile
STILE = 4096                       # LGW_LIST_STILE: keys per LSD tile
B24 = 1 << 24                      # the first index whose top byte (digit 8) is not 0
NEVER = "never"
I64_MIN, I64_MAX = int(np.iinfo(np.int64).min), int(np.iinfo(np.int64).max)
_FLIP = np.uint64(0x7FFF_FFFF_FFFF_FFFF)


def keys(ts) -> np.ndarray:
    """kd of every timestamp: ascending kd is descending ts"""
    return np.asarray(ts, np.int64).view(np.uint64) ^ _FLIP


def ts_of(kd) -> np.ndarray:
    return (np.asarray(kd, np.uint64) ^ _FLIP).view(np.int64)


def reference(ts) -> np.ndarray:
    """record indices newest first, equal timestamps in index order.  (~ts is descending ts without -ts's overflow at INT64_MIN)"""
    return np.argsort(~np.asarray(ts, np.int64), kind="stable")


def sort_path(count: int) -> str:
    return "bitonic" if count <= SMEM_SORT else "lsd"


# ---- model of the select's passes ----------------------------------------------------------------------------------------
@dataclass
class Trace:
    bounds: tuple                  # ((kd, index), (kd, index)) of the records at ranks first and first + count - 1
    digits: tuple                  # the 12 digits each pass fixed, per boundary
    under: list                    # per pass: records under the prefixes after the pick (one prefix counted once)
    compact: object                # the pass after which the select compacts, or NEVER
    wide: bool                     # pass 8 saw a record with index byte 3 != 0 under a boundary's prefix

    @property
    def depth(self) -> int:
        a, b = self.digits
        return next((d for d in range(DIGITS) if a[d] != b[d]), DIGITS)


class Model:
    """The select of k_list_hist / k_list_pick on one table.  Passes 0 - 7 histogram the distinct kd values under a boundary's
    prefix weighted by their counts, passes 8 - 11 the indices of the records whose kd is the boundary's; either way the
    records under a prefix are a contiguous range of a sorted array, which each pass narrows to its picked digit.  (Reading
    the candidate list instead of the column does not change a histogram: the candidates are the records under the prefixes.)"""

    def __init__(self, ts):
        self.kd = keys(ts)
        self.n = int(self.kd.size)
        self.uk, cnt = np.unique(self.kd, return_counts=True)
        self.cnt = cnt.astype(np.int64)
        self._members = {}
        self._hist = {}                        # (d, lo, hi, kd) -> histogram: pages of one table share their first passes

    def members(self, k) -> np.ndarray:
        k = int(k)
        if k not in self._members:
            self._members[k] = np.flatnonzero(self.kd == np.uint64(k))
        return self._members[k]

    def _sorted(self, d: int, kd):
        """the sorted array pass d reads and the shift of its digit"""
        return (self.uk, 56 - 8 * d) if d < 8 else (self.members(kd), 24 - 8 * (d - 8))

    def _histogram(self, d: int, lo: int, hi: int, kd) -> np.ndarray:
        key = (d, lo, hi, kd)
        if key not in self._hist:
            a, s = self._sorted(d, kd)
            dig = ((a[lo:hi] >> a.dtype.type(s)) & a.dtype.type(255)).astype(np.intp)
            h = np.bincount(dig, weights=self.cnt[lo:hi] if d < 8 else None, minlength=256)
            self._hist[key] = h.astype(np.int64)
        return self._hist[key]

    def _narrow(self, d: int, lo: int, hi: int, kd, g: int) -> tuple:
        """the part of [lo, hi) whose digit d is g: contiguous, as every element of [lo, hi) shares the digits before d"""
        a, s = self._sorted(d, kd)
        base = (int(a[lo]) >> (s + 8) << (s + 8)) | (g << s)
        top = base + (1 << s)
        part = a[lo:hi]
        z = hi if top >= 1 << 64 else lo + int(np.searchsorted(part, a.dtype.type(top), "left"))
        return lo + int(np.searchsorted(part, a.dtype.type(base), "left")), z

    def select(self, first: int, count: int) -> Trace:
        assert 0 < count and 0 <= first and first + count <= self.n
        cap = self.n // CAND_DIV
        rank = [first, first + count - 1]
        span = [(0, self.uk.size), (0, self.uk.size)]
        picked = ([], [])
        under, compact, wide, bound_kd = [], NEVER, False, None
        for d in range(DIGITS):
            if d == 8:                                                      # kd fixed: the records of each boundary's kd next
                bound_kd = [int(self.uk[span[b][0]]) for b in (0, 1)]
                span = [(0, self.members(k).size) for k in bound_kd]
            grp = [0, 0]
            for b in (0, 1):
                lo, hi = span[b]
                kd = None if d < 8 else bound_kd[b]
                h = self._histogram(d, lo, hi, kd)
                wide |= d == 8 and bool(h[1:].any())
                c = np.cumsum(h)
                g = int(np.searchsorted(c, rank[b], side="right"))          # first digit whose cumulative count covers the rank
                rank[b] -= int(c[g - 1]) if g else 0
                grp[b] = int(h[g])
                span[b] = self._narrow(d, lo, hi, kd, g)
                picked[b].append(g)
            u = grp[0] if picked[0] == picked[1] else grp[0] + grp[1]
            under.append(u)
            if compact == NEVER and d + 1 < DIGITS and u <= cap:
                compact = d
        idx = [int(self.members(bound_kd[b])[span[b][0]]) for b in (0, 1)]
        return Trace(((bound_kd[0], idx[0]), (bound_kd[1], idx[1])), (tuple(picked[0]), tuple(picked[1])), under, compact, wide)


# ---- tables ------------------------------------------------------------------------------------------------------------
@dataclass
class Page:
    first: int
    count: int
    depth: int | None = None       # claimed divergence depth
    compact: object = None         # claimed compaction pass (an int or NEVER); None: no claim
    wide: bool = False             # claimed: records with index byte 3 != 0 under a boundary prefix at pass 8


@dataclass
class Table:
    name: str
    family: str
    ts: np.ndarray
    pages: list = field(default_factory=list)
    identity: bool = False         # every timestamp equal: the reference is the identity

    @property
    def n(self) -> int:
        return int(self.ts.size)

    @cached_property
    def order(self) -> np.ndarray:
        return np.arange(self.n, dtype=np.int64) if self.identity else reference(self.ts)

    def expected(self, page: Page) -> np.ndarray:
        if self.identity:
            return np.arange(page.first, page.first + page.count, dtype=np.int64)
        return self.order[page.first:page.first + page.count]


def _pages(n: int, firsts, counts, **claim) -> list:
    out, seen = [], set()
    for f in firsts:
        for c in counts:
            c = min(c, n - f)
            if 0 <= f < n and c > 0 and (f, c) not in seen:
                seen.add((f, c))
                out.append(Page(f, c, **claim))
    return out


def _c5_ts(rng, n: int) -> np.ndarray:
    """BASELINE config 5's timestamps: uniform over the 400 days before NOW, microseconds"""
    return to_us(NOW) - rng.integers(0, 400 * DAY_US, n, dtype=np.int64)


def _bursts(rng, ts: np.ndarray, n_bursts: int, max_len: int) -> None:
    """runs of 2 .. max_len consecutive records that share their first record's whole second (in place)"""
    n = ts.size
    starts = rng.integers(0, n, n_bursts)
    lens = rng.integers(2, max_len + 1, n_bursts)
    pos = np.repeat(starts, lens) + np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens)
    val = np.repeat(ts[starts] // SEC * SEC, lens)
    keep = pos < n
    ts[pos[keep]] = val[keep]


def _rank_of(ts: np.ndarray, index_list, i: int) -> int:
    """rank of record i among records whose timestamp equals ts[i] is its position in index order"""
    return int((ts > ts[i]).sum()) + int(np.searchsorted(index_list, i))


def _run_page(ts: np.ndarray, a: int, b: int, **claim) -> Page:
    """the page from record a to record b (a < b, equal timestamps)"""
    assert ts[a] == ts[b] and a < b
    members = np.flatnonzero(ts == ts[a])
    ra = _rank_of(ts, members, a)
    return Page(ra, int(np.searchsorted(members, b)) - int(np.searchsorted(members, a)) + 1, **claim)


# -- past 2^24 records --
def equal_2_24() -> Table:
    """n = 2^24 + 2^20 + 3 records of one timestamp: every boundary key differs from the other only in its index"""
    n = B24 + (1 << 20) + 3
    ts = np.full(n, to_us(NOW) // SEC * SEC, np.int64)
    pages = _pages(n, (0, (1 << 16) - 1, (1 << 16) + 1, B24 - 25, B24 - 1, B24, n - 25, n - 1), (25,))
    pages += [Page(B24 + 1, 25, depth=11, compact=8, wide=True),               # both boundaries past 2^24: 2^20 + 3 <= n / 16
              Page(B24 - 12, 25, depth=8, compact=9, wide=True),               # across 2^24
              Page(B24 - 1, 2, depth=8, compact=9, wide=True),
              Page((1 << 16) - 1, 2, depth=9, compact=9),                      # 0x0000FFFF, 0x00010000
              Page(255, 2, depth=10, compact=9),                               # 0x000000FF, 0x00000100
              Page(259, 5, depth=11, compact=9),
              Page(B24 - (1 << 19), (1 << 20) + 1, depth=8, wide=True),        # a 2^20-row page across 2^24
              Page(0, n, depth=8, wide=True)]                                  # the full listing
    return Table("equal_2^24", "past_2^24", ts, pages, identity=True)


def c5_20m() -> Table:
    """20 M C5 timestamps with bursts of equal whole seconds; two runs of equal timestamps straddle index 2^24: the newest
    records (indices 2^24 - 40 .. 2^24 + 39) and a run in the middle (2^24 - 70 .. 2^24 - 41 and 2^24 + 40 .. 2^24 + 69)"""
    n = 20_000_003
    rng = np.random.default_rng([24, n])
    ts = _c5_ts(rng, n)
    _bursts(rng, ts, 400_000, 48)
    new = (int(ts.max()) // SEC + 1) * SEC
    ts[B24 - 40:B24 + 40] = new
    mid = int(np.median(ts[:1000])) // SEC * SEC + 1                              # (no burst is at an odd microsecond)
    ts[B24 - 70:B24 - 40] = mid
    ts[B24 + 40:B24 + 70] = mid
    pages = _pages(n, (0, (1 << 16) - 1, (1 << 16) + 1, B24 - 25, B24 - 1, B24, B24 + 1, n - 25, n - 1), (25,))
    pages += [Page(30, 20, depth=8, wide=True), Page(39, 2, depth=8, wide=True),
              _run_page(ts, B24 - 45 - 25, B24 + 45, depth=8, wide=True),
              _run_page(ts, B24 - 41, B24 + 40, depth=8, wide=True),
              Page(B24 - (1 << 19), (1 << 20) + 1), Page(0, n)]
    return Table("c5_20m", "past_2^24", ts, pages)


# -- divergence depth --
def depth_kd(d: int) -> Table:
    """divergence at digit d < 8: a cluster of records whose kd shares its first d bytes, the smallest with byte d = 0x00 and
    the largest with 0xFF, among records whose kd is random; pages from the cluster's first record and to its last"""
    n, m = 50_000 + d, 12_000
    rng = np.random.default_rng([31, d])
    kd = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    if d:
        top = np.uint64(~((1 << (64 - 8 * d)) - 1) & ((1 << 64) - 1))
        at = rng.choice(n, m, replace=False)
        kd[at] = (kd[at[0]] & top) | (kd[at] & ~top)
        byte = np.uint64(255 << (56 - 8 * d))
        kd[at[1]] &= ~byte
        kd[at[2]] |= byte
        inside = (kd & top) == (kd[at[0]] & top)
        first, size = int((kd[~inside] < kd[at[0]]).sum()), int(inside.sum())
    else:
        kd[0], kd[1] = 0, (1 << 64) - 1
        first, size = 0, n
    pages = [Page(first, size, depth=d, compact=d), Page(first, 8000, depth=d), Page(first + size - 8000, 8000, depth=d),
             Page(first + size // 2, 25)]
    return Table("depth_%d" % d, "depth", ts_of(kd), pages)


def depth_index() -> Table:
    """divergence at digits 9, 10 and 11: 10 000 records of one timestamp at indices 60 000 .. 69 999, pages whose boundaries
    are two of them across index 2^16 (0x0000FFFF / 0x00010000), across 0xF0FF / 0xF100 and inside 0xF1xx"""
    n = 70_000
    rng = np.random.default_rng(32)
    ts = _c5_ts(rng, n)
    ts[60_000:] = int(np.median(ts)) // SEC * SEC + 1
    pages = [_run_page(ts, 65_535, 65_536, depth=9, compact=10), _run_page(ts, 65_535 - 100, 65_536 + 200, depth=9, compact=10),
             _run_page(ts, 0xF0FF, 0xF100, depth=10, compact=10), _run_page(ts, 61_700, 61_710, depth=11, compact=10),
             _run_page(ts, 60_000, 69_999, depth=9), Page(0, 25), Page(0, n)]
    return Table("depth_index", "depth", ts, pages)


# -- compaction pass --
def full_range() -> Table:
    """timestamps over all of int64 (every top byte of kd), with INT64_MIN / MAX, datetime.min / max and -1, 0, 1: the records
    under a boundary's first digit are already at most n / 16, so the select compacts after pass 0"""
    n = 100_001
    rng = np.random.default_rng(40)
    ts = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    special = [I64_MIN, I64_MAX, to_us(datetime.min), to_us(datetime.max), -1, 0, 1]
    ts[rng.choice(n, 3 * len(special), replace=False)] = special * 3
    ts[0], ts[-1] = I64_MIN, I64_MAX
    return Table("full_range", "compaction", ts, _pages(n, (0, n // 2, n - 25), (25,), compact=0) + [Page(0, n), Page(n // 3, 9000)])


def prefix(p: int) -> Table:
    """every kd shares its first p bytes (those of NOW), the rest random: each digit-p group holds about n / 256 records, so the
    select compacts after pass p (p = 7: only 256 distinct timestamps, every one shared by ~390 records)"""
    n = 100_000 + p
    rng = np.random.default_rng([41, p])
    top = np.uint64(~((1 << (64 - 8 * p)) - 1) & ((1 << 64) - 1))
    kd = (keys(np.array([to_us(NOW)]))[0] & top) | (rng.integers(0, 1 << 64, n, dtype=np.uint64) & ~top)
    return Table("prefix_%d" % p, "compaction", ts_of(kd), _pages(n, (0, n // 2, n - 25), (25,), compact=p) + [Page(0, n)])


def every_8th() -> Table:
    """200 000 records, every 8th of one (newest) timestamp: 25 000 > n / 16 of them, 8 192 in each 2^16 block of indices, so a
    page inside one block compacts after pass 9 and a page across a block edge after pass 10"""
    n = 200_000
    rng = np.random.default_rng(42)
    ts = _c5_ts(rng, n)
    ts[::8] = (int(ts.max()) // SEC + 1) * SEC
    pages = [Page(0, 25, compact=9), Page(4000, 25, compact=9), Page(8190, 4, depth=9, compact=10), Page(24_990, 10, compact=9),
             Page(0, 25_000), Page(20_000, 10_000)]
    return Table("every_8th", "compaction", ts, pages)


def equal(n: int, compact) -> Table:
    """n records of one timestamp.  n = 40 000 and 4 096: the 256 records of one block of indices (digits 8 - 10 fixed) are at
    most n / 16, so a page inside a block compacts after pass 10; n = 4 095 and 1 000: they are more, and it never does --
    except in the last block of 4 095, which holds 255 = n / 16"""
    ts = np.full(n, to_us(NOW) // SEC * SEC, np.int64)
    pages = _pages(n, (0, 1, n // 2), (25,), compact=compact)
    pages += [Page(n - 25, 25, compact=10 if n == 4095 else compact), Page(255, 2, depth=10), Page(0, n)]
    return Table("equal_%d" % n, "compaction", ts, pages, identity=True)


def random_15() -> Table:
    """n < 16: the candidate list has room for none (n / 16 = 0), the select never compacts"""
    rng = np.random.default_rng(43)
    ts = _c5_ts(rng, 15)
    ts[3:6] = ts[10]
    return Table("random_15", "compaction", ts, [Page(f, c, compact=NEVER) for f in range(15) for c in range(1, 16 - f)])


# -- key extremes --
def extremes_10m() -> Table:
    """10 M C5 timestamps with INT64_MIN, INT64_MAX, -1, 0, 1, datetime.min / max and one value for every top byte of kd mixed
    in, three records each (INT64_MAX first and INT64_MIN last in the table)"""
    n = 10_000_001
    rng = np.random.default_rng(50)
    ts = _c5_ts(rng, n)
    c5_lo, c5_hi = int(ts.min()), int(ts.max())
    top = ts_of((np.arange(256, dtype=np.uint64) << np.uint64(56)) | rng.integers(0, 1 << 56, 256, dtype=np.uint64))
    special = np.array([I64_MIN, I64_MAX, -1, 0, 1, to_us(datetime.min), to_us(datetime.max)] + top.tolist(), np.int64)
    ts[rng.choice(n, 3 * special.size, replace=False)] = np.tile(special, 3)
    ts[0], ts[-1] = I64_MAX, I64_MIN
    above = int((ts > c5_hi).sum())
    below = int((ts >= c5_lo).sum())
    zero = int((ts > 0).sum())
    pages = [Page(0, 25, compact=0), Page(n - 25, 25, compact=0), Page(n - 1, 1), Page(0, 1000), Page(n - 1000, 1000),
             Page(above - 10, 20), Page(below - 10, 20), Page(zero - 5, 10), Page(n // 2, 25), Page(0, 65_537), Page(0, n)]
    return Table("extremes_10m", "extremes", ts, pages)


# -- table sizes at the kernels' edges --
SIZES = (1, 2, 3, 15, 16, 17, 31, 32, 33, 63, 64, 65, 2047, 2048, 2049, 4095, 4096, 4097, 65535, 65536, 65537)


def size_table(n: int) -> Table:
    """n records of heavily tied whole-second timestamps (about four per value); every page for n <= 33, a ladder above"""
    rng = np.random.default_rng([60, n])
    ts = to_us(NOW) // SEC * SEC - rng.integers(0, n // 4 + 1, n, dtype=np.int64) * SEC
    if n <= 33:
        pages = [Page(f, c) for f in range(n) for c in range(1, n - f + 1)]
    else:
        firsts = (0, 1, 31, 32, 33, n // 2, n - 33, n - 32, n - 31, n - 2, n - 1)
        pages = _pages(n, firsts, (1, 2, 31, 32, 33, 2047, 2048, 2049, 4095, 4096, 4097, 8192, 8193, n))
    return Table("size_%d" % n, "sizes", ts, pages)


# -- page sizes at the sort's edges --
SORT_COUNTS = (4095, 4096, 4097, 8191, 8192, 8193, 12_287, 12_288, 12_289, 16_384, 65_535, 65_536, 65_537, (1 << 20) + 1)


def ties_10m() -> Table:
    """10 M C5 timestamps cut to whole minutes (~17 records per value) and every 37th record of one timestamp (270 271 records):
    inside a page the LSD passes' stable order decides the order of equal keys"""
    n = 10_000_005
    rng = np.random.default_rng(70)
    ts = _c5_ts(rng, n) // (60 * SEC) * (60 * SEC)
    big = int(np.median(ts[:1000])) // (60 * SEC) * (60 * SEC) + SEC
    ts[::37] = big
    run = int((ts > big).sum())
    pages = []
    for c in SORT_COUNTS:
        pages += [Page(0, c), Page(n // 2 - c // 2, c), Page(n - c, c), Page(run + 1000, c)]
    pages += [Page(run - 3, 25), Page(n // 2, 25), Page(0, n)]
    return Table("ties_10m", "sort_edges", ts, pages)


BUILDERS = {"equal_2^24": equal_2_24, "c5_20m": c5_20m}
BUILDERS.update({"depth_%d" % d: (lambda d=d: depth_kd(d)) for d in range(8)})
BUILDERS["depth_index"] = depth_index
BUILDERS["full_range"] = full_range
BUILDERS.update({"prefix_%d" % p: (lambda p=p: prefix(p)) for p in range(1, 8)})
BUILDERS["every_8th"] = every_8th
BUILDERS.update({"equal_%d" % n: (lambda n=n, c=c: equal(n, c)) for n, c in ((40_000, 10), (4096, 10), (4095, NEVER), (1000, NEVER))})
BUILDERS["random_15"] = random_15
BUILDERS["extremes_10m"] = extremes_10m
BUILDERS.update({"size_%d" % n: (lambda n=n: size_table(n)) for n in SIZES})
BUILDERS["ties_10m"] = ties_10m
LARGE = ("equal_2^24", "c5_20m", "extremes_10m", "ties_10m")      # tables of 10 M records and more


def build(name: str) -> Table:
    return BUILDERS[name]()
