"""CPU: what the record listing's geometry cases (tests/listing_geometry_cases.py) reach, by the numpy model of the select's
passes -- every claimed divergence depth, compaction pass and index-byte-3 prefix holds, the cases together cover every depth
0 - 11 and every compaction pass 0 - 10 plus "never", both page sorts at their edges -- and the reference itself against a plain
Python sort.  The model's boundary keys are checked against the reference on every page, so that what it reports is about the
records the device has to select."""
import numpy as np
import pytest

import listing_geometry_cases as LG


@pytest.fixture(scope="module")
def traces():
    """name -> (family, n, [(page, trace)]): every page of every case through the model, its boundaries against the reference"""
    out = {}
    for name in LG.BUILDERS:
        t = LG.build(name)
        model = LG.Model(t.ts)
        rows = []
        for p in t.pages:
            tr = model.select(p.first, p.count)
            for (kd, i), rank in zip(tr.bounds, (p.first, p.first + p.count - 1)):
                assert int(t.order[rank]) == i and int(model.kd[i]) == kd, (name, p, rank)
            rows.append((p, tr))
        out[name] = (t.family, t.n, rows)
        del t, model
    return out


def test_reference_is_a_plain_sort_on_small_tables():
    for name in LG.BUILDERS:
        t = LG.build(name)
        if t.n > 110_000:
            continue
        ts = t.ts.tolist()
        want = sorted(range(t.n), key=lambda i: (-ts[i], i))
        assert t.order.tolist() == want, name
        if t.identity:
            assert np.array_equal(LG.reference(t.ts), np.arange(t.n)), name


def test_reference_at_int64_extremes():
    ts = np.array([0, LG.I64_MIN, LG.I64_MAX, -1, 1, LG.I64_MIN, LG.I64_MAX, 0], np.int64)
    assert LG.reference(ts).tolist() == [2, 6, 4, 0, 7, 3, 1, 5]
    assert np.array_equal(LG.ts_of(LG.keys(ts)), ts) and LG.keys(ts)[2] == 0 and LG.keys(ts)[1] == np.uint64(2 ** 64 - 1)


def test_every_claim_holds(traces):
    bad = []
    for name, (_, _, rows) in traces.items():
        for p, tr in rows:
            if p.depth is not None and tr.depth != p.depth:
                bad.append((name, p, "depth", tr.depth))
            if p.compact is not None and tr.compact != p.compact:
                bad.append((name, p, "compact", tr.compact, tr.under))
            if p.wide and not tr.wide:
                bad.append((name, p, "wide"))
    assert not bad, bad[:10]


@pytest.mark.parametrize("d", range(LG.DIGITS))
def test_divergence_depth_covered(traces, d):
    hits = [(name, p) for name, (_, _, rows) in traces.items() for p, tr in rows if p.depth == d and tr.depth == d and p.count > 1]
    assert hits, d
    if d < 8:
        assert any(name == "depth_%d" % d for name, _ in hits)


@pytest.mark.parametrize("p", list(range(LG.DIGITS - 1)) + [LG.NEVER])
def test_compaction_pass_covered(traces, p):
    hits = [(name, pg) for name, (_, _, rows) in traces.items() for pg, tr in rows if pg.compact == p and tr.compact == p]
    assert hits, p
    if p == LG.NEVER:                                              # with n < 16 (no room) and with many equal timestamps
        assert {"random_15", "equal_1000", "equal_4095"} <= {name for name, _ in hits}


def test_compaction_after_pass_0_at_10m(traces):
    _, n, rows = traces["extremes_10m"]
    assert n >= 10_000_000 and sum(tr.compact == 0 for _, tr in rows) >= 2


def test_past_2_24(traces):
    """tables past 2^24 records: pages at the named firsts, pages across rank 2^24, a full listing and a 2^20-row page each; a
    boundary prefix that holds records with index byte 3 != 0 (pass 8 decides), and the lo digit pass 8 picks not 0"""
    firsts = {0, (1 << 16) - 1, (1 << 16) + 1, LG.B24 - 25, LG.B24 - 1, LG.B24, LG.B24 + 1}
    for name in ("equal_2^24", "c5_20m"):
        _, n, rows = traces[name]
        assert n > LG.B24 and n % 2 == 1
        pages = [p for p, _ in rows]
        assert firsts | {n - 25, n - 1} <= {p.first for p in pages}, name
        assert any(p.first < LG.B24 < p.first + p.count for p in pages) and any(p.count >= 1 << 20 for p in pages), name
        assert any(p.first == 0 and p.count == n for p in pages), name
        wide = [tr for p, tr in rows if p.wide]
        assert wide and any(tr.digits[0][8] == 0 and tr.digits[1][8] == 1 for tr in wide), name


def test_table_sizes_at_kernel_edges(traces):
    for n in LG.SIZES:
        _, size, rows = traces["size_%d" % n]
        assert size == n
        pages = {(p.first, p.count) for p, _ in rows}
        if n <= 33:
            assert pages == {(f, c) for f in range(n) for c in range(1, n - f + 1)}
        else:
            assert (0, n) in pages and (n - 1, 1) in pages and (0, 1) in pages
    assert {n % LG.CTILE for n in LG.SIZES if n > LG.CTILE} == {LG.CTILE - 1, 0, 1} and {n % 32 for n in LG.SIZES} >= {31, 0, 1}


def test_page_sizes_at_sort_edges(traces):
    """the heavy-tie 10 M table pages at 4 096 k + {-1, 0, 1} of both sorts, the one-block bound, 2^20 + 1 and the whole table;
    inside the big tie run the stable order of the LSD passes alone orders the page"""
    _, n, rows = traces["ties_10m"]
    assert n >= 10_000_000
    counts = {p.count for p, _ in rows}
    assert set(LG.SORT_COUNTS) | {n} <= counts
    paths = {LG.sort_path(c) for c in counts}
    assert paths == {"bitonic", "lsd"}
    for k in (1, 2, 3, 4, 16):
        edge = {c for c in counts if abs(c - LG.STILE * k) <= 1}
        assert len(edge) >= (3 if k != 4 else 1), k
    assert LG.sort_path(LG.SMEM_SORT) == "bitonic" and LG.sort_path(LG.SMEM_SORT + 1) == "lsd"
    t = LG.build("ties_10m")
    run = int((t.ts > t.ts[0]).sum())                                   # (record 0 is in the big run)
    inside = [tr for p, tr in rows if p.first == run + 1000 and p.count > LG.SMEM_SORT and p.count < 200_000]
    assert len(inside) == 8 and all(tr.bounds[0][0] == tr.bounds[1][0] for tr in inside)   # one timestamp across the page
    assert t.n / np.unique(t.ts).size > 10


def test_key_extremes(traces):
    t = LG.build("extremes_10m")
    kd = LG.keys(t.ts)
    assert t.n >= 10_000_000 and t.ts[0] == LG.I64_MAX and t.ts[-1] == LG.I64_MIN
    assert set(np.unique(kd >> np.uint64(56)).tolist()) == set(range(256))
    assert np.isin([LG.I64_MIN, LG.I64_MAX, -1, 0, 1], t.ts).all()
