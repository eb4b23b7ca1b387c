"""GPU: UsageTable.save_tokens_usage_db lays out the `tokens_usage` file on the device (csrc/save.cuh).  The seeded families of
test_usage_save_cpu.py give the same bytes through the device as through the host build.  C5's 10 M records save with
integrity_check ok and within the density target, load back on the same engine into the same device columns, rollups and
listing pages; after cleanup_old_records(180) the file holds exactly the survivors.  Rank shifts, pending rows (no full
upload, the table resident and unchanged), a table past 2^24 records, two saves and saves between rollups on a side stream,
the scratch released after a save and after a failed one, and the ABI's argument checks."""
import ctypes as C
import sqlite3
from datetime import timedelta

import numpy as np
import pytest

import load_cases as L
import save_cases as S
from host_save import HostSaveTable
from llmapigateway_b200.usage import _EPOCH, UsageTable, stats_window, synth_usage_columns
from test_usage_retention_gpu import CountingLib, _download, _new_engine

pytestmark = pytest.mark.gpu
PERIODS = ("hour", "day", "week", "month")


@pytest.fixture(scope="module")
def engine():
    e = _new_engine()
    yield e
    e.close_engine()


def _host_bytes(fill, page_size, path) -> bytes:
    t = fill(HostSaveTable())
    t.save_tokens_usage_db(path, page_size)
    return path.read_bytes()


@pytest.mark.parametrize("page_size", [1024, 4096, 65536])
@pytest.mark.parametrize("name", S.FAMILIES)
def test_family_bytes_equal_host_build(engine, tmp_path, name, page_size):
    t = S.fill(UsageTable(engine), name)
    path = tmp_path / "dev.db"
    assert t.save_tokens_usage_db(path, page_size) == len(t)
    assert path.read_bytes() == _host_bytes(lambda h: S.fill(h, name), page_size, tmp_path / "host.db")
    t.close()


def _vacuum_bytes_per_record(tmp_path, ts, models, tok, cost, m=200_000) -> float:
    """VACUUM INTO of the first m records as a sink-style file writes them: bytes per record"""
    path, vac = tmp_path / "sample.db", tmp_path / "sample-vacuum.db"
    conn = L.create(str(path), 4096)
    stamps = [(_EPOCH + timedelta(microseconds=int(x))).isoformat() for x in ts[:m]]
    conn.executemany(L.INSERT, zip(stamps, *[a[:m].tolist() for a in tok], cost[:m].tolist(), models[:m].tolist(), [None] * m))
    conn.commit()
    conn.execute("VACUUM INTO ?", (str(vac),))
    conn.close()
    return vac.stat().st_size / m


def test_c5_save_load_cleanup(engine, tmp_path):
    n = 10_000_000
    ts, models, tok, cost = synth_usage_columns(n)
    t = UsageTable(engine)
    t.load_columns(ts, models, *tok, cost)
    t._upload()
    before = _download(t)
    path = tmp_path / "c5.db"
    assert t.save_tokens_usage_db(path, 4096) == n
    per = _vacuum_bytes_per_record(tmp_path, ts, models, tok, cost)
    assert path.stat().st_size <= 1.10 * per * n, (path.stat().st_size / n, per)
    conn = sqlite3.connect(path)
    assert conn.execute("PRAGMA integrity_check").fetchall() == [("ok",)]
    conn.close()
    u = UsageTable(engine)
    assert u.load_tokens_usage_db(path) == n and u.rejected == 0
    got = _download(u)
    for c in UsageTable.COLS:
        assert got[c].tobytes() == before[c].tobytes(), c
    now = _EPOCH + timedelta(microseconds=int(ts.max()))
    for period in PERIODS:
        for window in ((None, None), stats_window(period, now)):
            assert np.array_equal(u.rollup_rows(period, *window), t.rollup_rows(period, *window)), (period, window)
    for limit, offset in ((25, 0), (100, 12345), (10, n - 3)):
        assert u.get_latest_usage_records(limit, offset) == t.get_latest_usage_records(limit, offset)
    u.close()
    t.cleanup_old_records(180, now=now)
    assert 0 < len(t) < n
    after = tmp_path / "c5-180.db"
    assert t.save_tokens_usage_db(after, 4096) == len(t)
    conn = sqlite3.connect(after)
    ids = np.fromiter((r[0] for r in conn.execute("SELECT id FROM tokens_usage ORDER BY id")), np.int64)
    conn.close()
    assert np.array_equal(ids, t._ids)
    t.close()


def test_rank_shift_and_pending_rows(engine, tmp_path):
    def fill(t):
        S.fill(t, "c5like")
        t._upload()
        for k in range(20):                   # a name that sorts first moves every rank; the rows stay pending
            t.insert_usage({"prompt_tokens": k, "model": "aaa-first" if k % 2 else "zzz-last", "provider": "q"}, S.T0 + timedelta(seconds=k))
        return t
    t = fill(UsageTable(engine))
    lib = CountingLib(t._lib)
    t._lib = lib
    path = tmp_path / "dev.db"
    assert t.save_tokens_usage_db(path, 4096) == 3020
    assert lib.uploads == 0 and t._dev is not None and not t._pending_rows
    got = _download(t)
    for c in UsageTable.COLS:
        assert got[c].tobytes() == t._host[c][:t._dev_n].tobytes(), c
    assert path.read_bytes() == _host_bytes(fill, 4096, tmp_path / "host.db")
    S.check_file(path, t)
    t.close()


def test_past_2_24_records(engine, tmp_path):
    n = (1 << 24) + 4099
    ts, models, tok, cost = synth_usage_columns(n, seed=9)
    t = UsageTable(engine)
    t.load_columns(ts, models, *tok, cost)
    t._upload()
    path = tmp_path / "big.db"
    assert t.save_tokens_usage_db(path, 8192) == n
    u = UsageTable(engine)
    assert u.load_tokens_usage_db(path) == n
    a, b = _download(t), _download(u)
    for c in UsageTable.COLS:
        assert a[c].tobytes() == b[c].tobytes(), c
    assert np.array_equal(u._ids, t._ids)
    t.close()
    u.close()


def test_engine_reuse_side_stream_and_scratch(engine, tmp_path):
    import torch
    t = S.fill(UsageTable(engine), "spill")
    S.fill(t, "c5like")
    t._upload()
    want = {}
    fresh = _new_engine()
    try:
        f = S.fill(UsageTable(fresh), "spill")
        S.fill(f, "c5like")
        for ps in (1024, 65536):
            f.save_tokens_usage_db(tmp_path / "fresh.db", ps)
            want[ps] = (tmp_path / "fresh.db").read_bytes()
        f.close()
    finally:
        fresh.close_engine()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(2):
        for ps in (1024, 65536):
            t.save_tokens_usage_db(tmp_path / "a.db", ps)
            assert (tmp_path / "a.db").read_bytes() == want[ps]
    assert torch.cuda.mem_get_info()[0] >= free0 - (4 << 20)
    stream = torch.cuda.Stream()
    try:
        engine.set_stream(stream.cuda_stream)
        day = t.rollup_rows("day")
        for ps in (65536, 1024):
            t.save_tokens_usage_db(tmp_path / "b.db", ps)
            assert (tmp_path / "b.db").read_bytes() == want[ps]
            assert np.array_equal(t.rollup_rows("day"), day)
            t.rollup_rows("hour", S.T0 - timedelta(days=3), S.T0)
    finally:
        engine.set_stream(None)
    real = t._save_call
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]               # (the rollups above grew their own scratch)

    def fail(step, *args):
        real(step, *args)
        if step == "plan":
            raise RuntimeError("injected after the plan")
    t._save_call = fail
    with pytest.raises(RuntimeError):
        t.save_tokens_usage_db(tmp_path / "b.db", 4096)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] >= free1 - (4 << 20)
    assert (tmp_path / "b.db").read_bytes() == want[1024]
    t.close()


def test_abi_guards(engine):
    from llmapigateway_b200.usage import _save_text_table
    h = engine._h
    t = S.fill(UsageTable(engine), "c5like")
    t._upload()
    n = len(t)
    cols = t._save_cols()
    ids = np.ascontiguousarray(t._ids, np.int64)
    prov = np.zeros(n, np.int32)
    models, _m = _save_text_table(t._names)
    providers, _p = _save_text_table([None])
    out = np.zeros(5, np.uint64)

    def plan(cols_=cols, n_=n, ids_=ids.ctypes.data, prov_=prov.ctypes.data, m_=C.byref(models), p_=C.byref(providers), ps=4096, o=out.ctypes.data):
        return t._lib.lgw_usage_save_plan(h, cols_, n_, ids_, prov_, m_, p_, ps, o)
    assert t._lib.lgw_usage_save_write(h, out.ctypes.data, None) == -1           # write before a plan
    assert plan(n_=1 << 32) == -1
    assert plan(o=None) == -1 and plan(ids_=None) == -1 and plan(prov_=None) == -1 and plan(m_=None) == -1
    assert plan(ps=512) == -1 and plan(ps=3000) == -1 and plan(ps=131072) == -1
    shifted = (C.c_void_p * 8)(*[cols[k] for k in range(8)])
    shifted[0] = cols[0] + 8
    assert plan(cols_=shifted, n_=n - 1) == -1                                    # a misaligned ts_us column
    empty = type(models)(models.blob, models.off, models.len, 0, 0)
    assert plan(m_=C.byref(empty)) == -1
    bad_prov = prov.copy()
    bad_prov[5] = 1
    assert plan(prov_=bad_prov.ctypes.data) == -1                               # a code outside its text table
    back = ids.copy()
    back[9] = back[8]
    assert plan(ids_=back.ctypes.data) == -1                                    # ids not ascending
    assert plan() == 0 and int(out[3]) == n
    assert t._lib.lgw_usage_save_release(h) == 0
    assert t._lib.lgw_usage_save_write(h, out.ctypes.data, None) == -1           # released: nothing to write
    t.close()
