"""`tokens_usage` files written by the installed sqlite3 from a seed, for the loader's tests (test_usage_load_cpu.py,
test_usage_load_gpu.py), and what sqlite3 itself reads back from them under UsageTable.load_tokens_usage_db's record rules."""
from __future__ import annotations

import math
import random
import sqlite3
from datetime import datetime, timedelta

import numpy as np

from llmapigateway_b200.usage import UsageTable, to_us

SCHEMA = """CREATE TABLE tokens_usage (id INTEGER PRIMARY KEY AUTOINCREMENT, timestamp DATETIME NOT NULL,
    prompt_tokens INTEGER DEFAULT 0, completion_tokens INTEGER DEFAULT 0, total_tokens INTEGER DEFAULT 0,
    reasoning_tokens INTEGER DEFAULT 0, cached_tokens INTEGER DEFAULT 0, cost REAL DEFAULT 0.0, model TEXT, provider TEXT)"""
INSERT = ("INSERT INTO tokens_usage (timestamp, prompt_tokens, completion_tokens, total_tokens, reasoning_tokens, cached_tokens,"
          " cost, model, provider) VALUES (?,?,?,?,?,?,?,?,?)")
T0 = datetime(2026, 9, 21, 6, 57, 17, 47518)

GOOD_TS = ["2026-01-02T03:04:05", "2026-01-02T03:04:05.000001", "0001-01-01T00:00:00", "9999-12-31T23:59:59.999999",
           "2024-02-29T12:00:00", "1969-12-31T23:59:59.5".ljust(26, "0")]
BAD_TS = ["2026-01-02 03:04:05", "2026-01-02T03:04:05.000000", "2026-01-02T03:04:05+00:00", "2026-02-30T00:00:00",
          "2026-01-02T24:00:00", "2026-01-02T03:04:05 ", "2023-02-29T00:00:00", "0000-01-01T00:00:00", "2026-1-02T03:04:05",
          "2026-01-02T03:04:60", "2026-13-01T00:00:00", "2026-01-02T03:04:05.5", "x" * 19, ""]
NAMES = ["gpt-4o", "provider-00/model-00", "", "é-modèle", "模型", "zz", "a", "provider-03/model-03"]


def _ts(rng) -> str:
    return (T0 - timedelta(microseconds=int(rng.integers(0, 400 * 86400 * 10**6)))).isoformat()


def _row(rng, names=NAMES):
    tok = [int(x) for x in rng.integers(0, 2**17, 5)]
    m = names[int(rng.integers(0, len(names)))] if rng.random() > 0.05 else None
    p = names[int(rng.integers(0, len(names)))] if rng.random() > 0.3 else None
    return (_ts(rng), *tok, int(rng.integers(0, 10**6)) * 1e-6, m, p)


def create(path, page_size=4096, auto_vacuum=None) -> sqlite3.Connection:
    conn = sqlite3.connect(path)
    conn.execute(f"PRAGMA page_size = {page_size}")
    if auto_vacuum:
        conn.execute(f"PRAGMA auto_vacuum = {auto_vacuum}")
    conn.execute(SCHEMA)
    conn.execute("CREATE INDEX idx_tokens_usage_timestamp ON tokens_usage (timestamp)")
    return conn


def fill(path, n, seed, page_size=4096, auto_vacuum=None, names=NAMES):
    rng = np.random.default_rng(seed)
    conn = create(path, page_size, auto_vacuum)
    conn.executemany(INSERT, (_row(rng, names) for _ in range(n)))
    conn.commit()
    return conn


def fam_values(path, seed):
    """every storage class in every column: integers of each width and at +-2^31, REAL / TEXT / BLOB token counts, -0.0,
    +-inf, NULL and default costs, accepted and refused timestamps, invalid UTF-8, empty and non-ASCII names"""
    rng = np.random.default_rng(seed)
    conn = create(path, 1024)
    ints = [0, 1, -1, 127, -128, 128, 32767, -32768, 32768, 2**23 - 1, -2**23, 2**23, 2**31 - 1, -2**31, 2**31, -2**31 - 1,
            2**47, -2**47 - 5, 2**63 - 1, -2**63, None]
    rows = []
    for v in ints:
        for col in range(5):
            tok = [int(x) for x in rng.integers(0, 100, 5)]
            tok[col] = v
            rows.append((_ts(rng), *tok, 0.5, "m", "p"))
    for v in [1.5, 2.0, "12", b"\x01", "abc"]:
        rows.append((_ts(rng), v, 1, 2, 3, 4, 0.25, "m", None))
    for c in [-0.0, 0.0, math.inf, -math.inf, None, 3, -(2**63), 2**62 + 1, 1e-300, "0.5", b"\x00", 7.25]:
        rows.append((_ts(rng), 1, 2, 3, 4, 5, c, "m", "p"))
    for ts in GOOD_TS + BAD_TS + [b"2026-01-02T03:04:05", 20260102, 1.5, None]:
        if ts is None:
            continue
        rows.append((ts, 1, 2, 3, 4, 5, 0.5, "m", "p"))
    for m in NAMES + [b"blob", 42]:
        rows.append((_ts(rng), 1, 2, 3, 4, 5, 0.5, m, m))
    conn.executemany(INSERT, rows)
    conn.execute("INSERT INTO tokens_usage (timestamp) VALUES ('2026-03-04T05:06:07')")                # every default
    conn.execute("INSERT INTO tokens_usage (timestamp, model, provider) VALUES ('2026-03-04T05:06:08', CAST(x'ff' AS TEXT), 'p')")
    conn.execute("INSERT INTO tokens_usage (timestamp, model, provider) VALUES ('2026-03-04T05:06:09', 'm', CAST(x'c3' AS TEXT))")
    conn.execute("INSERT INTO tokens_usage (timestamp, model) VALUES ('2026-03-04T05:06:10', CAST(x'eda080' AS TEXT))")
    conn.execute("INSERT INTO tokens_usage (timestamp, model) VALUES ('2026-03-04T05:06:11', 'only-refused')")
    conn.execute("UPDATE tokens_usage SET prompt_tokens = 1.5 WHERE model = 'only-refused'")
    conn.commit()
    conn.close()


def fam_spill(path, seed, page_size):
    """model and provider texts spilling into 1, 2 and many overflow pages"""
    rng = np.random.default_rng(seed)
    conn = create(path, page_size)
    rows = []
    for k in range(60):
        ln = [page_size - 40, page_size + 100, 2 * page_size + 7, 9 * page_size + 3, int(rng.integers(1, 3 * page_size))][k % 5]
        m = "M%d" % (k % 7) + "é" * (ln // 2)
        p = "P" * int(rng.integers(0, 2 * page_size)) if k % 3 else None
        rows.append((_ts(rng), k, 2, 3, 4, 5, k * 0.5, m, p))
        rows.append(_row(rng))
    conn.executemany(INSERT, rows)
    conn.commit()
    conn.close()


def fam_deleted(path, seed, vacuum):
    """freelist pages and freeblocks after large deletes (and the same file after VACUUM)"""
    conn = fill(path, 6000, seed, 1024)
    conn.execute("DELETE FROM tokens_usage WHERE id % 3 = 0 OR (id > 1000 AND id < 3000)")
    conn.commit()
    if vacuum:
        conn.execute("VACUUM")
    conn.close()


def fam_short(path, seed):
    """short records: rows written before ALTER TABLE ... ADD COLUMN cost / model / provider"""
    rng = np.random.default_rng(seed)
    conn = sqlite3.connect(path)
    conn.execute(SCHEMA.split(", cost REAL")[0] + ")")
    conn.executemany("INSERT INTO tokens_usage (timestamp, prompt_tokens, completion_tokens, total_tokens, reasoning_tokens,"
                     " cached_tokens) VALUES (?,?,?,?,?,?)", [(_ts(rng), 1, 2, 3, 4, 5) for _ in range(50)])
    conn.execute("ALTER TABLE tokens_usage ADD COLUMN cost REAL DEFAULT 0.0")
    conn.executemany("INSERT INTO tokens_usage (timestamp, cost) VALUES (?,?)", [(_ts(rng), 0.25) for _ in range(20)])
    conn.execute("ALTER TABLE tokens_usage ADD COLUMN model TEXT")
    conn.execute("ALTER TABLE tokens_usage ADD COLUMN provider TEXT")
    conn.executemany(INSERT, (_row(rng) for _ in range(30)))
    conn.commit()
    conn.close()


def families():
    """(name, writer(path, seed)) of every family the tests run"""
    out = []
    for ps, n in ((512, 25000), (1024, 3000), (4096, 5000), (65536, 20000)):
        out.append((f"pages{ps}", lambda p, s, ps=ps, n=n: fill(p, n, s, ps).close()))
    out.append(("root_leaf", lambda p, s: fill(p, 3, s, 4096).close()))
    out.append(("empty", lambda p, s: fill(p, 0, s, 4096).close()))
    for av in ("FULL", "INCREMENTAL"):
        out.append((f"autovacuum_{av}", lambda p, s, av=av: fill(p, 4000, s, 1024, av).close()))
    out.append(("deleted", lambda p, s: fam_deleted(p, s, False)))
    out.append(("vacuumed", lambda p, s: fam_deleted(p, s, True)))
    out.append(("values", fam_values))
    for ps in (512, 4096):
        out.append((f"spill{ps}", lambda p, s, ps=ps: fam_spill(p, s, ps)))
    out.append(("short", fam_short))
    return out


def tree_depth(path) -> int:
    """levels of the tokens_usage b-tree, following the left-most child"""
    conn = sqlite3.connect(path)
    root = conn.execute("SELECT rootpage FROM sqlite_schema WHERE name = 'tokens_usage'").fetchone()[0]
    conn.close()
    data = open(path, "rb").read()
    ps = int.from_bytes(data[16:18], "big") or 65536
    ps = 65536 if ps == 1 else ps
    pg, depth = root, 1
    while True:
        p = data[(pg - 1) * ps:pg * ps]
        o = 100 if pg == 1 else 0
        if p[o] == 13:
            return depth
        c = int.from_bytes(p[o + 12:o + 14], "big")
        pg = int.from_bytes(p[c:c + 4], "big")
        depth += 1


def _iso_ok(s) -> bool:
    try:
        d = datetime.fromisoformat(s)
    except (TypeError, ValueError):
        return False
    return d.tzinfo is None and d.isoformat() == s


def sqlite_expect(path) -> dict:
    """What sqlite3 reads from the file, under the loader's record rules: kept records in id order (ids, the eight-column
    values, models, providers), refused ids, and the next id - 1"""
    conn = sqlite3.connect(path)
    q = ("SELECT id, CAST(timestamp AS BLOB), typeof(timestamp), " +
         ", ".join(f"{c}, typeof({c})" for c in ("prompt_tokens", "completion_tokens", "total_tokens", "reasoning_tokens", "cached_tokens", "cost")) +
         ", CAST(model AS BLOB), typeof(model), CAST(provider AS BLOB), typeof(provider) FROM tokens_usage ORDER BY id")
    kept, refused = [], []
    for r in conn.execute(q):
        rid, ts_b, ts_t = r[0], r[1], r[2]
        ok = ts_t == "text"
        ts = None
        if ok:
            try:
                s = ts_b.decode("utf-8")
                ok = _iso_ok(s)
                ts = to_us(datetime.fromisoformat(s)) if ok else None
            except UnicodeDecodeError:
                ok = False
        tok = []
        for k in range(5):
            v, t = r[3 + 2 * k], r[4 + 2 * k]
            if t == "null":
                v = 0
            elif t != "integer" or not -2**31 <= v < 2**31:
                ok = False
            tok.append(v)
        cost, ct = r[13], r[14]
        if ct == "null":
            cost = math.nan
        elif ct in ("integer", "real"):
            cost = float(cost)
        else:
            ok = False
        texts = []
        for b, t in ((r[15], r[16]), (r[17], r[18])):
            if t == "null":
                texts.append(None)
                continue
            try:
                texts.append(b.decode("utf-8") if t == "text" else None)
                ok = ok and t == "text"
            except UnicodeDecodeError:
                ok = False
        if ok:
            kept.append((rid, ts, tok, cost, texts[0], texts[1]))
        else:
            refused.append(rid)
    seq = conn.execute("SELECT seq FROM sqlite_sequence WHERE name = 'tokens_usage'").fetchone()
    seq = seq[0] if seq else (conn.execute("SELECT max(id) FROM tokens_usage").fetchone()[0] or 0)
    conn.close()
    return {"kept": kept, "refused": refused, "seq": seq}


def inserted_table(expect: dict, table_cls=UsageTable, **kw) -> UsageTable:
    """a table that got the kept records one by one through insert_usage with their stored timestamps, materialised"""
    t = table_cls(**kw)
    for rid, ts, tok, cost, m, p in expect["kept"]:
        d = dict(zip(("prompt_tokens", "completion_tokens", "total_tokens", "reasoning_tokens", "cached_tokens"), tok))
        d.update(cost=None if math.isnan(cost) else cost, model=m, provider=p)
        assert t.insert_usage(d, datetime(1970, 1, 1) + timedelta(microseconds=ts))
    t._materialise()
    return t


def assert_loaded(t: UsageTable, expect: dict):
    """the loaded table against sqlite3's reading of the same file and a table of the kept records inserted one by one"""
    kept = expect["kept"]
    n = len(kept)
    assert len(t) == n and t._dev_n == n and t._dev_cap == n and not t._pending_rows
    assert t._ids.tolist() == [k[0] for k in kept]
    assert t.rejected_ids.tolist() == expect["refused"]
    assert t._seq == expect["seq"]
    ref = inserted_table(expect, engine=object()) if n else None
    h = t._host
    assert h["ts_us"].tolist() == [k[1] for k in kept]
    for c, name in enumerate(UsageTable.COLS[2:7]):
        assert h[name].tolist() == [k[2][c] for k in kept], name
    assert np.array_equal(h["cost"].view(np.int64), np.array([k[3] for k in kept], np.float64).view(np.int64))
    assert t._models == [k[4] for k in kept]
    assert t._providers == [k[5] for k in kept]
    if ref is not None:
        for c in UsageTable.COLS:
            assert h[c].dtype == ref._host[c].dtype and h[c].tobytes() == ref._host[c].tobytes(), c
        assert t._names == ref._names and t._rank == ref._rank

