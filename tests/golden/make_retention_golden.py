"""Generate tests/golden/retention_cases.json with the UNMODIFIED reference method
(llm_gateway_core/db/tokens_usage_db.py TokensUsageDB.cleanup_old_records, :164-198) -- dev container only.

    python tests/golden/make_retention_golden.py

Every case starts from the same table: rows inserted by SQL with chosen ISO timestamps -- whole seconds (isoformat drops the
fraction) next to neighbours one microsecond later and earlier, records exactly at each cutoff, runs of equal timestamps at
and just below it, records in the future, and the oldest records inserted last (the newest ids are among the deleted).  The
module's `datetime` is patched so that `now` is fixed.  Recorded per case: the surviving ids, the id a following insert_usage
gets, and what the method logged.
"""
import json
import logging
import pathlib
import random
import sqlite3
import sys
import tempfile
from datetime import datetime, timedelta

sys.path.insert(0, "/root/reference")
import llm_gateway_core.db.tokens_usage_db as M  # noqa: E402
from llm_gateway_core.db.tokens_usage_db import TokensUsageDB  # noqa: E402

NOWS = (datetime(2026, 9, 21, 6, 57, 17, 47518), datetime(2026, 9, 21, 6, 57, 17))
RETENTIONS = (180, 0, -3, 1.5, True, 10**9, "x", None)


def _stamps():
    rng = random.Random(180)
    us = timedelta(microseconds=1)
    out = []
    for now in NOWS:
        for r in (180, 0, -3, 1.5, 1):
            c = now - timedelta(days=r)
            whole = c.replace(microsecond=0)
            out += [c - us, c, c + us, whole, whole + us, whole - us, whole + timedelta(seconds=1)]
            out += [c] * 3 + [c - us] * 3 + [whole] * 2
    out += [NOWS[0] - timedelta(seconds=rng.randrange(0, 400 * 86400), microseconds=rng.randrange(10**6)) for _ in range(150)]
    out += [NOWS[0] + timedelta(days=rng.randrange(4, 30), microseconds=rng.randrange(10**6)) for _ in range(10)]
    rng.shuffle(out)
    out += [NOWS[0] - timedelta(days=500 + k, microseconds=k) for k in range(6)]          # oldest last: the newest ids go
    return out


def _rows():
    models = ["gpt-4.1", "claude", None, "modèle-é"]
    return [[t.isoformat(), i % 97, (3 * i) % 101, i % 97 + (3 * i) % 101, i % 5, i % 3, (i % 11) * 1e-6, models[i % 4], "P%d" % (i % 3)]
            for i, t in enumerate(_stamps())]


class _Log(logging.Handler):
    def __init__(self):
        super().__init__(logging.DEBUG)
        self.records = []

    def emit(self, record):
        self.records.append([record.levelname, record.getMessage()])


def run_case(rows, now, retention):
    class FixedNow(datetime):
        @classmethod
        def now(cls, tz=None):
            return now

    db = TokensUsageDB.__new__(TokensUsageDB)          # the constructor hard-codes <reference>/db (read-only), :17-25
    db.db_path = pathlib.Path(tempfile.mkdtemp()) / "t.db"
    db._init_db()
    c = sqlite3.connect(db.db_path)
    c.executemany("INSERT INTO tokens_usage (timestamp, prompt_tokens, completion_tokens, total_tokens, reasoning_tokens, cached_tokens,"
                  " cost, model, provider) VALUES (?,?,?,?,?,?,?,?,?)", rows)
    c.commit(); c.close()
    log, root = _Log(), logging.getLogger()
    saved, level = M.datetime, root.level
    M.datetime = FixedNow
    root.addHandler(log); root.setLevel(logging.DEBUG)
    try:
        ret = db.cleanup_old_records(retention)
    finally:
        root.removeHandler(log); root.setLevel(level)
    try:
        c = sqlite3.connect(db.db_path)
        survivors = [r[0] for r in c.execute("SELECT id FROM tokens_usage ORDER BY id")]
        c.close()
        logging.disable(logging.CRITICAL)
        db.insert_usage({"prompt_tokens": 1})
        logging.disable(logging.NOTSET)
        c = sqlite3.connect(db.db_path)
        next_id = c.execute("SELECT max(id) FROM tokens_usage").fetchone()[0]
        c.close()
    finally:
        M.datetime = saved
    assert ret is None
    return {"now": now.isoformat(), "retention_days": retention, "survivors": survivors, "next_id": next_id, "log": log.records}


def main():
    rows = _rows()
    cases = [run_case(rows, now, r) for now in NOWS for r in RETENTIONS]
    out = pathlib.Path(__file__).resolve().parent / "retention_cases.json"
    json.dump({"generator": "tests/golden/make_retention_golden.py", "sqlite": sqlite3.sqlite_version, "rows": rows, "cases": cases},
              open(out, "w"), ensure_ascii=False)
    print("wrote", out, len(rows), "rows,", len(cases), "cases:", [len(c["survivors"]) for c in cases])


if __name__ == "__main__":
    main()
