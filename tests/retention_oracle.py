"""CPU oracle for deleting old usage records -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates TokensUsageDB.cleanup_old_records (llm_gateway_core/db/tokens_usage_db.py:164-198) over a connection made by
oracle.rollup_oracle.make_db: the cutoff is `(now - timedelta(days=retention_days)).isoformat()` and SQLite runs the
reference's statement, `DELETE FROM tokens_usage WHERE timestamp < ?`, on the ISO text.  Every exception deletes nothing.
Pinned to the unmodified reference by tests/golden/retention_cases.json (tests/test_usage_retention_cpu.py).
"""
from __future__ import annotations

import sqlite3
from datetime import datetime, timedelta


def cleanup_old_records(conn: sqlite3.Connection, retention_days=180, now: datetime | None = None) -> int | None:
    """the number of records deleted; None where the reference logs an error and deletes nothing"""
    try:
        cutoff = ((now if now is not None else datetime.now()) - timedelta(days=retention_days)).isoformat()
        n = conn.execute("DELETE FROM tokens_usage WHERE timestamp < ?", (cutoff,)).rowcount
        conn.commit()
        return n
    except Exception:
        conn.rollback()
        return None


def insert_usage(conn: sqlite3.Connection, timestamp: datetime) -> int:
    """insert_usage (:119-162) of an empty usage dict at `timestamp`: the id AUTOINCREMENT gives it"""
    cur = conn.execute("INSERT INTO tokens_usage (timestamp, prompt_tokens, completion_tokens, total_tokens, reasoning_tokens,"
                       " cached_tokens, cost, model, provider) VALUES (?,0,0,0,0,0,0.0,NULL,NULL)", (timestamp.isoformat(),))
    conn.commit()
    return cur.lastrowid


def ids(conn: sqlite3.Connection) -> list[int]:
    return [r[0] for r in conn.execute("SELECT id FROM tokens_usage ORDER BY id")]


def latest_ids(conn: sqlite3.Connection, limit: int, offset: int) -> list[int]:
    """ids of get_latest_usage_records (:69-117); equal timestamps in id order, the order UsageTable lists them in"""
    return [r[0] for r in conn.execute("SELECT id FROM tokens_usage ORDER BY timestamp DESC, id ASC LIMIT ? OFFSET ?", (limit, offset))]
