"""Usage records on the device and their rollup -- the host-side mirror of
llm_gateway_core/db/tokens_usage_db.py (TokensUsageDB) for rows a10/a11 of SURVEY.md section 8:

  UsageTable.insert_usage(d)         <- TokensUsageDB.insert_usage          (:119-162)  [GPU kernel: append at query time]
  UsageTable.get_aggregated_usage()  <- TokensUsageDB.get_aggregated_usage  (:222-304)  [GPU kernel]
  UsageTable.get_latest_usage_records() <- TokensUsageDB.get_latest_usage_records (:69-117) [GPU kernel: page selection]
  UsageTable.cleanup_old_records()   <- TokensUsageDB.cleanup_old_records   (:164-198)  [GPU kernel: stable compaction]
  UsageTable.load_tokens_usage_db()  <- the tokens_usage file itself        (:37-50)    [GPU kernels: SQLite pages decoded]
  stats_window(period, now)          <- llm_gateway_core/api/v1/stats.py:46-55

Records live as SoA columns (40 B/record) in HBM; `model` is dictionary-encoded at ingest and
ranked in byte order so that ascending rank == the SQL's `model ASC`.  Every accumulator of the
rollup is an integer (see csrc/rollup.cuh), so per-GPU partial tables merge with a plain sum.
"""
from __future__ import annotations

import ctypes as C
import logging
import math
from datetime import datetime, timedelta
from fractions import Fraction
from itertools import compress

import numpy as np

from . import _native

PERIODS = {"hour": 0, "day": 1, "week": 2, "month": 3}
_EPOCH = datetime(1970, 1, 1)
ROLLUP_CELLS = 10
# the record listing merges up to this many rows inserted since the last upload on the host; more, and it uploads the table again
LISTING_PENDING_MAX = 65536
APPEND_MAX = (1 << 32) - 1      # records a device table can hold (lgw_usage_append: n + m < 2^32)

ROW_DTYPE = np.dtype([("bucket", "<i8"), ("model_rank", "<i4"), ("inexact", "<u4"), ("prompt_tokens", "<i8"),
                      ("completion_tokens", "<i8"), ("total_tokens", "<i8"), ("reasoning_tokens", "<i8"),
                      ("cached_tokens", "<i8"), ("cost", "<f8"), ("count", "<i8")])
assert ROW_DTYPE.itemsize == 72


def to_us(dt: datetime) -> int:
    return (dt - _EPOCH) // timedelta(microseconds=1)


def period_label(period: str, bucket: int) -> str:
    """strftime(fmt, timestamp) of tokens_usage_db.py:242-250 for a bucket index."""
    if period == "hour":                      # bucket = day * 24 + hour of day (csrc/rollup.cuh)
        return (_EPOCH + timedelta(days=bucket // 24)).strftime("%Y-%m-%d") + " %02d:00:00" % (bucket % 24)
    if period == "day":
        return (_EPOCH + timedelta(days=bucket)).strftime("%Y-%m-%d")
    if period == "week":
        return "%04d-W%02d" % (bucket // 64, bucket % 64)
    return "%04d-%02d" % (bucket // 12, bucket % 12 + 1)


def _sql_value(cost: float):
    """a stored or summed cost as SQLite hands it out: NaN is NULL"""
    return None if math.isnan(cost) else cost


def sql_sum(costs: list[float]) -> float:
    """SUM(cost) of SQLite 3.45 over REAL values, NaN standing for NULL both ways: NULLs are skipped and nothing left gives
    NULL; +inf with -inf gives NULL, else an infinity gives itself; finite values give their correctly rounded sum, +-inf
    when that exceeds the double range.  (SQLite's compensated sum is within an ulp or so of the correctly rounded one.  When
    finite costs overflow, its result depends on record order -- inf or NULL; costs near 1e308 are out of any real use.)"""
    vals = [c for c in costs if not math.isnan(c)]
    if not vals:
        return math.nan
    pos, neg = math.inf in vals, -math.inf in vals
    if pos or neg:
        return math.nan if pos and neg else (math.inf if pos else -math.inf)
    try:
        return math.fsum(vals)
    except OverflowError:                         # an intermediate sum left the double range: sum exactly, then round
        exact = sum(map(Fraction, vals))
        try:
            return float(exact)
        except OverflowError:
            return math.inf if exact > 0 else -math.inf


class UsageDbNotModelled(Exception):
    """A `tokens_usage` file or table the loader does not decode: WAL mode, a text encoding other than UTF-8, reserved bytes
    per page, other payload fractions, another schema, or WITHOUT ROWID.  Nothing was loaded."""


class UsageDbCorrupt(Exception):
    """A structurally damaged `tokens_usage` file (see csrc/load.cuh LoadError).  Nothing was loaded."""


# PRAGMA table_info(tokens_usage) of tokens_usage_db.py:37-50 (and gateway.SqliteUsageSink)
TOKENS_USAGE_INFO = [(0, "id", "INTEGER", 0, None, 1), (1, "timestamp", "DATETIME", 1, None, 0)] + [
    (k, c, "INTEGER", 0, "0", 0) for k, c in enumerate(("prompt_tokens", "completion_tokens", "total_tokens", "reasoning_tokens", "cached_tokens"), 2)] + [
    (7, "cost", "REAL", 0, "0.0", 0), (8, "model", "TEXT", 0, None, 0), (9, "provider", "TEXT", 0, None, 0)]
LOAD_ERRORS = {1: "a page number outside the file", 2: "a b-tree page of another type", 3: "a cell outside its page",
               4: "a payload larger than the file or a broken overflow chain", 5: "a record header that does not fit its payload",
               6: "a page reached twice, a level mixing interior and leaf pages, or a tree too deep",
               8: "a rowid not above the one before it (duplicate or misordered cells)"}
LOAD_ID_STORED = 7
LOAD_MAX_BYTES = 1 << 33        # lgw_usage_load_decode takes files below this size


def db_geometry(header: bytes, size: int):
    """(page size, page count) of a SQLite file from its first 100 bytes and its size; UsageDbNotModelled for a file the
    loader does not decode, UsageDbCorrupt for a header that is not SQLite's.  The page count is the header's when bytes
    92-95 equal 24-27, else the file size's, and never more pages than the file holds."""
    if len(header) < 100 or header[:16] != b"SQLite format 3\x00":
        raise UsageDbCorrupt("not a SQLite 3 file")
    ps = int.from_bytes(header[16:18], "big")
    ps = 65536 if ps == 1 else ps
    if ps < 512 or ps & (ps - 1):
        raise UsageDbCorrupt(f"page size {ps}")
    if header[18] == 2 or header[19] == 2:
        raise UsageDbNotModelled("WAL-mode file")
    if header[20] != 0:
        raise UsageDbNotModelled(f"{header[20]} reserved bytes per page")
    if tuple(header[21:24]) != (64, 32, 32):
        raise UsageDbNotModelled(f"payload fractions {tuple(header[21:24])}")
    if int.from_bytes(header[56:60], "big") != 1:
        raise UsageDbNotModelled("text encoding other than UTF-8")
    n_pages = int.from_bytes(header[28:32], "big") if header[92:96] == header[24:28] else size // ps
    return ps, min(n_pages, size // ps)


def read_tokens_usage_snapshot(db_path, alloc, free) -> dict:
    """The bytes of a `tokens_usage` file as one consistent snapshot, with what the loader needs from SQLite itself.  Inside one
    read transaction (BEGIN, then a SELECT on tokens_usage: SQLite rolls back a hot journal and takes a SHARED lock, and in
    rollback-journal mode no writer can change the file while it is held) the schema row, PRAGMA table_info and
    sqlite_sequence are read, and the file is read into alloc(size) (a uint8 array; given to free() if the call fails).  A file
    the process may not write is opened read-only; SQLite then refuses to read it past a hot journal (UsageDbNotModelled).
    Files of 2^33 bytes (8 GiB) or more are not decoded either."""
    import os
    import sqlite3
    from urllib.parse import quote
    if os.path.getsize(db_path) >= LOAD_MAX_BYTES:
        raise UsageDbNotModelled(f"a file of {os.path.getsize(db_path)} bytes: the loader decodes files below 2^33 bytes")
    mode = "rw" if os.access(db_path, os.W_OK) else "ro"
    conn = sqlite3.connect(f"file:{quote(os.fspath(db_path))}?mode={mode}", uri=True, isolation_level=None)
    try:
        conn.execute("BEGIN")
        try:
            conn.execute("SELECT 1 FROM tokens_usage LIMIT 1").fetchall()
        except sqlite3.OperationalError as e:                 # no such table, or a hot journal a read-only file cannot roll back
            raise UsageDbNotModelled(str(e)) from None
        except sqlite3.DatabaseError as e:                    # SQLite itself finds the file malformed
            raise UsageDbCorrupt(str(e)) from None
        row = conn.execute("SELECT rootpage FROM sqlite_schema WHERE type = 'table' AND name = 'tokens_usage'").fetchone()
        if not row or not row[0]:
            raise UsageDbNotModelled("tokens_usage is not a table (a view or a virtual table)")
        root = row[0]
        info = conn.execute("PRAGMA table_info(tokens_usage)").fetchall()
        wr = conn.execute("SELECT wr FROM pragma_table_list WHERE schema = 'main' AND name = 'tokens_usage'").fetchone()
        if info != TOKENS_USAGE_INFO or (wr and wr[0]):
            raise UsageDbNotModelled("tokens_usage has another schema or is WITHOUT ROWID")
        try:
            seq = conn.execute("SELECT seq FROM sqlite_sequence WHERE name = 'tokens_usage'").fetchone()
        except sqlite3.OperationalError:
            seq = None
        seq = seq or conn.execute("SELECT max(id) FROM tokens_usage").fetchone()
        size = os.path.getsize(db_path)
        buf = alloc(max(size, 100))
        try:
            with open(db_path, "rb") as f:
                got = f.readinto(memoryview(buf)[:size])
            ps, n_pages = db_geometry(bytes(buf[:min(got, 100)]), got)
        except BaseException:
            free(buf)
            raise
    finally:
        conn.close()                      # (ends the read transaction)
    return {"buf": buf, "size": got, "page_size": ps, "n_pages": n_pages, "root": int(root), "seq": int(seq[0] or 0)}


SAVE_TEXT_NULL, SAVE_TEXT_BAD = 0xFFFFFFFF, 0xFFFFFFFE     # lgw_save_text lengths (include/llmgw_b200.h)
SQL_MAX_LENGTH = 1_000_000_000      # SQLite's default SQLITE_MAX_LENGTH: a longer text is not stored either


class SaveText(C.Structure):
    """lgw_save_text: text k of a table is bytes blob[off[k]:off[k] + len[k]], or NULL / not storable"""
    _fields_ = [("blob", C.c_void_p), ("off", C.c_void_p), ("len", C.c_void_p), ("n", C.c_uint32), ("pad", C.c_uint32)]


def _save_text_table(texts: list) -> tuple:
    """(SaveText, the arrays it points into) for a list of str | None: UTF-8 bytes, NULL for None, BAD for a str that is not
    encodable as UTF-8 (a lone surrogate) or longer than SQL_MAX_LENGTH bytes"""
    raw, lens = [], np.empty(len(texts), np.uint32)
    for k, s in enumerate(texts):
        if s is None:
            b, lens[k] = b"", SAVE_TEXT_NULL
        else:
            try:
                b = s.encode("utf-8")
            except UnicodeEncodeError:
                b = None
            if b is None or len(b) > SQL_MAX_LENGTH:
                b, lens[k] = b"", SAVE_TEXT_BAD
            else:
                lens[k] = len(b)
        raw.append(b)
    off = np.zeros(len(texts) + 1, np.uint64)
    np.cumsum([len(b) for b in raw], out=off[1:])
    blob = np.frombuffer(b"".join(raw) or b"\0", np.uint8)
    t = SaveText(blob.ctypes.data, off.ctypes.data, lens.ctypes.data, len(texts), 0)
    return t, (blob, off, lens)


def _varint(v: int) -> bytes:
    if v >> 56:
        out = [v & 0xFF]
        v >>= 8
        for i in range(8):
            out.append((v & 0x7F) | 0x80)
            v >>= 7
        return bytes(reversed(out))
    out = [v & 0x7F]
    v >>= 7
    while v:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    return bytes(reversed(out))


def _sql_record(values) -> bytes:
    """a SQLite record of ints, strs and None (schema format 4)"""
    types, body = [], b""
    for v in values:
        if v is None:
            types.append(0)
        elif isinstance(v, int):
            if v in (0, 1):
                types.append(8 + v)
                continue
            n, t = next((n, t) for n, t in ((1, 1), (2, 2), (3, 3), (4, 4), (6, 5), (8, 6)) if -(1 << (8 * n - 1)) <= v < 1 << (8 * n - 1))
            types.append(t)
            body += v.to_bytes(n, "big", signed=True)
        else:
            b = v.encode("utf-8")
            types.append(13 + 2 * len(b))
            body += b
    head = b"".join(_varint(t) for t in types)
    return _varint(len(head) + 1) + head + body        # (the schema's headers are short: their size takes one byte)


def _leaf_page(rows, ps: int, first: bool) -> bytes:
    """a table leaf page holding (rowid, record) cells that fit it without spilling; page 1 keeps its first 100 bytes for the
    file header"""
    hdr = 100 if first else 0
    page = bytearray(ps)
    at = ps
    for k, (rowid, rec) in enumerate(rows):
        cell = _varint(len(rec)) + _varint(rowid) + rec
        at -= len(cell)
        page[at:at + len(cell)] = cell
        page[hdr + 8 + 2 * k:hdr + 10 + 2 * k] = at.to_bytes(2, "big")
    assert hdr + 8 + 2 * len(rows) <= at
    page[hdr] = 13
    page[hdr + 3:hdr + 5] = len(rows).to_bytes(2, "big")
    page[hdr + 5:hdr + 7] = (at & 0xFFFF).to_bytes(2, "big")
    return bytes(page)


def _sink_schema() -> list:
    """(type, name, tbl_name, sql) of the sqlite_schema rows SqliteUsageSink creates, as the installed sqlite3 stores them"""
    from .gateway import SqliteUsageSink
    sink = SqliteUsageSink(":memory:")
    try:
        return sink.conn.execute("SELECT type, name, tbl_name, sql FROM sqlite_schema ORDER BY rowid").fetchall()
    finally:
        sink.conn.close()


def _head_pages(ps: int, n_pages: int, table_root: int, index_root: int, seq: int) -> bytes:
    """pages 1 (the 100-byte header and sqlite_schema) and 2 (sqlite_sequence) of a saved file"""
    import sqlite3
    roots = {"tokens_usage": table_root, "sqlite_sequence": 2, "idx_tokens_usage_timestamp": index_root}
    schema = [(k + 1, _sql_record((ty, name, tbl, roots[name], sql))) for k, (ty, name, tbl, sql) in enumerate(_sink_schema())]
    p1 = bytearray(_leaf_page(schema, ps, True))
    v = sqlite3.sqlite_version_info
    h = bytearray(100)
    h[0:16] = b"SQLite format 3\x00"
    h[16:18] = (ps if ps < 65536 else 1).to_bytes(2, "big")
    h[18] = h[19] = 1                                      # rollback journal
    h[21:24] = bytes((64, 32, 32))
    h[24:28] = (1).to_bytes(4, "big")                      # file change counter
    h[28:32] = n_pages.to_bytes(4, "big")
    h[40:44] = (1).to_bytes(4, "big")                      # schema cookie
    h[44:48] = (4).to_bytes(4, "big")                      # schema format
    h[56:60] = (1).to_bytes(4, "big")                      # UTF-8
    h[92:96] = (1).to_bytes(4, "big")                      # version-valid-for == the change counter
    h[96:100] = (v[0] * 1000000 + v[1] * 1000 + v[2]).to_bytes(4, "big")
    p1[:100] = h
    p2 = _leaf_page([(1, _sql_record(("tokens_usage", seq)))] if seq > 0 else [], ps, False)
    return bytes(p1) + p2


def _check_page_size(page_size) -> None:
    if isinstance(page_size, bool) or not isinstance(page_size, int) or not 1024 <= page_size <= 65536 or page_size & (page_size - 1):
        raise ValueError(f"page_size {page_size!r}: a power of two in [1024, 65536]")


class _ReplaceLock:
    """Held while a save replaces the file at db_path: an EXCLUSIVE lock on the file there (SQLite rolls back a hot journal
    when it takes it), nothing when there is none.  A WAL-mode file is refused before any connection is opened; a lock another
    connection holds raises sqlite3.OperationalError at once."""

    def __init__(self, db_path):
        self.db_path, self.conn = db_path, None

    def __enter__(self):
        import os
        import sqlite3
        from urllib.parse import quote
        if not os.path.exists(self.db_path):
            return self
        with open(self.db_path, "rb") as f:
            head = f.read(100)
        if len(head) >= 20 and head[:16] == b"SQLite format 3\x00" and 2 in (head[18], head[19]):
            raise UsageDbNotModelled("the file at the path is in WAL mode: a save writes rollback-journal files only")
        self.conn = sqlite3.connect(f"file:{quote(os.fspath(self.db_path))}?mode=rw", uri=True, isolation_level=None, timeout=0)
        try:
            self.conn.execute("BEGIN EXCLUSIVE")
        except BaseException:
            self.conn.close()
            raise
        return self

    def __exit__(self, *exc):
        if self.conn is not None:
            self.conn.close()                     # (ends the transaction; the lock was on the file that has been replaced)


def _write_replace(db_path, data) -> None:
    """data to a temporary file next to db_path, fsync'd, moved over db_path with os.replace, then the directory fsync'd.  A
    replaced file's permission bits carry over.  On a failure the temporary file is removed and db_path is as it was."""
    import os
    import tempfile
    path = os.path.abspath(os.fspath(db_path))
    d = os.path.dirname(path)
    try:
        mode = os.stat(path).st_mode & 0o7777
    except FileNotFoundError:
        umask = os.umask(0)
        os.umask(umask)
        mode = 0o666 & ~umask
    fd, tmp = tempfile.mkstemp(prefix="." + os.path.basename(path) + ".", suffix=".saving", dir=d)
    try:
        with os.fdopen(fd, "wb") as f:
            f.write(data)
            f.flush()
            os.fchmod(f.fileno(), mode)
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        try:
            os.unlink(tmp)
        except FileNotFoundError:
            pass
        raise
    dfd = os.open(d, os.O_RDONLY)
    try:
        os.fsync(dfd)
    finally:
        os.close(dfd)


def _utf8_or_none(b: bytes):
    try:
        return b.decode("utf-8")
    except UnicodeDecodeError:
        return None


def _object_array(items: list) -> np.ndarray:
    a = np.empty(len(items), dtype=object)
    a[:] = items
    return a


def stats_window(period: str, now: datetime):
    """stats.py:46-55: (start_date, end_date) the stats endpoint asks for."""
    delta = {"hour": timedelta(hours=24), "day": timedelta(weeks=2), "week": timedelta(weeks=15), "month": timedelta(days=365)}[period]
    return now - delta, now


class UsageTable:
    """Device-resident usage records + GPU rollup.  `engine` is an llmapigateway_b200.Engine."""

    COLS = ("ts_us", "model_rank", "prompt_tokens", "completion_tokens", "total_tokens", "reasoning_tokens", "cached_tokens", "cost")
    DTYPES = (np.int64, np.int32, np.int32, np.int32, np.int32, np.int32, np.int32, np.float64)
    # Record ids, as SQLite's AUTOINCREMENT gives them: _ids holds the id of each host record, a pending row carries its own,
    # and _seq is the largest id ever given out (sqlite_sequence) -- a deleted id is never given out again.
    _ids = np.zeros(0, np.int64)
    _seq = 0
    # Inserts append: _rank (model name -> rank, None: rank every record at the next _materialise) persists between
    # materialisations; _hbuf holds the buffers the host columns and ids are exact-length views of, with room to grow;
    # _dev_rank_map maps the ranks of the resident device records to the current ones when a new name shifted them (None: no
    # shift since the device was last brought up to date); _dev_cap is the capacity of the device columns, in records;
    # _ts_range is (the ts_us array it describes, min, max), kept across inserts so that a rollup needs no pass over the column.
    _rank = None
    _fixed_names = None
    _hbuf = None
    _dev_n = None
    _dev_rank_map = None
    _dev_cap = 0
    _ts_range = None
    rejected_ids = np.zeros(0, np.int64)      # ids of the records the last load_tokens_usage_db refused
    save_refused_ids = np.zeros(0, np.int64)  # ids of the records the last save_tokens_usage_db did not write

    def __init__(self, engine):
        self.eng = engine
        self._lib = _native.load()
        self._host = {c: np.zeros(0, dtype=d) for c, d in zip(self.COLS, self.DTYPES)}
        self._models: list[str | None] = []      # per record, until encoded
        self._providers: list[str | None] = []   # per record (listing only; the rollup does not group by provider)
        self._dev = None                          # (n, {col: device ptr}, names)
        self._dev_n = None                        # records [0, _dev_n) of the host copy are on the device (inserts only append)
        self._pending_rows: list[tuple] = []
        self.rejected = 0                         # records insert_usage refused (see there)

    # -- ingest ------------------------------------------------------------------------------------
    def insert_usage(self, tokens_usage: dict, timestamp: datetime | None = None):
        """One record, same dict shape as the reference's insert_usage (:136-143).  Like the reference (:155-159) this never
        raises: a value SQLite would have stored as NULL (JSON null), as REAL/TEXT (a non-integer where a count belongs), or
        that no INTEGER column of the device table can hold (|v| >= 2^31) makes the record unusable for the integer rollup
        and the row is REJECTED (counted in `rejected`), never half-inserted."""
        ts = to_us(timestamp or datetime.now())
        g = tokens_usage.get
        try:
            counts = []
            for k in ("prompt_tokens", "completion_tokens", "total_tokens", "reasoning_tokens", "cached_tokens"):
                v = g(k, 0)
                if v is None:
                    v = 0                                              # SUM() skips NULL
                if isinstance(v, bool) or not isinstance(v, int):
                    if isinstance(v, float) and v.is_integer():
                        v = int(v)
                    else:
                        raise ValueError(k)
                if not -(1 << 31) <= v < (1 << 31):
                    raise OverflowError(k)
                counts.append(v)
            cost = g("cost", 0.0)
            cost = math.nan if cost is None else float(cost)            # NaN == SQL NULL (SQLite stores a NaN as NULL too)
            model, provider = g("model"), g("provider")
            if model is not None and not isinstance(model, str):
                model = str(model)
        except Exception:
            self.rejected += 1
            return False
        self._seq += 1
        self._pending_rows.append((ts, model, *counts, cost, provider, self._seq))
        self._dev = None
        return True

    def load_columns(self, ts_us, models, prompt, completion, total, reasoning, cached, cost, names=None):
        """Bulk ingest of columns (models: sequence of str|None).  `names`: the model dictionary to encode against when several
        tables (one per GPU) are merged -- every rank must rank the models identically (sorted by UTF-8 bytes, NULL first)."""
        self._fixed_names = sorted(set(names), key=lambda s: s.encode("utf-8")) if names is not None else None
        self._host = {"ts_us": np.ascontiguousarray(ts_us, np.int64), "model_rank": None,
                      "prompt_tokens": np.ascontiguousarray(prompt, np.int32), "completion_tokens": np.ascontiguousarray(completion, np.int32),
                      "total_tokens": np.ascontiguousarray(total, np.int32), "reasoning_tokens": np.ascontiguousarray(reasoning, np.int32),
                      "cached_tokens": np.ascontiguousarray(cached, np.int32), "cost": np.ascontiguousarray(cost, np.float64)}
        self._models = list(models)
        self._providers = [None] * len(self._models)
        self._ids = np.arange(1, len(self._models) + 1, dtype=np.int64)
        self._seq = len(self._models)
        self._pending_rows = []
        self._dev = None
        self._dev_n = None
        self._rank = None
        self._dev_rank_map = None
        self._ts_range = None

    def load_tokens_usage_db(self, db_path) -> int:
        """Replace the table's contents with the records of the `tokens_usage` table of the SQLite file at db_path (as
        tokens_usage_db.py and gateway.SqliteUsageSink write it), decoded on the device (csrc/load.cuh); the number loaded.
        The table then equals one that got those records through insert_usage with their stored timestamps, in id order, and
        was brought up to date on the device: same columns, model ranks, ids (gaps included), model and provider strings, and
        the next id is sqlite_sequence's + 1.  The device columns are resident: the next query uploads nothing.
        A record the table cannot hold is refused whole: its id goes to `rejected_ids` and the count to `rejected`.  It holds
        a timestamp that is not TEXT exactly as datetime.isoformat() writes a naive datetime, a token count that is not an
        INTEGER in [-2^31, 2^31) or NULL, a cost that is TEXT or BLOB, or a model or provider that is not NULL or valid UTF-8
        TEXT.  Raises UsageDbNotModelled or UsageDbCorrupt (or the engine's error) and leaves the table as it was."""
        snap = read_tokens_usage_snapshot(db_path, self._load_alloc, self._load_free)
        try:
            got = self._load_records(snap)
        finally:
            self._load_free(snap["buf"])
        cols, ids, names, prov_names, prov, refused, dev = got
        n = int(ids.size)
        old = getattr(self, "_dev_ptrs", None)
        self._host = cols
        self._ids = ids
        self._seq = snap["seq"]
        self._names = [None] + names
        self._rank = {m: i for i, m in enumerate(self._names)}
        self._models = _object_array(self._names).take(cols["model_rank"]).tolist()
        self._providers = _object_array([None] + prov_names).take(prov).tolist()
        self._pending_rows = []
        self._fixed_names = None
        self._hbuf = None
        self._ts_range = None
        self._dev_rank_map = None
        self._dev_ptrs = dev
        self._dev = (n, dev)
        self._dev_n = self._dev_cap = n
        if old:
            self._free_ptrs(old)
        self.rejected += int(refused.size)
        self.rejected_ids = refused
        return n

    def _load_records(self, snap: dict):
        """csrc/load.cuh over the snapshot's bytes: (host columns, ids, ranked model names, provider names, provider codes,
        refused ids, device columns).  Distinct texts come back once each; a text that is not valid UTF-8 refuses its records."""
        try:
            return self._load_steps(snap)
        finally:
            self._load_call("release")                # (the load's device scratch is only needed until finish)

    def _load_steps(self, snap: dict):
        buf = snap["buf"]
        bp = buf.ctypes.data_as(C.c_void_p)
        out = np.zeros(6, np.uint64)
        self._load_call("decode", bp, snap["size"], snap["page_size"], snap["n_pages"], snap["root"], out.ctypes.data_as(C.c_void_p))
        err, n, counts, nbytes = int(out[0]), int(out[1]), (int(out[2]), int(out[3])), (int(out[4]), int(out[5]))
        if err == LOAD_ID_STORED:
            raise UsageDbNotModelled("tokens_usage stores its id column: id is not a rowid alias")
        if err:
            raise UsageDbCorrupt(LOAD_ERRORS.get(err, f"load error {err}"))
        texts = []
        for field in (0, 1):
            raw = np.zeros(max(nbytes[field], 1), np.uint8)
            offs = np.zeros(counts[field] + 1, np.uint64)
            self._load_call("names", bp, field, raw.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p))
            blob, o = raw.tobytes(), offs.tolist()
            texts.append([_utf8_or_none(blob[o[k]:o[k + 1]]) for k in range(counts[field])])
        mm = np.array([0 if t is not None else -1 for t in texts[0]] or [0], np.int32)
        pm = np.array([k + 1 if t is not None else -1 for k, t in enumerate(texts[1])] or [0], np.int32)
        used = np.zeros(max(counts[0], 1), np.uint8)
        n_keep = C.c_uint64(0)
        self._load_call("mark", mm.ctypes.data_as(C.c_void_p), pm.ctypes.data_as(C.c_void_p), used.ctypes.data_as(C.c_void_p), C.byref(n_keep))
        k = n_keep.value
        names = sorted({texts[0][c] for c in np.flatnonzero(used[:counts[0]]).tolist()}, key=lambda s: s.encode("utf-8"))
        rank = {m: i + 1 for i, m in enumerate(names)}
        mm = np.array([rank.get(t, 0) if t is not None else -1 for t in texts[0]] or [0], np.int32)
        cols = {c: np.empty(k, d) for c, d in zip(self.COLS, self.DTYPES)}
        ids, prov, refused = np.empty(k, np.int64), np.empty(k, np.int32), np.empty(n - k, np.int64)
        dev = self._load_cols_alloc(k)
        try:
            d_cols = (C.c_void_p * 8)(*[dev[c].value if dev else None for c in self.COLS])
            h_cols = (C.c_void_p * 8)(*[cols[c].ctypes.data for c in self.COLS])
            self._load_call("finish", mm.ctypes.data_as(C.c_void_p), pm.ctypes.data_as(C.c_void_p), d_cols, h_cols,
                            ids.ctypes.data_as(C.c_void_p), prov.ctypes.data_as(C.c_void_p), refused.ctypes.data_as(C.c_void_p))
        except BaseException:
            self._free_ptrs(dev)
            raise
        return cols, ids, names, texts[1], prov, refused, dev

    # the loader's seams: a CPU stand-in replaces these with the host build of csrc/load.cuh and numpy buffers
    def _load_call(self, step: str, *args):
        self.eng._ck(getattr(self._lib, "lgw_usage_load_" + step)(self.eng._h, *args), "usage_load_" + step)

    def _load_alloc(self, nbytes: int) -> np.ndarray:
        return self.eng.alloc_pinned(nbytes)

    def _load_free(self, buf: np.ndarray):
        self._lib.lgw_free_pinned(self.eng._h, C.c_void_p(buf.ctypes.data))

    def _load_cols_alloc(self, n: int) -> dict:
        ptrs = {}
        try:
            for c, d in zip(self.COLS, self.DTYPES):
                p = C.c_void_p()
                self.eng._ck(self._lib.lgw_device_alloc(self.eng._h, max(n * np.dtype(d).itemsize, 8), C.byref(p)), "device_alloc")
                ptrs[c] = p
        except BaseException:
            self._free_ptrs(ptrs)
            raise
        return ptrs

    def load_last_ms(self) -> dict:
        """device times of the last load_tokens_usage_db, milliseconds"""
        ms = (C.c_float * 4)()
        self.eng._ck(self._lib.lgw_usage_load_last_ms(self.eng._h, C.byref(ms)), "usage_load_last_ms")
        return {"copy": ms[0], "decode": ms[1], "dictionary": ms[2], "compaction": ms[3]}

    # -- saving the table as a tokens_usage file ---------------------------------------------------------------------------
    def save_tokens_usage_db(self, db_path, page_size: int = 4096) -> int:
        """Write every record of the table (pending rows included: _upload() first) to a new `tokens_usage` SQLite file at
        db_path, laid out on the device (csrc/save.cuh); the number written.  The file has SqliteUsageSink's schema, its
        `tokens_usage` rows in id order with rowid = id (gaps kept), the timestamps as datetime.isoformat() text, costs as
        8-byte REALs bit for bit (NaN as NULL), sqlite_sequence holding _seq (no row when it is 0) and a complete
        idx_tokens_usage_timestamp; load_tokens_usage_db reads it back as this table.
        A record the file cannot hold -- a model or provider that is not encodable as UTF-8, a timestamp with no isoformat text
        (only load_columns can give one) -- is not written: its id goes to `save_refused_ids` and a warning is logged.
        The file is written next to db_path, fsync'd and moved into place with os.replace.  An existing file is first locked
        EXCLUSIVE through sqlite3 (which rolls back a hot journal) until it is replaced.  A busy lock (sqlite3.OperationalError),
        a WAL-mode file there or a file of LOAD_MAX_BYTES or more (UsageDbNotModelled), a page_size that is not a power of two
        in [1024, 65536] (ValueError) or any other failure leave the old file, and the table, as they were.  Replacing a file
        that another connection still has open (a live SqliteUsageSink) is the caller's to avoid: that connection keeps
        writing to the replaced file, and its rows are lost."""
        _check_page_size(page_size)
        self._upload()
        n = int(self._host["ts_us"].size)
        models, _m = _save_text_table(self._names)
        codes: dict = {None: 0}
        prov = np.fromiter((codes.setdefault(p, len(codes)) for p in self._providers), np.int32, count=n)
        providers, _p = _save_text_table(list(codes))
        ids = np.ascontiguousarray(self._ids[:n], np.int64)
        with _ReplaceLock(db_path):
            try:
                out = np.zeros(5, np.uint64)
                self._save_call("plan", self._save_cols(), n, ids.ctypes.data_as(C.c_void_p), prov.ctypes.data_as(C.c_void_p),
                                C.byref(models), C.byref(providers), page_size, out.ctypes.data_as(C.c_void_p))
                pages, table_root, index_root, kept, refused_n = (int(x) for x in out)
                if pages * page_size >= LOAD_MAX_BYTES:
                    raise UsageDbNotModelled(f"a file of {pages * page_size} bytes: load_tokens_usage_db reads files below 2^33 bytes")
                buf = self._save_alloc(pages * page_size)
                try:
                    refused = np.zeros(refused_n, np.int64)
                    self._save_call("write", buf.ctypes.data_as(C.c_void_p), refused.ctypes.data_as(C.c_void_p))
                    buf[:2 * page_size] = np.frombuffer(_head_pages(page_size, pages, table_root, index_root, self._seq), np.uint8)
                    _write_replace(db_path, memoryview(buf)[:pages * page_size])
                finally:
                    self._save_free(buf)
            finally:
                self._save_call("release")
        self.save_refused_ids = refused
        if refused.size:
            logging.warning(f"save_tokens_usage_db: {refused.size} records the file cannot hold were not written "
                            "(a text that is not UTF-8, or a timestamp with no isoformat text); their ids are in save_refused_ids")
        return kept

    # the save's seams: a CPU stand-in replaces these with the host build of csrc/save.cuh and numpy buffers
    def _save_call(self, step: str, *args):
        self.eng._ck(getattr(self._lib, "lgw_usage_save_" + step)(self.eng._h, *args), "usage_save_" + step)

    def _save_cols(self):
        return (C.c_void_p * 8)(*[self._dev_ptrs[c].value for c in self.COLS])

    def _save_alloc(self, nbytes: int) -> np.ndarray:
        return self.eng.alloc_pinned(nbytes)

    def _save_free(self, buf: np.ndarray):
        self._lib.lgw_free_pinned(self.eng._h, C.c_void_p(buf.ctypes.data))

    def save_last_ms(self) -> dict:
        """device times of the last save_tokens_usage_db, milliseconds"""
        ms = (C.c_float * 6)()
        self.eng._ck(self._lib.lgw_usage_save_last_ms(self.eng._h, C.byref(ms)), "usage_save_last_ms")
        return dict(zip(("upload", "keep", "sort", "pack", "write", "download"), ms))

    def _grow(self, key: str, a: np.ndarray, new: np.ndarray) -> np.ndarray:
        """a followed by new, as an exact-length view of a buffer of this table with room to grow (doubling): when a is the
        view of that buffer and it has room, the values already there are not touched"""
        if self._hbuf is None:
            self._hbuf = {}
        n, m = a.size, new.size
        buf = self._hbuf.get(key)
        if buf is None or a.base is not buf or n + m > buf.size:
            buf = self._hbuf[key] = np.empty(max(2 * (n + m), 1024), a.dtype)
            buf[:n] = a
        buf[n:n + m] = new
        return buf[:n + m]

    def _materialise(self):
        """Move the pending rows into the host columns and rank their model names.  Only the new rows are visited, except
        when a new name shifts the ranks of the old ones (see _rank_new)."""
        if self._pending_rows:
            cols = list(zip(*self._pending_rows))
            h = self._host
            new = {"ts_us": np.array(cols[0], np.int64), "cost": np.array(cols[7], np.float64)}      # built completely
            for k, name in enumerate(self.COLS[2:7]):                                                  # before anything is
                new[name] = np.array(cols[2 + k], np.int32)                                            # replaced
            ids = np.array(cols[9], np.int64)
            fresh = {c: (self._grow(c, h[c], new[c]) if c in new else h[c]) for c in self.COLS}
            self._ids = self._grow("ids", self._ids, ids)
            self._host = fresh
            rng, t = self._ts_range, new["ts_us"]
            if h["ts_us"].size == 0:
                rng = (fresh["ts_us"], int(t.min()), int(t.max()))
            elif rng is not None and rng[0] is h["ts_us"]:
                rng = (fresh["ts_us"], min(rng[1], int(t.min())), max(rng[2], int(t.max())))
            self._ts_range = rng if rng is not None and rng[0] is fresh["ts_us"] else None
            self._models.extend(cols[1])
            self._providers.extend(cols[8])
            self._pending_rows = []
        mr = self._host["model_rank"]
        if mr is None or self._rank is None:
            self._rank_all()
        elif mr.size < len(self._models):
            self._rank_new(mr)

    def _rank_all(self):
        """rank every record's model name (a table loaded with load_columns, or one never ranked)"""
        names = self._fixed_names or sorted({m for m in self._models if m is not None}, key=lambda s: s.encode("utf-8"))
        rank = {m: i + 1 for i, m in enumerate(names)}
        rank[None] = 0
        self._host["model_rank"] = np.fromiter((rank[m] for m in self._models), dtype=np.int32, count=len(self._models))
        self._names = [None] + names
        self._rank = rank

    def _rank_new(self, mr: np.ndarray):
        """rank the records [mr.size, n) whose names have no rank yet.  A name not ranked before is merged into the byte-ordered
        names; when that moves an old name, the host ranks are rewritten through the old -> new map and the map is kept for the
        device records (_dev_rank_map).  A table with a fixed dictionary (load_columns(names=...)) never adds a name."""
        new_models = self._models[mr.size:]
        rank = self._rank
        if not self._fixed_names:
            unranked = {m for m in new_models if m not in rank}
            if unranked:
                old_names = self._names
                self._names = [None] + sorted(old_names[1:] + list(unranked), key=lambda s: s.encode("utf-8"))
                rank = self._rank = {m: i for i, m in enumerate(self._names)}
                step = np.fromiter((rank[m] for m in old_names), dtype=np.int32, count=len(old_names))
                if np.any(step != np.arange(len(old_names), dtype=np.int32)):
                    mr[...] = step[mr]
                    if self._dev_n is not None:
                        self._dev_rank_map = step if self._dev_rank_map is None else step[self._dev_rank_map]
        new_rank = np.fromiter((rank[m] for m in new_models), dtype=np.int32, count=len(new_models))
        self._host["model_rank"] = self._grow("model_rank", mr, new_rank)

    def _free_device(self):
        """Give the device copy of the columns back (an insert makes it stale; without this every re-upload would leak the last one)."""
        ptrs, self._dev_ptrs = getattr(self, "_dev_ptrs", None), None
        self._dev = None
        self._dev_n = None
        self._dev_rank_map = None
        self._dev_cap = 0
        if ptrs and getattr(self.eng, "_h", None):
            self._free_ptrs(ptrs)

    def _free_ptrs(self, ptrs: dict):
        for p in ptrs.values():
            self._lib.lgw_device_free(self.eng._h, p)

    def close(self):
        self._free_device()

    def _upload(self):
        """Bring the device copy up to date.  With one resident (device records [0, _dev_n) are host records [0, _dev_n)), the
        host records past _dev_n, pending rows included, are appended to it (_append_on_device), growing the columns by
        doubling when they are full; without one (a fresh table, or after load_columns) every column is uploaded."""
        if self._dev is not None:
            return
        if self._dev_n is None:
            self._upload_all()
            return
        self._materialise()
        n_dev, n = self._dev_n, int(self._host["ts_us"].size)
        rank_map = self._dev_rank_map
        if n > n_dev or rank_map is not None:
            cap = min(max(2 * self._dev_cap, n, 1024), APPEND_MAX) if n > self._dev_cap else None
            try:
                ptrs = self._append_on_device(n_dev, n - n_dev, rank_map, cap)
            except BaseException:
                self._free_device()               # (the next query uploads the table again: device ranks never disagree with the host)
                raise
            old, self._dev_ptrs = self._dev_ptrs, ptrs
            if cap is not None:
                self._dev_cap = cap
                self._free_ptrs(old)
            self._dev_n = n
            self._dev_rank_map = None
        self._dev = (n, self._dev_ptrs)

    def _upload_all(self):
        self._free_device()
        self._materialise()
        n = int(self._host["ts_us"].size)
        ptrs = {}
        self._dev_ptrs = ptrs                     # (registered before the first allocation: a failed upload frees what it got)
        for c in self.COLS:
            a = self._host[c]
            p = C.c_void_p()
            self.eng._ck(self._lib.lgw_device_alloc(self.eng._h, max(a.nbytes, 8), C.byref(p)), "device_alloc")
            self.eng._ck(self._lib.lgw_device_upload(self.eng._h, p, a.ctypes.data_as(C.c_void_p), a.nbytes), "device_upload")
            ptrs[c] = p
        self._dev = (n, ptrs)
        self._dev_n = n
        self._dev_cap = n

    def _append_on_device(self, n: int, m: int, rank_map, cap) -> dict:
        """host records [n, n + m) after the n resident ones (lgw_usage_append), the resident model ranks mapped through rank_map
        (or None): in place when cap is None, else into fresh columns with room for cap records (the old ones stay as they
        were, and on a failure the fresh ones are freed).  A new dict of the column pointers either way."""
        lib, h = self._lib, self.eng._h
        fresh = {}
        try:
            if cap is not None:
                for c, d in zip(self.COLS, self.DTYPES):
                    p = C.c_void_p()
                    self.eng._ck(lib.lgw_device_alloc(h, max(cap * np.dtype(d).itemsize, 8), C.byref(p)), "device_alloc")
                    fresh[c] = p
            cols = (C.c_void_p * 8)(*[self._dev_ptrs[c].value for c in self.COLS])
            grow = (C.c_void_p * 8)(*[fresh[c].value for c in self.COLS]) if cap is not None else None
            new = [self._host[c][n:n + m] for c in self.COLS]
            h_new = (C.c_void_p * 8)(*[a.ctypes.data for a in new])
            rmap = np.ascontiguousarray(rank_map, np.int32) if rank_map is not None else None
            self.eng._ck(lib.lgw_usage_append(h, cols, grow, n, h_new, m, rmap.ctypes.data_as(C.c_void_p) if rmap is not None else None,
                                              rmap.size if rmap is not None else 0), "usage_append")
        except BaseException:
            self._free_ptrs(fresh)
            raise
        return fresh if cap is not None else dict(self._dev_ptrs)

    def __len__(self):
        return int(self._host["ts_us"].size) + len(self._pending_rows)

    # -- rollup ---------------------------------------------------------------------------------------
    def geometry(self, period: str, start: datetime | None, end: datetime | None):
        self._materialise() if self._host.get("model_rank") is None or self._pending_rows else None
        ts = self._host["ts_us"]
        p = PERIODS[period]
        rng = self._ts_range
        if rng is None or rng[0] is not ts:
            rng = self._ts_range = (ts, int(ts.min()) if ts.size else 0, int(ts.max()) if ts.size else 0)
        lo, hi = rng[1], rng[2]
        if start is not None:
            lo = max(lo, to_us(start))
        if end is not None:
            hi = min(hi, to_us(end))
        if hi < lo:
            hi = lo
        # SQLite's millisecond rounding (csrc/rollup.cuh bucket_of) makes buckets not monotone in time.  At the top it can push a
        # record one day ahead: slack.  At the bottom: a `lo` in the last half millisecond of a 29th..31st has the NEXT day's 23:00
        # hour while the records after it are in that day's 00:00 hour (lo + 1 ms is past the rounding window); and a Monday's
        # rounded records take Tuesday's weekday, which puts them one %W week BELOW the rest of that Monday.
        b0 = min(int(self._lib.lgw_rollup_bucket_of(lo, p)), int(self._lib.lgw_rollup_bucket_of(lo + 1000, p))) - (period == "week")
        b1 = int(self._lib.lgw_rollup_bucket_of(hi, p))
        slack = 25 if period == "hour" else 1
        return b0, b1 - b0 + 1 + slack, len(self._names)

    def accumulate(self, period: str, start, end, bucket0: int, n_buckets: int, n_models: int, d_table, d_inexact, d_oob):
        """Add this table's records into a caller-owned dense device table (multi-GPU merge)."""
        self._upload()
        n, ptr = self._dev
        self.eng._ck(self._lib.lgw_usage_rollup_accum(
            self.eng._h, ptr["ts_us"], ptr["model_rank"], ptr["prompt_tokens"], ptr["completion_tokens"], ptr["total_tokens"],
            ptr["reasoning_tokens"], ptr["cached_tokens"], ptr["cost"], n, PERIODS[period],
            int(start is not None), to_us(start) if start is not None else 0, int(end is not None), to_us(end) if end is not None else 0,
            bucket0, n_buckets, n_models, d_table, d_inexact, d_oob), "usage_rollup_accum")

    def emit(self, bucket0: int, n_buckets: int, n_models: int, d_table, d_inexact, pinned: bool = False) -> np.ndarray:
        """Rows of a dense device table (this GPU's, or the all-reduced sum of every GPU's), time_period DESC, model ASC.
        pinned=True: the rows land in a page-locked buffer owned by this table (grown on demand, REUSED by the next pinned emit:
        consume or copy them first) -- a full `hour` table over 400 days is 45 MB of rows, 10 ms into pageable memory, < 1 ms pinned.
        The cost of a row with `inexact` set is NOT the group's sum (rollup_rows sums such groups again from the host copy of the
        records; a merged multi-GPU table has no single copy of them to do that with): the caller has to treat it as unknown."""
        groups = n_buckets * n_models
        if pinned:
            need = groups * ROW_DTYPE.itemsize
            buf = getattr(self, "_pinned_rows", None)
            if buf is None or buf.size < need:
                buf = self._pinned_rows = self.eng.alloc_pinned(need)
            rows = buf[:need].view(ROW_DTYPE)
        else:
            rows = np.zeros(groups, dtype=ROW_DTYPE)
        n_rows = C.c_uint64(0)
        self.eng._ck(self._lib.lgw_usage_rollup_emit(self.eng._h, d_table, d_inexact, bucket0, n_buckets, n_models,
                                                     rows.ctypes.data_as(C.c_void_p), groups, C.byref(n_rows)), "usage_rollup_emit")
        return rows[:n_rows.value]

    def rows_to_dicts(self, period: str, rows) -> list[dict]:
        return [{"time_period": period_label(period, int(r["bucket"])), "model": self._names[int(r["model_rank"])],
                 "prompt_tokens": int(r["prompt_tokens"]), "completion_tokens": int(r["completion_tokens"]),
                 "total_tokens": int(r["total_tokens"]), "reasoning_tokens": int(r["reasoning_tokens"]),
                 "cached_tokens": int(r["cached_tokens"]), "cost": _sql_value(float(r["cost"])), "count": int(r["count"])} for r in rows]

    def rollup_rows(self, period: str, start: datetime | None = None, end: datetime | None = None) -> np.ndarray:
        """Rows (ROW_DTYPE) ordered time_period DESC, model ASC.  `cost` is SQLite's SUM(cost) of the group: the correctly
        rounded sum, NaN where SQLite gives NULL (see sql_sum).  Rows with `inexact` set were summed on the host."""
        self._upload()
        b0, nb, nm = self.geometry(period, start, end)
        groups = nb * nm
        lib, h = self._lib, self.eng._h
        tab, inx, oob = C.c_void_p(), C.c_void_p(), C.c_void_p()
        for p, nbytes in ((tab, groups * ROLLUP_CELLS * 8), (inx, groups * 4), (oob, 8)):
            self.eng._ck(lib.lgw_device_alloc(h, nbytes, C.byref(p)), "device_alloc")
            self.eng._ck(lib.lgw_device_zero(h, p, nbytes), "device_zero")
        try:
            self.accumulate(period, start, end, b0, nb, nm, tab, inx, oob)
            rows = np.zeros(groups, dtype=ROW_DTYPE)
            n_rows = C.c_uint64(0)
            self.eng._ck(lib.lgw_usage_rollup_emit(h, tab, inx, b0, nb, nm, rows.ctypes.data_as(C.c_void_p), groups, C.byref(n_rows)), "usage_rollup_emit")
            lost = np.zeros(1, np.uint32)
            self.eng._ck(lib.lgw_device_download(h, lost.ctypes.data_as(C.c_void_p), oob, 4), "device_download")
            # records outside the table are exactly those the window excludes only when no window was given; never expected
            assert int(lost[0]) == 0 or start is not None or end is not None, "records fell outside the rollup table"
            rows = rows[:n_rows.value]
        finally:
            for p in (tab, inx, oob):
                lib.lgw_device_free(h, p)
        if rows["inexact"].any():
            self._sum_flagged_groups(rows, period, start, end)
        return rows

    def _sum_flagged_groups(self, rows, period: str, start, end):
        """Replace the device cost of every flagged row (a cost the fixed point cannot hold, csrc/rollup.cuh cost_to_limbs) with
        sql_sum() of the group's records, found with the kernel's own bucket arithmetic.  The flag stays set: it now says that
        the host summed the group.  Runs only when a group is flagged."""
        ts, mr = self._host["ts_us"], self._host["model_rank"]
        sel = np.ones(ts.size, bool)
        if start is not None:
            sel &= ts >= to_us(start)
        if end is not None:
            sel &= ts <= to_us(end)
        idx = np.flatnonzero(sel)
        tsel = np.ascontiguousarray(ts[idx])
        bucket = np.empty(idx.size, np.int64)
        self.eng._ck(self._lib.lgw_rollup_buckets_of(tsel.ctypes.data_as(C.c_void_p), idx.size, PERIODS[period],
                                                     bucket.ctypes.data_as(C.c_void_p)), "rollup_buckets_of")
        nm = len(self._names)
        key = bucket * nm + mr[idx]
        flagged = np.flatnonzero(rows["inexact"])
        want = rows["bucket"][flagged] * nm + rows["model_rank"][flagged]
        keep = np.isin(key, want)
        key, idx = key[keep], idx[keep]
        order = np.argsort(key, kind="stable")
        key, idx = key[order], idx[order]
        lo = np.searchsorted(key, want, "left")
        hi = np.searchsorted(key, want, "right")
        cost = self._host["cost"]
        for r, a, b in zip(flagged, lo, hi):
            rows["cost"][r] = sql_sum(cost[idx[a:b]].tolist())

    def get_aggregated_usage(self, period: str, start_date: datetime | None = None, end_date: datetime | None = None) -> list[dict]:
        """Same result shape and order as TokensUsageDB.get_aggregated_usage (:289-291); [] for a bad period (:296-298).
        A group whose costs are all NULL has cost None, as SUM(cost) in SQLite."""
        if period not in PERIODS:
            return []
        if len(self) == 0:
            return []
        return self.rows_to_dicts(period, self.rollup_rows(period, start_date, end_date))

    # -- record listing: /v1/api/usage-records (stats.py:69-87) ---------------------------------------------
    def get_total_records_count(self) -> int:
        """tokens_usage_db.py:200-220"""
        return len(self)

    def get_latest_usage_records(self, limit: int = 25, offset: int = 0) -> list[dict]:
        """tokens_usage_db.py:69-117: newest first (`ORDER BY timestamp DESC LIMIT ? OFFSET ?`), same keys.  Records with
        equal timestamps come in insertion order (SQLite leaves their order unspecified).  With an engine the page is
        selected on the device (_latest_on_device) from the uploaded timestamps, and rows inserted since the upload are
        merged on the host; without one, from the host copy of the columns."""
        if self.eng is not None:
            return self._latest_records_device(limit, offset)
        self._materialise()
        h = self._host
        n = int(h["ts_us"].size)
        if limit < 0:
            limit = n                                           # SQLite: a negative LIMIT means no limit
        order = np.argsort(-h["ts_us"], kind="stable")[max(offset, 0):max(offset, 0) + limit]
        return [self._record(int(i)) for i in order]

    def _record(self, i: int) -> dict:
        """record i as a listing row; i may be a row inserted since the host columns were last built"""
        h = self._host
        n_host = int(h["ts_us"].size)
        if i < n_host:
            ts, model, provider, rid = int(h["ts_us"][i]), self._models[i], self._providers[i], int(self._ids[i])
            tok = [int(h[c][i]) for c in self.COLS[2:7]]
            cost = float(h["cost"][i])
        else:
            ts, model, *tok, cost, provider, rid = self._pending_rows[i - n_host]
        return {"id": rid, "timestamp": (_EPOCH + timedelta(microseconds=int(ts))).isoformat(),
                "prompt_tokens": int(tok[0]), "completion_tokens": int(tok[1]), "total_tokens": int(tok[2]),
                "reasoning_tokens": int(tok[3]), "cached_tokens": int(tok[4]), "cost": _sql_value(float(cost)),
                "model": model, "provider": provider}

    def _latest_on_device(self, n: int, first: int, count: int) -> np.ndarray:
        """indices of the uploaded records [0, n) at ranks [first, first + count) of (ts_us DESC, index ASC)"""
        idx = np.empty(count, np.uint64)
        self.eng._ck(self._lib.lgw_usage_latest(self.eng._h, self._dev_ptrs["ts_us"], n, first, count,
                                                idx.ctypes.data_as(C.c_void_p)), "usage_latest")
        return idx

    def _latest_records_device(self, limit: int, offset: int) -> list[dict]:
        total = len(self)
        if limit < 0:
            limit = total                                       # SQLite: a negative LIMIT means no limit
        offset = max(offset, 0)
        if limit == 0 or offset >= total:
            return []
        if self._dev_n is None or total - self._dev_n > LISTING_PENDING_MAX:
            self._upload()                                      # (both cases have _dev None: a load, or inserts since the upload)
        n_dev = self._dev_n
        p = total - n_dev
        if p == 0:
            return [self._record(int(i)) for i in self._latest_on_device(n_dev, offset, min(limit, total - offset))]
        # Rows n_dev .. total-1 are not on the device; all of them sort after the uploaded ones on equal timestamps.  A page
        # row from the device has an uploaded rank in [offset - p, offset + limit): select those, merge with the pending rows.
        lo = max(0, offset - p)
        hi = min(n_dev, offset + limit)
        dev_idx = self._latest_on_device(n_dev, lo, hi - lo).astype(np.int64) if hi > lo else np.zeros(0, np.int64)
        h_ts = self._host["ts_us"]
        pend_ts = np.concatenate([h_ts[n_dev:], np.array([r[0] for r in self._pending_rows], np.int64)])
        idx = np.concatenate([dev_idx, np.arange(n_dev, total, dtype=np.int64)])
        ts = np.concatenate([h_ts[dev_idx], pend_ts])
        merged = idx[np.lexsort((idx, ~ts))]                   # (~ts: descending, without -ts's overflow at INT64_MIN)
        # merged position j >= p holds global rank lo + j when lo > 0 (pending rows before uploaded rank lo rank below offset);
        # every position holds global rank j when lo == 0
        start = offset - lo
        return [self._record(int(i)) for i in merged[start:start + limit]]

    # -- deleting old records (tokens_usage_db.py:164-198) ---------------------------------------------------------------
    def cleanup_old_records(self, retention_days: int = 180, now: datetime | None = None) -> None:
        """tokens_usage_db.py:164-198: delete the records older than `now - retention_days` (`now` defaults to
        datetime.now()).  A record goes exactly when ts_us < to_us(cutoff); one at the cutoff stays.  For every timestamp a
        datetime can express this is SQLite's `timestamp < cutoff.isoformat()` on the text (isoformat drops a zero microsecond
        part, which sorts the same); timestamps with no text form (only load_columns can give them, e.g. INT64_MIN) compare as
        the integers they are.  Ids survive, and the next insert gets the largest id ever given out + 1, as AUTOINCREMENT does.
        Like the reference this never raises and returns None: a bad `retention_days`, a cutoff outside datetime's range or a
        failed device call is logged and deletes nothing.  Uploaded records are compacted on the device (_retain_on_device);
        the table stays resident, model names keep their ranks until the next re-rank, and nothing is uploaded again."""
        try:
            cutoff = to_us((now if now is not None else datetime.now()) - timedelta(days=retention_days))
            deleted = self._retain(cutoff)
        except Exception as e:
            logging.error(f"Error cleaning up old token usage records: {str(e)}")
            return None
        if deleted > 0:
            logging.info(f"Cleaned up {deleted} old token usage records (older than {retention_days} days)")
        else:
            logging.debug("No old token usage records to clean up")
        return None

    def _retain(self, cutoff: int) -> int:
        """delete every record with ts_us < cutoff; the number deleted.  The device call comes first: if it fails, host and
        device are as they were.  Rows not on the device (host rows past _dev_n, pending rows) are deleted on the host only."""
        h = self._host
        keep = h["ts_us"] >= cutoff
        pend_keep = [r[0] >= cutoff for r in self._pending_rows]
        deleted = int(keep.size - np.count_nonzero(keep)) + pend_keep.count(False)
        if deleted == 0:
            return 0
        n_dev = self._dev_n
        if n_dev is not None:
            n_keep = int(np.count_nonzero(keep[:n_dev]))
            if n_keep < n_dev:
                fresh = self._retain_on_device(n_dev, cutoff, n_keep)
                old, self._dev_ptrs = self._dev_ptrs, fresh
                self._free_ptrs(old)
                if self._dev is not None:
                    self._dev = (n_keep, fresh)
                self._dev_n = n_keep
                self._dev_cap = n_keep
        idx = np.flatnonzero(keep)                # (take() with indices is several times faster than a boolean mask here)
        self._host = {c: (a.take(idx) if a is not None else None) for c, a in h.items()}
        self._ts_range = None
        self._ids = self._ids.take(idx)
        mask = keep.tolist()                      # (compress() over a list of bools, not over numpy bools: far faster)
        self._models = list(compress(self._models, mask))
        self._providers = list(compress(self._providers, mask))
        self._pending_rows = list(compress(self._pending_rows, pend_keep))
        return deleted

    def _retain_on_device(self, n: int, cutoff: int, n_keep: int) -> dict:
        """the n uploaded records with ts_us >= cutoff, compacted into fresh device columns (lgw_usage_retain); the old
        columns stay as they were, and on a failure the fresh ones are freed"""
        lib, h = self._lib, self.eng._h
        fresh = {}
        try:
            for c, d in zip(self.COLS, self.DTYPES):
                p = C.c_void_p()
                self.eng._ck(lib.lgw_device_alloc(h, max(n_keep * np.dtype(d).itemsize, 8), C.byref(p)), "device_alloc")
                fresh[c] = p
            src = (C.c_void_p * 8)(*[self._dev_ptrs[c].value for c in self.COLS])
            dst = (C.c_void_p * 8)(*[fresh[c].value for c in self.COLS])
            self.eng._ck(lib.lgw_usage_retain(h, src, dst, n, cutoff, n_keep), "usage_retain")
        except BaseException:
            self._free_ptrs(fresh)
            raise
        return fresh

    def retain_last_ms(self) -> float:
        """device time of the last lgw_usage_retain, milliseconds (a cleanup that deletes no uploaded record makes no device
        call and leaves it as it was)"""
        ms = C.c_float()
        self.eng._ck(self._lib.lgw_usage_retain_last_ms(self.eng._h, C.byref(ms)), "usage_retain_last_ms")
        return ms.value

    def append_last_ms(self) -> float:
        """device time of the last lgw_usage_append (the copy of the new rows and k_usage_append), milliseconds"""
        ms = C.c_float()
        self.eng._ck(self._lib.lgw_usage_append_last_ms(self.eng._h, C.byref(ms)), "usage_append_last_ms")
        return ms.value

    def last_ms(self):
        ms = (C.c_float * 2)()
        self.eng._ck(self._lib.lgw_rollup_last_ms(self.eng._h, C.byref(ms)), "rollup_last_ms")
        return {"accum": ms[0], "emit": ms[1]}

    def listing_last_ms(self) -> float:
        """device time of the last page selected on the device (0 when the last listing needed none)"""
        ms = C.c_float()
        self.eng._ck(self._lib.lgw_usage_latest_last_ms(self.eng._h, C.byref(ms)), "usage_latest_last_ms")
        return ms.value


def synth_usage_columns(n: int, seed: int = 5, end: datetime = datetime(2026, 9, 21, 6, 57, 17, 47518), days: int = 400, n_models: int = 64):
    """SURVEY 8(d) C5: timestamps uniform over a 400-day window, 64 model names (Zipf s=1.1) + 1% NULL,
    token ints < 2^17, cost = k x 1e-6."""
    rng = np.random.default_rng([seed, n])
    ts = to_us(end) - rng.integers(0, days * 86400 * 10**6, n, dtype=np.int64)
    w = 1.0 / np.arange(1, n_models + 1) ** 1.1
    mid = rng.choice(n_models, size=n, p=w / w.sum())
    names = np.array(["provider-%02d/model-%02d" % (i % 7, i) for i in range(n_models)], dtype=object)
    models = names[mid]
    models[rng.random(n) < 0.01] = None
    tok = [rng.integers(0, 2**17, n, dtype=np.int32) for _ in range(5)]
    cost = rng.integers(0, 10**6, n).astype(np.float64) * 1e-6
    return ts, models, tok, cost
