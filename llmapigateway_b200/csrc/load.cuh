// Loading the usage table from the `tokens_usage` SQLite file (llm_gateway_core/db/tokens_usage_db.py:37-50 writes it): the
// file's pages are copied to the device whole and decoded there.  SQLite's documented file format is all this relies on.
//
//  1. Walk, one b-tree level at a time from the table's root page.  k_load_count checks each page of the level (number in
//     range, never visited before, type 0x05 or 0x0D, cell pointer array inside the page) and counts its children (interior:
//     cells + the right-most pointer) or its cells (leaf).  k_list_scan places the next level; k_load_children writes it in key
//     order.  A level holds one page type only; the host stops after LGW_LOAD_MAX_DEPTH levels, and the visited bitmap bounds
//     the pages visited by the page count, so a cycle or a stray pointer ends as a status, never as a hang.
//  2. Decode (k_load_decode, a block per leaf page, a thread per cell): the leaf scan's offset + cell index is the record's
//     index in rowid order.  Payload and rowid varints, the record header's serial types, then each field, read through a
//     PayCursor that follows the overflow chain when the record spilled (the chain is checked first: every page in range, as
//     many pages as the payload needs, the last one ending the chain).  Each record gets its id, ts_us, five token columns,
//     cost, a refusal status and where its model and provider texts lie.
//  3. Dictionary (k_load_dict): model and provider texts of unrefused records go into two open-addressing hash tables keyed on
//     their bytes (FNV-1a; a tag match is confirmed by comparing bytes).  The first record to claim a slot gives the text a
//     dense provisional code and its location; the host reads those few texts from its own copy of the file.
//  4. The host sends back provisional code -> model rank and -> provider code maps, -1 for a text it refuses (invalid UTF-8).
//     k_load_mark counts each tile's kept records and marks the model codes they use; k_list_scan; k_load_finish writes the
//     kept records, in id order, into the eight UsageTable.COLS columns plus ids and provider codes, and the refused ids.
//
// Structural damage is a LoadError (the largest one seen); a record the table cannot hold is refused whole (RecStatus).
// Every read of the file is bounded by the page count the caller gives, which the caller checks against the bytes it copied.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#include "scan.cuh"
#endif

#if defined(__CUDACC__)
#define LGW_LOAD __host__ __device__ __forceinline__
#else
#define LGW_LOAD static inline
#endif

#define LGW_LOAD_MAX_DEPTH 20u      /* b-tree levels walked at most (SQLite's own cursors stop at 20) */
#define LGW_LOAD_NONE 0xFFFFFFFFu   /* TextRef.off of a NULL text; slot of a record without that text */
#define LGW_LOAD_TILE 2048u         /* mark / finish tile: 1024 threads x two records */

namespace lgw {

enum LoadError : uint32_t {
    LOAD_OK = 0, LOAD_BAD_PAGE = 1,     // a page number outside [1, page count]
    LOAD_BAD_TYPE = 2,                  // a b-tree page that is not a table interior or leaf page
    LOAD_BAD_CELL = 3,                  // a cell pointer or cell outside its page
    LOAD_BAD_PAYLOAD = 4,               // a payload larger than the file, or a broken overflow chain
    LOAD_BAD_RECORD = 5,                // a record header that does not fit its payload, or a reserved serial type
    LOAD_BAD_TREE = 6,                  // a page reached twice, a level mixing interior and leaf pages, or too deep
    LOAD_ID_STORED = 7,                 // the id column is stored in the record: `id` is not a rowid alias
    LOAD_BAD_ORDER = 8,                 // a rowid not above the one before it (duplicate or misordered cells)
};
// REC_DAMAGED: a record decode_cell could not read (the load fails with a LoadError; the record holds no text to index)
enum RecStatus : uint32_t { REC_OK = 0, REC_TIMESTAMP = 1, REC_TOKENS = 2, REC_COST = 3, REC_MODEL = 4, REC_PROVIDER = 5, REC_DAMAGED = 6 };

struct DbGeom { const uint8_t* f; uint32_t ps, n_pages; };      // the file; page size (== usable size: no reserved bytes)
struct CellRef { uint64_t pay; uint32_t P, ovfl; };            // payload start (file offset), payload size, first overflow page
struct TextRef { uint32_t off, len; };                          // payload offset and length of a text; off == NONE: NULL
struct NameRef { CellRef cell; TextRef t; };

// per record, in rowid order
struct LoadRecs {
    int64_t *id, *ts; double* cost; int32_t* tok[5]; uint32_t* status;
    CellRef* cell; TextRef* text[2]; uint32_t* slot[2];
};
struct LoadDict { uint64_t* table; uint32_t* slot_code; NameRef* names; uint32_t cap; uint32_t* n_codes; unsigned long long* n_bytes; };

#if defined(__CUDA_ARCH__)
#define LGW_LOAD_CAS64(p, c, v) atomicCAS((unsigned long long*)(p), (unsigned long long)(c), (unsigned long long)(v))
#define LGW_LOAD_INC(p) atomicAdd((p), 1u)
#define LGW_LOAD_ADD64(p, v) atomicAdd((p), (unsigned long long)(v))
#define LGW_LOAD_VOLATILE volatile
#else                               // the host build runs the items one after another
LGW_LOAD uint64_t load_cas_(uint64_t* p, uint64_t c, uint64_t v) { const uint64_t o = *p; if (o == c) *p = v; return o; }
#define LGW_LOAD_CAS64(p, c, v) load_cas_((p), (c), (v))
#define LGW_LOAD_INC(p) ((*(p))++)
#define LGW_LOAD_ADD64(p, v) (*(p) += (v))
#define LGW_LOAD_VOLATILE
#endif

LGW_LOAD uint32_t be16(const uint8_t* p) { return (uint32_t)p[0] << 8 | p[1]; }
LGW_LOAD uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
LGW_LOAD bool page_ok(const DbGeom& g, uint64_t pg) { return pg >= 1 && pg <= g.n_pages; }
LGW_LOAD const uint8_t* page_at(const DbGeom& g, uint32_t pg) { return g.f + (uint64_t)(pg - 1) * g.ps; }

// a varint of at most `avail` bytes at p: its length, 0 when it would run past avail
LGW_LOAD uint32_t varint(const uint8_t* p, uint64_t avail, uint64_t& v) {
    v = 0;
    for (uint32_t i = 0; i < 8; ++i) {
        if (i >= avail) return 0;
        v = (v << 7) | (p[i] & 0x7Fu);
        if (!(p[i] & 0x80u)) return i + 1;
    }
    if (avail < 9) return 0;
    v = (v << 8) | p[8];
    return 9;
}

struct PageHdr { uint32_t type, ncells, right, ptrs, hdr_end; };   // ptrs: offset of the cell pointer array in the page

// the b-tree header of page pg; LOAD_OK or the error
LGW_LOAD uint32_t read_page(const DbGeom& g, uint64_t pg, PageHdr& h) {
    if (!page_ok(g, pg)) return LOAD_BAD_PAGE;
    const uint8_t* p = page_at(g, (uint32_t)pg);
    const uint32_t o = pg == 1 ? 100 : 0;
    h.type = p[o];
    if (h.type != 5 && h.type != 13) return LOAD_BAD_TYPE;
    h.ncells = be16(p + o + 3);
    h.right = h.type == 5 ? be32(p + o + 8) : 0;
    h.ptrs = o + (h.type == 5 ? 12 : 8);
    h.hdr_end = h.ptrs + 2 * h.ncells;
    return h.hdr_end > g.ps ? (uint32_t)LOAD_BAD_CELL : (uint32_t)LOAD_OK;
}

// offset of cell k of a page whose header read_page accepted; 0 when it lies outside the page
LGW_LOAD uint32_t cell_at(const DbGeom& g, const uint8_t* p, const PageHdr& h, uint32_t k) {
    const uint32_t c = be16(p + h.ptrs + 2 * k);
    return c >= h.hdr_end && c < g.ps ? c : 0;
}

// child k (k <= ncells) of an interior page; 0 on a cell outside the page (the caller's check of the child page reports it)
LGW_LOAD uint32_t interior_child(const DbGeom& g, uint32_t pg, const PageHdr& h, uint32_t k, uint32_t& err) {
    if (k == h.ncells) return h.right;
    const uint8_t* p = page_at(g, pg);
    const uint32_t c = cell_at(g, p, h, k);
    if (!c || c + 4 > g.ps) { err = LOAD_BAD_CELL; return 0; }
    return be32(p + c);
}

LGW_LOAD uint32_t local_size(uint32_t P, uint32_t U) {
    const uint32_t X = U - 35, M = ((U - 12) * 32 / 255) - 23;
    if (P <= X) return P;
    const uint32_t K = M + (P - M) % (U - 4);
    return K <= X ? K : M;
}
// the same for a cell of an index b-tree page: its own maximum local size X
LGW_LOAD uint32_t index_local_size(uint32_t P, uint32_t U) {
    const uint32_t X = ((U - 12) * 64 / 255) - 23, M = ((U - 12) * 32 / 255) - 23;
    if (P <= X) return P;
    const uint32_t K = M + (P - M) % (U - 4);
    return K <= X ? K : M;
}

// Sequential reader of one cell's payload: the local part, then each overflow page's U - 4 bytes after its next-page number.
struct PayCursor { const uint8_t* p; uint32_t left, next; bool bad; };

LGW_LOAD void cur_piece(const DbGeom& g, PayCursor& c) {
    if (!page_ok(g, c.next)) { c.bad = true; c.left = 0; return; }
    const uint8_t* pg = page_at(g, c.next);
    c.next = be32(pg);
    c.p = pg + 4;
    c.left = g.ps - 4;
}
LGW_LOAD void cur_skip(const DbGeom& g, PayCursor& c, uint32_t n) {
    while (n > c.left && !c.bad) { n -= c.left; cur_piece(g, c); }
    if (!c.bad) { c.p += n; c.left -= n; }
}
LGW_LOAD PayCursor cur_at(const DbGeom& g, const CellRef& r, uint32_t off) {
    PayCursor c{g.f + r.pay, local_size(r.P, g.ps), r.ovfl, false};
    cur_skip(g, c, off);
    return c;
}
LGW_LOAD uint32_t cur_get(const DbGeom& g, PayCursor& c) {
    if (!c.left) cur_piece(g, c);
    if (c.bad) return 0;
    --c.left;
    return *c.p++;
}
// a varint read through the cursor, at most `avail` bytes; its length, 0 when it would run past avail
LGW_LOAD uint32_t cur_varint(const DbGeom& g, PayCursor& c, uint64_t avail, uint64_t& v) {
    v = 0;
    for (uint32_t i = 0; i < 9; ++i) {
        if (i >= avail) return 0;
        const uint32_t b = cur_get(g, c);
        if (i == 8) { v = (v << 8) | b; return 9; }
        v = (v << 7) | (b & 0x7Fu);
        if (!(b & 0x80u)) return i + 1;
    }
    return 0;
}

// the overflow chain of a payload that spills `spill` bytes: every page in range, no more and no fewer than it needs
LGW_LOAD bool chain_ok(const DbGeom& g, uint32_t first, uint64_t spill) {
    const uint64_t pages = (spill + g.ps - 5) / (g.ps - 4);
    uint32_t pg = first;
    for (uint64_t i = 0; i < pages; ++i) {
        if (!page_ok(g, pg)) return false;
        pg = be32(page_at(g, pg));
    }
    return pg == 0;
}

// serial type -> body size; 10 and 11 are reserved (~0)
LGW_LOAD uint64_t serial_size(uint64_t t) {
    if (t <= 4) return t;
    if (t == 5) return 6;
    if (t == 6 || t == 7) return 8;
    if (t == 8 || t == 9) return 0;
    if (t < 12) return ~0ull;
    return (t - 12) / 2;
}

LGW_LOAD int64_t days_from_civil(int64_t y, uint32_t m, uint32_t d) {    // proleptic Gregorian, days since 1970-01-01
    y -= m <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const uint32_t yoe = (uint32_t)(y - era * 400);
    const uint32_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    const uint32_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int64_t)doe - 719468;
}

// `YYYY-MM-DDTHH:MM:SS[.ffffff]` exactly as datetime.isoformat() writes a naive datetime (a microsecond part only when it is
// not zero), years 0001-9999, a real calendar date: its microseconds since 1970-01-01 (usage.py to_us)
LGW_LOAD bool iso_to_us(const uint8_t* s, uint32_t n, int64_t& us) {
    if (n != 19 && n != 26) return false;
    uint32_t v[7] = {0, 0, 0, 0, 0, 0, 0};
    const uint8_t pos[7] = {0, 5, 8, 11, 14, 17, 20}, len[7] = {4, 2, 2, 2, 2, 2, 6};
    const uint8_t sep[6] = {'-', '-', 'T', ':', ':', '.'};
    for (uint32_t k = 0; k < 7; ++k) {
        if (k == 6 && n == 19) break;
        if (k && s[pos[k] - 1] != sep[k - 1]) return false;
        for (uint32_t i = 0; i < len[k]; ++i) {
            const uint32_t d = (uint32_t)s[pos[k] + i] - '0';
            if (d > 9) return false;
            v[k] = v[k] * 10 + d;
        }
    }
    const uint32_t y = v[0], mo = v[1], d = v[2];
    if (y < 1 || mo < 1 || mo > 12 || d < 1 || v[3] > 23 || v[4] > 59 || v[5] > 59 || (n == 26 && v[6] == 0)) return false;
    const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
    const uint32_t dim = mo == 2 ? 28 + leap : 30 + ((mo + (mo > 7)) & 1);
    if (d > dim) return false;
    us = ((days_from_civil(y, mo, d) * 86400 + v[3] * 3600 + v[4] * 60 + v[5]) * 1000000) + v[6];
    return true;
}

// Cell k of leaf page pg into record i: LOAD_OK or the structural error.  A value the table cannot hold sets recs.status[i].
LGW_LOAD uint32_t decode_cell(const DbGeom& g, uint32_t pg, uint32_t k, const LoadRecs& r, uint64_t i) {
    r.status[i] = REC_DAMAGED;                                      // until the record is read whole: no later pass follows
    r.cell[i] = CellRef{0, 0, 0};                                   // its (unset) text locations
    r.text[0][i] = r.text[1][i] = TextRef{LGW_LOAD_NONE, 0};
    PageHdr h;
    uint32_t err = read_page(g, pg, h);
    if (err) return err;
    const uint8_t* p = page_at(g, pg);
    const uint32_t c = cell_at(g, p, h, k);
    if (!c) return LOAD_BAD_CELL;
    uint64_t P, rowid;
    const uint32_t n1 = varint(p + c, g.ps - c, P);
    const uint32_t n2 = n1 ? varint(p + c + n1, g.ps - c - n1, rowid) : 0;
    if (!n2) return LOAD_BAD_CELL;
    if (P >= (1ull << 31) || P > (uint64_t)g.n_pages * (g.ps - 4)) return LOAD_BAD_PAYLOAD;
    const uint32_t L = local_size((uint32_t)P, g.ps), spilled = P > L;
    if ((uint64_t)c + n1 + n2 + L + 4 * spilled > g.ps) return LOAD_BAD_CELL;
    CellRef cell{(uint64_t)(pg - 1) * g.ps + c + n1 + n2, (uint32_t)P, spilled ? be32(p + c + n1 + n2 + L) : 0u};
    if (spilled && !chain_ok(g, cell.ovfl, P - L)) return LOAD_BAD_PAYLOAD;
    // record header: its size, then the serial types of the first ten fields (the table's columns; more are ignored)
    PayCursor cur = cur_at(g, cell, 0);
    uint64_t hs, t[10];
    uint32_t used = cur_varint(g, cur, P, hs), nf = 0;
    if (!used || hs < used || hs > P) return LOAD_BAD_RECORD;
    uint64_t body = 0;
    while (used < hs && nf < 10) {
        const uint32_t b = cur_varint(g, cur, hs - used, t[nf]);
        const uint64_t sz = serial_size(t[nf]);
        if (!b || sz > P) return LOAD_BAD_RECORD;
        used += b;
        body += sz;
        ++nf;
    }
    if (cur.bad || body > P - hs) return LOAD_BAD_RECORD;
    if (nf && t[0] != 0) return LOAD_ID_STORED;
    // the fields, in order
    cur = cur_at(g, cell, (uint32_t)hs);
    uint32_t st = nf < 2 ? (uint32_t)REC_TIMESTAMP : (uint32_t)REC_OK;
    int64_t ts = 0;
    int32_t tok[5] = {0, 0, 0, 0, 0};
    double cost = 0.0;
    TextRef text[2] = {{LGW_LOAD_NONE, 0}, {LGW_LOAD_NONE, 0}};
    uint32_t off = (uint32_t)hs;
    for (uint32_t f = 1; f < nf; ++f) {
        const uint64_t ty = t[f];
        const uint32_t sz = (uint32_t)serial_size(ty);
        if (f == 1) {                                               // timestamp
            uint8_t s[26];
            if (ty >= 13 && (ty & 1) && (sz == 19 || sz == 26)) {
                for (uint32_t b = 0; b < sz; ++b) s[b] = (uint8_t)cur_get(g, cur);
                if (!iso_to_us(s, sz, ts) && !st) st = REC_TIMESTAMP;
            } else {
                cur_skip(g, cur, sz);
                if (!st) st = REC_TIMESTAMP;
            }
        } else if (f <= 7) {                                        // the five token columns, then cost
            const bool is_cost = f == 7;
            uint64_t u = 0;
            if (ty >= 1 && ty <= 7) { for (uint32_t b = 0; b < sz; ++b) u = (u << 8) | cur_get(g, cur); }
            else cur_skip(g, cur, sz);
            if (ty == 7) {                                          // REAL: a cost; never a token count
                if (is_cost) memcpy(&cost, &u, 8);
                else if (!st) st = REC_TOKENS;
            } else if (ty == 0) {                                   // NULL: a token count of 0 (SUM skips it), a NaN cost
                if (is_cost) { const uint64_t nan = 0x7FF8000000000000ull; memcpy(&cost, &nan, 8); }
            } else if (ty <= 9) {                                   // INTEGER
                const int64_t v = ty >= 8 ? (int64_t)ty - 8 : sz == 8 ? (int64_t)u : (int64_t)(u << (64 - 8 * sz)) >> (64 - 8 * sz);
                if (is_cost) cost = (double)v;
                else if (v < -(1ll << 31) || v >= (1ll << 31)) { if (!st) st = REC_TOKENS; }
                else tok[f - 2] = (int32_t)v;
            } else if (!st) {                                       // TEXT, BLOB
                st = is_cost ? REC_COST : REC_TOKENS;
            }
        } else {                                                    // model, provider
            if (ty >= 13 && (ty & 1)) text[f - 8] = TextRef{off, sz};
            else if (ty != 0 && !st) st = f == 8 ? REC_MODEL : REC_PROVIDER;
            cur_skip(g, cur, sz);
        }
        off += sz;
    }
    if (cur.bad) return LOAD_BAD_PAYLOAD;
    r.id[i] = (int64_t)rowid;
    r.ts[i] = ts;
    for (int c5 = 0; c5 < 5; ++c5) r.tok[c5][i] = tok[c5];
    r.cost[i] = cost;
    r.status[i] = st;
    r.cell[i] = cell;
    r.text[0][i] = text[0];
    r.text[1][i] = text[1];
    return LOAD_OK;
}

LGW_LOAD uint64_t text_hash(const DbGeom& g, const CellRef& c, const TextRef& t) {
    PayCursor cur = cur_at(g, c, t.off);
    uint64_t h = 0xCBF29CE484222325ull;
    for (uint32_t b = 0; b < t.len; ++b) h = (h ^ cur_get(g, cur)) * 0x100000001B3ull;
    return h;
}
LGW_LOAD bool text_eq(const DbGeom& g, const CellRef& ca, const TextRef& ta, const CellRef& cb, const TextRef& tb) {
    if (ta.len != tb.len) return false;
    PayCursor a = cur_at(g, ca, ta.off), b = cur_at(g, cb, tb.off);
    for (uint32_t k = 0; k < ta.len; ++k) if (cur_get(g, a) != cur_get(g, b)) return false;
    return true;
}
LGW_LOAD void text_copy(const DbGeom& g, const CellRef& c, const TextRef& t, uint8_t* out) {
    PayCursor cur = cur_at(g, c, t.off);
    for (uint32_t b = 0; b < t.len; ++b) out[b] = (uint8_t)cur_get(g, cur);
}

// text `field` of record i into the dictionary: its slot (LGW_LOAD_NONE for a NULL text).  A slot word is the hash's high 32
// bits above (owner record + 1); 0 is empty.  The table has at least twice as many slots as records, so a probe finds one.
LGW_LOAD uint32_t dict_insert(const DbGeom& g, const LoadRecs& r, uint32_t field, const LoadDict& d, uint32_t i) {
    const TextRef t = r.text[field][i];
    if (t.off == LGW_LOAD_NONE) return LGW_LOAD_NONE;
    const CellRef c = r.cell[i];
    const uint64_t h = text_hash(g, c, t), mine = (h >> 32) << 32 | (uint64_t)(i + 1);
    uint32_t s = (uint32_t)h & (d.cap - 1);
    for (uint32_t probe = 0; probe < d.cap; ++probe, s = (s + 1) & (d.cap - 1)) {
        uint64_t w = ((LGW_LOAD_VOLATILE uint64_t*)d.table)[s];
        if (w == 0) {
            w = LGW_LOAD_CAS64(d.table + s, 0ull, mine);
            if (w == 0) {
                const uint32_t code = LGW_LOAD_INC(d.n_codes);
                d.slot_code[s] = code;
                d.names[code] = NameRef{c, t};
                LGW_LOAD_ADD64(d.n_bytes, t.len);
                return s;
            }
        }
        if ((w >> 32) == (h >> 32)) {
            const uint32_t o = (uint32_t)w - 1;
            if (text_eq(g, r.cell[o], r.text[field][o], c, t)) return s;
        }
    }
    return LGW_LOAD_NONE;
}

// record i's dictionary step: its two texts into their dictionaries when none of its values is refused (a REC_DAMAGED record
// has none); LOAD_BAD_ORDER when its rowid is not above the previous record's (record order is rowid order)
LGW_LOAD uint32_t dict_record(const DbGeom& g, const LoadRecs& r, uint32_t i, const LoadDict& dm, const LoadDict& dp) {
    const bool ok = r.status[i] == REC_OK;
    r.slot[0][i] = ok ? dict_insert(g, r, 0, dm, i) : LGW_LOAD_NONE;
    r.slot[1][i] = ok ? dict_insert(g, r, 1, dp, i) : LGW_LOAD_NONE;
    return i && r.id[i] <= r.id[i - 1] ? (uint32_t)LOAD_BAD_ORDER : (uint32_t)LOAD_OK;
}

// record i stays: no refused value, and neither text refused by the host's maps (-1)
LGW_LOAD bool load_keep(const LoadRecs& r, const uint32_t* const code[2], const int32_t* const map[2], uint32_t i) {
    if (r.status[i]) return false;
    for (int f = 0; f < 2; ++f) {
        const uint32_t s = r.slot[f][i];
        if (s != LGW_LOAD_NONE && map[f][code[f][s]] < 0) return false;
    }
    return true;
}

struct LoadOut { int64_t* ts; int32_t* i32[6]; double* cost; int64_t* id; int32_t* prov; int64_t* refused; };

// kept record i at place `to`: the eight columns (model rank from map[0], 0 for NULL), its id and provider code (map[1], 0: NULL)
LGW_LOAD void load_store(const LoadRecs& r, const uint32_t* const code[2], const int32_t* const map[2], uint32_t i, uint32_t to, const LoadOut& o) {
    const uint32_t sm = r.slot[0][i], sp = r.slot[1][i];
    o.ts[to] = r.ts[i];
    o.i32[0][to] = sm == LGW_LOAD_NONE ? 0 : map[0][code[0][sm]];
    for (int c = 0; c < 5; ++c) o.i32[1 + c][to] = r.tok[c][i];
    o.cost[to] = r.cost[i];
    o.id[to] = r.id[i];
    o.prov[to] = sp == LGW_LOAD_NONE ? 0 : map[1][code[1][sp]];
}

#if defined(__CUDACC__)
// each page of a level: checked, marked visited, its children (interior) or cells (leaf) counted; kinds |= 1 interior, 2 leaf
__global__ void __launch_bounds__(256) k_load_count(const DbGeom g, const uint32_t* __restrict__ level, uint32_t m, uint32_t* __restrict__ cnt,
                                                    uint32_t* visited, uint32_t* kinds, uint32_t* err) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        PageHdr h;
        const uint32_t pg = level[i];
        uint32_t e = read_page(g, pg, h);
        if (!e && (atomicOr(visited + (pg >> 5), 1u << (pg & 31)) >> (pg & 31) & 1)) e = LOAD_BAD_TREE;
        if (e) { atomicMax(err, e); cnt[i] = 0; continue; }
        cnt[i] = h.ncells + (h.type == 5);
        atomicOr(kinds, h.type == 5 ? 1u : 2u);
    }
}

// the children of each interior page of a level, in key order, at the places k_list_scan gave: a block per page
__global__ void __launch_bounds__(128) k_load_children(const DbGeom g, const uint32_t* __restrict__ level, uint32_t m, const uint32_t* __restrict__ off,
                                                       uint32_t* __restrict__ next, uint32_t* err) {
    for (uint32_t i = blockIdx.x; i < m; i += gridDim.x) {
        PageHdr h;
        const uint32_t pg = level[i];
        if (read_page(g, pg, h)) continue;
        for (uint32_t k = threadIdx.x; k <= h.ncells; k += blockDim.x) {
            uint32_t e = 0;
            next[off[i] + k] = interior_child(g, pg, h, k, e);
            if (e) atomicMax(err, e);
        }
    }
}

// every cell of the leaf level: a block per page, a thread per cell; record index = the page's scan offset + cell index
__global__ void __launch_bounds__(128) k_load_decode(const DbGeom g, const uint32_t* __restrict__ level, uint32_t m, const uint32_t* __restrict__ off,
                                                     const LoadRecs r, uint32_t* err) {
    for (uint32_t i = blockIdx.x; i < m; i += gridDim.x) {
        PageHdr h;
        const uint32_t pg = level[i];
        if (read_page(g, pg, h)) continue;
        for (uint32_t k = threadIdx.x; k < h.ncells; k += blockDim.x) {
            const uint32_t e = decode_cell(g, pg, k, r, (uint64_t)off[i] + k);
            if (e) atomicMax(err, e);
        }
    }
}

// model and provider texts of the records not refused so far into their dictionaries, and the rowid order checked.  Nothing
// after a structural error of the decode: the load fails, so there is nothing to index.
__global__ void __launch_bounds__(256) k_load_dict(const DbGeom g, const LoadRecs r, uint32_t n, const LoadDict dm, const LoadDict dp, uint32_t* err) {
    if (*(volatile uint32_t*)err) return;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t e = dict_record(g, r, i, dm, dp);
        if (e) atomicMax(err, e);
    }
}

// kept records of each tile; used[code] = 1 for each model code a kept record has
__global__ void __launch_bounds__(1024) k_load_mark(const LoadRecs r, uint32_t n, const uint32_t* const code0, const uint32_t* const code1,
                                                    const int32_t* map0, const int32_t* map1, uint8_t* used, uint32_t* __restrict__ tile_count) {
    __shared__ WarpSums<uint32_t> warp_sums;
    const uint32_t* const code[2] = {code0, code1};
    const int32_t* const map[2] = {map0, map1};
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t c = 0;
    for (uint32_t i = 2 * j; i < 2 * j + 2 && i < n; ++i) {
        if (!load_keep(r, code, map, i)) continue;
        ++c;
        const uint32_t s = r.slot[0][i];
        if (s != LGW_LOAD_NONE) used[code0[s]] = 1;
    }
    c = block_sum(c, threadIdx.x, blockDim.x, warp_sums);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = c;
}

// kept records at their places (tile offset + the kept records before them in the tile); a refused record's id at its index
// minus the kept records before it.  Places at or past n_keep / n - n_keep are not stored.
__global__ void __launch_bounds__(1024) k_load_finish(const LoadRecs r, uint32_t n, const uint32_t* const code0, const uint32_t* const code1,
                                                      const int32_t* map0, const int32_t* map1, const uint32_t* __restrict__ tile_off,
                                                      uint32_t n_keep, const LoadOut o) {
    __shared__ WarpSums<uint32_t> warp_sums;
    const uint32_t* const code[2] = {code0, code1};
    const int32_t* const map[2] = {map0, map1};
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const bool ka = 2 * j < n && load_keep(r, code, map, 2 * j), kb = 2 * j + 1 < n && load_keep(r, code, map, 2 * j + 1);
    uint32_t pos = tile_off[blockIdx.x] + warp_place(ka, kb, threadIdx.x, warp_sums);
    for (uint32_t i = 2 * j; i < 2 * j + 2 && i < n; ++i) {
        const bool keep = i == 2 * j ? ka : kb;
        if (keep) { if (pos < n_keep) load_store(r, code, map, i, pos, o); ++pos; }
        else if (i - pos < n - n_keep) o.refused[i - pos] = r.id[i];
    }
}
#endif

}  // namespace lgw
