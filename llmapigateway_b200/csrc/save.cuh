// Saving the usage table as a `tokens_usage` SQLite file (the file load.cuh reads): every b-tree page and overflow page of the
// table and of idx_tokens_usage_timestamp is composed on the device; the host adds page 1 (header and sqlite_schema) and page 2
// (sqlite_sequence).  SQLite's documented file format is all this relies on.
//
// File layout, pages in this order: 1 schema, 2 sqlite_sequence, then the "pool" -- the table's leaves, its interior levels
// bottom up, the index's leaves, its interior levels -- then the overflow pages, each record's chain on consecutive pages in
// record order.  Pool page g is page LGW_SAVE_POOL0 + g of this order; its file page is save_page() of that, which steps over
// the lock-byte page (the page holding file offset 2^30, which SQLite never uses and refuses to read) in files that reach it.
//
//  1. Keep (k_save_count, k_list_scan, k_save_keep; tiles of LGW_LOAD_TILE records): a record is kept when it has an
//     isoformat text (years 0001-9999) and UTF-8 model and provider texts (the host marks the others).  Kept records get
//     their table cell size, overflow page count and sort key (ts_us - the smallest kept ts_us); refused ones give their ids.
//  2. Sort: the stable LSD radix sort of listing.cuh over the 8-bit digits the key range needs, so that the index entries
//     (timestamp text, rowid) come in BINARY order: text order is ts_us order, and ties stay in id order.
//  3. Pack (k_save_pack, a thread per tile of save_tile(page size) items; k_list_scan; k_save_gather): each tile fills pages
//     greedily in item order, so pages never cross a tile (at most one partly filled page per tile) and the result has no
//     atomics.  Table leaves hold records; a table interior page holds children, the last one as its right-most pointer; an
//     index page is followed by the entry that divides it from the next page, which moves up a level (a non-last tile keeps
//     its last entry for that).  One level per round, until a level has one page: the root.
//  4. Write (k_save_pages, a block per pool page): cells built in shared memory, packed at the end of the page in cell order
//     with no freeblocks, then the page out with 16-byte stores; k_save_chains writes the overflow chains.
#pragma once
#include <stdint.h>
#include <string.h>

#include "load.cuh"
#include "rollup.cuh"

#define LGW_SAVE LGW_LOAD
#define LGW_SAVE_TILE 2048u                       /* pack tile at 4 KiB pages and below: items a thread packs into pages */
#define LGW_SAVE_NULL 0xFFFFFFFFu                 /* SaveText.len of NULL */
#define LGW_SAVE_BAD 0xFFFFFFFEu                  /* SaveText.len of a text the file cannot hold (not UTF-8) */
#define LGW_SAVE_POOL0 3u                         /* file page of pool page 0 */
#define LGW_SAVE_MAX_LEVELS 16u
#define LGW_SAVE_TS_MIN (-62135596800000000ll)    /* 0001-01-01T00:00:00 in ts_us */
#define LGW_SAVE_TS_MAX 253402300799999999ll      /* 9999-12-31T23:59:59.999999 */

namespace lgw {

enum SaveKind : uint32_t { SAVE_TABLE_LEAF = 0, SAVE_TABLE_INTERIOR = 1, SAVE_INDEX_LEAF = 2, SAVE_INDEX_INTERIOR = 3 };

struct SaveText { const uint8_t* blob; const uint64_t* off; const uint32_t* len; uint32_t n, pad; };   // == lgw_save_text
struct SaveIn { const int64_t* ts; const int32_t* i32[6]; const double* cost; const int64_t* id; const int32_t* prov; SaveText text[2]; };
struct PageDesc { uint64_t up; uint32_t start, cnt; };     // cells [start, start + cnt) of its level's items; up: see gather_page

// what the page writers read: kept record of each kept place, kept place of each sorted entry, table cell sizes and first
// overflow pages of the kept places, the pool, where each level of each tree starts in it
struct SaveCtx {
    SaveIn in; uint32_t U;
    const uint32_t *kidx, *sidx, *lsz, *lov;
    const PageDesc* pool;
    uint32_t base[2][LGW_SAVE_MAX_LEVELS + 1], levels[2];
    uint32_t lock;                                          // the lock-byte page: 2^30 / U + 1
};

// file page of page p of the layout: the pages from the lock-byte page on move up by one
LGW_SAVE uint32_t save_page(const SaveCtx& c, uint32_t p) { return p >= c.lock ? p + 1 : p; }

LGW_SAVE uint32_t varint_len(uint64_t v) {
    if (v >> 56) return 9;
    uint32_t n = 1;
    while (v >= 128) { v >>= 7; ++n; }
    return n;
}
LGW_SAVE uint32_t put_varint(uint8_t* p, uint64_t v) {
    if (v >> 56) {
        p[8] = (uint8_t)v;
        v >>= 8;
        for (int i = 7; i >= 0; --i) { p[i] = (uint8_t)((v & 0x7F) | 0x80); v >>= 7; }
        return 9;
    }
    const uint32_t n = varint_len(v);
    for (int i = (int)n - 1; i >= 0; --i) { p[i] = (uint8_t)((v & 0x7F) | (i == (int)n - 1 ? 0 : 0x80)); v >>= 7; }
    return n;
}
LGW_SAVE void put_be(uint8_t* p, uint64_t v, uint32_t bytes) { for (uint32_t i = 0; i < bytes; ++i) p[i] = (uint8_t)(v >> (8 * (bytes - 1 - i))); }

// serial type of an integer as SQLite stores it (schema format 4: 0 and 1 take no body bytes), and its body size
LGW_SAVE uint32_t int_type(int64_t v) {
    if (v == 0) return 8;
    if (v == 1) return 9;
    const uint64_t u = v < 0 ? ~(uint64_t)v : (uint64_t)v;
    return u < 0x80ull ? 1 : u < 0x8000ull ? 2 : u < 0x800000ull ? 3 : u < 0x80000000ull ? 4 : u < 0x800000000000ull ? 5 : 6;
}
LGW_SAVE uint32_t int_bytes(uint32_t t) { return t >= 8 ? 0 : t == 5 ? 6 : t == 6 ? 8 : t; }

// datetime.isoformat() of a ts_us in [LGW_SAVE_TS_MIN, LGW_SAVE_TS_MAX]: `YYYY-MM-DDTHH:MM:SS`, `.ffffff` when not zero
LGW_SAVE uint32_t iso_text(int64_t us, uint8_t* s) {
    const int64_t days = fdiv(us, 86400000000ll), rem = us - days * 86400000000ll;
    int64_t y; int m, d;
    civil_from_days(days, y, m, d);
    const uint32_t sec = (uint32_t)(rem / 1000000), frac = (uint32_t)(rem % 1000000);
    const uint32_t v[7] = {(uint32_t)y, (uint32_t)m, (uint32_t)d, sec / 3600, sec / 60 % 60, sec % 60, frac};
    const uint8_t pos[7] = {0, 5, 8, 11, 14, 17, 20}, len[7] = {4, 2, 2, 2, 2, 2, 6}, sep[6] = {'-', '-', 'T', ':', ':', '.'};
    const uint32_t n = frac ? 26 : 19;
    for (uint32_t k = 0; k < 7; ++k) {
        if (k == 6 && !frac) break;
        if (k) s[pos[k] - 1] = sep[k - 1];
        uint32_t x = v[k];
        for (int i = len[k] - 1; i >= 0; --i) { s[pos[k] + i] = (uint8_t)('0' + x % 10); x /= 10; }
    }
    return n;
}
LGW_SAVE uint32_t iso_len(int64_t us) { return us % 1000000 ? 26 : 19; }

// One record's payload: `pre` (the record header, the timestamp text, the token and cost bytes) and the model and provider texts.
struct SaveRec { uint8_t pre[80]; uint32_t npre, P; const uint8_t* t[2]; uint32_t tl[2]; };

enum SaveStatus : uint32_t { SAVE_KEEP = 0, SAVE_REFUSE = 1, SAVE_BAD_CODE = 2 };

// record i's payload; SAVE_REFUSE for a record the file cannot hold, SAVE_BAD_CODE for a model rank or provider code outside
// its text table (a caller's error)
LGW_SAVE uint32_t save_rec(const SaveIn& in, uint32_t i, SaveRec& r) {
    const int64_t ts = in.ts[i];
    uint32_t st[10];
    const int32_t code[2] = {in.i32[0][i], in.prov[i]};
    uint32_t status = ts < LGW_SAVE_TS_MIN || ts > LGW_SAVE_TS_MAX ? (uint32_t)SAVE_REFUSE : (uint32_t)SAVE_KEEP;
    for (int f = 0; f < 2; ++f) {
        const SaveText& x = in.text[f];
        if (code[f] < 0 || (uint32_t)code[f] >= x.n) return SAVE_BAD_CODE;
        const uint32_t len = x.len[code[f]];
        if (len == LGW_SAVE_BAD) status = SAVE_REFUSE;
        r.t[f] = len >= LGW_SAVE_BAD ? nullptr : x.blob + x.off[code[f]];
        r.tl[f] = len >= LGW_SAVE_BAD ? 0 : len;
        st[8 + f] = len >= LGW_SAVE_BAD ? 0 : 13 + 2 * len;
    }
    if (status) return status;
    uint8_t txt[26];
    const uint32_t tl = iso_text(ts, txt);
    st[0] = 0;                                              // id: the rowid alias, NULL in the record
    st[1] = 13 + 2 * tl;
    int32_t tok[5];
    for (int c = 0; c < 5; ++c) { tok[c] = in.i32[1 + c][i]; st[2 + c] = int_type(tok[c]); }
    const double cost = in.cost[i];
    st[7] = cost != cost ? 0 : 7;                           // NaN: NULL; anything else as the 8-byte REAL it is
    uint32_t hs = 1;
    for (int k = 0; k < 10; ++k) hs += varint_len(st[k]);  // (< 128: the header size takes one byte)
    uint8_t* p = r.pre;
    uint32_t o = put_varint(p, hs);
    for (int k = 0; k < 10; ++k) o += put_varint(p + o, st[k]);
    memcpy(p + o, txt, tl);
    o += tl;
    for (int c = 0; c < 5; ++c) { const uint32_t b = int_bytes(st[2 + c]); put_be(p + o, (uint64_t)(int64_t)tok[c], b); o += b; }
    if (st[7]) { uint64_t u; memcpy(&u, &cost, 8); put_be(p + o, u, 8); o += 8; }
    r.npre = o;
    r.P = o + r.tl[0] + r.tl[1];
    return SAVE_KEEP;
}

// payload bytes [lo, hi) of a record to dst
LGW_SAVE void rec_bytes(const SaveRec& r, uint32_t lo, uint32_t hi, uint8_t* dst) {
    const uint8_t* piece[3] = {r.pre, r.t[0], r.t[1]};
    const uint32_t len[3] = {r.npre, r.tl[0], r.tl[1]};
    uint32_t at = 0;
    for (int k = 0; k < 3; ++k) {
        const uint32_t a = lo > at ? lo : at, b = hi < at + len[k] ? hi : at + len[k];
        for (uint32_t x = a; x < b; ++x) dst[x - lo] = piece[k][x - at];
        at += len[k];
    }
}

// a table leaf cell: its size and overflow pages
LGW_SAVE uint32_t table_cell_size(const SaveRec& r, int64_t id, uint32_t U, uint32_t& ovfl) {
    const uint32_t L = local_size(r.P, U);
    ovfl = r.P > L ? (r.P - L + U - 5) / (U - 4) : 0;
    return varint_len(r.P) + varint_len((uint64_t)id) + L + (r.P > L ? 4 : 0);
}

// index entry (timestamp, rowid) of record r: its payload size.  At most 37 bytes: below any page's index_local_size limit,
// so an index cell never spills.
LGW_SAVE uint32_t entry_payload(const SaveIn& in, uint32_t r) { return 3 + iso_len(in.ts[r]) + int_bytes(int_type(in.id[r])); }
LGW_SAVE uint32_t entry_write(const SaveIn& in, uint32_t r, uint8_t* p) {
    const int64_t ts = in.ts[r], id = in.id[r];
    const uint32_t t = int_type(id), b = int_bytes(t);
    p[0] = 3;
    const uint32_t tl = iso_text(ts, p + 3);
    p[1] = (uint8_t)(13 + 2 * tl);
    p[2] = (uint8_t)t;
    put_be(p + 3 + tl, (uint64_t)id, b);
    return 3 + tl + b;
}

// ---- packing -------------------------------------------------------------------------------------------------------------
// Items [s, e) of a level (sizes isz, pointer excluded) into pages; the page count.  Page j of the tile: its cells are items
// [pstart[j], pstart[j] + pcnt[j]).  The item after them is a table interior page's right-most child, or the entry between an
// index page and the next.  `last`: the level's last tile.  An empty level gives one empty page (an empty tree's root).
LGW_SAVE uint32_t pack_tile(const uint32_t* isz, uint32_t s, uint32_t e, bool last, uint32_t kind, uint32_t U, uint32_t* pstart, uint32_t* pcnt) {
    const uint32_t hdr = kind == SAVE_TABLE_LEAF || kind == SAVE_INDEX_LEAF ? 8 : 12;
    const bool divides = kind >= SAVE_INDEX_LEAF;
    if (s == e) { pstart[0] = s; pcnt[0] = 0; return 1; }
    if (divides && !last) --e;                              // the tile's last entry divides it from the next tile
    uint32_t np = 0, k = s;
    while (k < e) {
        const uint32_t st = k;
        uint32_t used = hdr;
        if (kind == SAVE_TABLE_INTERIOR) {                  // cells while they fit; the next child is the right-most pointer
            while (k + 1 < e && used + isz[k] + 2 <= U) { used += isz[k] + 2; ++k; }
            pstart[np] = st; pcnt[np] = k - st; ++np; ++k;
            if (k == e && pcnt[np - 1] == 0 && np > 1) {    // a last page with one child takes the one before it
                --pcnt[np - 2];
                pstart[np - 1] = st - 1; pcnt[np - 1] = 1;
            }
            continue;
        }
        while (k < e && used + isz[k] + 2 <= U) { used += isz[k] + 2; ++k; }
        if (!divides || k == e) { pstart[np] = st; pcnt[np] = k - st; ++np; continue; }
        if (k + 1 == e) {                                   // the entry that does not fit is the last one: the entry before it
            pstart[np] = st; pcnt[np] = k - 1 - st; ++np;   // divides, and it fills the last page alone
            pstart[np] = k; pcnt[np] = 1; ++np;
            k = e;
            continue;
        }
        pstart[np] = st; pcnt[np] = k - st; ++np; ++k;      // entry k divides this page from the next
    }
    return np;
}

// items per pack tile: LGW_SAVE_TILE, grown with pages above 4 KiB so that a tile spans about as many pages at any size
LGW_SAVE uint32_t save_tile(uint32_t U) { return U > 4096 ? LGW_SAVE_TILE * (U / 4096) : LGW_SAVE_TILE; }
// tiles of a level of m items: whole tiles, the last one taking the rest (so every tile has `tile` items or more, or is the only one)
LGW_SAVE uint32_t pack_tiles(uint32_t m, uint32_t tile) { const uint32_t t = m / tile; return t ? t : 1; }
LGW_SAVE void tile_range(uint32_t t, uint32_t tiles, uint32_t m, uint32_t tile, uint32_t& s, uint32_t& e) { s = t * tile; e = t + 1 == tiles ? m : s + tile; }

// overflow pages of the kept places [s, e): lov holds each one's count, then its exclusive offset within the tile; the total
LGW_SAVE uint32_t ovfl_tile(uint32_t* lov, uint32_t s, uint32_t e) {
    uint32_t run = 0;
    for (uint32_t k = s; k < e; ++k) { const uint32_t c = lov[k]; lov[k] = run; run += c; }
    return run;
}

// Page g_local of a level (tree 0 table, 1 index; m items) from its tile slot into the pool at `at`.  up: a table page's largest
// rowid; an index page's following entry (the sorted place of the entry that divides it from the next page).  isz_next gets
// the page's item of the next level: a table interior cell (child, key), or an index interior cell (child, entry).
LGW_SAVE void gather_page(const SaveCtx& c, uint32_t tree, uint32_t level, uint32_t m, uint32_t slot, uint32_t g_local, const uint32_t* pstart,
                          const uint32_t* pcnt, PageDesc* pool, uint32_t at, uint32_t* isz_next) {
    PageDesc d{0, pstart[slot], pcnt[slot]};
    const uint32_t nx = d.start + d.cnt;
    const PageDesc* below = level ? pool + c.base[tree][level - 1] : nullptr;
    if (tree == 0) d.up = level ? below[nx].up : d.cnt ? (uint64_t)c.in.id[c.kidx[nx - 1]] : 0;
    else d.up = nx < m ? (level ? below[nx].up : nx) : 0;
    pool[at + g_local] = d;
    if (tree == 0) isz_next[g_local] = 4 + varint_len(d.up);
    else isz_next[g_local] = nx < m ? 5 + entry_payload(c.in, c.kidx[c.sidx[d.up]]) : 0;
}

// ---- writing -------------------------------------------------------------------------------------------------------------
LGW_SAVE uint32_t page_kind(const SaveCtx& c, uint32_t g, uint32_t& level) {
    const uint32_t tree = g >= c.base[1][0];
    level = 0;
    while (level + 1 < c.levels[tree] && g >= c.base[tree][level + 1]) ++level;
    return tree ? (level ? SAVE_INDEX_INTERIOR : SAVE_INDEX_LEAF) : (level ? SAVE_TABLE_INTERIOR : SAVE_TABLE_LEAF);
}

// cell `item` of a page of this kind and level: its size, and its bytes at dst
LGW_SAVE uint32_t cell_size(const SaveCtx& c, uint32_t kind, uint32_t level, uint32_t item) {
    if (kind == SAVE_TABLE_LEAF) return c.lsz[item];
    if (kind == SAVE_INDEX_LEAF) return 1 + entry_payload(c.in, c.kidx[c.sidx[item]]);
    const PageDesc& child = c.pool[c.base[kind == SAVE_INDEX_INTERIOR][level - 1] + item];
    if (kind == SAVE_TABLE_INTERIOR) return 4 + varint_len(child.up);
    return 5 + entry_payload(c.in, c.kidx[c.sidx[child.up]]);
}
LGW_SAVE void cell_write(const SaveCtx& c, uint32_t kind, uint32_t level, uint32_t item, uint8_t* dst) {
    if (kind == SAVE_TABLE_LEAF) {
        const uint32_t r = c.kidx[item];
        SaveRec rec;
        save_rec(c.in, r, rec);
        const uint32_t L = local_size(rec.P, c.U);
        uint32_t o = put_varint(dst, rec.P);
        o += put_varint(dst + o, (uint64_t)c.in.id[r]);
        rec_bytes(rec, 0, L, dst + o);
        if (rec.P > L) put_be(dst + o + L, save_page(c, c.lov[item]), 4);
        return;
    }
    if (kind == SAVE_INDEX_LEAF) {
        const uint32_t r = c.kidx[c.sidx[item]];
        dst[0] = (uint8_t)entry_payload(c.in, r);
        entry_write(c.in, r, dst + 1);
        return;
    }
    const uint32_t tree = kind == SAVE_INDEX_INTERIOR, b = c.base[tree][level - 1];
    put_be(dst, save_page(c, LGW_SAVE_POOL0 + b + item), 4);
    const uint64_t up = c.pool[b + item].up;
    if (!tree) { put_varint(dst + 4, up); return; }
    const uint32_t r = c.kidx[c.sidx[up]];
    dst[4] = (uint8_t)entry_payload(c.in, r);
    entry_write(c.in, r, dst + 5);
}
LGW_SAVE uint32_t page_hdr(uint32_t kind) { return kind == SAVE_TABLE_LEAF || kind == SAVE_INDEX_LEAF ? 8 : 12; }
// the b-tree page header, for cells taking `total` bytes at the end of the page
LGW_SAVE void page_header(const SaveCtx& c, uint32_t kind, uint32_t level, const PageDesc& d, uint32_t total, uint8_t* p) {
    const uint8_t type[4] = {13, 5, 10, 2};
    p[0] = type[kind];
    p[1] = p[2] = 0;
    put_be(p + 3, d.cnt, 2);
    put_be(p + 5, (c.U - total) & 0xFFFF, 2);              // (65536: 0)
    p[7] = 0;
    if (kind == SAVE_TABLE_INTERIOR || kind == SAVE_INDEX_INTERIOR)
        put_be(p + 8, save_page(c, LGW_SAVE_POOL0 + c.base[kind == SAVE_INDEX_INTERIOR][level - 1] + d.start + d.cnt), 4);
}

// the overflow chain of kept place k, if it has one, on its pages (img: file page LGW_SAVE_POOL0 at offset 0)
LGW_SAVE uint8_t* page_in(const SaveCtx& c, uint8_t* img, uint32_t p) { return img + (uint64_t)(save_page(c, p) - LGW_SAVE_POOL0) * c.U; }
LGW_SAVE void write_chain(const SaveCtx& c, uint32_t k, uint8_t* img) {
    SaveRec rec;
    save_rec(c.in, c.kidx[k], rec);
    const uint32_t U = c.U, L = local_size(rec.P, U);
    if (rec.P <= L) return;
    const uint32_t n = (rec.P - L + U - 5) / (U - 4);
    for (uint32_t j = 0; j < n; ++j) {
        const uint32_t pg = c.lov[k] + j, lo = L + j * (U - 4), hi = rec.P - lo > U - 4 ? lo + U - 4 : rec.P;
        uint8_t* p = page_in(c, img, pg);
        put_be(p, j + 1 < n ? save_page(c, pg + 1) : 0, 4);
        rec_bytes(rec, lo, hi, p + 4);
        memset(p + 4 + (hi - lo), 0, U - 4 - (hi - lo));
    }
}

#if defined(__CUDACC__)
// kept records of each tile of LGW_LOAD_TILE; the smallest and largest kept sort key (ts_us - LGW_SAVE_TS_MIN); rowid order
// and text codes checked (err |= 1: a rowid not above the one before it, 2: a code outside its text table)
__global__ void __launch_bounds__(1024) k_save_count(const SaveIn in, uint32_t n, uint32_t* __restrict__ tile_count, unsigned long long* kmin,
                                                     unsigned long long* kmax, uint32_t* err) {
    __shared__ WarpSums<uint32_t> warp_sums;
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t c = 0, e = 0;
    unsigned long long lo = ~0ull, hi = 0;
    for (uint32_t i = 2 * j; i < 2 * j + 2 && i < n; ++i) {
        SaveRec r;
        const uint32_t s = save_rec(in, i, r);
        if (s == SAVE_BAD_CODE) e |= 2;
        if (i && in.id[i] <= in.id[i - 1]) e |= 1;
        if (s != SAVE_KEEP) continue;
        ++c;
        const unsigned long long k = (unsigned long long)(in.ts[i] - LGW_SAVE_TS_MIN);
        lo = k < lo ? k : lo;
        hi = k > hi ? k : hi;
    }
    for (int o = 16; o; o >>= 1) {                         // a warp's extremes, then one atomic each
        const unsigned long long a = __shfl_xor_sync(0xFFFFFFFFu, lo, o), b = __shfl_xor_sync(0xFFFFFFFFu, hi, o);
        lo = a < lo ? a : lo;
        hi = b > hi ? b : hi;
    }
    if ((threadIdx.x & 31u) == 0 && lo != ~0ull) { atomicMin(kmin, lo); atomicMax(kmax, hi); }
    if (e) atomicOr(err, e);
    c = block_sum(c, threadIdx.x, blockDim.x, warp_sums);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = c;
}

// kept records at their places: kidx, table cell size (lsz), overflow page count (lov), sort key and identity index; a refused
// record's id at its index minus the kept records before it
__global__ void __launch_bounds__(1024) k_save_keep(const SaveIn in, uint32_t n, uint32_t U, const uint32_t* __restrict__ tile_off,
                                                    const unsigned long long* kmin, uint32_t* kidx, uint32_t* lsz, uint32_t* lov,
                                                    uint64_t* key, uint32_t* idx, int64_t* refused) {
    __shared__ WarpSums<uint32_t> warp_sums;
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    SaveRec ra, rb;
    const bool ka = 2 * j < n && save_rec(in, 2 * j, ra) == SAVE_KEEP, kb = 2 * j + 1 < n && save_rec(in, 2 * j + 1, rb) == SAVE_KEEP;
    uint32_t pos = tile_off[blockIdx.x] + warp_place(ka, kb, threadIdx.x, warp_sums);
    const unsigned long long k0 = *kmin;
    for (uint32_t i = 2 * j; i < 2 * j + 2 && i < n; ++i) {
        const bool keep = i == 2 * j ? ka : kb;
        if (keep) {
            uint32_t ov;
            kidx[pos] = i;
            lsz[pos] = table_cell_size(i == 2 * j ? ra : rb, in.id[i], U, ov);
            lov[pos] = ov;
            key[pos] = (uint64_t)(in.ts[i] - LGW_SAVE_TS_MIN) - k0;
            idx[pos] = pos;
            ++pos;
        } else refused[i - pos] = in.id[i];
    }
}

// entry e's index leaf cell size, in sorted order
__global__ void __launch_bounds__(256) k_save_entry_sizes(const SaveIn in, const uint32_t* __restrict__ kidx, const uint32_t* __restrict__ sidx,
                                                          uint32_t m, uint32_t* isz) {
    for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < m; e += gridDim.x * blockDim.x) isz[e] = 1 + entry_payload(in, kidx[sidx[e]]);
}

// a thread per tile: its pages (tile_pages[t]) and their slots; for the table's leaves also each tile's overflow pages
__global__ void __launch_bounds__(128) k_save_pack(const uint32_t* __restrict__ isz, uint32_t m, uint32_t tiles, uint32_t kind, uint32_t U,
                                                   uint32_t* pstart, uint32_t* pcnt, uint32_t* tile_pages, uint32_t* lov, uint32_t* tile_ovfl) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= tiles) return;
    uint32_t s, e;
    tile_range(t, tiles, m, save_tile(U), s, e);
    tile_pages[t] = pack_tile(isz, s, e, t + 1 == tiles, kind, U, pstart + s, pcnt + s);
    if (lov) tile_ovfl[t] = ovfl_tile(lov, s, e);
}

// the pages of each tile into the pool, at the level's start `at` + the tile's page offset
__global__ void __launch_bounds__(128) k_save_gather(const SaveCtx c, uint32_t tree, uint32_t level, uint32_t m, uint32_t tiles,
                                                     const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ pstart,
                                                     const uint32_t* __restrict__ pcnt, PageDesc* pool, uint32_t at, uint32_t* isz_next) {
    for (uint32_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        uint32_t s, e;
        tile_range(t, tiles, m, save_tile(c.U), s, e);
        const uint32_t np = tile_off[t + 1] - tile_off[t];
        for (uint32_t jj = threadIdx.x; jj < np; jj += blockDim.x)
            gather_page(c, tree, level, m, s + jj, tile_off[t] + jj, pstart, pcnt, pool, at, isz_next);
    }
}

// each kept record's first overflow page: base + its tile's offset + its offset within the tile
__global__ void __launch_bounds__(256) k_save_ovfl_abs(uint32_t* lov, uint32_t m, uint32_t tiles, uint32_t tile, const uint32_t* __restrict__ tile_off, uint32_t base) {
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        const uint32_t t = k / tile;
        lov[k] += base + tile_off[t < tiles ? t : tiles - 1];
    }
}

// a block per pool page: cells built in shared memory (dynamic, U bytes), packed at the end in cell order, then written out
__global__ void __launch_bounds__(256) k_save_pages(const SaveCtx c, uint32_t n_pages, uint8_t* __restrict__ img) {
    extern __shared__ uint4 page4[];
    __shared__ WarpSums<uint32_t> warp_sums;
    uint8_t* page = reinterpret_cast<uint8_t*>(page4);
    const uint32_t U = c.U;
    for (uint32_t g = blockIdx.x; g < n_pages; g += gridDim.x) {
        for (uint32_t w = threadIdx.x; w < U / 16; w += blockDim.x) page4[w] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        uint32_t level;
        const uint32_t kind = page_kind(c, g, level), hdr = page_hdr(kind);
        const PageDesc d = c.pool[g];
        const uint32_t total = block_scan<uint32_t>(d.cnt, threadIdx.x, blockDim.x, warp_sums,
            [&](uint32_t k) { return cell_size(c, kind, level, d.start + k); },
            [&](uint32_t k, uint32_t off) {
                const uint32_t at = U - off - cell_size(c, kind, level, d.start + k);
                cell_write(c, kind, level, d.start + k, page + at);
                put_be(page + hdr + 2 * k, at, 2);
            });
        if (threadIdx.x == 0) page_header(c, kind, level, d, total, page);
        __syncthreads();
        uint4* out = reinterpret_cast<uint4*>(page_in(c, img, LGW_SAVE_POOL0 + g));
        for (uint32_t w = threadIdx.x; w < U / 16; w += blockDim.x) out[w] = page4[w];
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_save_chains(const SaveCtx c, uint32_t m, uint8_t* img) {
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) write_chain(c, k, img);
}
#endif

}  // namespace lgw
