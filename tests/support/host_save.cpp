// TEST AID ONLY: the usage-table writer of csrc/save.cuh (save_rec, table_cell_size, pack_tile, ovfl_tile, gather_page,
// cell_size / cell_write / page_header, write_chain) built with g++ and driven item by item in the order the kernels run
// them, behind the same calls as lgw_usage_save_plan / _write / _release (without the engine; d_cols are host columns).  The
// sort is std::stable_sort on the same key, which orders exactly as the stable LSD passes do.  Built as a shared library for
// the CPU tests and, with LGWT_MAIN, as a program run under -fsanitize=address.  Never linked into the product library; the
// product has no CPU path.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../llmapigateway_b200/csrc/save.cuh"

using namespace lgw;

namespace {
struct State {
    std::vector<int64_t> ids; std::vector<int32_t> prov;
    std::vector<uint64_t> off[2]; std::vector<uint32_t> len[2]; std::vector<uint8_t> blob[2];
    std::vector<uint32_t> kidx, lsz, lov, sidx, pstart, pcnt, isz[2], tpages, tovfl;
    std::vector<int64_t> refused;
    std::vector<PageDesc> pool;
    SaveCtx c{};
    uint32_t n = 0, kept = 0, n_pool = 0, n_ovfl = 0;
    uint64_t pages = 0;
    bool planned = false;
} S;

// k_list_scan: exclusive offsets in place; the total
uint32_t scan(std::vector<uint32_t>& v, uint32_t len) {
    uint32_t run = 0;
    for (uint32_t k = 0; k < len; ++k) { const uint32_t x = v[k]; v[k] = run; run += x; }
    v[len] = run;
    return run;
}
}

extern "C" int lgwt_save_release() {
    S = State();
    return 0;
}

extern "C" int lgwt_save_plan(void* const cols[8], uint64_t n, const int64_t* h_ids, const int32_t* h_prov, const SaveText* models,
                              const SaveText* providers, uint32_t U, uint64_t out[5]) {
    if (n >= (1ull << 32) || U < 1024 || U > 65536 || (U & (U - 1))) return -1;
    lgwt_save_release();
    const uint32_t N = (uint32_t)n, M = N ? N : 1;
    // the inputs copied as the device's are (exactly their sizes, so that a read past them is seen under ASan)
    S.ids.assign(h_ids, h_ids + N);
    S.prov.assign(h_prov, h_prov + N);
    const SaveText* tx[2] = {models, providers};
    SaveIn in{};
    in.ts = (const int64_t*)cols[0]; in.cost = (const double*)cols[7];
    for (int c = 0; c < 6; ++c) in.i32[c] = (const int32_t*)cols[1 + c];
    in.id = S.ids.data(); in.prov = S.prov.data();
    for (int f = 0; f < 2; ++f) {
        const uint32_t k = tx[f]->n;
        S.off[f].assign(tx[f]->off, tx[f]->off + k + 1);
        S.len[f].assign(tx[f]->len, tx[f]->len + k);
        S.blob[f].assign(tx[f]->blob, tx[f]->blob + tx[f]->off[k]);
        in.text[f] = SaveText{S.blob[f].data(), S.off[f].data(), S.len[f].data(), k, 0};
    }
    // k_save_count: rowid order, codes, the key range
    uint64_t kmin = ~0ull, kmax = 0;
    uint32_t K = 0;
    for (uint32_t i = 0; i < N; ++i) {
        SaveRec r;
        const uint32_t s = save_rec(in, i, r);
        if (s == SAVE_BAD_CODE || (i && in.id[i] <= in.id[i - 1])) return -2;
        if (s != SAVE_KEEP) continue;
        ++K;
        const uint64_t k = (uint64_t)(in.ts[i] - LGW_SAVE_TS_MIN);
        kmin = std::min(kmin, k);
        kmax = std::max(kmax, k);
    }
    // k_save_keep
    S.kidx.assign(M, 0); S.lsz.assign(M, 0); S.lov.assign(M, 0); S.refused.assign(N - K + 1, 0);
    std::vector<uint64_t> key(M, 0);
    uint32_t pos = 0;
    for (uint32_t i = 0; i < N; ++i) {
        SaveRec r;
        if (save_rec(in, i, r) != SAVE_KEEP) { S.refused[i - pos] = in.id[i]; continue; }
        uint32_t ov;
        S.kidx[pos] = i;
        S.lsz[pos] = table_cell_size(r, in.id[i], U, ov);
        S.lov[pos] = ov;
        key[pos] = (uint64_t)(in.ts[i] - LGW_SAVE_TS_MIN) - kmin;
        ++pos;
    }
    // the sort
    S.sidx.resize(M);
    for (uint32_t k = 0; k < M; ++k) S.sidx[k] = k;
    std::stable_sort(S.sidx.begin(), S.sidx.begin() + K, [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
    // pack, level by level
    const uint32_t tile = save_tile(U), ptiles = pack_tiles(K, tile), pool_cap = 4 * M + 4 * LGW_SAVE_MAX_LEVELS;
    S.pstart.assign(M, 0); S.pcnt.assign(M, 0); S.isz[0].assign(M, 0); S.isz[1].assign(M, 0);
    S.tpages.assign(ptiles + 1, 0); S.tovfl.assign(ptiles + 1, 0);
    S.pool.assign(pool_cap, PageDesc{0, 0, 0});
    SaveCtx& c = S.c;
    c.in = in; c.U = U; c.kidx = S.kidx.data(); c.sidx = S.sidx.data(); c.lsz = S.lsz.data(); c.lov = S.lov.data(); c.pool = S.pool.data();
    c.lock = (1u << 30) / U + 1;
    uint32_t used = 0, n_ovfl = 0;
    for (uint32_t tree = 0; tree < 2; ++tree) {
        const uint32_t* isz = S.lsz.data();
        uint32_t* next = S.isz[0].data();
        if (tree == 1) {                                              // k_save_entry_sizes
            for (uint32_t e = 0; e < K; ++e) S.isz[0][e] = 1 + entry_payload(in, S.kidx[S.sidx[e]]);
            isz = S.isz[0].data(); next = S.isz[1].data();
        }
        uint32_t m = K, kind = tree ? SAVE_INDEX_LEAF : SAVE_TABLE_LEAF;
        for (uint32_t level = 0;; ++level) {
            if (level == LGW_SAVE_MAX_LEVELS) return -3;
            const uint32_t tiles = pack_tiles(m, tile);
            const bool ovfl = tree == 0 && level == 0;
            for (uint32_t t = 0; t < tiles; ++t) {                     // k_save_pack
                uint32_t s, e;
                tile_range(t, tiles, m, tile, s, e);
                S.tpages[t] = pack_tile(isz, s, e, t + 1 == tiles, kind, U, S.pstart.data() + s, S.pcnt.data() + s);
                if (ovfl) S.tovfl[t] = ovfl_tile(S.lov.data(), s, e);
            }
            const uint32_t P = scan(S.tpages, tiles);
            if (ovfl) n_ovfl = scan(S.tovfl, tiles);
            if ((uint64_t)used + P > pool_cap) return -4;
            c.base[tree][level] = used;
            for (uint32_t t = 0; t < tiles; ++t) {                     // k_save_gather
                uint32_t s, e;
                tile_range(t, tiles, m, tile, s, e);
                for (uint32_t j = 0; j < S.tpages[t + 1] - S.tpages[t]; ++j)
                    gather_page(c, tree, level, m, s + j, S.tpages[t] + j, S.pstart.data(), S.pcnt.data(), S.pool.data(), used, next);
            }
            used += P;
            if (P == 1) { c.levels[tree] = level + 1; c.base[tree][level + 1] = used; break; }
            m = tree ? P - 1 : P;
            kind = tree ? SAVE_INDEX_INTERIOR : SAVE_TABLE_INTERIOR;
            isz = next;
            next = next == S.isz[0].data() ? S.isz[1].data() : S.isz[0].data();
        }
    }
    for (uint32_t k = 0; k < K; ++k) {                                 // k_save_ovfl_abs
        const uint32_t t = k / tile;
        S.lov[k] += LGW_SAVE_POOL0 + used + S.tovfl[t < ptiles ? t : ptiles - 1];
    }
    const uint64_t laid = 2ull + used + n_ovfl;
    S.n = N; S.kept = K; S.n_pool = used; S.n_ovfl = n_ovfl; S.pages = laid + (laid >= c.lock); S.planned = true;
    out[0] = S.pages;
    out[1] = save_page(c, LGW_SAVE_POOL0 + c.base[0][c.levels[0] - 1]);
    out[2] = save_page(c, LGW_SAVE_POOL0 + c.base[1][c.levels[1] - 1]);
    out[3] = K; out[4] = N - K;
    return 0;
}

extern "C" int lgwt_save_write(uint8_t* h_file, int64_t* h_refused) {
    if (!S.planned) return -1;
    const SaveCtx& c = S.c;
    const uint32_t U = c.U;
    uint8_t* img = h_file + 2ull * U;
    std::vector<uint8_t> page(U);
    if (S.pages > c.lock) memset(img + (uint64_t)(c.lock - LGW_SAVE_POOL0) * U, 0, U);       // the lock-byte page
    for (uint32_t g = 0; g < S.n_pool; ++g) {                         // k_save_pages: one page at a time
        memset(page.data(), 0, U);
        uint32_t level;
        const uint32_t kind = page_kind(c, g, level), hdr = page_hdr(kind);
        const PageDesc d = c.pool[g];
        uint32_t off = 0;
        for (uint32_t k = 0; k < d.cnt; ++k) {
            const uint32_t sz = cell_size(c, kind, level, d.start + k), at = U - off - sz;
            cell_write(c, kind, level, d.start + k, page.data() + at);
            put_be(page.data() + hdr + 2 * k, at, 2);
            off += sz;
        }
        page_header(c, kind, level, d, off, page.data());
        memcpy(page_in(c, img, LGW_SAVE_POOL0 + g), page.data(), U);
    }
    for (uint32_t k = 0; S.n_ovfl && k < S.kept; ++k) write_chain(c, k, img);      // k_save_chains
    if (S.n > S.kept) memcpy(h_refused, S.refused.data(), 8ull * (S.n - S.kept));
    return lgwt_save_release();
}

#ifdef LGWT_MAIN
// host_save <columns file> <page size> <out file>: the columns file holds n, then the eight columns, ids, provider codes, and
// for models and providers the text count k, k + 1 offsets, k lengths and the blob -- every array read into a buffer of
// exactly its size.  Writes pages 3 .. of the file (pages 1 and 2 zero) and prints "pages table_root index_root kept refused".
static uint8_t* slurp(FILE* fp, uint64_t bytes) {
    uint8_t* p = (uint8_t*)malloc(bytes ? bytes : 1);
    if (bytes && fread(p, 1, bytes, fp) != bytes) exit(2);
    return p;
}
int main(int argc, char** argv) {
    if (argc != 4) return 2;
    FILE* fp = fopen(argv[1], "rb");
    if (!fp) return 2;
    uint64_t n;
    if (fread(&n, 8, 1, fp) != 1) return 2;
    static const uint32_t width[8] = {8, 4, 4, 4, 4, 4, 4, 8};
    void* cols[8];
    for (int c = 0; c < 8; ++c) cols[c] = slurp(fp, width[c] * n);
    int64_t* ids = (int64_t*)slurp(fp, 8 * n);
    int32_t* prov = (int32_t*)slurp(fp, 4 * n);
    SaveText t[2];
    for (int f = 0; f < 2; ++f) {
        uint64_t k;
        if (fread(&k, 8, 1, fp) != 1) return 2;
        uint64_t* off = (uint64_t*)slurp(fp, 8 * (k + 1));
        uint32_t* len = (uint32_t*)slurp(fp, 4 * k);
        t[f] = SaveText{slurp(fp, off[k]), off, len, (uint32_t)k, 0};
    }
    fclose(fp);
    uint64_t out[5];
    const int rc = lgwt_save_plan(cols, n, ids, prov, &t[0], &t[1], (uint32_t)atoi(argv[2]), out);
    if (rc) { printf("plan %d\n", rc); return 0; }
    const uint64_t bytes = out[0] * (uint64_t)atoi(argv[2]);
    uint8_t* file = (uint8_t*)calloc(bytes, 1);
    int64_t* refused = (int64_t*)malloc(8 * (out[4] + 1));
    lgwt_save_write(file, refused);
    FILE* fo = fopen(argv[3], "wb");
    if (!fo || fwrite(file, 1, bytes, fo) != bytes) return 2;
    fclose(fo);
    printf("%llu %llu %llu %llu %llu\n", (unsigned long long)out[0], (unsigned long long)out[1], (unsigned long long)out[2],
           (unsigned long long)out[3], (unsigned long long)out[4]);
    for (int c = 0; c < 8; ++c) free(cols[c]);
    free(ids); free(prov); free(file); free(refused);
    for (int f = 0; f < 2; ++f) { free((void*)t[f].blob); free((void*)t[f].off); free((void*)t[f].len); }
    return 0;
}
#endif
