// TEST AID ONLY: the usage-table loader of csrc/load.cuh (read_page, interior_child, decode_cell, dict_insert, load_keep,
// load_store) built with g++ and driven item by item in the order the kernels run them, behind the same four calls as
// lgw_usage_load_decode / _names / _mark / _finish (without the engine; d_cols is ignored).  Built as a shared library for the
// CPU tests and, with LGWT_MAIN, as a program the damaged-file tests run under -fsanitize=address.  Never linked into the
// product library; the product has no CPU path.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../llmapigateway_b200/csrc/load.cuh"

using namespace lgw;

namespace {
struct State {
    DbGeom g{};
    uint32_t n = 0, n_names[2]{};
    uint64_t n_keep = 0;
    std::vector<int64_t> id, ts; std::vector<double> cost; std::vector<int32_t> tok[5]; std::vector<uint32_t> status;
    std::vector<CellRef> cell; std::vector<TextRef> text[2]; std::vector<uint32_t> slot[2];
    std::vector<uint64_t> table[2]; std::vector<uint32_t> slot_code[2]; std::vector<NameRef> names[2];
    uint32_t codes[2]{}; unsigned long long bytes[2]{};
    LoadRecs r{};
} S;
}

extern "C" int lgwt_load_decode(const uint8_t* file, uint64_t n_bytes, uint32_t ps, uint32_t n_pages, uint32_t root, uint64_t out[6]) {
    if (ps < 512 || ps > 65536 || (ps & (ps - 1)) || n_pages == 0 || (uint64_t)n_pages * ps > n_bytes) return -1;
    S = State();
    const DbGeom g{file, ps, n_pages};
    S.g = g;
    std::vector<uint32_t> level{root}, cnt;
    std::vector<uint32_t> visited(n_pages / 32 + 1, 0);
    uint32_t err = 0, seen = 1, total = 0;
    for (uint32_t depth = 0;; ++depth) {                 // k_load_count, k_list_scan, k_load_children
        if (depth == LGW_LOAD_MAX_DEPTH) { err = LOAD_BAD_TREE; break; }
        uint32_t kinds = 0;
        cnt.assign(level.size(), 0);
        for (size_t i = 0; i < level.size(); ++i) {
            PageHdr h;
            const uint32_t pg = level[i];
            uint32_t e = read_page(g, pg, h);
            if (!e && (visited[pg >> 5] >> (pg & 31) & 1)) e = LOAD_BAD_TREE;
            if (!e) visited[pg >> 5] |= 1u << (pg & 31);
            if (e) { if (e > err) err = e; continue; }
            cnt[i] = h.ncells + (h.type == 5);
            kinds |= h.type == 5 ? 1u : 2u;
        }
        total = 0;
        for (auto& c : cnt) { const uint32_t v = c; c = total; total += v; }
        if (err) break;
        if (kinds == 3) { err = LOAD_BAD_TREE; break; }
        if (kinds == 2) break;
        seen += total;
        if (seen > n_pages) { err = LOAD_BAD_TREE; break; }
        std::vector<uint32_t> next(total, 0);
        for (size_t i = 0; i < level.size(); ++i) {
            PageHdr h;
            if (read_page(g, level[i], h)) continue;
            for (uint32_t k = 0; k <= h.ncells; ++k) {
                uint32_t e = 0;
                next[cnt[i] + k] = interior_child(g, level[i], h, k, e);
                if (e > err) err = e;
            }
        }
        level.swap(next);
    }
    const uint32_t n = err ? 0 : total;
    S.n = n;
    // the record arrays start as stale memory would: an unread record looks valid, with a text far outside the file
    const uint64_t far = (uint64_t)n_pages * ps + (1ull << 20);
    S.id.assign(n, 0); S.ts.assign(n, 0); S.cost.assign(n, 0); S.status.assign(n, REC_OK); S.cell.assign(n, CellRef{far, 64, 0});
    LoadRecs& r = S.r;
    r.id = S.id.data(); r.ts = S.ts.data(); r.cost = S.cost.data(); r.status = S.status.data(); r.cell = S.cell.data();
    for (int k = 0; k < 5; ++k) { S.tok[k].assign(n, 0); r.tok[k] = S.tok[k].data(); }
    uint32_t cap = 64;
    while (cap < 2ull * n) cap <<= 1;
    LoadDict d[2];
    for (int f = 0; f < 2; ++f) {
        S.text[f].assign(n, TextRef{0, 48}); S.slot[f].assign(n, LGW_LOAD_NONE);
        r.text[f] = S.text[f].data(); r.slot[f] = S.slot[f].data();
        S.table[f].assign(cap, 0); S.slot_code[f].assign(cap, 0); S.names[f].assign(n ? n : 1, NameRef{});
        d[f] = LoadDict{S.table[f].data(), S.slot_code[f].data(), S.names[f].data(), cap, &S.codes[f], &S.bytes[f]};
    }
    if (n) {                                              // k_load_decode
        for (size_t i = 0; i < level.size(); ++i) {
            PageHdr h;
            if (read_page(g, level[i], h)) continue;
            for (uint32_t k = 0; k < h.ncells; ++k) {
                const uint32_t e = decode_cell(g, level[i], k, r, (uint64_t)cnt[i] + k);
                if (e > err) err = e;
            }
        }
    }
    // k_load_dict skips its pass after a decode error; the host build runs it regardless, so that the records decode_cell
    // failed on are read here as the kernel would read them without that check
    const uint32_t decode_err = err;
    for (uint32_t i = 0; i < n; ++i) {                    // k_load_dict
        const uint32_t e = dict_record(g, r, i, d[0], d[1]);
        if (e > err) err = e;
    }
    if (decode_err) err = decode_err;
    S.n_names[0] = S.codes[0]; S.n_names[1] = S.codes[1];
    out[0] = err; out[1] = n; out[2] = S.codes[0]; out[3] = S.codes[1]; out[4] = S.bytes[0]; out[5] = S.bytes[1];
    return 0;
}

extern "C" int lgwt_load_names(const uint8_t* file, int field, uint8_t* buf, uint64_t* offs) {
    const DbGeom hg{file, S.g.ps, S.g.n_pages};
    uint64_t at = 0;
    for (uint32_t c = 0; c < S.n_names[field]; ++c) {
        offs[c] = at;
        text_copy(hg, S.names[field][c].cell, S.names[field][c].t, buf + at);
        at += S.names[field][c].t.len;
    }
    offs[S.n_names[field]] = at;
    return 0;
}

extern "C" int lgwt_load_mark(const int32_t* mm, const int32_t* pm, uint8_t* used, uint64_t* n_keep) {
    const uint32_t* code[2] = {S.slot_code[0].data(), S.slot_code[1].data()};
    const int32_t* map[2] = {mm, pm};
    if (S.n_names[0]) memset(used, 0, S.n_names[0]);
    uint64_t k = 0;
    for (uint32_t i = 0; i < S.n; ++i) {
        if (!load_keep(S.r, code, map, i)) continue;
        ++k;
        if (S.r.slot[0][i] != LGW_LOAD_NONE) used[code[0][S.r.slot[0][i]]] = 1;
    }
    S.n_keep = *n_keep = k;
    return 0;
}

extern "C" int lgwt_load_finish(const int32_t* mm, const int32_t* pm, void* const* d_cols, void* const h_cols[8], int64_t* ids, int32_t* prov, int64_t* refused) {
    (void)d_cols;
    const uint32_t* code[2] = {S.slot_code[0].data(), S.slot_code[1].data()};
    const int32_t* map[2] = {mm, pm};
    LoadOut o{(int64_t*)h_cols[0], {}, (double*)h_cols[7], ids, prov, refused};
    for (int c = 0; c < 6; ++c) o.i32[c] = (int32_t*)h_cols[1 + c];
    uint32_t pos = 0;
    for (uint32_t i = 0; i < S.n; ++i) {
        if (load_keep(S.r, code, map, i)) { if (pos < S.n_keep) load_store(S.r, code, map, i, pos, o); ++pos; }
        else if (i - pos < S.n - S.n_keep) refused[i - pos] = S.r.id[i];
    }
    return 0;
}

extern "C" int lgwt_load_release() {
    S = State();
    return 0;
}

#ifdef LGWT_MAIN
// host_load <file> <page size> <page count> <root page>: the file read into a buffer of exactly its size, every call run with
// maps that refuse nothing; prints "err records kept models providers"
int main(int argc, char** argv) {
    if (argc != 5) return 2;
    FILE* fp = fopen(argv[1], "rb");
    if (!fp) return 2;
    fseek(fp, 0, SEEK_END);
    const long size = ftell(fp);
    fseek(fp, 0, SEEK_SET);
    uint8_t* file = (uint8_t*)malloc(size ? size : 1);
    if (fread(file, 1, size, fp) != (size_t)size) return 2;
    fclose(fp);
    uint64_t out[6];
    if (lgwt_load_decode(file, size, atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), out)) { printf("arg\n"); free(file); return 0; }
    uint64_t kept = 0;
    if (!out[0]) {
        std::vector<uint8_t> mb(out[4] + 1), pb(out[5] + 1);
        std::vector<uint64_t> mo(out[2] + 1), po(out[3] + 1);
        lgwt_load_names(file, 0, mb.data(), mo.data());
        lgwt_load_names(file, 1, pb.data(), po.data());
        std::vector<int32_t> mm(out[2] + 1, 0), pm(out[3] + 1, 1);
        std::vector<uint8_t> used(out[2] + 1);
        lgwt_load_mark(mm.data(), pm.data(), used.data(), &kept);
        std::vector<int64_t> c64[2] = {std::vector<int64_t>(kept + 1), std::vector<int64_t>(kept + 1)};
        std::vector<int32_t> c32[7];
        for (auto& v : c32) v.assign(kept + 1, 0);
        void* h[8] = {c64[0].data(), c32[0].data(), c32[1].data(), c32[2].data(), c32[3].data(), c32[4].data(), c32[5].data(), c64[1].data()};
        std::vector<int64_t> ids(kept + 1), refused(out[1] - kept + 1);
        lgwt_load_finish(mm.data(), pm.data(), nullptr, h, ids.data(), c32[6].data(), refused.data());
    }
    printf("%llu %llu %llu %llu %llu\n", (unsigned long long)out[0], (unsigned long long)out[1], (unsigned long long)kept,
           (unsigned long long)out[2], (unsigned long long)out[3]);
    free(file);
    return 0;
}
#endif
