// Bulk path of the SSE step, round 2:  k_relay2 -> k_commit2.
// (included from sse_kernels.cuh, inside namespace lgw)
//
// What changed against round 1 (relay_kernels.cuh, thread-per-chunk walk of a staged tile):
//   * The re-emit is done by the TMA engine: every warp owns a contiguous byte range and runs its own ring of
//     3 KiB shared-memory buffers -- cp.async.bulk global -> shared (mbarrier complete_tx), cp.async.bulk shared ->
//     global straight from the same buffer.  No byte of the copy passes through a register.
//   * The parse is warp-cooperative and driven by bytes, not by chunks: 16 bytes per lane, 512 bytes per pass.  SSE
//     deltas of a stream are the same JSON skeleton over and over, so the event text is compared against a PERIODIC
//     image of a validated event template (text ++ LF LF ++ text ...): one unaligned 16-byte load of the image per lane
//     (16 pre-shifted copies of the default template in shared memory make it an aligned LDS.128), one XOR/AND per word
//     against the literal mask, a SWAR test of the bytes that lie in string-value spans (control, quote, backslash)
//     and one ballot.  A pass that matches proves the boundaries and the validity of every event it covers
//     (the LF LF separators are literal bytes of the image).  A mismatch is classified by its template offset: inside
//     a string or number VALUE span the value's own end is found (ballot scan for the closing quote, number automaton)
//     and the comparison is re-anchored behind it; anywhere else the event is tried against the other template slots
//     and finally walked by the byte-wise recogniser (lean_json.cuh).  Same judgement as round 1's matcher: an event
//     that equals a template outside value spans, holds plain bytes / valid escapes inside string spans and a valid JSON
//     number in number spans drives the recogniser through the same states as the template.
//   * Usage extraction is on the clock: an event that follows a usage-bearing template has its eight fields read
//     straight from the value spans the match located (number text -> decimal.cuh, strings decoded like the full
//     machine does) into a per-segment candidate record that k_commit2 installs.  Usage events without such a template
//     are staged in shared memory by k_commit2 and read with the full machine right there: reading a stream's state is a
//     plain copy, nothing is deferred.
//
// Regular streams -- committed (or committing on their first chunk), carries empty and equal at the start of the bulk
// region, every chunk valid UTF-8 and non-empty, no run of three or more LFs, no event the tap turns into an extra row
// ("error"), at most one usage event per step, no event longer than the carry capacity -- are exactly the streams for
// which the reference's chunk-by-chunk split (request_handler.py:111-115, chat_logging.py:108-112) equals a split of
// the CONCATENATED text on every LF LF pair.  Everything else is flagged irregular and redone by k_commit2 with the
// exact sequential machine, so the result never depends on which path ran (tests run both and the oracle).
//
// The file also compiles with g++ against tests/support/simt_emu.h (fibers as lanes) so that the CPU test-suite can run
// these very kernels; that build is a test aid, the product has no CPU path.
#pragma once

#if defined(__CUDACC__)
#define R2_DEV __device__ __forceinline__
#define R2_MEM __device__ __forceinline__
#define R2_DEV_NOINLINE __device__ __noinline__
#define R2_GLOBAL __global__
#define R2_TID (threadIdx.x)
#define R2_BID (blockIdx.x)
#define R2_NBLK (gridDim.x)
#define R2_NTHR (blockDim.x)
#define R2_HOST_EMU 0
#else
#define R2_DEV static inline
#define R2_MEM inline
#define R2_DEV_NOINLINE static
#define R2_GLOBAL static
#define R2_TID (simt::tid())
#define R2_BID (simt::bid())
#define R2_NBLK (simt::nblocks())
#define R2_NTHR (simt::nthreads())
#define R2_HOST_EMU 1
#endif

#ifndef R2_WARPS                        /* (overridable for geometry experiments: make EXTRA="-DR2_WARPS=24u -DR2_TILE=2048u") */
#define R2_WARPS 16u
#endif
#define R2_THREADS (R2_WARPS * 32u)
#ifndef R2_TILE
#define R2_TILE 3072u                   /* a multiple of 512 (the fast loop walks whole 512-byte windows of a tile) */
#endif
#ifndef R2_NBUF
#define R2_NBUF 2u                      /* ring depth per warp.  2 x 3 KiB x 16 warps = 96 KiB: with the 33 KiB of tables the block takes the 132 KiB
                                           carve-out and leaves ~96 KiB of L1 for the out-of-line paths' local memory (672 B of stack per thread);
                                           on the H100 a 3-deep ring (144 KiB) was no faster (DESIGN 9.8) */
#endif
#define R2_SLOTS 4u
#define R2_TPL_MAX 504u                 /* longest event kept as a template (text without its LF LF) */
#define R2_TPL_MIN 16u
#define R2_TEXT 544u                    /* periodic image: period <= 506, + 16 + 15 bytes of run-over, rounded to 16 */
#define R2_SPANS 32u
#define R2_FULL 0xFFFFFFFFu
#define R2_NONE 0xFFFFFFFFu
#define R2_MAX_STR 8192u                /* longest string value the matcher follows (as in round 1) */

struct TplMeta {
    uint32_t len, P, recip, flags, cls, n_spans, usage_ok, full_flags;
    uint16_t sstart[R2_SPANS], send[R2_SPANS];     // value span: first content byte / first number char .. closing quote / terminator
    uint8_t skind[R2_SPANS];                       // 0 string value, 1 number value
    uint8_t field_span[8];                         // usage field (UsageField) -> span id, 0xff: the template's own value
};
struct Tpl2 {
    TplMeta m;
    uint8_t text[R2_TEXT];       // periodic image: text ++ LF LF ++ text ...
    uint8_t lit[R2_TEXT];        // 0xff: byte must equal the image; 0x00: content of a string value span
    uint8_t span_id[R2_TPL_MAX + 8];   // per text position: id of the value span it belongs to (sstart..send inclusive), 0xff none
};
// Event templates survive across launches (any validated event is a sound template wherever it came from).
// state: 0 empty, 1 being written, 2 ready.
struct TemplateCache2 {
    uint32_t state[R2_SLOTS];
    uint32_t hits[R2_SLOTS];         // events matched per slot (decayed once per launch set: tpl_cache_upkeep)
    uint32_t general;                // events that matched no slot
    uint32_t lock;                   // publication lock
    uint32_t _pad[2];
    Tpl2 tpl[R2_SLOTS];
    UsageRaw raw[R2_SLOTS];          // the template event's own UsageRaw (usage_ok slots)
};

// ---- shared memory of k_relay2 -------------------------------------------------------------------------------------
struct R2Shared {
    alignas(16) uint8_t fast_text[16 * R2_TEXT];     // default slot: copy c holds image[c ..], so image[t .. t+16) is an aligned vector of copy t & 15
    alignas(16) uint8_t fast_lit[16 * R2_TEXT];
    alignas(16) Tpl2 tpl[R2_SLOTS];
    alignas(8) UsageRaw raw_tpl[R2_SLOTS];           // the template events' own UsageRaw (usage_ok slots)
    alignas(8) unsigned long long mbar[R2_WARPS * R2_NBUF];
    uint32_t slot_state[R2_SLOTS];                   // 0 empty, 1 being built, 2 ready
    uint32_t slot_gidx[R2_SLOTS];                    // the same template's slot in the engine-wide cache (R2_NONE: local to this block)
    uint32_t hits[R2_SLOTS];
    uint32_t general;
    uint32_t dflt, fast_ready;
    uint32_t learn_lock;                             // one warp of the block learns a template at a time
    uint32_t plan_win[R2_WARPS][3][32];              // per warp: relay_begin / seg_end / kept_end of 32 consecutive segments (SegStatic)
    StepArgs args;                                   // the kernel's arguments (read through a pointer by the out-of-line paths: taking the
                                                     //   address of the parameter itself would move it to local memory)
    alignas(4) uint8_t cls[256];
    alignas(4) uint8_t trans[LGW_LEAN_ROWS * 32];
};
#define R2_RING_BYTES (R2_WARPS * R2_NBUF * R2_TILE)
#define R2_SMEM_BYTES (R2_RING_BYTES + sizeof(R2Shared) + 128)

// ---- platform layer: shared-window addresses, TMA, mbarrier ----------------------------------------------------------
#if !R2_HOST_EMU
typedef uint32_t SPtr;                         // 32-bit shared-window address
R2_DEV SPtr sptr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
R2_DEV uint4 sld128(SPtr a) { uint4 v; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)); return v; }
R2_DEV uint32_t sld32(SPtr a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
R2_DEV uint32_t sld8(SPtr a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
R2_DEV void sst8(SPtr a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
R2_DEV uint4 gld128(const uint8_t* p) { uint4 v; asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)); return v; }
R2_DEV void mbar_init(SPtr a, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(a), "r"(n)); }
R2_DEV void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
R2_DEV void mbar_expect(SPtr a, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(a), "r"(bytes) : "memory"); }
R2_DEV void mbar_wait(SPtr a, uint32_t parity) {
    asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}" :: "r"(a), "r"(parity) : "memory");
}
R2_DEV void tma_load(SPtr dst, const void* src, uint32_t bytes, SPtr mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" :: "r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
R2_DEV void tma_store(void* dst, SPtr src, uint32_t bytes) {
    asm volatile("fence.proxy.async.shared::cta;\ncp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\ncp.async.bulk.commit_group;" :: "l"(dst), "r"(src), "r"(bytes) : "memory");
}
R2_DEV void tma_store_commit_empty() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
R2_DEV void tma_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
R2_DEV void tma_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
R2_DEV uint8_t* smem_base() { extern __shared__ __align__(128) uint8_t r2_smem[]; return r2_smem; }
// programmatic dependent launch: the next kernel of the step may start its prologue while this one still runs; it waits here
// before it touches anything this one writes
R2_DEV void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
R2_DEV void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#else
typedef uint8_t* SPtr;
R2_DEV SPtr sptr(const void* p) { return (uint8_t*)p; }
R2_DEV uint4 sld128(SPtr a) { uint4 v; memcpy(&v, a, 16); return v; }
R2_DEV uint32_t sld32(SPtr a) { uint32_t v; memcpy(&v, a, 4); return v; }
R2_DEV uint32_t sld8(SPtr a) { return *a; }
R2_DEV void sst8(SPtr a, uint32_t v) { *a = (uint8_t)v; }
R2_DEV uint4 gld128(const uint8_t* p) { uint4 v; memcpy(&v, p, 16); return v; }
R2_DEV void mbar_init(SPtr a, uint32_t) { memset(a, 0, 8); }
R2_DEV void mbar_fence_init() {}
R2_DEV void mbar_expect(SPtr, uint32_t) {}
R2_DEV void mbar_wait(SPtr, uint32_t) {}
R2_DEV void tma_load(SPtr dst, const void* src, uint32_t bytes, SPtr) { memcpy(dst, src, bytes); }
R2_DEV void tma_store(void* dst, SPtr src, uint32_t bytes) { memcpy(dst, src, bytes); }
R2_DEV void tma_store_commit_empty() {}
R2_DEV void tma_wait_read1() {}
R2_DEV void tma_wait_all() {}
R2_DEV uint8_t* smem_base() { return simt::g_dyn_smem; }
R2_DEV void griddep_wait() {}
R2_DEV void griddep_launch() {}
#endif
R2_DEV uint32_t r2_min(uint32_t a, uint32_t b) { return a < b ? a : b; }
R2_DEV uint32_t r2_max(uint32_t a, uint32_t b) { return a > b ? a : b; }

// bit 7 of every byte: set <=> the byte is plain string content (>= 0x20, not '"', not '\\'; bytes >= 0x80 are plain) or lies
// outside a string span (m byte = 0xff)
R2_DEV uint32_t span_ok(uint32_t w, uint32_t m) {
    const uint32_t w7 = w & 0x7f7f7f7fu;
    const uint32_t a = w7 + 0x60606060u;
    const uint32_t b = (w7 ^ 0x22222222u) + 0x7f7f7f7fu;
    const uint32_t c = (w7 ^ 0x5c5c5c5cu) + 0x7f7f7f7fu;
    return (a & b & c) | w | m;
}
// bit 7 of every byte: set <=> byte != 0
R2_DEV uint32_t nonzero_bytes(uint32_t x) { return (((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x) & 0x80808080u; }
// bits 7/15/23/31 -> bits 0..3
R2_DEV uint32_t movemask4(uint32_t m) { return (((m >> 7) * 0x00204081u) >> 21) & 0xFu; }
// 16-bit mask of the bytes of a vector equal to LF
R2_DEV uint32_t lf_mask16(const uint4& d) {
    const uint32_t a = ~nonzero_bytes(d.x ^ 0x0a0a0a0au) & 0x80808080u, b = ~nonzero_bytes(d.y ^ 0x0a0a0a0au) & 0x80808080u;
    const uint32_t c = ~nonzero_bytes(d.z ^ 0x0a0a0a0au) & 0x80808080u, e = ~nonzero_bytes(d.w ^ 0x0a0a0a0au) & 0x80808080u;
    return movemask4(a) | (movemask4(b) << 4) | (movemask4(c) << 8) | (movemask4(e) << 12);
}

// ---- per-warp context --------------------------------------------------------------------------------------------------
struct R2Ctx {
    const StepArgs* a;
    R2Shared* sh;
    uint32_t lane;
    // pipeline
    SPtr ring; SPtr bars;
    uint32_t base;               // byte offset of this warp's tile 0 (16-byte aligned)
    uint32_t n_tiles;            // tiles of the range
    uint32_t k;                  // resident tile (R2_NONE before the first)
    uint32_t tile_lo, tile_hi;   // bytes of the resident tile [tile_lo, tile_hi): tile_hi is clamped to n_bytes
    SPtr buf;                    // its buffer
    uint32_t n_bytes;            // end of the valid bytes
    // segment
    uint32_t seg, tb, te, kept_end;    // text of the current segment [tb, te); kept_end: end of the speculatively kept chunk (0: none)
    uint32_t in_kept, primed, kept_tried;   // in_kept: 0 no kept chunk (any more), 1 walking it on its own, 2 walking it optimistically
    uint32_t ev_a, ev_b, a_usage;
    uint32_t high;               // some byte >= 0x80 was seen in the current segment's text
    uint32_t walk_lo;            // first text position this warp walked in the current segment
    // matcher
    uint32_t t, pos, s_open;
    uint32_t dflt, fast;         // default (periodic) slot of the block; its pre-shifted copies are ready
    uint32_t ready, free_slots;  // bit per slot: template usable / slot empty (refreshed by refresh_slots, the same in every lane)
    uint32_t last_ra;            // position of the last number re-anchor (a mismatch right there is final)
    uint32_t hits_d;             // events matched by the default slot
    uint32_t single;             // the stream's events follow the default slot but not its period (value spans of varying length):
                                 //   judge them one by one, span by span (match_single), instead of window passes that re-anchor
};

// Where bytes are read from: the resident tile in shared memory, global memory outside it.  A small value type: the
// out-of-line slow paths take a COPY, so that the warp context itself never has its address taken and stays in registers.
struct R2Io {
    const uint8_t* data; const R2Shared* sh;
    uint32_t n_bytes, tile_lo, tile_hi; SPtr buf;
};
R2_DEV R2Io io_of(const R2Ctx& c) { R2Io io; io.data = c.a->data; io.sh = c.sh; io.n_bytes = c.n_bytes; io.tile_lo = c.tile_lo; io.tile_hi = c.tile_hi; io.buf = c.buf; return io; }
R2_DEV uint8_t io_byte(const R2Io& io, uint32_t p) {
    if (p >= io.tile_lo && p < io.tile_hi) return (uint8_t)sld8(io.buf + (p - io.tile_lo));
    return p < io.n_bytes ? __ldg(io.data + p) : (uint8_t)0;
}
R2_DEV uint8_t ring_byte(const R2Ctx& c, uint32_t p) {
    if (p >= c.tile_lo && p < c.tile_hi) return (uint8_t)sld8(c.buf + (p - c.tile_lo));
    return p < c.n_bytes ? __ldg(c.a->data + p) : (uint8_t)0;
}
// byte source for the single-lane walks (recogniser, template builder, field readers)
struct R2Bytes {
    R2Io io;
    R2_MEM uint32_t at(uint32_t p) const { return io_byte(io, p); }
    R2_MEM uint32_t cls(uint32_t ch) const { return io.sh->cls[ch]; }
    R2_MEM uint32_t trans(uint32_t i) const { return io.sh->trans[i]; }
};
// plain global-memory reader (field extraction: a handful of bytes per lane, L1/L2 hits)
struct R2Glob {
    const uint8_t* data; uint32_t n_bytes;
    R2_MEM uint32_t at(uint32_t p) const { return p < n_bytes ? (uint32_t)__ldg(data + p) : 0u; }
};
// 16 bytes at the 16-byte aligned position p: resident tile, else global memory; bytes at or after n_bytes read as 0
R2_DEV uint4 ld16(const R2Ctx& c, uint32_t p) {
    if (p >= c.tile_lo && p + 16 <= c.tile_hi) return sld128(c.buf + (p - c.tile_lo));
    if (p + 16 <= c.n_bytes) return gld128(c.a->data + p);
    uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
    for (uint32_t i = 0; i < 16 && p + i < c.n_bytes; ++i) {
        const uint32_t v = (uint32_t)ring_byte(c, p + i) << (8 * (i & 3));
        if (i < 4) w0 |= v; else if (i < 8) w1 |= v; else if (i < 12) w2 |= v; else w3 |= v;
    }
    return make_uint4(w0, w1, w2, w3);
}

// ---- pipeline ----------------------------------------------------------------------------------------------------------
R2_DEV uint32_t tile_bytes(const R2Ctx& c, uint32_t k) {              // valid bytes of tile k
    const uint32_t lo = c.base + k * R2_TILE;
    return c.n_bytes - lo < R2_TILE ? c.n_bytes - lo : R2_TILE;
}
R2_DEV void pipe_issue_load(const R2Ctx& c, uint32_t k) {            // lane 0
    const uint32_t b = k % R2_NBUF, n16 = tile_bytes(c, k) & ~15u;
    if (n16) { mbar_expect(c.bars + 8 * b, n16); tma_load(c.ring + b * R2_TILE, c.a->data + c.base + k * R2_TILE, n16, c.bars + 8 * b); }
}
R2_DEV void pipe_start(R2Ctx& c) {
    c.k = R2_NONE; c.tile_lo = c.tile_hi = c.base; c.buf = c.ring;
    if (c.lane == 0) for (uint32_t k = 0; k < R2_NBUF - 1 && k < c.n_tiles; ++k) pipe_issue_load(c, k);
}
// make tile k resident (k = previous + 1): wait for its bytes, hand it to the store engine, refill the buffer that just became free
struct PipeState { uint32_t k, tile_lo, tile_hi; SPtr buf; };
R2_DEV PipeState pipe_advance_impl(const StepArgs* ap, SPtr ring, SPtr bars, uint32_t base, uint32_t n_tiles, uint32_t n_bytes, uint32_t k_prev, uint32_t lane) {
    const uint32_t k = k_prev == R2_NONE ? 0u : k_prev + 1u;
    __syncwarp();                                   // every lane is done with the buffers of the earlier tiles
    const uint32_t lo = base + k * R2_TILE;
    const uint32_t b = k % R2_NBUF, nb = n_bytes - lo < R2_TILE ? n_bytes - lo : R2_TILE, n16 = nb & ~15u;
    PipeState ps; ps.k = k; ps.tile_lo = lo; ps.tile_hi = lo + nb; ps.buf = ring + b * R2_TILE;
    if (n16) mbar_wait(bars + 8 * b, (k / R2_NBUF) & 1u);
    if (nb != n16) {                                // ragged end of the buffer: the last bytes move by hand
        const uint32_t i = n16 + lane;
        if (lane < 16) {
            const uint32_t v = i < nb ? (uint32_t)__ldg(ap->data + lo + i) : 0u;
            sst8(ps.buf + i, v);
            if (i < nb) ap->out[lo + i] = (uint8_t)v;
        }
        __syncwarp();
    }
    if (lane == 0) {
        if (n16) tma_store(ap->out + lo, ps.buf, n16); else tma_store_commit_empty();
        tma_wait_read1();                           // the store of tile k-1 has read its buffer
        const uint32_t kn = k + R2_NBUF - 1;
        if (kn < n_tiles) {
            const uint32_t bn = kn % R2_NBUF, lon = base + kn * R2_TILE, nn = (n_bytes - lon < R2_TILE ? n_bytes - lon : R2_TILE) & ~15u;
            if (nn) { mbar_expect(bars + 8 * bn, nn); tma_load(ring + bn * R2_TILE, ap->data + lon, nn, bars + 8 * bn); }
        }
    }
    return ps;
}
R2_DEV void pipe_advance(R2Ctx& c) {
    const PipeState ps = pipe_advance_impl(c.a, c.ring, c.bars, c.base, c.n_tiles, c.n_bytes, c.k, c.lane);
    c.k = ps.k; c.tile_lo = ps.tile_lo; c.tile_hi = ps.tile_hi; c.buf = ps.buf;
}

// ---- templates ---------------------------------------------------------------------------------------------------------
// the 16 pre-shifted copies of slot `slot` (whole warp)
R2_DEV void build_fast_tables(R2Shared* sh, uint32_t slot, uint32_t lane, uint32_t step) {
    const Tpl2& tp = sh->tpl[slot];
    const uint32_t P = tp.m.P, recip = tp.m.recip;
    for (uint32_t i4 = lane; i4 < 16 * R2_TEXT / 4; i4 += step) {                 // four bytes per trip (R2_TEXT is a multiple of 4)
        const uint32_t i = i4 * 4u, cpy = i / R2_TEXT, j = i - cpy * R2_TEXT;
        uint32_t x = j + cpy; x -= __umulhi(x, recip) * P;
        uint32_t wt = 0, wl = 0;
        for (uint32_t b = 0; b < 4; ++b) { wt |= (uint32_t)tp.text[x] << (8 * b); wl |= (uint32_t)tp.lit[x] << (8 * b); if (++x == P) x = 0; }
        reinterpret_cast<uint32_t*>(sh->fast_text)[i4] = wt; reinterpret_cast<uint32_t*>(sh->fast_lit)[i4] = wl;
    }
}

// One lane validates the event [ps, LF LF) and, when it qualifies, fills `tp` with it.  limit = end of the segment's text.
template <class RD>
R2_DEV_NOINLINE bool build_template2(const RD& rd, Tpl2* tp, UsageRaw* raw_out, uint32_t ps, uint32_t limit) {
    uint32_t cls = PC_NONE;
    const uint32_t c0 = rd.at(ps);
    if (c0 == '{') cls = PC_BRACE;
    else if (c0 == 'd' && rd.at(ps + 1) == 'a' && rd.at(ps + 2) == 't' && rd.at(ps + 3) == 'a' && rd.at(ps + 4) == ':' && rd.at(ps + 5) == ' ' && rd.at(ps + 6) == '{') cls = PC_DATA;
    if (cls == PC_NONE) return false;
    TplMeta& m = tp->m;
    LeanMachine lm;
    lm.reset(cls == PC_DATA);
    const uint32_t skip = cls == PC_DATA ? 6u : 0u;
    for (uint32_t k = 0; k < R2_TPL_MAX + 8; ++k) tp->span_id[k] = 0xff;
    for (uint32_t k = 0; k < R2_TEXT; ++k) tp->lit[k] = 0xff;
    uint32_t pos = ps + skip, n_ids = 0, cur_s = 0xff, cur_n = 0xff;
    for (;;) {
        if (pos + 1 >= limit || pos - ps >= R2_TPL_MAX) return false;
        const uint32_t c = rd.at(pos);
        if (c == '\n' && rd.at(pos + 1) == '\n') break;
        const uint32_t prev = lm.st;
        const bool in_str = (prev == L_STR || prev == L_STR_ESC || prev == L_STR_U) && !lm.in_key;
        const bool in_num = prev >= L_NUM_MINUS && prev <= L_NUM_EXP;
        const uint32_t x = pos - ps;
        if (in_str && cur_s != 0xff) {
            tp->span_id[x] = (uint8_t)cur_s;
            if (prev == L_STR && c == '"') m.send[cur_s] = (uint16_t)x;         // the closing quote: literal
            else tp->lit[x] = 0x00;                                              // content
        }
        lm.step(c, pos, rd);
        const bool now_num = lm.st >= L_NUM_MINUS && lm.st <= L_NUM_EXP;
        if (in_num && cur_n != 0xff) {
            tp->span_id[x] = (uint8_t)cur_n;                                    // number characters and the terminator
            if (!now_num) { m.send[cur_n] = (uint16_t)x; cur_n = 0xff; }
        }
        if (prev < LGW_LEAN_ROWS && lm.st == L_STR && !lm.in_key) {              // a string VALUE opens
            cur_s = n_ids < R2_SPANS ? n_ids++ : 0xffu;
            if (cur_s != 0xff) { m.skind[cur_s] = 0; m.sstart[cur_s] = (uint16_t)(x + 1); m.send[cur_s] = 0xffff; }
        }
        if (!in_num && now_num) {                                               // a number opens
            cur_n = n_ids < R2_SPANS ? n_ids++ : 0xffu;
            if (cur_n != 0xff) { m.skind[cur_n] = 1; m.sstart[cur_n] = (uint16_t)x; m.send[cur_n] = 0xffff; tp->span_id[x] = (uint8_t)cur_n; }
        }
        if (lm.st == L_ERR) return false;
        ++pos;
    }
    const uint32_t f = lm.finish();
    if (!(f & PF_VALID_A) || (f & (TK_ERROR | TK_DETAIL | TK_CODE))) return false;
    if (pos + 2 < limit && rd.at(pos + 2) == '\n') return false;
    const uint32_t len = pos - ps;
    if (len < R2_TPL_MIN) return false;
    for (uint32_t k = 0; k < n_ids; ++k) if (m.send[k] >= len) return false;        // every span must be closed inside the event
    const uint32_t P = len + 2;
    for (uint32_t k = 0; k < R2_TEXT; ++k) {
        uint32_t x = k; while (x >= P) x -= P;
        tp->text[k] = x < len ? (uint8_t)rd.at(ps + x) : (uint8_t)'\n';
        if (k >= len) tp->lit[k] = x < len ? tp->lit[x] : (uint8_t)0xff;
    }
    m.len = len; m.P = P; m.recip = (uint32_t)((0x100000000ull + P - 1) / P); m.flags = f; m.cls = cls; m.n_spans = n_ids;
    m.usage_ok = 0; m.full_flags = 0;
    for (uint32_t k = 0; k < 8; ++k) m.field_span[k] = 0xff;
    if (f & TK_USAGE) {
        // the full machine over the template, tracking where the eight usage fields sit: events that follow the template
        // can then have their fields read straight from the matched value spans
        JsonMachine<true> jm; ValueTrack trk; trk.reset();
        jm.reset(raw_out, cls == PC_DATA); jm.trk = &trk;
        for (uint32_t i = skip; i < len; ++i) { trk.pos = i; jm.feed(rd.at(ps + i)); if (jm.failed()) break; }
        const uint32_t ff = jm.finish();
        m.full_flags = ff;
        bool ok = !jm.failed() && (ff & PF_VALID_B) && !(ff & PF_EXOTIC) && !((ff & TK_CHOICES) && (ff & PF_TYPE_ERROR)) && !trk.dup && n_ids <= R2_SPANS;
        if (ok && (ff & TK_CHOICES)) for (uint32_t k = 0; k < n_ids; ++k) if (m.send[k] >= trk.choices_lo && m.sstart[k] <= trk.choices_hi) ok = false;
        for (uint32_t fi = 0; ok && fi < UF_N; ++fi) {
            if (trk.fstart[fi] == 0xFFFFFFFFu) continue;                          // field absent: the template's (absent) value stands
            if (trk.fstart[fi] == 0xFFFFFFFEu) { ok = false; break; }            // a container where a usage field goes: not read from spans
            uint32_t j = 0xff;
            for (uint32_t k = 0; k < n_ids; ++k) {
                if (m.skind[k] == 1 && m.sstart[k] == trk.fstart[fi] && m.send[k] == trk.fend[fi]) j = k;
                if (m.skind[k] == 0 && (uint32_t)m.sstart[k] == trk.fstart[fi] + 1 && (uint32_t)m.send[k] + 1 == trk.fend[fi]) j = k;
            }
            if (j != 0xff && (m.skind[j] == 1) != (fi < UF_MODEL)) ok = false;      // a string where a number goes (or the reverse): not modelled here
            m.field_span[fi] = (uint8_t)j;
            // a field whose value is not a span (null, true, a container ...) is part of the literal text: same value in every match
            if (j == 0xff) for (uint32_t k = 0; k < n_ids; ++k) if (m.sstart[k] < trk.fend[fi] && m.send[k] >= trk.fstart[fi]) ok = false;   // spans inside a container value
        }
        m.usage_ok = ok ? 1u : 0u;
    }
    return true;
}

// ---- field extraction from matched value spans (usage_ok templates) ---------------------------------------------------------
// number text [p, p+n) (already validated by the number automaton) -> value exactly as json_machine.cuh reads it
template <class RD>
R2_DEV_NOINLINE Val parse_number_span(const RD& rd, uint32_t p, uint32_t n) {
    DecAcc num; num.reset();
    uint32_t i = 0;
    if (i < n && rd.at(p) == '-') { num.neg = 1; ++i; }
    for (; i < n; ++i) { const uint32_t c = rd.at(p + i); if (c - '0' >= 10u) break; num.digit(c - '0', false); }
    if (i < n && rd.at(p + i) == '.') { ++i; for (; i < n; ++i) { const uint32_t c = rd.at(p + i); if (c - '0' >= 10u) break; num.is_float = 1; num.digit(c - '0', true); } }
    if (i < n && (rd.at(p + i) | 0x20u) == 'e') {
        num.is_float = 1; ++i;
        if (i < n && rd.at(p + i) == '+') ++i; else if (i < n && rd.at(p + i) == '-') { num.exp_neg = 1; ++i; }
        for (; i < n; ++i) num.exp_digit(rd.at(p + i) - '0');
    }
    uint8_t kind; int64_t bits; bool truthy;
    num.finish(kind, bits, truthy);
    Val v; v.kind = kind; v.bits = bits;
    return v;
}
// string content [p, p+n) (validated: plain bytes and valid escapes) -> the capture json_machine.cuh makes of it
template <class RD>
R2_DEV_NOINLINE void decode_string_span(const RD& rd, uint32_t p, uint32_t n, char* dst, uint8_t& dlen, uint8_t& dflags) {
    uint32_t len = 0, flags = 0, pending_high = 0;
    auto put = [&](uint32_t b) { if (len < LGW_STR_CAP) dst[len++] = (char)b; else flags |= 1; };
    auto put_cp = [&](uint32_t cp) {
        if (cp < 0x80) put(cp);
        else if (cp < 0x800) { put(0xC0 | (cp >> 6)); put(0x80 | (cp & 63)); }
        else if (cp < 0x10000) { put(0xE0 | (cp >> 12)); put(0x80 | ((cp >> 6) & 63)); put(0x80 | (cp & 63)); }
        else { put(0xF0 | (cp >> 18)); put(0x80 | ((cp >> 12) & 63)); put(0x80 | ((cp >> 6) & 63)); put(0x80 | (cp & 63)); }
    };
    auto flush_high = [&]() { if (pending_high) { flags |= 2; pending_high = 0; } };
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t c = rd.at(p + i);
        if (c != '\\') { flush_high(); put(c); continue; }
        const uint32_t e = rd.at(p + ++i);
        if (e != 'u') { c = e == 'b' ? 8u : e == 'f' ? 12u : e == 'n' ? 10u : e == 'r' ? 13u : e == 't' ? 9u : e; flush_high(); put(c); continue; }
        uint32_t cp = 0;
        for (int d = 0; d < 4; ++d) { const uint32_t h = rd.at(p + ++i); cp = (cp << 4) | (h - '0' < 10u ? h - '0' : (h | 0x20u) - 'a' + 10u); }
        if (cp < 0x80) { flush_high(); put(cp); }
        else if (cp >= 0xD800 && cp <= 0xDBFF) { flush_high(); pending_high = cp; }
        else if (cp >= 0xDC00 && cp <= 0xDFFF) { if (pending_high) { put_cp(0x10000 + ((pending_high - 0xD800) << 10) + (cp - 0xDC00)); pending_high = 0; } else flags |= 2; }
        else { flush_high(); put_cp(cp); }
    }
    flush_high();
    dlen = (uint8_t)len; dflags = (uint8_t)flags;
}

// ---- the static plan of a segment ----------------------------------------------------------------------------------------
// Where a segment's bulk region lies, and whether its stream is SPECULATED to commit on its first non-empty chunk (a fresh
// stream; the bulk kernel verifies, k_commit2 applies or falls back).  A pure function of the segment's chunks, their offsets
// and the stream's state at the start of the launch set: k_relay2's warps and the segment's k_commit2 warp each compute it,
// and they must reach the same verdict, so this is the one place that decides it.
struct SegStatic {
    uint32_t resume_chunk;     // first chunk the sequential path would have to (re)do
    uint32_t relay_begin;      // byte offset where the bulk region starts (tap view); seg_end when none
    uint32_t seg_end;          // byte offset of the end of the segment
    uint32_t emit_chunk_begin;
    uint32_t kept_chunk;       // the speculated stream's first non-empty chunk (request_handler.py:69-95); R2_NONE: no speculation
    uint32_t kept_end;         // byte offset of the end of the kept chunk = where the handler's text starts; 0: none
    uint32_t irregular;        // 1: no bulk region, k_commit2 redoes [resume_chunk, end)
};
R2_DEV SegStatic seg_static(const uint32_t* chunk_off, uint32_t c0, uint32_t c1, uint32_t phase, uint32_t flags, uint32_t carry_a_len) {
    SegStatic p;
    p.seg_end = __ldg(chunk_off + c1); p.relay_begin = p.seg_end; p.irregular = 0;
    p.kept_chunk = R2_NONE; p.kept_end = 0;
    p.resume_chunk = c0; p.emit_chunk_begin = phase == PH_COMMITTED ? c0 : c1;
    if (phase == PH_COMMITTED && c0 < c1) {
        if ((flags & SF_SYNCED) && carry_a_len == 0) p.relay_begin = __ldg(chunk_off + c0);
        else p.irregular = 1;
    } else if (phase == PH_PRIMING && c0 < c1) {
        uint32_t c = c0;
        while (c < c1 && __ldg(chunk_off + c + 1) == __ldg(chunk_off + c)) ++c;     // empty chunks are never yielded (:60-63)
        if (c < c1 && carry_a_len == 0) {
            p.kept_chunk = c; p.kept_end = __ldg(chunk_off + c + 1); p.relay_begin = __ldg(chunk_off + c); p.emit_chunk_begin = c;
        } else if (c < c1) p.irregular = 1;                                    // an event is open from an earlier step
    }
    return p;
}
// segment `seg`'s static plan into the warp's window, column i
R2_DEV void put_plan(const StepArgs& a, uint32_t* win, uint32_t i, uint32_t seg) {
    const uint32_t c0 = __ldg(a.seg_chunk + seg), c1 = __ldg(a.seg_chunk + seg + 1);
    const StreamHdr* h = &a.t.state[__ldg(a.seg_slot + seg)].h;
    const SegStatic p = seg_static(a.chunk_off, c0, c1, h->phase, h->flags, h->carry_a_len);
    win[i] = p.relay_begin; win[32 + i] = p.seg_end; win[64 + i] = p.kept_end;
}
// the window holds segments [lo, lo + 32): lane i computes segment lo + i
R2_DEV_NOINLINE void load_plans(const StepArgs* ap, uint32_t* win, uint32_t lane, uint32_t lo) {
    __syncwarp();                                                              // (every lane is done with the old window)
    if (lo + lane < ap->n_segs) put_plan(*ap, win, lane, lo + lane);
    __syncwarp();
}
// The first segment whose text ends past byte x (the one that holds x; n_segs: none), with the warp's plan window filled from
// at most 31 segments before it.  Streams of a step tend to be of similar length, so the first round reads the 32 segments
// around the one the byte position suggests, each lane its candidate's whole plan: when they bracket the answer, that round
// was the search and the window load at once.  Otherwise strided rounds (two dependent reads each) narrow the answer down,
// and the window is loaded from it.
// Returns (the segment, the window's first segment).
R2_DEV_NOINLINE uint2 first_segment(const StepArgs* ap, uint32_t* win, uint32_t lane, uint32_t x) {
    const StepArgs& a = *ap;
    const uint32_t n = a.n_segs;
    const uint32_t nb = a.n_bytes - a.tile_base;
    const uint32_t g = nb ? (uint32_t)((unsigned long long)n * (x - a.tile_base) / nb) : 0u;
    const uint32_t w0 = n <= 32u ? 0u : r2_min(g > 16u ? g - 16u : 0u, n - 32u);
    if (w0 + lane < n) put_plan(a, win, lane, w0 + lane);
    __syncwarp();
    const bool past = w0 + lane < n && win[32 + lane] > x;
    const uint32_t pm = __ballot_sync(R2_FULL, past);
    uint32_t lo, hi;
    if (pm) {
        const uint32_t k = (uint32_t)__ffs(pm) - 1u;
        if (k || w0 == 0u) return make_uint2(w0 + k, w0);                                    // bracketed (or the very first segment)
        lo = 0; hi = w0;
    } else {
        if (w0 + 32u >= n) return make_uint2(n, w0);                                       // every segment ends at or before x
        lo = w0 + 32u; hi = n;
    }
    while (lo < hi) {
        const uint32_t s = lo + (uint32_t)((unsigned long long)(hi - lo) * lane / 32u);     // (nondecreasing in the lane)
        const bool e_past = __ldg(a.chunk_off + __ldg(a.seg_chunk + s + 1)) > x;
        const uint32_t m = __ballot_sync(R2_FULL, e_past);
        if (!m) { lo = __shfl_sync(R2_FULL, s, 31) + 1u; continue; }
        const uint32_t k = (uint32_t)__ffs(m) - 1u;
        const uint32_t sk = __shfl_sync(R2_FULL, s, (int)k), sp = __shfl_sync(R2_FULL, s, k ? (int)k - 1 : 0);
        hi = sk;
        if (k) lo = sp + 1u;
    }
    load_plans(ap, win, lane, lo);
    return make_uint2(lo, lo);
}

// ---- helpers of the walk ---------------------------------------------------------------------------------------------------
R2_DEV void flush_counts(R2Ctx& c) {
    if (c.lane == 0 && c.seg != R2_NONE) {
        SegPlan* pl = c.a->s.plan + c.seg;
        if (c.ev_a) atomicAdd(&pl->n_events_a, c.ev_a);
        if (c.ev_b) atomicAdd(&pl->n_events_b, c.ev_b);
        if (c.a_usage) pl->a_usage = 1;
    }
    c.ev_a = c.ev_b = c.a_usage = 0;
}
R2_DEV void mark_irregular(R2Ctx& c) { if (c.lane == 0 && c.seg != R2_NONE) c.a->s.plan[c.seg].irregular = 1; }

// chunk-level UTF-8 (request_handler.py:111 decodes every chunk on its own): the chunks of segment `seg` that overlap [lo, hi)
R2_DEV_NOINLINE bool chunks_utf8_ok(const StepArgs* ap, uint32_t lane, uint32_t seg, uint32_t lo, uint32_t hi) {
    const StepArgs& a = *ap;
    uint32_t c0 = __ldg(a.seg_chunk + seg), c1 = __ldg(a.seg_chunk + seg + 1);
    {   // first chunk that ends after lo
        uint32_t l = c0, h = c1;
        while (l < h) { const uint32_t mid = (l + h) >> 1; if (__ldg(a.chunk_off + mid + 1) <= lo) l = mid + 1; else h = mid; }
        c0 = l;
    }
    bool ok = true;
    for (uint32_t ch = c0 + lane; ch < c1; ch += 32) {
        const uint32_t o = __ldg(a.chunk_off + ch), e = __ldg(a.chunk_off + ch + 1);
        if (o >= hi) break;
        if (e > a.n_bytes) { ok = false; break; }
        if (!utf8_valid(a.data + o, e - o)) ok = false;
    }
    return __all_sync(R2_FULL, ok);
}

// first LF LF pair at or after `from` whose second LF lies before `end`: position of its first LF, R2_NONE when there is none
R2_DEV uint32_t find_lflf(R2Ctx& c, uint32_t from, uint32_t end, uint32_t& high) {
    uint32_t wb = from & ~15u;
    for (;;) {
        if (wb >= end) return R2_NONE;
        const uint32_t lp = wb + 16 * c.lane;
        const uint4 d = lp < end ? ld16(c, lp) : make_uint4(0, 0, 0, 0);
        high |= d.x | d.y | d.z | d.w;
        const uint32_t lf = lf_mask16(d);
        const uint32_t nxt = __shfl_down_sync(R2_FULL, lf, 1);
        uint32_t pair = lf & ((lf >> 1) | ((c.lane < 31 ? nxt & 1u : 0u) << 15));      // bit i: LF at i and at i+1
        if (lp < from) pair &= from - lp >= 16 ? 0u : (0xFFFFu << (from - lp));
        if (lp + 17 > end) pair &= end <= lp + 1 ? 0u : (0xFFFFu >> (lp + 17 - end));   // the second LF must lie before end
        const uint32_t any = __ballot_sync(R2_FULL, pair != 0);
        if (any) {
            const uint32_t fl = (uint32_t)__ffs(any) - 1u;
            const uint32_t pr = __shfl_sync(R2_FULL, pair, (int)fl);
            return wb + 16 * fl + ((uint32_t)__ffs(pr) - 1u);
        }
        wb += 31 * 16;                                                                   // the last lane is looked at again (pairs across windows)
    }
}

// the recogniser over one event starting at ps (single lane does the walk): finds its LF LF (e) or runs into `end`.
// out: cls, flags; returns e, or R2_NONE when the event is still open at `end`.
struct LeanOut { uint32_t e, cls, f, high; };
R2_DEV_NOINLINE LeanOut lean_event(R2Io io, uint32_t lane, uint32_t ps, uint32_t end) {
    uint32_t e = R2_NONE, cls = PC_NONE, f = 0, hi = 0;
    if (lane == 0) {
        R2Bytes rd{io};
        const uint32_t c0 = ps < end ? rd.at(ps) : 0u;
        if (c0 == '{') cls = PC_BRACE;
        else if (c0 == 'd' && ps + 7 <= end && rd.at(ps + 1) == 'a' && rd.at(ps + 2) == 't' && rd.at(ps + 3) == 'a' && rd.at(ps + 4) == ':' && rd.at(ps + 5) == ' ' && rd.at(ps + 6) == '{') cls = PC_DATA;
        LeanMachine lm; lm.reset(cls == PC_DATA);
        uint32_t pos = ps;
        const uint32_t body = ps + (cls == PC_DATA ? 6u : 0u);
        for (; pos < end; ++pos) {
            const uint32_t ch = rd.at(pos);
            hi |= ch;
            if (ch == '\n' && pos + 1 < end && rd.at(pos + 1) == '\n') { e = pos; break; }
            if (cls != PC_NONE && pos >= body) lm.step(ch, pos, rd);
        }
        if (e != R2_NONE && cls != PC_NONE) f = lm.finish();
    }
    LeanOut o;
    o.e = __shfl_sync(R2_FULL, e, 0); o.cls = __shfl_sync(R2_FULL, cls, 0); o.f = __shfl_sync(R2_FULL, f, 0); o.high = __shfl_sync(R2_FULL, hi, 0);
    return o;
}

// Slot states as one lane sees them, handed to all (other warps of the block publish templates while this one runs; every
// lane of a warp must act on the same view).
R2_DEV void refresh_slots(R2Ctx& c) {
    uint32_t r = 0, f = 0, fast = 0;
    if (c.lane == 0) {
        for (uint32_t k = 0; k < R2_SLOTS; ++k) { const uint32_t st = *(volatile uint32_t*)&c.sh->slot_state[k]; if (st == 2u) r |= 1u << k; else if (st == 0u) f |= 1u << k; }
        fast = *(volatile uint32_t*)&c.sh->fast_ready;
    }
    c.ready = __shfl_sync(R2_FULL, r, 0); c.free_slots = __shfl_sync(R2_FULL, f, 0); c.fast = __shfl_sync(R2_FULL, fast, 0);
}
// ---- template learning ---------------------------------------------------------------------------------------------------------
R2_DEV bool tpl_same(const Tpl2& x, const Tpl2& y) {
    if (x.m.len != y.m.len || x.m.cls != y.m.cls) return false;
    for (uint32_t k = 0; k < x.m.len; ++k) if (x.lit[k] != y.lit[k] || (x.lit[k] && x.text[k] != y.text[k])) return false;
    return true;
}
// The event [ps, LF LF) was walked by the recogniser and is valid: install it in a free slot of this block and, when the
// engine-wide cache has room and does not hold the same skeleton yet, publish it there.  One warp of a block learns at a
// time, and not when another warp has just made a template ready that this event was not tried against (it may be the very
// same skeleton: in a cold step every warp meets the first delta at the same moment).
R2_DEV_NOINLINE void learn_template(const StepArgs* ap, R2Shared* sh, R2Io io, UsageRaw* block_raw, uint32_t lane, uint32_t ready_before, uint32_t ps, uint32_t end) {
    uint32_t got = 0;
    if (lane == 0) got = atomicCAS(&sh->learn_lock, 0u, 1u) == 0u ? 1u : 0u;
    got = __shfl_sync(R2_FULL, got, 0);
    if (!got) return;
    uint32_t ready = 0, free_slots = 0;
    if (lane == 0) for (uint32_t k = 0; k < R2_SLOTS; ++k) { const uint32_t st = *(volatile uint32_t*)&sh->slot_state[k]; if (st == 2u) ready |= 1u << k; else if (st == 0u) free_slots |= 1u << k; }
    ready = __shfl_sync(R2_FULL, ready, 0); free_slots = __shfl_sync(R2_FULL, free_slots, 0);
    uint32_t slot = R2_NONE;
    if (ready == ready_before && free_slots) {
        if (lane == 0) {
            slot = (uint32_t)__ffs(free_slots) - 1u;
            atomicExch(&sh->slot_state[slot], 1u);
            R2Bytes rd{io};
            TemplateCache2* tc = ap->s.tpl_cache2;
            UsageRaw* raw = block_raw + slot;
            if (build_template2(rd, &sh->tpl[slot], raw, ps, end)) {
                sh->slot_gidx[slot] = R2_NONE;
                if (atomicCAS(&tc->lock, 0u, 1u) == 0u) {                        // (busy: the template stays local to this block for this launch)
                    bool dup = false; uint32_t dst = R2_NONE;
                    for (uint32_t k = 0; k < R2_SLOTS; ++k) {
                        const uint32_t st = *(volatile uint32_t*)&tc->state[k];
                        if (st == 2u) { if (tpl_same(tc->tpl[k], sh->tpl[slot])) dup = true; }
                        else if (st == 0u && dst == R2_NONE) dst = k;
                    }
                    sh->slot_gidx[slot] = R2_NONE;
                    if (!dup && dst != R2_NONE) {
                        tc->tpl[dst] = sh->tpl[slot]; tc->raw[dst] = *raw; tc->hits[dst] = 0;
                        __threadfence();
                        atomicExch(&tc->state[dst], 2u);
                        sh->slot_gidx[slot] = dst;
                    }
                    __threadfence();
                    atomicExch(&tc->lock, 0u);
                }
            } else { atomicExch(&sh->slot_state[slot], 0u); slot = R2_NONE; }
        }
        slot = __shfl_sync(R2_FULL, slot, 0);
    }
    if (slot != R2_NONE) {
        uint32_t need_fast = 0;
        if (lane == 0) need_fast = (slot == sh->dflt && !*(volatile uint32_t*)&sh->fast_ready) ? 1u : 0u;
        need_fast = __shfl_sync(R2_FULL, need_fast, 0);
        if (need_fast) {                                                        // a cold block: its first template becomes the default
            build_fast_tables(sh, slot, lane, 32);
            __threadfence_block();
            __syncwarp();
            if (lane == 0) *(volatile uint32_t*)&sh->fast_ready = 1u;
        }
        __threadfence_block();
        if (lane == 0) atomicExch(&sh->slot_state[slot], 2u);
    }
    __syncwarp();
    if (lane == 0) { __threadfence_block(); atomicExch(&sh->learn_lock, 0u); }
    __syncwarp();
}

// Enter segment `seg` (static plan: bulk region [tb, te), kept = end of the kept chunk, 0: none); `from` = the warp's range
// start when the segment's bytes begin before it, else the segment's first byte.  Sets the text range and the first event start
// this warp owns in it; false: the warp owns nothing here.
R2_DEV bool enter_segment(R2Ctx& c, uint32_t seg, uint32_t tb, uint32_t te, uint32_t kept, uint32_t from, uint32_t range_hi) {
    const SegPlan* pl = c.a->s.plan + seg;
    c.seg = seg; c.ev_a = c.ev_b = c.a_usage = 0; c.high = 0; c.in_kept = 0; c.primed = 0; c.kept_tried = 0;
    c.tb = tb; c.te = te;
    c.kept_end = kept;
    c.pos = te; c.walk_lo = te;
    c.t = 0;
    // `irregular` is a finding other warps write while this kernel runs (mark_irregular): one lane reads it and hands
    // it to all -- lanes reading it on their own could see different values and part ways before the next collective
    uint32_t irr = 0;
    if (c.lane == 0) irr = *(volatile const uint32_t*)&pl->irregular;
    irr = __shfl_sync(R2_FULL, irr, 0);
    if (irr || tb >= te) return false;
    if (from <= tb) {
        if (tb >= range_hi) return false;
        if (kept) c.in_kept = 1u;                            // the kept chunk is walked by ONE warp, the one that owns its first byte (beyond its range if need be)
        c.pos = c.s_open = c.walk_lo = tb;
        c.last_ra = R2_NONE;
        return true;
    }
    // the range starts inside the segment's text: the event that is open there belongs to the previous warp; ours start
    // behind the first separator that ends at or after `from`
    if (from >= te) return false;
    c.walk_lo = from;
    if (kept && from < kept) {                                                   // the range starts inside the kept chunk: the warp before walks that to its end;
        if (kept >= range_hi || kept >= te) return false;                        //   the speculation holds only if the chunk ends on a separator, so ours begin right there
        c.pos = c.s_open = kept;
        c.last_ra = R2_NONE;
        return true;
    }
    const uint32_t p = find_lflf(c, from - tb >= 2u ? from - 2u : tb, te, c.high);
    if (p == R2_NONE) return false;
    const uint32_t s = p + 2u;
    if (s >= range_hi && s != te) return false;                                  // its first event starts in a later range
    if ((p > tb && ring_byte(c, p - 1) == '\n') || (s < te && ring_byte(c, s) == '\n')) { mark_irregular(c); return false; }   // LF run >= 3
    if (s >= te) return false;                                                   // the text ends on this separator (the previous warp posts the tail)
    c.pos = c.s_open = s;
    c.last_ra = R2_NONE;
    return true;
}


// leave the current segment (its text is done as far as this warp is concerned)
R2_DEV void leave_segment(R2Ctx& c, uint32_t range_hi) {
    if (c.seg == R2_NONE) return;
    if (__any_sync(R2_FULL, (c.high & 0x80808080u) != 0)) {
        if (!chunks_utf8_ok(c.a, c.lane, c.seg, c.walk_lo, r2_min(c.te, r2_max(c.pos, range_hi)))) mark_irregular(c);
    }
    flush_counts(c);
    c.seg = R2_NONE;
}

// ---- one event against one (non-periodic) slot: hop from value span to value span ------------------------------------------------
// The judgement of the compare pass for a single event, made span by span instead of window by window: the literal text
// between two value spans is compared byte for byte (a lane per byte), a number span ends at the first byte that no JSON
// number holds and must be a valid number (a plain run of digits is judged from the ballot, anything else by the
// recogniser's number rows), a string span holds plain bytes and valid escapes up to its closing quote.  Usage events and
// the odd chunks of a stream (role, finish) take this path: ~30 warp-instructions per span instead of a pass per span.
// ok: the event follows the slot; e = position of its LF LF.  Lanes 0..7 also learn where their usage field sits.
struct SingleOut { uint32_t ok, e, high, f_start, f_len, f_esc; };
R2_DEV_NOINLINE SingleOut match_single(R2Io io, const Tpl2* tp, uint32_t lane, uint32_t ps, uint32_t ev_end) {
    const TplMeta& m = tp->m;
    SingleOut o; o.ok = 0; o.e = 0; o.high = 0; o.f_start = 0; o.f_len = 0; o.f_esc = 0;
    const uint32_t my_span = lane < 8u ? (uint32_t)m.field_span[lane] : 0xffu;
    const uint32_t n_spans = m.n_spans, len = m.len;
    uint32_t pos = ps, ta = 0, high = 0;
    for (uint32_t j = 0; j <= n_spans; ++j) {
        const uint32_t tb = j < n_spans ? (uint32_t)m.sstart[j] : len + 2u;          // literal text [ta, tb) of the image (the last piece ends with LF LF)
        bool same = true;
        for (uint32_t off = lane; off < tb - ta; off += 32) {
            const uint32_t c = pos + off < ev_end ? (uint32_t)io_byte(io, pos + off) : 0x100u;
            if (c != (uint32_t)tp->text[ta + off]) same = false;
            high |= c;
        }
        if (!__all_sync(R2_FULL, same)) return o;
        pos += tb - ta;
        if (j == n_spans) break;
        uint32_t span_len = 0, esc = 0;
        if (m.skind[j] == 1) {                                                         // number value
            const uint32_t c = pos + lane < ev_end ? (uint32_t)io_byte(io, pos + lane) : 0u;
            const uint32_t cl = io.sh->cls[c & 0xffu];
            const uint32_t isnum = __ballot_sync(R2_FULL, cl >= C_MINUS && cl <= C_EXP);
            const uint32_t isdig = __ballot_sync(R2_FULL, cl == C_ZERO || cl == C_DIGIT);
            const uint32_t run = (uint32_t)__ffs(~isnum) - 1u;                            // (32 number characters in a row: not followed here)
            if (run == 0u || run >= 32u) return o;
            const uint32_t runmask = (1u << run) - 1u;
            const uint32_t first = __shfl_sync(R2_FULL, c, 0);
            if ((isdig & runmask) != runmask || (run > 1u && first == '0')) {           // sign, fraction, exponent, leading zero: the recogniser's number rows
                uint32_t good = 0;
                if (lane == 0) {
                    uint32_t st = L_VALUE;
                    for (uint32_t k = 0; k < run && st != L_ERR; ++k) st = io.sh->trans[st * 32 + io.sh->cls[io_byte(io, pos + k)]] & 31u;
                    good = (st == L_NUM_ZERO || st == L_NUM_INT || st == L_NUM_FRAC || st == L_NUM_EXP) ? 1u : 0u;
                }
                if (!__shfl_sync(R2_FULL, good, 0)) return o;
            }
            span_len = run;
        } else {                                                                       // string value
            uint32_t q = pos;
            for (;;) {
                const uint32_t c = q + lane < ev_end ? (uint32_t)io_byte(io, q + lane) : 0u;   // (past the end: reads as a control byte, the scan stops)
                high |= c;
                const uint32_t sp = __ballot_sync(R2_FULL, c < 0x20u || c == '"' || c == '\\');
                if (!sp) { q += 32; if (q - pos > R2_MAX_STR) return o; continue; }
                const uint32_t k = (uint32_t)__ffs(sp) - 1u, x = q + k;
                const uint32_t ch = __shfl_sync(R2_FULL, c, (int)k);
                if (ch == '"') { q = x; break; }
                if (ch != '\\') return o;                                            // a control byte (or the end of the readable text)
                const uint32_t e1 = x + 1 < ev_end ? (uint32_t)io_byte(io, x + 1) : 0u;
                uint32_t el = 0;
                if (e1 == 'u') { el = 6; for (uint32_t h4 = 2; h4 < 6; ++h4) { const uint32_t h = x + h4 < ev_end ? (uint32_t)io_byte(io, x + h4) : 0u; if (!(h - '0' < 10u || (h | 0x20u) - 'a' < 6u)) el = 0; } }
                else if (e1 == '"' || e1 == '\\' || e1 == '/' || e1 == 'b' || e1 == 'f' || e1 == 'n' || e1 == 'r' || e1 == 't') el = 2;
                if (el == 0) return o;
                esc = 1; q = x + el;
                if (q - pos > R2_MAX_STR) return o;
            }
            span_len = q - pos;
        }
        if (my_span == j) { o.f_start = pos; o.f_len = span_len; o.f_esc = esc; }
        pos += span_len; ta = m.send[j];
    }
    o.ok = 1; o.e = pos - 2u; o.high = high;
    return o;
}

// ---- the two out-of-line steps of the walk ---------------------------------------------------------------------------------------
// Both take a handful of scalars and return a handful: the walk's own values stay in registers across the calls (passing the
// whole context by value cost ~90 local-memory words per call, and with 180 KB of shared memory there is next to no L1 left
// to hide that behind).

// what one completed event (or n events of a template) adds to the segment's counters
struct Acct { uint32_t ok, ev_a, ev_b, a_usage, primed; };
R2_DEV Acct account(const StepArgs* ap, uint32_t lane, uint32_t seg, uint32_t in_kept, uint32_t primed, uint32_t cls, uint32_t f, uint32_t n, uint32_t ps, uint32_t e) {
    Acct r; r.ok = 1; r.ev_a = 0; r.ev_b = 0; r.a_usage = 0; r.primed = primed;
    if (cls == PC_NONE) return r;
    if (cls == PC_DATA) {
        if (in_kept) {                                        // priming loop on the kept chunk, request_handler.py:82-91
            if (!primed) { if (!(f & PF_VALID_A) || (f & (TK_ERROR | TK_DETAIL))) { r.ok = 0; return r; } r.primed = 1; }
        } else {                                              // handler loop, request_handler.py:122-134
            r.ev_a = n;
            if ((f & PF_VALID_A) && !(f & TK_CODE) && (f & TK_USAGE)) r.a_usage = 1;
        }
    }
    if (f & PF_VALID_B) {                                     // tap loop, chat_logging.py:123-141
        r.ev_b = n;
        if (f & TK_ERROR) { r.ok = 0; return r; }             // extra DB row: sequential path
        if ((f & TK_USAGE) && lane == 0) {
            SegPlan* pl = ap->s.plan + seg;
            atomicAdd(&pl->n_usage_b, n);
            atomicMax(&pl->last_usage, ((unsigned long long)(ps + 1) << 32) | (e - ps));
        }
    }
    return r;
}

// The hot loop of the kernel.  Whole 16-byte aligned windows of the resident tile against the default slot's periodic image,
// two windows per trip while two fit (two independent chains of loads and byte tests in flight), moving the TMA pipeline on
// from tile to tile.  No boundary lanes, no limits other than `stop` (end of the text / of the range); a mismatch, or a window
// that does not fit before `stop`, ends the run -- the caller's pass finds out where and why, from the same position.  Out of
// line with scalar arguments so that nothing but the loop's own values lives in registers here (no spill code in the loop).
struct FastOut { uint32_t k, tile_lo, tile_hi; SPtr buf; uint32_t pos, t, s_open, nfast, high; };
R2_DEV_NOINLINE FastOut fast_run(const StepArgs* ap, const R2Shared* sh, SPtr ring, SPtr bars, uint32_t base, uint32_t n_tiles, uint32_t n_bytes,
                                 uint32_t k, uint32_t tile_lo, uint32_t tile_hi, SPtr buf, uint32_t pos, uint32_t t, uint32_t s_open,
                                 const uint32_t stop, const uint32_t P, const uint32_t recip, const uint32_t lane) {
    const SPtr ft = sptr(sh->fast_text), fl = sptr(sh->fast_lit);
    uint32_t nfast = 0, high = 0;
    for (;;) {
        if (pos >= tile_hi) {
            if (k + 1 >= n_tiles) break;
            const PipeState ps = pipe_advance_impl(ap, ring, bars, base, n_tiles, n_bytes, k, lane);
            k = ps.k; tile_lo = ps.tile_lo; tile_hi = ps.tile_hi; buf = ps.buf;
        }
        const uint32_t u = t + 16u * lane;
        const uint32_t tl = u - __umulhi(u, recip) * P;
        const uint32_t ad = (tl & 15u) * R2_TEXT + (tl & ~15u);
        const SPtr dp = buf + (pos + 16u * lane - tile_lo);
        if (pos + 1024u <= tile_hi && pos + 1024u <= stop) {
            const uint32_t ub = u + 512u;
            const uint32_t tlb = ub - __umulhi(ub, recip) * P;
            const uint32_t adb = (tlb & 15u) * R2_TEXT + (tlb & ~15u);
            const uint4 d = sld128(dp), e = sld128(dp + 512u);
            const uint4 tx = sld128(ft + ad), mk = sld128(fl + ad), txb = sld128(ft + adb), mkb = sld128(fl + adb);
            high |= d.x | d.y | d.z | d.w | e.x | e.y | e.z | e.w;
            const uint32_t lit = ((d.x ^ tx.x) & mk.x) | ((d.y ^ tx.y) & mk.y) | ((d.z ^ tx.z) & mk.z) | ((d.w ^ tx.w) & mk.w);
            const uint32_t litb = ((e.x ^ txb.x) & mkb.x) | ((e.y ^ txb.y) & mkb.y) | ((e.z ^ txb.z) & mkb.z) | ((e.w ^ txb.w) & mkb.w);
            const uint32_t ok = span_ok(d.x, mk.x) & span_ok(d.y, mk.y) & span_ok(d.z, mk.z) & span_ok(d.w, mk.w);
            const uint32_t okb = span_ok(e.x, mkb.x) & span_ok(e.y, mkb.y) & span_ok(e.z, mkb.z) & span_ok(e.w, mkb.w);
            if (!__ballot_sync(R2_FULL, (lit | litb | (~(ok & okb) & 0x80808080u)) != 0)) {
                const uint32_t u2 = t + 1024u;
                const uint32_t nwr = __umulhi(u2, recip);
                t = u2 - nwr * P; pos += 1024u; nfast += nwr;
                if (nwr) s_open = pos - t;
                continue;
            }
        }
        // one window (the last of a tile, or the first of a pair that did not match)
        const uint32_t lim = r2_min(pos + 512u, tile_hi);
        if (lim > stop || (lim & 15u)) break;
        uint32_t bad = 0;
        if (pos + 16u * lane < lim) {
            const uint4 d = sld128(dp);
            const uint4 tx = sld128(ft + ad), mk = sld128(fl + ad);
            high |= d.x | d.y | d.z | d.w;
            const uint32_t lit = ((d.x ^ tx.x) & mk.x) | ((d.y ^ tx.y) & mk.y) | ((d.z ^ tx.z) & mk.z) | ((d.w ^ tx.w) & mk.w);
            const uint32_t ok = span_ok(d.x, mk.x) & span_ok(d.y, mk.y) & span_ok(d.z, mk.z) & span_ok(d.w, mk.w);
            bad = lit | (~ok & 0x80808080u);
        }
        if (__ballot_sync(R2_FULL, bad != 0)) break;
        const uint32_t u2 = t + (lim - pos);
        const uint32_t nwr = __umulhi(u2, recip);
        t = u2 - nwr * P; pos = lim; nfast += nwr;
        if (nwr) s_open = pos - t;
    }
    FastOut o; o.k = k; o.tile_lo = tile_lo; o.tile_hi = tile_hi; o.buf = buf; o.pos = pos; o.t = t; o.s_open = s_open; o.nfast = nfast; o.high = high;
    return o;
}

// One compare pass of up to 512 bytes from pos against the default slot's periodic image, boundary lanes and limits
// included, and -- on a mismatch inside a value span -- the re-anchoring behind the value's own end.
//   kind 0: fine (ran to its limit, or re-anchored): go on from (pos, t)
//   kind 1: the event that starts at s_open does not follow the default slot
struct PassOut { uint32_t pos, t, s_open, nwr, kind, last_ra, high, reanchored; };
R2_DEV_NOINLINE PassOut pass_step(R2Io io, uint32_t lane, uint32_t slot, uint32_t fast, uint32_t pos0, uint32_t t0, uint32_t s_open0, uint32_t last_ra,
                                  uint32_t sub_end, uint32_t range_hi, uint32_t in_kept, uint32_t carry_cap) {
    const R2Shared* sh = io.sh;
    const TplMeta& m = sh->tpl[slot].m;
    const uint32_t P = m.P;
    PassOut o; o.pos = pos0; o.t = t0; o.s_open = s_open0; o.nwr = 0; o.kind = 0; o.last_ra = last_ra; o.high = 0; o.reanchored = 0;
    const uint32_t wbase = pos0 & ~15u;
    uint32_t lim = r2_min(sub_end, wbase + 512u);
    if (pos0 >= io.tile_lo && pos0 < io.tile_hi) lim = r2_min(lim, io.tile_hi);             // windows do not straddle the resident tile's end
    if (wbase + 512u > range_hi && !in_kept) {                                               // stop at the first event boundary in the next range
        const uint32_t nb = pos0 + (P - t0);
        uint32_t b = nb;
        if (b < range_hi) b = nb + __umulhi(range_hi - nb + P - 1u, m.recip) * P;
        lim = r2_min(lim, b);
    }
    const uint32_t lp = wbase + 16u * lane;
    const uint32_t u = t0 + P + 16u * lane - (pos0 & 15u);
    const uint32_t tl = u - __umulhi(u, m.recip) * P;
    uint4 tx, mk;
    if (fast) {
        const uint32_t ad = (tl & 15u) * R2_TEXT + (tl & ~15u);
        tx = sld128(sptr(sh->fast_text) + ad); mk = sld128(sptr(sh->fast_lit) + ad);
    } else {
        const SPtr tp = sptr(sh->tpl[slot].text) + (tl & ~3u), lpm = sptr(sh->tpl[slot].lit) + (tl & ~3u);
        const uint32_t shf = 8 * (tl & 3u);
        const uint32_t a0 = sld32(tp), a1 = sld32(tp + 4), a2 = sld32(tp + 8), a3 = sld32(tp + 12), a4 = sld32(tp + 16);
        const uint32_t b0 = sld32(lpm), b1 = sld32(lpm + 4), b2 = sld32(lpm + 8), b3 = sld32(lpm + 12), b4 = sld32(lpm + 16);
        tx = make_uint4(__funnelshift_r(a0, a1, shf), __funnelshift_r(a1, a2, shf), __funnelshift_r(a2, a3, shf), __funnelshift_r(a3, a4, shf));
        mk = make_uint4(__funnelshift_r(b0, b1, shf), __funnelshift_r(b1, b2, shf), __funnelshift_r(b2, b3, shf), __funnelshift_r(b3, b4, shf));
    }
    const bool active = lp < lim;
    uint4 d = make_uint4(0, 0, 0, 0);
    if (active) {
        if (lp >= io.tile_lo && lp + 16 <= io.tile_hi) d = sld128(io.buf + (lp - io.tile_lo));
        else if (lp + 16 <= io.n_bytes) d = gld128(io.data + lp);
        else { uint32_t w[4] = {0, 0, 0, 0}; for (uint32_t i = 0; i < 16; ++i) w[i >> 2] |= (uint32_t)io_byte(io, lp + i) << (8 * (i & 3)); d = make_uint4(w[0], w[1], w[2], w[3]); }
    }
    o.high = d.x | d.y | d.z | d.w;
    const uint32_t r0 = (d.x ^ tx.x) & mk.x, r1 = (d.y ^ tx.y) & mk.y, r2 = (d.z ^ tx.z) & mk.z, r3 = (d.w ^ tx.w) & mk.w;
    const uint32_t s0 = ~span_ok(d.x, mk.x) & 0x80808080u, s1 = ~span_ok(d.y, mk.y) & 0x80808080u;
    const uint32_t s2 = ~span_ok(d.z, mk.z) & 0x80808080u, s3 = ~span_ok(d.w, mk.w) & 0x80808080u;
    uint32_t bm = 0xFFFFu;                                                                  // bytes of this lane that count
    if (lp < pos0) bm &= pos0 - lp >= 16u ? 0u : (0xFFFFu << (pos0 - lp));
    if (lp + 16u > lim) bm &= lp >= lim ? 0u : (0xFFFFu >> (lp + 16u - lim));
    const uint32_t bb = (movemask4(nonzero_bytes(r0) | s0) | (movemask4(nonzero_bytes(r1) | s1) << 4) | (movemask4(nonzero_bytes(r2) | s2) << 8) | (movemask4(nonzero_bytes(r3) | s3) << 12)) & bm;
    const uint32_t any = __ballot_sync(R2_FULL, active && bb != 0);
    uint32_t mpos = lim;
    if (any) {
        const uint32_t fl = (uint32_t)__ffs(any) - 1u;
        const uint32_t b1 = __shfl_sync(R2_FULL, bb, (int)fl);
        mpos = wbase + 16u * fl + ((uint32_t)__ffs(b1) - 1u);
    }
    // ---- events completed by the pass ----
    const uint32_t u2 = t0 + (mpos - pos0);
    const uint32_t nwr = __umulhi(u2, m.recip);                                               // separators passed
    const uint32_t t2 = u2 - nwr * P;
    o.nwr = nwr; o.pos = mpos; o.t = t2;
    if (nwr) o.s_open = mpos - t2;                                                          // start of the event that is open now
    if (!any) return o;                                                                     // the pass ran to its limit
    // ---- a mismatch at mpos, template offset t2: inside a value span? ----
    const uint32_t id = (t2 < m.len && mpos != last_ra) ? sh->tpl[slot].span_id[t2] : 0xffu;
    if (id != 0xffu) {
        const uint32_t sstart = m.sstart[id], send = m.send[id];
        const uint32_t ev_end = r2_min(sub_end, o.s_open + carry_cap + 2u);
        if (m.skind[id] == 0) {                                                              // string value: plain bytes and valid escapes up to the closing quote
            uint32_t q = mpos;
            for (;;) {
                // first byte at or after q that is not plain string content, a lane per byte
                const uint32_t c = q + lane < ev_end ? (uint32_t)io_byte(io, q + lane) : 0u;   // (past the end: reads as a control byte, the scan stops)
                o.high |= c;
                const uint32_t sp = __ballot_sync(R2_FULL, c < 0x20u || c == '"' || c == '\\');
                if (!sp) { q += 32; if (q - mpos > R2_MAX_STR) break; continue; }
                const uint32_t k = (uint32_t)__ffs(sp) - 1u, x = q + k;
                const uint32_t ch = __shfl_sync(R2_FULL, c, (int)k);
                if (ch == '"') { o.pos = x; o.t = send; o.reanchored = 1; return o; }        // (the closing quote itself is compared by the next pass)
                if (ch != '\\') break;                                                       // a control byte (or the end of the readable text)
                const uint32_t e1 = x + 1 < ev_end ? (uint32_t)io_byte(io, x + 1) : 0u;
                uint32_t el = 0;
                if (e1 == 'u') { el = 6; for (uint32_t h4 = 2; h4 < 6; ++h4) { const uint32_t h = x + h4 < ev_end ? (uint32_t)io_byte(io, x + h4) : 0u; if (!(h - '0' < 10u || (h | 0x20u) - 'a' < 6u)) el = 0; } }
                else if (e1 == '"' || e1 == '\\' || e1 == '/' || e1 == 'b' || e1 == 'f' || e1 == 'n' || e1 == 'r' || e1 == 't') el = 2;
                if (el == 0) break;
                q = x + el;
                if (q - mpos > R2_MAX_STR) break;
            }
        } else {                                                                              // number value: the event's own number must be valid
            const uint32_t bs = mpos - (t2 - sstart);
            uint32_t x2 = 0, good = 0;
            if (lane == 0) {
                uint32_t st = L_VALUE, p = bs;
                for (;;) {
                    if (p >= ev_end) break;
                    const uint32_t cl = sh->cls[io_byte(io, p)];
                    if (cl < C_MINUS || cl > C_EXP) break;
                    st = sh->trans[st * 32 + cl] & 31u;
                    if (st == L_ERR) break;
                    ++p;
                }
                good = (st == L_NUM_ZERO || st == L_NUM_INT || st == L_NUM_FRAC || st == L_NUM_EXP) ? 1u : 0u;
                x2 = p;
            }
            x2 = __shfl_sync(R2_FULL, x2, 0); good = __shfl_sync(R2_FULL, good, 0);
            if (good && x2 >= mpos) { o.pos = x2; o.t = send; o.last_ra = x2; o.reanchored = 1; return o; }
        }
    }
    // the event does not follow this slot: back to its start
    o.kind = 1; o.pos = o.s_open; o.t = 0; o.last_ra = R2_NONE;
    return o;
}

// the first eight bytes of the event at ps against the first eight of a template (literal positions only): true = they part
R2_DEV bool head_differs(const R2Io& io, const Tpl2* tp, uint32_t lane, uint32_t ps, uint32_t ev_end) {
    bool diff = false;                  // one byte per lane over the template's first 32 bytes (events of different kinds share "data: {" and more)
    if (lane < tp->m.len && tp->lit[lane]) diff = ps + lane >= ev_end || (uint32_t)io_byte(io, ps + lane) != (uint32_t)tp->text[lane];
    return __any_sync(R2_FULL, diff) != 0;
}

// One event that does not follow the default slot: the other slots span by span (usage events read their fields on the
// way), else the byte-wise recogniser (which may leave a new template behind).
//   e: position of the event's LF LF; R2_NONE: still open at the end of the text
//   status 1: the stream goes to the sequential path
struct OddOut { uint32_t e, status, ev_a, ev_b, a_usage, primed, high; };
R2_DEV_NOINLINE OddOut odd_event(const StepArgs* ap, R2Shared* sh, R2Io io, uint32_t lane, uint32_t seg, uint32_t tb, uint32_t ps, uint32_t sub_end,
                                 uint32_t in_kept, uint32_t primed, uint32_t skip_slot) {
    OddOut o; o.e = R2_NONE; o.status = 0; o.ev_a = o.ev_b = o.a_usage = 0; o.primed = primed; o.high = 0;
    TemplateCache2* tc = ap->s.tpl_cache2;
    const uint32_t ev_end = r2_min(sub_end, ps + ap->t.carry_cap + 2u);
    uint32_t ready = 0, free_slots = 0;
    if (lane == 0) for (uint32_t k = 0; k < R2_SLOTS; ++k) { const uint32_t st = *(volatile uint32_t*)&sh->slot_state[k]; if (st == 2u) ready |= 1u << k; else if (st == 0u) free_slots |= 1u << k; }
    ready = __shfl_sync(R2_FULL, ready, 0); free_slots = __shfl_sync(R2_FULL, free_slots, 0);
    // the stream terminator `data: [DONE]` LF LF, byte for byte (not JSON: no class, nothing to account; chat_logging.py:116-121,
    // request_handler.py:122-131 skip it) -- the one non-JSON event every stream has
    {
        const uint32_t want = lane < 14u ? (uint32_t)(uint8_t)"data: [DONE]\n\n"[lane] : 0u;
        const bool fits = ps + 14u <= ev_end;
        const bool same = lane >= 14u || (fits && (uint32_t)io_byte(io, ps + lane) == want);
        if (__all_sync(R2_FULL, same)) {
            const bool third_lf = ps + 14u < sub_end && io_byte(io, ps + 14u) == '\n';           // LF run >= 3: the sequential path's case
            if (!third_lf) { o.e = ps + 12u; return o; }
        }
    }
    for (uint32_t slot = 0; slot < R2_SLOTS; ++slot) {
        if (!(ready & (1u << slot)) || slot == skip_slot) continue;
        if (head_differs(io, &sh->tpl[slot], lane, ps, ev_end)) continue;            // (most wrong slots part within the first bytes)
        const TplMeta& m = sh->tpl[slot].m;
        const SingleOut so = match_single(io, &sh->tpl[slot], lane, ps, ev_end);
        if (!so.ok) continue;
        o.high |= so.high;
        if (lane == 0 && sh->slot_gidx[slot] != R2_NONE) atomicAdd(&tc->hits[sh->slot_gidx[slot]], 1u);
        const Acct ac = account(ap, lane, seg, in_kept, primed, m.cls, m.flags, 1, ps, so.e);
        if (!ac.ok) { o.status = 1; return o; }
        if ((m.flags & TK_USAGE) && (m.flags & PF_VALID_B) && m.usage_ok && so.e - ps <= LGW_PENDING_CAP && sh->slot_gidx[slot] != R2_NONE) {
            // where its eight usage fields sit: k_commit2 reads the values out (one warp per segment there, nothing serial here)
            uint2* uf = ap->s.usage_fields + (size_t)seg * 9u;
            if (lane < 8u) uf[lane] = m.field_span[lane] != 0xffu ? make_uint2(so.f_start, so.f_len | (so.f_esc << 31)) : make_uint2(0u, 0xFFFFFFFFu);
            if (lane == 0) { uf[8] = make_uint2(sh->slot_gidx[slot], m.full_flags); ap->s.plan[seg].cand_ps = ps + 1u; }
        }
        o.e = so.e; o.ev_a = ac.ev_a; o.ev_b = ac.ev_b; o.a_usage = ac.a_usage; o.primed = ac.primed;
        return o;
    }
    // ---- no template fits: the byte-wise recogniser walks the event ----
    if (ps > tb && io_byte(io, ps) == '\n') { o.status = 1; return o; }                       // LF run >= 3
    const LeanOut lo = lean_event(io, lane, ps, ev_end);
    o.high |= lo.high;
    if (lo.e == R2_NONE) { if (ev_end < sub_end) o.status = 1; return o; }                    // longer than the carry capacity / open at the end of the text
    if (lo.e + 2 < sub_end && io_byte(io, lo.e + 2) == '\n') { o.status = 1; return o; }
    if (lo.cls != PC_NONE && lane == 0) atomicAdd(&tc->general, 1u);
    const Acct ac = account(ap, lane, seg, in_kept, primed, lo.cls, lo.f, 1, ps, lo.e);
    if (!ac.ok) { o.status = 1; return o; }
    if (lo.cls != PC_NONE && (lo.f & PF_VALID_A) && !(lo.f & (TK_ERROR | TK_DETAIL | TK_CODE)) && lo.e - ps >= R2_TPL_MIN && lo.e - ps <= R2_TPL_MAX && free_slots)
        learn_template(ap, sh, io, sh->raw_tpl, lane, ready, ps, sub_end);
    o.e = lo.e; o.ev_a = ac.ev_a; o.ev_b = ac.ev_b; o.a_usage = ac.a_usage; o.primed = ac.primed;
    return o;
}

// Walk the current segment from c.pos.  Returns true when the warp is done (the open event starts in the next warp's
// range); false when the segment's text is finished for this warp (go on with the next segment).  The caller leaves the
// segment (counters, chunk-level UTF-8) either way.
R2_DEV bool walk_segment(R2Ctx& c, const uint32_t range_hi) {
    R2Shared* sh = c.sh;
    const uint32_t lane = c.lane;
    for (;;) {
        // The kept chunk of a freshly speculated stream (in_kept 1) is walked on its own: its events are the priming loop's and the
        // tap's, not the handler's, and it must end on a separator.  When the chunk is a whole number of default-slot periods
        // long it is first walked OPTIMISTICALLY (in_kept 2) as part of the periodic run: if nothing but rigid default events
        // happened up to its end, that end is a separator and the events before it were valid real events -- accounts are
        // corrected and the chunk is done; any surprise before its end rewinds to the segment's start and walks it the careful way.
        if (c.in_kept == 2u && c.s_open >= c.kept_end) {
            const TplMeta& dm = sh->tpl[c.dflt].m;
            c.ev_a -= __umulhi(c.kept_end - c.tb, dm.recip);                   // the kept chunk's events are not the handler's
            if (lane == 0) c.a->s.plan[c.seg].prime_ok = 1;
            c.in_kept = 0;
        }
        const uint32_t sub_end = c.in_kept == 1u ? c.kept_end : c.te;          // the text the current phase may read
        if (c.pos >= sub_end) {
            // ---- end of the kept chunk / of the segment's text ----
            if (c.in_kept == 2u) { c.in_kept = 1u; c.pos = c.s_open = c.tb; c.t = 0; c.ev_a = c.ev_b = c.a_usage = 0; c.primed = 0; c.last_ra = R2_NONE; continue; }
            if (c.in_kept) {                                                   // the speculation holds when a real event was accepted
                if (c.s_open != c.kept_end || !c.primed) { mark_irregular(c); return false; }   //   and the chunk ends on a separator
                if (lane == 0) c.a->s.plan[c.seg].prime_ok = 1;
                c.in_kept = 0;
                continue;
            }
            if (lane == 0) c.a->s.plan[c.seg].tail_start = c.s_open + 1u;      // the open event is the new carry
            return false;
        }
        if (c.s_open >= range_hi && c.pos == c.s_open && !c.in_kept) return true;   // the open event starts in the next warp's range
        while (c.pos >= c.tile_hi && c.k + 1 < c.n_tiles) pipe_advance(c);      // (slow paths may have run ahead of the resident tile)

        const bool have_dflt = (c.ready & (1u << c.dflt)) != 0u && !(sh->tpl[c.dflt].m.flags & TK_USAGE);
        if (c.in_kept == 1u && c.pos == c.tb && have_dflt && c.kept_end > c.tb && c.kept_end < c.te) {
            const TplMeta& dm = sh->tpl[c.dflt].m;
            const uint32_t n = c.kept_end - c.tb, q = __umulhi(n, dm.recip);
            if (dm.cls == PC_DATA && q * dm.P == n && !c.kept_tried) { c.in_kept = 2u; c.kept_tried = 1u; }
        }
        // ---- fast run: whole 16-byte aligned windows against the default slot's periodic image, tile after tile (out of line) ----
        if (have_dflt && c.fast && c.in_kept != 1u && (c.pos & 15u) == 0u && c.pos >= c.tile_lo && c.pos < c.tile_hi) {
            const TplMeta& dm = sh->tpl[c.dflt].m;
            const FastOut fo = fast_run(c.a, sh, c.ring, c.bars, c.base, c.n_tiles, c.n_bytes, c.k, c.tile_lo, c.tile_hi, c.buf,
                                        c.pos, c.t, c.s_open, r2_min(sub_end, range_hi), dm.P, dm.recip, lane);
            c.k = fo.k; c.tile_lo = fo.tile_lo; c.tile_hi = fo.tile_hi; c.buf = fo.buf;
            c.high |= fo.high;
            if (fo.nfast) {
                c.single = 0u;
                c.hits_d += fo.nfast; c.s_open = fo.s_open;
                if (dm.cls == PC_DATA) c.ev_a += fo.nfast;
                if (dm.flags & PF_VALID_B) c.ev_b += fo.nfast;
            }
            if (fo.pos != c.pos) { c.pos = fo.pos; c.t = fo.t; continue; }
        }
        // ---- events that follow the default slot but not its period: one event per step, span by span ----
        bool try_pass = have_dflt;
        if (have_dflt && c.single && c.t == 0u && c.pos == c.s_open && c.in_kept != 2u) {
            const SingleOut so = match_single(io_of(c), &sh->tpl[c.dflt], lane, c.pos, r2_min(sub_end, c.pos + c.a->t.carry_cap + 2u));
            if (so.ok) {
                const TplMeta& dm = sh->tpl[c.dflt].m;
                c.high |= so.high; ++c.hits_d;
                if (dm.cls == PC_DATA) { if (c.in_kept == 1u) c.primed = 1; else ++c.ev_a; }
                if (dm.flags & PF_VALID_B) ++c.ev_b;
                c.pos = c.s_open = so.e + 2u; c.last_ra = R2_NONE;
                continue;
            }
            try_pass = false;                                                  // not a default event at all: the other slots / the recogniser
        }
        // ---- one pass with its boundary lanes, limits and re-anchoring (out of line) ----
        if (try_pass && c.t == 0u && c.pos == c.s_open && head_differs(io_of(c), &sh->tpl[c.dflt], lane, c.pos, sub_end)) try_pass = false;   // not a default event: no pass
        if (try_pass) {
            const PassOut po = pass_step(io_of(c), lane, c.dflt, c.fast, c.pos, c.t, c.s_open, c.last_ra, sub_end, range_hi, c.in_kept == 1u ? 1u : 0u, c.a->t.carry_cap);
            c.high |= po.high;
            if (po.nwr) {
                const TplMeta& dm = sh->tpl[c.dflt].m;
                c.hits_d += po.nwr;
                if (dm.cls == PC_DATA) { if (c.in_kept == 1u) c.primed = 1; else c.ev_a += po.nwr; }      // (a template is a valid event without error/detail)
                if (dm.flags & PF_VALID_B) c.ev_b += po.nwr;
            }
            c.pos = po.pos; c.t = po.t; c.s_open = po.s_open; c.last_ra = po.last_ra;
            if (po.reanchored) c.single = 1u;                                  // a value span of another length than the template's
            if (c.in_kept == 2u && (po.kind || po.reanchored) && c.s_open < c.kept_end) {      // a surprise inside the kept chunk: walk it the careful way
                c.in_kept = 1u; c.pos = c.s_open = c.tb; c.t = 0; c.ev_a = c.ev_b = c.a_usage = 0; c.primed = 0; c.last_ra = R2_NONE;
                continue;
            }
            // single-event mode and the pass ran on into a LATER event before it met a value span of another length: that event is
            // judged from its start by match_single (one step per event) -- going on from the re-anchor would keep the stream in
            // pass mode for good, because every pass ends inside the next event and never at an event start
            if (po.kind == 0 && po.reanchored && po.nwr && c.in_kept != 2u) { c.pos = c.s_open; c.t = 0u; c.last_ra = R2_NONE; continue; }
            if (po.kind == 0) continue;
        } else if (c.in_kept == 2u && c.s_open < c.kept_end) {
            c.in_kept = 1u; c.pos = c.s_open = c.tb; c.t = 0; c.ev_a = c.ev_b = c.a_usage = 0; c.primed = 0; c.last_ra = R2_NONE;
            continue;
        }
        // ---- the event at s_open does not follow the default slot ----
        {
            const OddOut oo = odd_event(c.a, sh, io_of(c), lane, c.seg, c.tb, c.s_open, sub_end, c.in_kept == 1u ? 1u : 0u, c.primed, have_dflt ? c.dflt : R2_NONE);
            c.high |= oo.high;
            if (oo.status) { mark_irregular(c); return false; }
            refresh_slots(c);
            if (oo.e == R2_NONE) { c.pos = sub_end; continue; }             // open at the end of the text: the carry
            c.ev_a += oo.ev_a; c.ev_b += oo.ev_b; c.a_usage |= oo.a_usage; c.primed = oo.primed;
            c.pos = c.s_open = oo.e + 2u; c.t = 0; c.last_ra = R2_NONE;
        }
    }
}

R2_GLOBAL void
#if !R2_HOST_EMU
#ifdef R2_MAXREG                        /* experiment: a register cap below 65536 / R2_THREADS leaves room for the commit kernel's blocks beside this one */
__maxnreg__(R2_MAXREG)
#else
__launch_bounds__(R2_THREADS, 1)
#endif
#endif
k_relay2(StepArgs a, uint32_t n_tiles_total, uint32_t tiles_per_warp, uint32_t base0) {
    uint8_t* smem = smem_base();
    R2Shared* sh = reinterpret_cast<R2Shared*>(smem + R2_RING_BYTES);
    const uint32_t tid = R2_TID, warp = tid >> 5, lane = tid & 31u;
    TemplateCache2* tc = a.s.tpl_cache2;
    UsageRaw* block_raw = sh->raw_tpl;

    // ---- block prologue: recogniser tables, barriers, the first tiles.  This is the launch set's first kernel, ordered behind the
    // previous one's k_commit2 (and any k_streams_open) by the stream: nothing to wait for ----
    griddep_launch();
    if (R2_BID == 0 && tid == 0 && a.reset_rows) *a.rowq_count = 0;        // (only k_commit2 appends rows, after this kernel)
    for (uint32_t k = tid; k < 64 + LGW_LEAN_ROWS * 8; k += R2_THREADS) {
        if (k < 64) reinterpret_cast<uint32_t*>(sh->cls)[k] = reinterpret_cast<const uint32_t*>(lean_tables().cls)[k];
        else reinterpret_cast<uint32_t*>(sh->trans)[k - 64] = reinterpret_cast<const uint32_t*>(lean_tables().trans)[k - 64];
    }
    if (tid == 0) { sh->fast_ready = 0; sh->learn_lock = 0; sh->args = a; }
    if (lane == 0) for (uint32_t b = 0; b < R2_NBUF; ++b) mbar_init(sptr(&sh->mbar[warp * R2_NBUF + b]), 1);
    mbar_fence_init();
    __syncthreads();
    // this warp's byte range; its first tiles are requested now, they travel while the block sets up its tables
    const uint32_t gw = R2_BID * R2_WARPS + warp;
    const uint32_t t_first = gw * tiles_per_warp;
    R2Ctx c;
    c.a = &sh->args; c.sh = sh; c.lane = lane;
    c.ring = sptr(smem) + warp * R2_NBUF * R2_TILE; c.bars = sptr(&sh->mbar[warp * R2_NBUF]);
    c.n_bytes = a.n_bytes;
    c.base = base0 + t_first * R2_TILE;
    c.n_tiles = t_first >= n_tiles_total ? 0u : r2_min(tiles_per_warp, n_tiles_total - t_first);
    pipe_start(c);
    if (tid < R2_SLOTS) { sh->slot_state[tid] = (*(volatile uint32_t*)&tc->state[tid] == 2u) ? 2u : 0u; sh->slot_gidx[tid] = tid; }
    __syncthreads();
    for (uint32_t s = 0; s < R2_SLOTS; ++s) {
        if (sh->slot_state[s] != 2u) continue;
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&tc->tpl[s]);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sh->tpl[s]);
        for (uint32_t k = tid; k < sizeof(Tpl2) / 4; k += R2_THREADS) dst[k] = src[k];
        const uint32_t* rs = reinterpret_cast<const uint32_t*>(&tc->raw[s]);
        uint32_t* rd = reinterpret_cast<uint32_t*>(&block_raw[s]);
        for (uint32_t k = tid; k < sizeof(UsageRaw) / 4; k += R2_THREADS) rd[k] = rs[k];
    }
    if (tid == 0) {
        uint32_t d = 0, best = 0; bool have = false;
        for (uint32_t s = 0; s < R2_SLOTS; ++s) if (sh->slot_state[s] == 2u) { const uint32_t h = tc->hits[s]; if (!have || h > best) { d = s; best = h; have = true; } }
        sh->dflt = d;
    }
    __syncthreads();
    if (sh->slot_state[sh->dflt] == 2u) {
        build_fast_tables(sh, sh->dflt, tid, R2_THREADS);
        __syncthreads();
        if (tid == 0) sh->fast_ready = 1;
    }
    __syncthreads();

    c.dflt = sh->dflt; c.last_ra = R2_NONE; c.hits_d = 0; c.single = 0;
    refresh_slots(c);
    c.seg = R2_NONE; c.ev_a = c.ev_b = c.a_usage = 0; c.high = 0;
    c.t = 0; c.pos = c.s_open = 0;
    c.in_kept = c.primed = c.kept_tried = 0; c.tb = c.te = c.kept_end = 0; c.walk_lo = 0;
    if (c.n_tiles == 0) return;
    const uint32_t range_lo = r2_max(c.base, a.tile_base);          // (tile_base = first byte of this launch; a slice starts inside tile 0)
    const uint32_t range_hi = r2_min(c.base + c.n_tiles * R2_TILE, a.n_bytes);
    uint32_t* win = &sh->plan_win[warp][0][0];
    const uint2 fs = first_segment(&sh->args, win, lane, range_lo);              // the segment that holds the range's first byte
    const uint32_t seg0 = fs.x;
    uint32_t win_lo = fs.y;
    pipe_advance(c);

    uint32_t seg_first = range_lo;                                                // (seg0's text begins at or before range_lo)
    for (uint32_t seg = seg0; seg < a.n_segs; ++seg) {
        if (seg_first >= range_hi) break;
        if (seg - win_lo >= 32u) { win_lo = seg; load_plans(&sh->args, win, lane, seg); }   // the walk has left the window
        const uint32_t i = seg - win_lo, tb = win[i], te = win[32 + i], kept = win[64 + i];
        const bool done = enter_segment(c, seg, tb, te, kept, r2_max(range_lo, seg_first), range_hi) && walk_segment(c, range_hi);
        leave_segment(c, range_hi);
        if (done) break;
        seg_first = te;
    }
    // ---- the rest of the range is copy only ----
    while (c.k + 1 < c.n_tiles) pipe_advance(c);
    __syncwarp();
    if (lane == 0) {
        tma_wait_all();
        if (c.hits_d && sh->slot_gidx[c.dflt] != R2_NONE) atomicAdd(&tc->hits[sh->slot_gidx[c.dflt]], c.hits_d);
    }
}

#if R2_HOST_EMU
// The emulator's step driver (tests/support/host_relay2.cpp) still launches a planning kernel before the bulk kernel, as the
// device step did before each kernel began to compute its segments' static plans itself (seg_static): nothing is left for it.
R2_GLOBAL void k_prime2(StepArgs) {}
#endif

// ---- template-cache upkeep: once per launch set, between its k_relay2 and the next launch set's (k_commit2's block 0) ----------------
R2_DEV void tpl_cache_upkeep(TemplateCache2* tc) {
    uint32_t total = 0, full = 1, lo = 0;
    for (uint32_t s = 0; s < R2_SLOTS; ++s) { total += tc->hits[s]; if (tc->state[s] != 2u) full = 0; if (tc->hits[s] < tc->hits[lo]) lo = s; }
    // most events of the last steps matched no template although every slot is taken: forget the least useful one
    // -- or one slot has not matched anything for many steps while events go unmatched
    if (full && tc->general && (tc->hits[lo] == 0 || (tc->general > 64u && tc->general > total / 2u))) { tc->state[lo] = 0; tc->hits[lo] = 0; }
    for (uint32_t s = 0; s < R2_SLOTS; ++s) tc->hits[s] >>= 1;
    tc->general >>= 1;
}

// ---- k_commit2 (one warp per segment) ----------------------------------------------------------------------------------------------
#define R2_CWARPS 8u
#ifndef R2_CBLOCKS                      /* resident blocks per SM the commit kernel is compiled for: 6 -> 40 registers, 4 -> 64, 3 -> 80.
                                           4 x 8 warps x 132 SMs hold a warp for each of C3's 4 096 segments at once, and with 64
                                           registers ptxas reports 12 B of spill stores instead of 140 (DESIGN 4.3)
                                           (3 blocks: two waves, no faster than 6; DESIGN 9.12) */
#define R2_CBLOCKS 4
#endif
// the exact sequential machine over a stream's chunks (streams the bulk kernel could not vouch for), out of line
R2_DEV_NOINLINE uint32_t commit_sequential(StepIO io, const uint8_t* data, const uint32_t* chunk_off, uint32_t c_from, uint32_t c_to, uint32_t emit_begin) {
    run_chunks(io, data, chunk_off, c_from, c_to, emit_begin, false);
    return emit_begin;
}
// a usage event that followed no usage template: the full machine over its staged text (chat_logging.py:123-135 ->
// get_token_usage :233-272), exactly what the sequential path does for the event
R2_DEV_NOINLINE void commit_usage_event(StepIO io, const uint8_t* text, uint32_t n) {
    StreamHdr& st = *io.st;
    Rope r{nullptr, 0, text, n};
    const uint8_t cls = classify_part(r, 0, n);
    UsageRaw raw;
    const uint32_t f = parse_part<true>(r, 0, n, cls, &raw);
    if (f & PF_EXOTIC) { ++st.n_exotic; st.flags |= SF_EXOTIC_SEEN; return; }
    if ((f & TK_CHOICES) && (f & PF_TYPE_ERROR)) return;
    normalise_usage(raw, f, *io.rec);
    st.flags |= SF_REC_VALID; ++st.n_usage_b;
    if (io.rec->exotic) { ++st.n_exotic; st.flags |= SF_EXOTIC_SEEN; }
}
// usage fields of a template-following usage event straight from the value spans the bulk kernel's match located (usage_ok
// templates): numbers through decimal.cuh, strings copied (decoded like the full machine does when they hold escapes),
// get_token_usage's arithmetic (normalise_usage) on the assembled record, which lands in the stream's tap record.
// `text` holds the event's bytes (staged in shared memory), text[0] = the byte at position `ups` of the step's buffer.
struct TextReader {
    const uint8_t* text; uint32_t base, n;
    R2_MEM uint32_t at(uint32_t p) const { return p - base < n ? (uint32_t)text[p - base] : 0u; }
};
R2_DEV_NOINLINE uint32_t commit_usage_fields(const uint8_t* text, uint32_t ups, uint32_t ulen, uint32_t full_flags, UsageRaw* raw, UsageRec* cand, uint32_t lane,
                                             uint32_t f_start, uint32_t f_word) {
    TextReader rd{text, ups, ulen};
    const bool has_span = lane < 8u && f_word != 0xFFFFFFFFu;
    const uint32_t f_len = f_word & 0x7FFFFFFFu, f_esc = has_span ? f_word >> 31 : 0u;
    const uint32_t span_mask = __ballot_sync(R2_FULL, has_span);
    Val v; v.kind = KD_ABSENT; v.bits = 0;
    __syncwarp();
    const uint32_t slow_str = __ballot_sync(R2_FULL, has_span && lane >= UF_MODEL && f_esc != 0u);
    if (has_span) {
        if (lane < UF_MODEL) v = parse_number_span(rd, f_start, f_len);
        else if (f_esc) {                                                              // escapes: decode like json_machine.cuh does
            if (lane == UF_MODEL) decode_string_span(rd, f_start, f_len, raw->model, raw->model_len, raw->model_flags);
            else decode_string_span(rd, f_start, f_len, raw->provider, raw->provider_len, raw->provider_flags);
        } else if (lane == UF_MODEL) { raw->model_len = 0; raw->model_flags = 0; }
        else { raw->provider_len = 0; raw->provider_flags = 0; }
    }
    __syncwarp();
    for (uint32_t fi = 0; fi < UF_MODEL; ++fi) {
        const unsigned long long vb = __shfl_sync(R2_FULL, (unsigned long long)v.bits, (int)fi);
        const uint32_t vk = __shfl_sync(R2_FULL, (uint32_t)v.kind, (int)fi);
        if (lane == 0 && (span_mask & (1u << fi))) {
            Val x; x.bits = (int64_t)vb; x.kind = (uint8_t)vk;
            if (fi == UF_PROMPT) raw->prompt = x; else if (fi == UF_COMPLETION) raw->completion = x; else if (fi == UF_TOTAL) raw->total = x;
            else if (fi == UF_COST) raw->cost = x; else if (fi == UF_REASONING) raw->reasoning = x; else raw->cached = x;
        }
    }
    uint32_t has = 0, exotic = 0;                                                      // has bit 0: the record carries "model" as a string, bit 1: "provider"
    if (lane == 0) {
        normalise_usage(*raw, full_flags, *cand);
        has = (cand->model_val.kind == KD_STR ? 1u : 0u) | (cand->provider_val.kind == KD_STR ? 2u : 0u);
        exotic = cand->exotic;
    }
    has = __shfl_sync(R2_FULL, has, 0);
    // plain strings (no escapes): the span's bytes ARE the decoded text -- copy them into the record, a lane per byte
    for (uint32_t which = 0; which < 2; ++which) {
        const uint32_t fl = UF_MODEL + which;
        const uint32_t st = __shfl_sync(R2_FULL, f_start, (int)fl), ln = __shfl_sync(R2_FULL, f_len, (int)fl);
        if (!(span_mask & (1u << fl)) || (slow_str & (1u << fl)) || !(has & (1u << which))) continue;
        const uint32_t n = ln < LGW_STR_CAP ? ln : (uint32_t)LGW_STR_CAP;
        char* dst = which == 0 ? cand->model : cand->provider;
        for (uint32_t k = lane; k < n; k += 32) dst[k] = (char)rd.at(st + k);
        if (lane == 0) {
            if (which == 0) cand->model_len = (uint8_t)n; else cand->provider_len = (uint8_t)n;
            if (ln > LGW_STR_CAP) { cand->str_flags |= which == 0 ? 1u : 4u; cand->exotic = 1; exotic = 1; }   // truncated: reported, like the full machine's capture
        }
    }
    __syncwarp();
    return __shfl_sync(R2_FULL, exotic, 0);                                            // (the record's `exotic`, without reading it back)
}

R2_DEV_NOINLINE void commit_settle_pending(StepIO io) { resolve_pending(io); }
#if !R2_HOST_EMU
R2_DEV uint4 commit_ld16(const uint8_t* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
#else
R2_DEV uint4 commit_ld16(const uint8_t* p) { uint4 v; memcpy(&v, p, 16); return v; }
#endif

// the commit of segment `seg` (one warp)
R2_DEV void commit_one(const StepArgs& a, uint32_t seg, uint32_t lane, uint8_t* stage, UsageRaw* stage_raw, uint32_t* counts) {
    const uint32_t c0 = __ldg(a.seg_chunk + seg), c1 = __ldg(a.seg_chunk + seg + 1);
    const uint32_t slot = __ldg(a.seg_slot + seg);
    // Everything that does not depend on the bulk kernel runs BEFORE the wait, while that kernel is still at work (this kernel's
    // blocks become resident as soon as the bulk kernel's blocks have all started): the stream's state (written only by the
    // commit of an earlier step) and the scan of the segment's chunk offsets for empty chunks.
    StreamHdr st = a.t.state[slot].h;                     // (every lane holds a copy; lane 0's is the one written back)
    // an empty chunk is never yielded (request_handler.py:60-63): the concatenation argument does not cover it
    bool empty = false;
    if ((st.phase == PH_COMMITTED || st.phase == PH_PRIMING) && c0 < c1) {
        for (uint32_t c = c0 + lane; c < c1; c += 32 * 8) {                 // eight independent trips in flight (a plain loop is one DRAM round trip per trip)
            uint32_t lo[8], hi[8];
#pragma unroll
            for (uint32_t j = 0; j < 8; ++j) { const uint32_t cc = c + 32 * j; lo[j] = cc < c1 ? __ldg(a.chunk_off + cc) : 0u; hi[j] = cc < c1 ? __ldg(a.chunk_off + cc + 1) : 1u; }
#pragma unroll
            for (uint32_t j = 0; j < 8; ++j) if (lo[j] == hi[j]) empty = true;
        }
    }
    const bool any_empty = __any_sync(R2_FULL, empty);
    // the plan the bulk kernel worked to (its chunk offsets were just read by the scan)
    const SegStatic p = seg_static(a.chunk_off, c0, c1, st.phase, st.flags, st.carry_a_len);
    griddep_wait();                                       // (the bulk kernel's findings from here on)
    SegPlan* const fp = a.s.plan + seg;
    const SegPlan f = *fp;
    const uint2 fw = lane < 9u ? a.s.usage_fields[(size_t)seg * 9u + lane] : make_uint2(0u, 0xFFFFFFFFu);   // (requested with the findings, used when has_cand)
    __syncwarp();
    if (lane < sizeof(SegPlan) / 4) reinterpret_cast<uint32_t*>(fp)[lane] = 0u;   // read: zero again for the next launch set
    const StepIO io = make_io(a, slot, &st);
    uint32_t emit_begin = p.emit_chunk_begin;
    const bool speculated = p.kept_chunk != 0xFFFFFFFFu;
    if ((st.phase == PH_COMMITTED || st.phase == PH_PRIMING) && p.resume_chunk < c1) {
        const uint8_t* __restrict__ d = a.data;
        // the winning usage event: its text (and, when the bulk kernel matched it against a usage template, where its fields sit)
        // is requested now, together with the chunk offsets below -- one round trip for all of it
        const uint32_t ups = (uint32_t)(f.last_usage >> 32) - 1u, ulen = (uint32_t)f.last_usage;
        const bool staged = f.last_usage && ulen <= LGW_PENDING_CAP && (uint64_t)ups + ulen <= a.n_bytes;
        const bool has_cand = staged && f.cand_ps == ups + 1u;
        const uint2 fld = has_cand && lane < 8u ? fw : make_uint2(0u, 0xFFFFFFFFu);
        const uint32_t g_slot = __shfl_sync(R2_FULL, fw.x, 8), g_flags = __shfl_sync(R2_FULL, fw.y, 8);
        if (has_cand) {                                   // the template event's own UsageRaw, requested together with the text
            const uint32_t* src = reinterpret_cast<const uint32_t*>(&a.s.tpl_cache2->raw[g_slot]);
            for (uint32_t k = lane; k < sizeof(UsageRaw) / 4; k += 32) reinterpret_cast<uint32_t*>(stage_raw)[k] = src[k];
        }
        // staged as whole 16-byte vectors around the text (the step's buffer is 16-byte aligned: the bulk kernel's TMA needs that too);
        // a vector that would reach beyond the step's bytes is read byte by byte
        const uint32_t ab = ups & ~15u, skew = ups - ab;
        const bool d_aligned = (reinterpret_cast<uintptr_t>(d) & 15u) == 0u;
        const uint8_t* const utext = stage + skew;
        if (staged) {
            const uint32_t nvec = (skew + ulen + 15u) >> 4;
            for (uint32_t k = lane; k < nvec; k += 32) {
                const uint32_t o = ab + (k << 4);
                if (o + 16u <= a.n_bytes && d_aligned) *reinterpret_cast<uint4*>(stage + (k << 4)) = commit_ld16(d + o);
                else for (uint32_t j = 0; j < 16u && o + j < a.n_bytes; ++j) stage[(k << 4) + j] = __ldg(d + o + j);
            }
        }
        bool sequential = p.irregular || f.irregular || f.n_usage_b > 1 || any_empty;   // several usage candidates: let the exact path count them
        if (st.phase == PH_PRIMING && !(speculated && f.prime_ok)) sequential = true;
        if (!sequential && f.last_usage && !staged) sequential = true;
        if (!sequential && f.tail_start == 0u) sequential = true;                                // (nobody reached the end of the text)
        if (lane == 0) atomicAdd(&counts[sequential ? 0 : 1], 1u);
        if (sequential) {
            if (lane == 0) emit_begin = commit_sequential(io, a.data, a.chunk_off, p.resume_chunk, c1, (st.phase == PH_COMMITTED) ? p.resume_chunk : c1);
        } else {
            uint32_t first = p.resume_chunk;
            if (speculated) {                       // apply the verified commit (request_handler.py:89-90, chat_logging.py:200)
                st.phase = PH_COMMITTED; st.verdict = VD_OK;
                st.flags |= SF_EMITTED_ANY | SF_SYNCED;
                st.carry_a_len = st.carry_b_len = 0;
                ++st.n_events_a;                    // the priming parse of the first real event
                first = p.kept_chunk;
            }
            const uint32_t nch = c1 - first, nby = p.seg_end - p.relay_begin;
            st.n_chunks_in += nch; st.n_chunks_emitted += nch; st.bytes_in += nby; st.bytes_emitted += nby;
            st.n_events_a += f.n_events_a; st.n_events_b += f.n_events_b;
            if (f.a_usage) st.flags |= SF_A_USAGE_BOUND;
            if (f.last_usage) {                     // the last usage-bearing event wins (chat_logging.py:134-135)
                if (lane == 0 && (st.flags & SF_PENDING)) commit_settle_pending(io);   // (a stash left by an older engine version of this stream)
                __syncwarp();
                if (has_cand) {
                    // the bulk kernel matched it against a usage template and noted where the eight fields sit: read them out
                    const uint32_t exotic = commit_usage_fields(utext, ups, ulen, g_flags, stage_raw, io.rec, lane, fld.x, fld.y);
                    st.flags |= SF_REC_VALID; ++st.n_usage_b;
                    if (exotic) { ++st.n_exotic; st.flags |= SF_EXOTIC_SEEN; }
                    if (lane == 0) atomicAdd(&counts[2], 1u);
                } else {
                    // no usage template: read the values out of the staged text with the full machine now
                    if (lane == 0) { commit_usage_event(io, utext, ulen); atomicAdd(&counts[3], 1u); }
                }
            }
            // new carry = text after the last separator (both loops: SF_SYNCED)
            const uint32_t tail = f.tail_start - 1u, n = p.seg_end - tail;
            if (n > a.t.carry_cap) { st.carry_a_len = 0; st.flags |= SF_CARRY_OVERFLOW; }
            else { for (uint32_t k = lane; k < n; k += 32) io.carry_a[k] = d[tail + k]; st.carry_a_len = n; }
        }
        __syncwarp();
        if (lane == 0) a.t.state[slot].h = st;
    }
    if (lane == 0) {
        SegResult res;
        fill_seg_result(st, emit_begin, c1, res);
        a.seg_out[seg] = res;
    }
}

R2_GLOBAL void
#if !R2_HOST_EMU
__launch_bounds__(R2_CWARPS * 32, R2_CBLOCKS)      // (the full machine behind commit_usage_event / commit_sequential spills instead of costing every warp 142 registers)
#endif
k_commit2(StepArgs a) {
#if !R2_HOST_EMU
    __shared__ __align__(16) uint8_t stage[R2_CWARPS][LGW_PENDING_STRIDE];           // the winning usage event's text
    __shared__ __align__(16) UsageRaw stage_raw[R2_CWARPS];                           // the record being assembled from it
    __shared__ uint32_t counts[4];                                                  // the block's share of StepScratch::counters, added to them once
#else
    alignas(16) static uint8_t stage[R2_CWARPS][LGW_PENDING_STRIDE];
    static UsageRaw stage_raw[R2_CWARPS];
    static uint32_t counts[4];
#endif
    const uint32_t seg = (R2_BID * R2_NTHR + R2_TID) >> 5, lane = R2_TID & 31u, warp = (R2_TID >> 5) % R2_CWARPS;
    if (R2_TID < 4) counts[R2_TID] = 0;
    __syncthreads();
    if (seg < a.n_segs) commit_one(a, seg, lane, stage[warp], &stage_raw[warp], counts);
    __syncthreads();
    if (R2_TID < 4 && counts[R2_TID]) atomicAdd(a.s.counters + R2_TID, counts[R2_TID]);
    if (R2_BID == 0 && R2_TID == 0) tpl_cache_upkeep(a.s.tpl_cache2);   // (segment 0's lane 0: past griddep_wait, the bulk kernel is done)
}

#if !R2_HOST_EMU
// The two kernels of a launch set.  k_relay2 is launched plainly: stream order puts it behind the previous launch set and any
// k_streams_open, whose writes (stream states, findings zeroed, template cache) it reads from its first instruction on.
// per_kernel = true: CUDA events between the kernels (ev[1] = ev[0]: nothing runs before the bulk kernel); false: k_commit2 is
// launched with programmatic stream serialisation, so that its prologue (and its launch latency) overlaps the bulk kernel -- it
// waits (griddepcontrol.wait) before it reads what that kernel wrote.
static inline cudaError_t launch_step_fast(const StepArgs& a, int sm_count, cudaStream_t stream, cudaEvent_t* ev, int* launched, bool per_kernel) {
    cudaError_t r;
    const uint32_t base0 = a.tile_base & ~15u;
    const uint32_t n_tiles = a.n_bytes > base0 ? (a.n_bytes - base0 + R2_TILE - 1) / R2_TILE : 0u;
    if (per_kernel && (r = cudaEventRecord(ev[1], stream)) != cudaSuccess) return r;
    if (n_tiles) {
        const uint32_t max_warps = (uint32_t)sm_count * R2_WARPS;
        const uint32_t tpw = (n_tiles + max_warps - 1) / max_warps;
        const uint32_t warps = (n_tiles + tpw - 1) / tpw;
        const uint32_t blocks = (warps + R2_WARPS - 1) / R2_WARPS;
        k_relay2<<<blocks, R2_THREADS, R2_SMEM_BYTES, stream>>>(a, n_tiles, tpw, base0);
        ++*launched;
    } else if (a.reset_rows && (r = cudaMemsetAsync(a.rowq_count, 0, 4, stream)) != cudaSuccess) return r;   // (no bulk kernel to do it)
    if (per_kernel && (r = cudaEventRecord(ev[2], stream)) != cudaSuccess) return r;
    if (a.n_segs) {
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((a.n_segs + R2_CWARPS - 1) / R2_CWARPS); cfg.blockDim = dim3(R2_CWARPS * 32); cfg.dynamicSmemBytes = 0; cfg.stream = stream;
        cfg.attrs = attr; cfg.numAttrs = per_kernel ? 0 : 1;
        if ((r = cudaLaunchKernelEx(&cfg, k_commit2, a)) != cudaSuccess) return r;
        ++*launched;
    }
    if (per_kernel && (r = cudaEventRecord(ev[3], stream)) != cudaSuccess) return r;
    if ((r = cudaEventRecord(ev[4], stream)) != cudaSuccess) return r;
    return cudaGetLastError();
}
#endif
