// Argument and scratch structures of the SSE step kernels (shared by sse_kernels.cuh and, as a test aid, the host
// build of relay2.cuh in tests/support).
#pragma once
#include "stream_machine.cuh"
#include "lean_json.cuh"

namespace lgw {

struct DeviceTables {
    StreamState* state;
    uint8_t* carry_a; uint8_t* carry_b; uint8_t* detail; uint8_t* pending;
    uint32_t carry_cap, detail_cap, max_streams;
};

// The bulk path's per-segment record: what k_relay2 found in the segment.  Zero is "nothing found": the scratch is zeroed when
// it is allocated, and k_commit2 zeroes each segment's record again once it has read it, so every launch set starts from zeros.
// (The segment's static plan -- bulk region, speculation -- is not stored: SegStatic in relay2.cuh, computed where it is used.)
struct SegPlan {
    uint32_t irregular;        // 1: the bulk kernel's findings are void, k_commit2 redoes the segment
    uint32_t a_usage;          // handler bound `tokens_usage` (request_handler.py:134)
    unsigned long long last_usage;   // (1 + byte offset) << 32 | length of the last usage-bearing event (atomicMax)
    uint32_t n_events_a, n_events_b, n_usage_b;
    uint32_t prime_ok;         // set by the warp that walks the kept chunk when the speculation holds
    uint32_t tail_start;       // 1 + where the event that is open at the end of the text begins (= new carry); 0: not reached
    uint32_t cand_ps;          // 1 + start of the usage event whose field spans sit in usage_fields[9 * seg ..] (0: none)
};
static_assert(sizeof(SegPlan) == 40, "SegPlan");

struct TemplateCache2;     // relay2.cuh

struct StepScratch {
    SegPlan* plan;             // [max_streams] what k_relay2 found per segment; all zero between launch sets
#ifndef __CUDACC__
    uint32_t* tile_seg;        // host build only, never read: the emulator's step driver (tests/support/host_relay2.cpp) still
                               //   hands the kernels a tile table, which the device step no longer has
#endif
    TemplateCache2* tpl_cache2;  // event templates, persistent across steps
    uint2* usage_fields;       // [max_streams][9] a template-following usage event of this step: (start, length | escapes << 31) of its eight
                               //   usage fields as the match located them, [8].x = the template's slot in the engine-wide cache
    uint32_t* counters;        // diagnostics since engine creation: [0] segments redone sequentially, [1] segments folded from the bulk
                               //   kernel's findings, [2] usage records read from template spans, [3] usage events stashed
};

struct StepArgs {
    DeviceTables t;
    const uint8_t* data; uint32_t n_bytes;     // n_bytes = end of the valid bytes (a slice of a pipelined step ends earlier)
    const uint32_t* chunk_off; uint32_t n_chunks;
    uint32_t tile_base;                        // first byte of the launch (a slice's start: any offset); tile 0 starts at tile_base & ~15
    uint32_t chunk_lo, chunk_hi;               // chunks of this launch: [chunk_lo, chunk_hi).  No kernel reads them: they describe the
                                               //   launch to a debugger, and the host build of the kernels (tests/support) fills them
    const uint32_t* seg_chunk; const uint32_t* seg_slot; uint32_t n_segs;
    uint8_t* out; SegResult* seg_out;
    RowEvent* rowq; uint32_t* rowq_count; uint32_t rowq_cap;
    uint32_t reset_rows;                       // 1: k_relay2 empties the row queue (the first launch of a step)
    StepScratch s;
};

// The slices of a host-buffer step (lgw_sse_step): slice j is segments [cut[j], cut[j + 1]), cut[j] = the first segment whose
// start byte is >= n_bytes * j / n_slices.  So a slice may be empty, and a cut lands on a segment without bytes when one starts
// there.  Fewer segments than slices: one slice.  Returns the number of slices; cut has room for n_slices + 1 entries.
// (The host build of the kernels in tests/support slices with this same function.)
static inline uint32_t step_slice_cuts(uint64_t n_bytes, const uint32_t* chunk_off, const uint32_t* seg_chunk, uint32_t n_segs,
                                       uint32_t n_slices, uint32_t* cut) {
    if (n_segs < n_slices) n_slices = 1;
    cut[0] = 0;
    for (uint32_t j = 1; j < n_slices; ++j) {
        const uint64_t want = n_bytes * j / n_slices;
        uint32_t lo = cut[j - 1], hi = n_segs;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((uint64_t)chunk_off[seg_chunk[mid]] < want) lo = mid + 1; else hi = mid; }
        cut[j] = lo;
    }
    cut[n_slices] = n_segs;
    return n_slices;
}

LGW_HD StepIO make_io(const StepArgs& a, uint32_t slot, StreamHdr* local_hdr) {
    StepIO io;
    io.st = local_hdr;
    io.rec = &a.t.state[slot].rec;
    io.pending = a.t.pending + (size_t)slot * LGW_PENDING_STRIDE;
    io.carry_a = a.t.carry_a + (size_t)slot * a.t.carry_cap;
    io.carry_b = a.t.carry_b + (size_t)slot * a.t.carry_cap;
    io.detail = a.t.detail + (size_t)slot * a.t.detail_cap;
    io.carry_cap = a.t.carry_cap; io.detail_cap = a.t.detail_cap;
    io.rowq = a.rowq; io.rowq_count = a.rowq_count; io.rowq_cap = a.rowq_cap; io.slot = slot;
    return io;
}

}  // namespace lgw
