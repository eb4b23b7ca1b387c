// Transcript tap: the text the reference's response tap accumulates in `llm_response_accum` (SURVEY.md 8(f) rank 3).
//
//   chat_logging.py:108-112   per relayed chunk: decode, buffer += text, split on LF LF, carry
//   chat_logging.py:116-123   per part: "data: {" / "{" prefix test, strip, json5.loads
//   chat_logging.py:124-133   for every choice: delta.content, else message.content -- appended when truthy
//   chat_logging.py:137-139   a top-level "error": the event's own (stripped) text is appended and write_log runs NOW with
//                             the text so far (a "mark": the host cuts the stream's transcript at that position)
//   chat_logging.py:140-143   any exception skips the rest of the part / the chunk (what was appended stays appended)
//
// The relay step (k_prime2 / k_relay2 / k_commit2) decides WHICH chunks are relayed; this pass runs after it over the same
// packed step (`emit_chunk_begin` of every segment) and is decoupled from the relay state: the tap's buffer is re-derived from
// the relayed chunks with its own carry, exactly like the reference's tap thread, which sees nothing but the relayed chunks.
// It is optional (lgw_transcripts_enable): the reference only taps when LOG_CHAT_ENABLED is set (chat_logging.py:166-168).
//
// Kernels (one warp per segment):
//   k_text_extract   regular segments -- tap carry empty, every relayed chunk valid UTF-8 and ending on LF LF, no "error" event --
//                    are parsed one chunk per lane (the split of such a stream never crosses a chunk); the decoded text of chunk c
//                    goes to the chunk's own footprint of a sparse buffer (decoded content is never longer than its JSON spelling).
//                    Anything else is redone by lane 0 with the exact sequential walk (carry, marks).
//   k_text_scan      exclusive scan of the per-segment text lengths (one block).
//   k_text_pack      compacts the sparse pieces into the step's text, segment after segment.
//
// Host/device portable like stream_machine.cuh (tests compile it with g++ over the SIMT emulator; the product has no CPU path).
#pragma once
#include "stream_machine.cuh"
#include "scan.cuh"

namespace lgw {

enum TextFlag : uint32_t {
    TF_LONE_SURROGATE = 1u << 0,   // the text holds a lone surrogate (encoded like Python's 'surrogatepass'): the reference's f.write raises
    TF_EXOTIC = 1u << 1,           // an event had a shape whose Python behaviour the device does not model: the text is not authoritative
    TF_CARRY_OVERFLOW = 1u << 2,   // an unterminated event outgrew carry_cap (engine limit)
    TF_MARKQ_OVERFLOW = 1u << 3,
    TF_SEQUENTIAL = 1u << 4,       // (per step) the segment took the sequential walk
    TF_DOC_ERROR_LOG = 1u << 5     // (per document, doc_text) the document made the tap call write_log at chat_logging.py:139
};

struct TextTap {               // per-stream state of the transcript tap
    uint32_t carry_len;
    uint32_t flags;
    uint32_t n_marks;          // mid-stream write_log calls so far (chat_logging.py:139)
    uint32_t _pad;
    uint64_t text_total;       // bytes of llm_response_accum so far (UTF-8)
};
struct TextMark { uint32_t slot, seq; uint64_t text_pos; };     // == lgw_text_mark

struct TextOut { uint8_t* p; uint32_t pos; uint32_t flags; };

LGW_HD void text_put_cp(TextOut& o, uint32_t cp) {
    uint8_t* q = o.p + o.pos;
    if (cp < 0x80) { q[0] = (uint8_t)cp; o.pos += 1; }
    else if (cp < 0x800) { q[0] = (uint8_t)(0xC0 | (cp >> 6)); q[1] = (uint8_t)(0x80 | (cp & 63)); o.pos += 2; }
    else if (cp < 0x10000) { q[0] = (uint8_t)(0xE0 | (cp >> 12)); q[1] = (uint8_t)(0x80 | ((cp >> 6) & 63)); q[2] = (uint8_t)(0x80 | (cp & 63)); o.pos += 3; }
    else { q[0] = (uint8_t)(0xF0 | (cp >> 18)); q[1] = (uint8_t)(0x80 | ((cp >> 12) & 63)); q[2] = (uint8_t)(0x80 | ((cp >> 6) & 63)); q[3] = (uint8_t)(0x80 | (cp & 63)); o.pos += 4; }
}

LGW_HD uint32_t text_hex4(const Rope& r, uint32_t i) {
    uint32_t v = 0;
    for (uint32_t k = 0; k < 4; ++k) {
        const uint32_t c = r.at(i + k);
        v = (v << 4) | (c - '0' < 10u ? c - '0' : (c | 0x20) - 'a' + 10);
    }
    return v;
}

// Decode the JSON string content r[lo, hi) (already validated by the machine) the way json.loads does: escapes resolved, a high
// surrogate escape directly followed by a low surrogate escape makes one code point, any other surrogate stays alone (Python keeps
// it in the str; here it is written in 'surrogatepass' form and flagged).  Every escape is at least as long as what it decodes to
// (\uXXXX: 6 -> <= 3 bytes, a pair: 12 -> 4), so the output never outgrows the input.
LGW_HD void text_unescape(const Rope& r, uint32_t lo, uint32_t hi, TextOut& o) {
    uint32_t i = lo;
    while (i < hi) {
        const uint32_t c = r.at(i);
        if (c != '\\') { o.p[o.pos++] = (uint8_t)c; ++i; continue; }
        const uint32_t e = r.at(i + 1);
        i += 2;
        switch (e) {
        case 'b': o.p[o.pos++] = 8; break;   case 'f': o.p[o.pos++] = 12; break;  case 'n': o.p[o.pos++] = 10; break;
        case 'r': o.p[o.pos++] = 13; break;  case 't': o.p[o.pos++] = 9; break;
        case 'u': {
            uint32_t cp = text_hex4(r, i); i += 4;
            if (cp >= 0xD800 && cp <= 0xDBFF && i + 6 <= hi && r.at(i) == '\\' && r.at(i + 1) == 'u') {
                const uint32_t lo2 = text_hex4(r, i + 2);
                if (lo2 >= 0xDC00 && lo2 <= 0xDFFF) { cp = 0x10000 + ((cp - 0xD800) << 10) + (lo2 - 0xDC00); i += 6; }
            }
            if (cp >= 0xD800 && cp <= 0xDFFF) o.flags |= TF_LONE_SURROGATE;
            text_put_cp(o, cp);
            break; }
        default: o.p[o.pos++] = (uint8_t)e; break;       // \" \\ \/
        }
    }
}

// One classified part [s, e) through the tap's per-part code (chat_logging.py:120-139).  Appends to `o`; returns true when the
// part makes the tap call write_log (a mark).  Content pieces never outgrow the event's own bytes; the text of an "error" event
// comes on top of them (an event can append up to twice its length), so the one-chunk-per-lane path, whose room is the chunk's own
// footprint, passes with_error_text = false and leaves such events to the sequential walk.
LGW_HD_NOINLINE bool text_part(const Rope& r, uint32_t s, uint32_t e, uint8_t cls, TextOut& o, bool with_error_text) {
    const uint32_t ev_pos = o.pos, ev_flags = o.flags;
    JsonMachine<false, true> m;
    m.reset(nullptr, cls == PC_DATA);
    const uint32_t t0 = s + (cls == PC_DATA ? 6u : 0u);
    for (uint32_t i = t0; i < e; ++i) {
        m.tpos = i;
        m.feed(r.at(i));
        if (m.failed()) break;
        if (m.rollback) { m.rollback = 0; o.pos = ev_pos; o.flags = ev_flags; }
        if (m.emit_pending) { m.emit_pending = 0; text_unescape(r, m.emit_lo, m.emit_hi, o); }
    }
    const uint32_t f = m.finish();
    if (!(f & PF_VALID_B)) { o.pos = ev_pos; o.flags = ev_flags; return false; }       // json5.loads raised: nothing was walked
    if (f & PF_EXOTIC) { o.flags |= TF_EXOTIC; return false; }
    if ((f & TK_CHOICES) && (f & PF_TYPE_ERROR)) return false;                          // :140-141, the pieces before the exception stay
    if (!(f & TK_ERROR)) return false;
    if (!with_error_text) return true;
    uint32_t te = e;                                                                    // :121 .strip() (the text starts with '{')
    if (cls == PC_DATA) while (te > t0 && JsonMachine<false>::is_py_ws(r.at(te - 1))) --te;
    for (uint32_t i = t0; i < te; ++i) o.p[o.pos++] = (uint8_t)r.at(i);               // :138 accum += decoded_chunk
    return true;
}

// The tap of a non-streaming response (chat_logging.py:97-150 with is_real_streaming=False): the joined chunks are ONE part
// (:105-106), walked by the per-part code above.  Appends the document's llm_response_accum to `o` (room: twice the document);
// returns true when the tap calls write_log at :139 as well as at :150.  Both calls write the same text.
LGW_HD bool doc_text(const Rope& r, uint32_t len, TextOut& o) {
    const uint8_t cls = classify_part(r, 0, len);                                       // :116-121
    if (cls == PC_NONE) return false;
    return text_part(r, 0, len, cls, o, true);
}

struct TextIO {
    TextTap* tap;              // local copy, written back by the caller
    uint8_t* carry; uint32_t carry_cap;
    TextMark* markq; uint32_t* markq_count; uint32_t markq_cap;
    uint32_t slot;
};

LGW_HD void text_push_mark(const TextIO& io, uint64_t pos) {
    TextTap& tp = *io.tap;
    ++tp.n_marks;
#if defined(__CUDA_ARCH__)
    const uint32_t k = atomicAdd(io.markq_count, 1u);
#else
    const uint32_t k = (*io.markq_count)++;
#endif
    if (k >= io.markq_cap) { tp.flags |= TF_MARKQ_OVERFLOW; return; }
    io.markq[k].slot = io.slot; io.markq[k].seq = tp.n_marks; io.markq[k].text_pos = pos;
}

// The relayed chunks [c_from, c_to) of one stream, sequentially, with the tap's carry.  Text goes to out[0 ..); returns its length.
LGW_HD uint32_t text_walk(const TextIO& io, const uint8_t* data, const uint32_t* chunk_off, uint32_t c_from, uint32_t c_to, uint8_t* out) {
    TextTap& tp = *io.tap;
    TextOut o{out, 0, 0};
    for (uint32_t c = c_from; c < c_to; ++c) {
        const uint32_t off = chunk_off[c], n = chunk_off[c + 1] - off;
        if (n == 0) continue;                                   // never yielded (request_handler.py:60-63)
        const uint8_t* p = data + off;
        if (!utf8_valid(p, n)) continue;                        // :142-143 (decode raised before the buffer changed)
        Rope r{io.carry, tp.carry_len, p, n};
        bool stopped;
        const uint32_t tail = split_scan(r, [&](uint32_t s, uint32_t e) {
            const uint8_t cls = classify_part(r, s, e);
            if (cls == PC_NONE) return true;
            if (text_part(r, s, e, cls, o, true)) text_push_mark(io, tp.text_total + o.pos);
            return true; }, stopped);
        if (!store_carry(io.carry, tp.carry_len, io.carry_cap, r, tail)) tp.flags |= TF_CARRY_OVERFLOW;
    }
    tp.flags |= o.flags;
    tp.text_total += o.pos;
    return o.pos;
}

// ---- kernels ----------------------------------------------------------------------------------------------------------
#if defined(__CUDACC__)
#define TX_GLOBAL __global__
#define TX_TID (threadIdx.x)
#define TX_BID (blockIdx.x)
#define TX_NTHR (blockDim.x)
#define TX_SHARED __shared__
#else
#define TX_GLOBAL static
#define TX_TID (simt::tid())
#define TX_BID (simt::bid())
#define TX_NTHR (simt::nthreads())
#define TX_SHARED static
#endif

#define TX_WARPS 8u
#define TX_FULL 0xFFFFFFFFu

struct TextArgs {
    const uint8_t* data; const uint32_t* chunk_off;
    const uint32_t* seg_chunk; const uint32_t* seg_slot; uint32_t n_segs;
    const SegResult* seg_res;          // the relay step's results: emit_chunk_begin
    TextTap* tap; uint8_t* carry; uint32_t carry_cap;      // [max_streams], [max_streams][carry_cap]
    uint8_t* sparse;                   // segment s writes from 2 * (s * carry_cap + chunk_off[seg_chunk[s]]); room: 2 * (carry_cap + segment bytes)
                                       //   (the sequential walk may append up to twice the bytes it reads: content pieces + "error" event texts)
    uint32_t* piece_len;               // [n_chunks] text bytes of the piece that starts at the chunk's footprint
    uint32_t* seg_len;                 // [n_segs]
    uint32_t* seg_flags;               // [n_segs] TextFlag bits of this step
    unsigned long long* seg_off;       // [n_segs + 1] filled by k_text_scan
    uint8_t* text;                     // compact text of the step
    TextMark* markq; uint32_t* markq_count; uint32_t markq_cap;
};

TX_GLOBAL void k_text_open(TextTap* tap, const uint32_t* slots, uint32_t n) {
    const uint32_t i = TX_BID * TX_NTHR + TX_TID;
    if (i >= n) return;
    TextTap z; z.carry_len = 0; z.flags = 0; z.n_marks = 0; z._pad = 0; z.text_total = 0;
    tap[slots[i]] = z;
}

#ifndef TX_BLOCKS                        /* resident 256-thread blocks per SM k_text_extract is compiled for (register budget 65536 / (256 * TX_BLOCKS)) */
#define TX_BLOCKS 4                     /* 64 registers: 32 warps per SM, the 4 096 warps of a C3 step are one wave (2.27 -> 2.03 ms; 3 -> 2.57, 5 -> 2.46, 6 -> 2.44) */
#endif
TX_GLOBAL void
#if defined(__CUDACC__)
__launch_bounds__(TX_WARPS * 32, TX_BLOCKS)
#endif
k_text_extract(TextArgs a) {
    const uint32_t seg = TX_BID * TX_WARPS + (TX_TID >> 5), lane = TX_TID & 31u;
    if (seg >= a.n_segs) return;
    const uint32_t slot = a.seg_slot[seg];
    const uint32_t c0 = a.seg_chunk[seg], c1 = a.seg_chunk[seg + 1];
    uint32_t cb = a.seg_res[seg].emit_chunk_begin;
    if (cb < c0) cb = c0;
    if (cb > c1) cb = c1;
    const uint32_t seg_byte0 = a.chunk_off[c0];
    uint8_t* const region = a.sparse + 2 * ((size_t)seg * a.carry_cap + seg_byte0);   // room: 2 * (carry_cap + the segment's bytes)
    TextTap tp = a.tap[slot];
    for (uint32_t c = c0 + lane; c < cb; c += 32) a.piece_len[c] = 0;             // dropped chunks: the tap never sees them
    // ---- regular attempt: one chunk per lane -------------------------------------------------------------------------------
    bool regular = tp.carry_len == 0;
    uint32_t total = 0, flags = 0;
    if (regular) {
        for (uint32_t base = cb; base < c1; base += 32) {
            const uint32_t c = base + lane;
            uint32_t len = 0; bool bad = false;
            if (c < c1) {
                const uint32_t off = a.chunk_off[c], n = a.chunk_off[c + 1] - off;
                if (n) {
                    const uint8_t* p = a.data + off;
                    if (n < 2 || p[n - 1] != '\n' || p[n - 2] != '\n' || !utf8_valid(p, n)) bad = true;
                    else {
                        Rope r{nullptr, 0, p, n};
                        TextOut o{region + 2 * (size_t)a.carry_cap + (off - seg_byte0), 0, 0};
                        bool stopped;
                        split_scan(r, [&](uint32_t s, uint32_t e) {
                            const uint8_t cls = classify_part(r, s, e);
                            if (cls == PC_NONE) return true;
                            if (text_part(r, s, e, cls, o, false)) { bad = true; return false; }   // a mark: position and room need the sequential walk
                            return true; }, stopped);
                        len = o.pos; flags |= o.flags;
                    }
                }
                a.piece_len[c] = len;
            }
            if (__any_sync(TX_FULL, bad)) { regular = false; break; }
            total += len;
        }
    }
    if (regular) {
        total = __reduce_add_sync(TX_FULL, total);
        flags = __reduce_or_sync(TX_FULL, flags);
        if (lane == 0) { tp.text_total += total; tp.flags |= flags; }
    } else {
        // ---- exact sequential walk by lane 0 (the regular attempt changed nothing but scratch) ------------------------------
        for (uint32_t c = cb + lane; c < c1; c += 32) a.piece_len[c] = 0;
        __syncwarp(TX_FULL);
        if (lane == 0) {
            const uint32_t before = tp.flags;
            TextIO io{&tp, a.carry + (size_t)slot * a.carry_cap, a.carry_cap, a.markq, a.markq_count, a.markq_cap, slot};
            total = text_walk(io, a.data, a.chunk_off, cb, c1, region);
            flags = (tp.flags & ~before) | TF_SEQUENTIAL;
            if (total) {
                // the piece starts at the segment's region, not at a chunk footprint: pack finds it through the first relayed chunk
                if (cb < c1) a.piece_len[cb] = total;
            }
        }
        total = __shfl_sync(TX_FULL, total, 0);
        flags = __shfl_sync(TX_FULL, flags, 0);
    }
    if (lane == 0) {
        a.tap[slot] = tp;
        a.seg_len[seg] = total;
        a.seg_flags[seg] = flags | (tp.flags & (TF_LONE_SURROGATE | TF_EXOTIC | TF_CARRY_OVERFLOW | TF_MARKQ_OVERFLOW));
    }
}

// exclusive scan of seg_len -> seg_off[0 .. n_segs] (one block of 1024 threads)
TX_GLOBAL void k_text_scan(const uint32_t* seg_len, uint32_t n_segs, unsigned long long* seg_off) {
    TX_SHARED WarpSums<unsigned long long> warp_sums;
    const unsigned long long total = block_scan(n_segs, TX_TID, TX_NTHR, warp_sums, [&](uint32_t i) { return seg_len[i]; },
                                                [&](uint32_t i, unsigned long long off) { seg_off[i] = off; });
    if (TX_TID == 0) seg_off[n_segs] = total;
}

// compaction: the pieces of segment s, in chunk order, to text[seg_off[s] ..)
TX_GLOBAL void k_text_pack(TextArgs a) {
    const uint32_t seg = TX_BID * TX_WARPS + (TX_TID >> 5), lane = TX_TID & 31u;
    if (seg >= a.n_segs) return;
    if (a.seg_len[seg] == 0) return;
    const uint32_t c0 = a.seg_chunk[seg], c1 = a.seg_chunk[seg + 1];
    uint32_t cb = a.seg_res[seg].emit_chunk_begin;
    if (cb < c0) cb = c0;
    if (cb > c1) cb = c1;
    const uint32_t seg_byte0 = a.chunk_off[c0];
    const uint8_t* const region = a.sparse + 2 * ((size_t)seg * a.carry_cap + seg_byte0);
    uint8_t* dst = a.text + a.seg_off[seg];
    if (a.seg_flags[seg] & TF_SEQUENTIAL) {                       // one piece at the start of the region
        const uint32_t n = a.seg_len[seg];
        for (uint32_t i = lane; i < n; i += 32) dst[i] = region[i];
        return;
    }
    uint32_t done = 0;
    for (uint32_t base = cb; base < c1; base += 32) {
        const uint32_t c = base + lane;
        const uint32_t len = c < c1 ? a.piece_len[c] : 0;
        uint32_t x = len;
        for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(TX_FULL, x, d); if (lane >= d) x += y; }
        if (len) {
            const uint8_t* src = region + 2 * (size_t)a.carry_cap + (a.chunk_off[c] - seg_byte0);
            uint8_t* q = dst + done + (x - len);
            for (uint32_t i = 0; i < len; ++i) q[i] = src[i];
        }
        done += __shfl_sync(TX_FULL, x, 31);
    }
}

}  // namespace lgw
