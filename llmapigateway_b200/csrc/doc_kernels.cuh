// Response tap of non-streaming responses (SURVEY.md row a8, non-stream mode): chat_logging.py:98-103 concatenates the
// chunks, :105-106 makes the whole text ONE part, :113-141 parses it once and reads usage / error like the streaming tap.
// One warp per document: the lanes stage the text in shared memory, one lane runs the full machine (json_machine.cuh) over
// it -- the same machine and the same tap rules (tap_part, stream_machine.cuh) as the streaming path, so the two modes cannot
// drift apart.  Documents longer than the stage are read from global memory.
// k_docs_text reads out the text the same tap accumulates (transcript.cuh doc_text) for the log files of chat transcripts.
#pragma once
#include <cuda_runtime.h>
#include "stream_machine.cuh"
#include "error_detail.cuh"
#include "transcript.cuh"

namespace lgw {

struct DocUsage {
    uint32_t flags;
    uint8_t rec_valid, error_row, exotic, _pad;
    UsageRec rec;
};

#define LGW_DOC_WARPS 4
#define LGW_DOC_STAGE 6144u

__global__ void __launch_bounds__(LGW_DOC_WARPS * 32) k_docs_usage(const uint8_t* __restrict__ docs, const uint64_t* __restrict__ off, uint32_t n, DocUsage* __restrict__ out) {
    __shared__ __align__(16) uint8_t stage[LGW_DOC_WARPS][LGW_DOC_STAGE];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (uint32_t i = blockIdx.x * LGW_DOC_WARPS + warp; i < n; i += gridDim.x * LGW_DOC_WARPS) {
        const uint8_t* src = docs + off[i];
        const uint64_t len64 = off[i + 1] - off[i];
        const uint32_t len = len64 > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)len64;
        const bool staged = len <= LGW_DOC_STAGE;
        if (staged) for (uint32_t k = lane; k < len; k += 32) stage[warp][k] = src[k];
        __syncwarp();
        if (lane == 0) {
            DocUsage* o = out + i;
            o->flags = 0; o->rec_valid = 0; o->error_row = 0; o->exotic = 0; o->_pad = 0;
            default_usage(o->rec);
            Rope r{nullptr, 0, staged ? stage[warp] : src, len};
            const uint8_t cls = classify_part(r, 0, len);                       // chat_logging.py:116-121
            if (cls != PC_NONE) {
                UsageRaw raw;
                const uint32_t f = parse_part<true>(r, 0, len, cls, &raw);      // :123
                o->flags = f;
                if ((f & PF_VALID_B) && (f & (TK_USAGE | TK_ERROR))) {
                    if (f & PF_EXOTIC) o->exotic = 1;
                    else if (!((f & TK_CHOICES) && (f & PF_TYPE_ERROR))) {      // (a TypeError in the choices walk skips the rest of the part, :140-141)
                        if (f & TK_USAGE) { normalise_usage(raw, f, o->rec); o->rec_valid = 1; if (o->rec.exotic) o->exotic = 1; }   // :134-135
                        if (f & TK_ERROR) o->error_row = 1;                     // :137-139
                    }
                }
            }
        }
        __syncwarp();
    }
}

// error detail of failing non-streaming responses (request_handler.py:167-169): one warp per document stages it, lane 0 walks it
// (error_detail.cuh); documents longer than the stage are walked in global memory.  Failing responses are the rare case.
__global__ void __launch_bounds__(LGW_DOC_WARPS * 32) k_docs_error_detail(const uint8_t* __restrict__ docs, const uint64_t* __restrict__ off, uint32_t n, DocError* __restrict__ out,
                                                                          uint8_t* __restrict__ text, uint32_t text_stride) {
    __shared__ __align__(16) uint8_t stage[LGW_DOC_WARPS][LGW_DOC_STAGE];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    for (uint32_t i = blockIdx.x * LGW_DOC_WARPS + warp; i < n; i += gridDim.x * LGW_DOC_WARPS) {
        const uint8_t* src = docs + off[i];
        const uint64_t len64 = off[i + 1] - off[i];
        const uint32_t len = len64 > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)len64;
        const bool staged = len <= LGW_DOC_STAGE;
        if (staged) for (uint32_t k = lane; k < len; k += 32) stage[warp][k] = src[k];
        __syncwarp();
        if (lane == 0) error_detail_of(staged ? stage[warp] : src, len, out[i], text + (size_t)i * text_stride, text_stride);
        __syncwarp();
    }
}

// text the tap accumulates for each non-streaming response (chat_logging.py:124-139, transcript.cuh doc_text), in k_docs_usage's
// geometry.  Document i writes its text to the sparse buffer at 2 * (off[i] - off[0]) (room: twice its length), its length to len[i]
// and its TextFlag bits to flags[i].  k_text_scan turns the lengths into offsets and k_docs_text_pack packs the pieces.
__global__ void __launch_bounds__(LGW_DOC_WARPS * 32) k_docs_text(const uint8_t* __restrict__ docs, const uint64_t* __restrict__ off, uint32_t n,
                                                                  uint8_t* __restrict__ sparse, uint32_t* __restrict__ len_out, uint32_t* __restrict__ flags_out) {
    __shared__ __align__(16) uint8_t stage[LGW_DOC_WARPS][LGW_DOC_STAGE];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t base = off[0];
    for (uint32_t i = blockIdx.x * LGW_DOC_WARPS + warp; i < n; i += gridDim.x * LGW_DOC_WARPS) {
        const uint8_t* src = docs + off[i];
        const uint32_t len = (uint32_t)(off[i + 1] - off[i]);              // (the engine limits documents to 2^31 bytes: 2 * len fits)
        const bool staged = len <= LGW_DOC_STAGE;
        if (staged) for (uint32_t k = lane; k < len; k += 32) stage[warp][k] = src[k];
        __syncwarp();
        if (lane == 0) {
            Rope r{nullptr, 0, staged ? stage[warp] : src, len};
            TextOut o{sparse + 2 * (off[i] - base), 0, 0};
            const bool logged = doc_text(r, len, o);
            len_out[i] = o.pos;
            flags_out[i] = o.flags | (logged ? (uint32_t)TF_DOC_ERROR_LOG : 0u);
        }
        __syncwarp();
    }
}

// the pieces of k_docs_text, document after document: text[text_off[i] ..) = sparse[2 * (off[i] - off[0]) ..), one warp per document
__global__ void __launch_bounds__(LGW_DOC_WARPS * 32) k_docs_text_pack(const uint64_t* __restrict__ off, uint32_t n, const uint8_t* __restrict__ sparse,
                                                                       const uint32_t* __restrict__ len, const unsigned long long* __restrict__ text_off,
                                                                       uint8_t* __restrict__ text) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint64_t base = off[0];
    for (uint32_t i = blockIdx.x * LGW_DOC_WARPS + warp; i < n; i += gridDim.x * LGW_DOC_WARPS) {
        const uint8_t* src = sparse + 2 * (off[i] - base);
        uint8_t* dst = text + text_off[i];
        const uint32_t m = len[i];
        for (uint32_t k = lane; k < m; k += 32) dst[k] = src[k];
    }
}

}  // namespace lgw
