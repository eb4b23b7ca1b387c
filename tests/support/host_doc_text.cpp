// TEST AID ONLY: the per-document walk of k_docs_text (transcript.cuh doc_text) built with g++, so that the CPU test-suite runs
// the very code the kernel runs for one document.  transcript.cuh also holds the transcript kernels, which build for the host
// over the SIMT emulator (simt_emu.h), as in host_relay2.cpp.  Never linked into the product library; the product has no CPU path.
#include <stddef.h>
#include <stdint.h>

#include "simt_emu.h"
#include "../../include/llmgw_b200.h"
#include "../../llmapigateway_b200/csrc/transcript.cuh"

using namespace lgw;

// what lane 0 of k_docs_text does for one document: its text into `text` (room: 2 * len bytes), its length into *text_len;
// returns the TextFlag bits k_docs_text stores (TF_DOC_ERROR_LOG when write_log also runs at chat_logging.py:139)
extern "C" uint32_t lgwt_doc_text(const uint8_t* doc, uint32_t len, uint8_t* text, uint32_t* text_len) {
    Rope r{nullptr, 0, doc, len};
    TextOut o{text, 0, 0};
    const bool logged = doc_text(r, len, o);
    *text_len = o.pos;
    return o.flags | (logged ? (uint32_t)TF_DOC_ERROR_LOG : 0u);
}
