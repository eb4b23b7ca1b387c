// Kernels of the SSE step (sm_90a).  See DESIGN.md for the data layout and the roofline of each.
//
// A launch set of the bulk path is two kernels, k_relay2 then k_commit2.  Neither needs a planning pass before it: each
// segment's static plan (seg_static: its bulk region, and whether a fresh stream is speculated to commit on its first
// non-empty chunk) is computed where it is used, and the bulk kernel's findings start at zero.
//   k_relay2   bulk kernel (relay2.cuh): one persistent block per SM, every warp owns a byte range and finds its first segment
//              itself (a 32-lane search over the segment table); the re-emit is a
//              TMA pipeline through shared memory (cp.async.bulk in, cp.async.bulk out), the parse compares the
//              staged bytes against periodic event templates, 16 bytes per lane, and reads the usage fields of
//              template-following usage events straight from the matched value spans.
//   k_commit2  one warp per segment: folds the bulk kernel's findings into the persistent stream state and zeroes them;
//              streams the bulk kernel flagged irregular (or whose speculation failed) are redone sequentially with the
//              exact machine.  Its block 0 decays the template cache's hit counts for the next launch set.
//   k_general  (mode 1 / fix-up) the exact sequential machine over whole segments.
#pragma once
#include <cuda_runtime.h>
#include "stream_machine.cuh"
#include "lean_json.cuh"
#include "step_types.cuh"

namespace lgw {

// ---- stream table maintenance -------------------------------------------------------------------
__global__ void k_streams_open(DeviceTables t, const uint32_t* slots, const int32_t* status, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    init_stream(t.state[slots[i]], status[i]);
}

__global__ void k_streams_gather(DeviceTables t, const uint32_t* slots, uint32_t n, StreamState* out, int free_after) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t slot = slots[i];
    StreamState* s = t.state + slot;
    if (s->h.flags & SF_PENDING) {            // extract the stashed usage event now (deferred by the bulk path)
        StreamHdr st = s->h;
        StepIO io;
        io.st = &st; io.rec = &s->rec; io.pending = t.pending + (size_t)slot * LGW_PENDING_STRIDE;
        io.carry_a = io.carry_b = io.detail = nullptr; io.carry_cap = io.detail_cap = 0;
        io.rowq = nullptr; io.rowq_count = nullptr; io.rowq_cap = 0; io.slot = slot;
        resolve_pending(io);
        s->h = st;
    }
    out[i] = *s;
    if (free_after) s->h.phase = PH_FREE;
}

// ---- exact sequential path ------------------------------------------------------------------------
__global__ void __launch_bounds__(64) k_general(StepArgs a) {
    const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= a.n_segs) return;
    const uint32_t slot = a.seg_slot[seg];
    StreamHdr st = a.t.state[slot].h;
    const StepIO io = make_io(a, slot, &st);
    SegResult res;
    run_segment(io, a.data, a.chunk_off, a.seg_chunk[seg], a.seg_chunk[seg + 1], res);
    a.t.state[slot].h = st;
    a.seg_out[seg] = res;
}

// ---- plain re-emit (used with k_general): out[i] = in[i], 16 bytes per thread per trip ---------------
__global__ void __launch_bounds__(256) k_copy(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, uint32_t n) {
    const uint32_t nvec = n >> 4;
    const uint4* __restrict__ vi = reinterpret_cast<const uint4*>(in);
    uint4* __restrict__ vo = reinterpret_cast<uint4*>(out);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) vo[i] = __ldg(vi + i);
    const uint32_t tail = nvec << 4;
    if (blockIdx.x == 0 && threadIdx.x < (n - tail)) out[tail + threadIdx.x] = in[tail + threadIdx.x];
}

#include "relay2.cuh"

// The step's scratch.  alloc(pointer, bytes) -> cudaError_t is the caller's allocator: the memory is the caller's to release.
template <class Alloc>
static inline cudaError_t scratch_alloc(StepScratch& s, size_t max_streams, Alloc alloc) {
    cudaError_t r;
    if ((r = alloc(s.plan, max_streams * sizeof(SegPlan))) != cudaSuccess) return r;
    if ((r = cudaMemset(s.plan, 0, max_streams * sizeof(SegPlan))) != cudaSuccess) return r;     // (k_commit2 keeps it zero)
    if ((r = alloc(s.tpl_cache2, sizeof(TemplateCache2))) != cudaSuccess) return r;
    if ((r = cudaMemset(s.tpl_cache2, 0, sizeof(TemplateCache2))) != cudaSuccess) return r;
    if ((r = alloc(s.usage_fields, max_streams * 9 * sizeof(uint2))) != cudaSuccess) return r;
    if ((r = alloc(s.counters, 64)) != cudaSuccess) return r;
    if ((r = cudaMemset(s.counters, 0, 64)) != cudaSuccess) return r;
    if ((r = cudaFuncSetAttribute(k_relay2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)R2_SMEM_BYTES)) != cudaSuccess) return r;
    return cudaSuccess;
}

// Launch one step on `stream`.  ev[0..3] bracket prime (nothing: ev[1] = ev[0]) / relay / commit (ev[4] = ev[3]: usage extraction is
// inside relay and commit).
static inline cudaError_t launch_step(const StepArgs& a, int mode, int sm_count, cudaStream_t stream, cudaEvent_t* ev, int* launched, bool per_kernel) {
    *launched = 0;
    cudaError_t r;
    if ((r = cudaEventRecord(ev[0], stream)) != cudaSuccess) return r;
    if (mode == 1) {
        if ((r = cudaEventRecord(ev[1], stream)) != cudaSuccess) return r;
        if (a.n_bytes) { k_copy<<<sm_count * 8, 256, 0, stream>>>(a.data, a.out, a.n_bytes); ++*launched; }
        if ((r = cudaEventRecord(ev[2], stream)) != cudaSuccess) return r;
        if (a.n_segs) { k_general<<<(a.n_segs + 63) / 64, 64, 0, stream>>>(a); ++*launched; }
        if ((r = cudaEventRecord(ev[3], stream)) != cudaSuccess) return r;
        if ((r = cudaEventRecord(ev[4], stream)) != cudaSuccess) return r;
        return cudaGetLastError();
    }
    return launch_step_fast(a, sm_count, stream, ev, launched, per_kernel);
}

}  // namespace lgw
