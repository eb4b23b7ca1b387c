// Block-wide exclusive scan, sum and ordered placement: the one implementation behind the engine's offsets (k_list_scan,
// k_rollup_scan, k_text_scan, k_body_offsets, k_lsd_scatter's digit totals) and its stable compactions (k_list_tile_count /
// k_list_tile_write, k_retain_count / k_retain_write, k_rollup_write).  An offset is the sum of the entries before it; a place is
// the kept items before it in thread order.
//
// Host/device portable: the CPU tests compile k_text_scan with g++ over the SIMT emulator (tests/support/simt_emu.h, included
// first), so the thread index, the block size and the shared warp-sums array are arguments.  Every thread of the block calls
// each helper; the block is a multiple of 32 threads, at most 1024.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define LGW_SCAN __device__ __forceinline__
#else
#define LGW_SCAN static inline
#endif

namespace lgw {

template <class Acc> using WarpSums = Acc[32];    // one entry per warp of a block: declare __shared__ and pass to the helpers

// x's exclusive offset within the block (thread order); block_total gets the sum over the block.  Other threads may still be
// reading warp_sums when this returns: a caller that uses it again passes a __syncthreads() first.
template <class Acc>
LGW_SCAN Acc block_exclusive_scan(Acc x, uint32_t tid, uint32_t nthr, Acc* warp_sums, Acc& block_total) {
    const uint32_t lane = tid & 31u, warp = tid >> 5;
    Acc s = x;                                                        // inclusive within the warp
    for (uint32_t d = 1; d < 32; d <<= 1) { const Acc y = __shfl_up_sync(0xFFFFFFFFu, s, d); if (lane >= d) s += y; }
    if (lane == 31) warp_sums[warp] = s;
    __syncthreads();
    if (warp == 0) {                                                  // inclusive scan of the warp sums, in place
        Acc w = lane < (nthr >> 5) ? warp_sums[lane] : (Acc)0;
        for (uint32_t d = 1; d < 32; d <<= 1) { const Acc y = __shfl_up_sync(0xFFFFFFFFu, w, d); if (lane >= d) w += y; }
        warp_sums[lane] = w;
    }
    __syncthreads();
    block_total = warp_sums[(nthr >> 5) - 1];
    return (warp ? warp_sums[warp - 1] : (Acc)0) + s - x;
}

// exclusive scan of `len` entries in rounds of nthr, the sum of the rounds before carried: entry k is load(k), its offset goes to
// store(k, offset).  Returns the total.
template <class Acc, class Load, class Store>
LGW_SCAN Acc block_scan(uint32_t len, uint32_t tid, uint32_t nthr, Acc* warp_sums, Load load, Store store) {
    Acc carry = 0;
    for (uint32_t start = 0; start < len; start += nthr) {
        const uint32_t k = start + tid;
        Acc all;
        const Acc off = block_exclusive_scan<Acc>(k < len ? (Acc)load(k) : (Acc)0, tid, nthr, warp_sums, all);
        if (k < len) store(k, carry + off);
        carry += all;
        __syncthreads();
    }
    return carry;
}

// the sum of x over the block, in thread 0 (a tile's count, where no thread needs its offset)
LGW_SCAN uint32_t block_sum(uint32_t x, uint32_t tid, uint32_t nthr, uint32_t* warp_sums) {
    const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, x);
    if ((tid & 31u) == 0) warp_sums[tid >> 5] = w;
    __syncthreads();
    return tid < 32 ? __reduce_add_sync(0xFFFFFFFFu, tid < (nthr >> 5) ? warp_sums[tid] : 0u) : 0u;
}

// a thread's first place within its tile when each thread keeps up to two items (keep_a before keep_b): the kept items of the
// warps before it and of the lanes before it.  One item per thread: keep_b = false.
LGW_SCAN uint32_t warp_place(bool keep_a, bool keep_b, uint32_t tid, uint32_t* warp_sums) {
    const uint32_t lane = tid & 31u, warp = tid >> 5, lt = (1u << lane) - 1u;
    const uint32_t ma = __ballot_sync(0xFFFFFFFFu, keep_a), mb = __ballot_sync(0xFFFFFFFFu, keep_b);
    if (lane == 0) warp_sums[warp] = __popc(ma) + __popc(mb);
    __syncthreads();
    uint32_t pos = __popc(ma & lt) + __popc(mb & lt);
    for (uint32_t w = 0; w < warp; ++w) pos += warp_sums[w];
    return pos;
}

}  // namespace lgw
