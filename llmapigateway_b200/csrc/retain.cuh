// Deleting old usage records on the device: `DELETE FROM tokens_usage WHERE timestamp < ?` of
// llm_gateway_core/db/tokens_usage_db.py:164-198 (cleanup_old_records) over the usage table's device-resident columns.
//
// A record survives when ts_us >= cutoff_us.  The survivors of all eight columns (UsageTable.COLS) are written, in index order,
// into fresh columns: a stable compaction with the listing's tile pattern (csrc/listing.cuh).
//  1. k_retain_count: survivors of each tile of LGW_LIST_CTILE records, from one 16-byte timestamp load per thread.
//  2. k_list_scan (listing.cuh): exclusive scan of the tile counts; its total is the number of survivors.
//  3. k_retain_write: each survivor's place from the tile offset, the warps before it and a ballot / popcount inside its warp.
//     It reads the other seven columns of survivors only, and stores only places below n_keep (the survivor count the caller
//     computed from its own copy of the timestamps): a device count that differs is caught by the host's check of the total,
//     never by writing past the output.
// Out of place on purpose: compacting in place would let block k overwrite input that block j < k has not read yet.
// HBM bytes: 16 per record (the timestamps, read by both kernels) + 72 per survivor (32 read: the other seven columns; 40 written).
#pragma once
#include <stdint.h>

#include "listing.cuh"

namespace lgw {

#if defined(__CUDACC__)
// the eight columns in UsageTable.COLS order: ts_us, model_rank, prompt, completion, total, reasoning, cached (int32), cost
struct RetainCols {
    int64_t* ts;
    int32_t* i32[6];
    double* cost;
};

// survivors of each compaction tile
__global__ void __launch_bounds__(1024) k_retain_count(const int64_t* __restrict__ ts, uint32_t n, int64_t cutoff, uint32_t* __restrict__ tile_count) {
    __shared__ uint32_t warp_sums[32];
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    int64_t a, b;
    list_load_pair(ts, n, j, a, b);
    const uint32_t c = (2 * j < n && a >= cutoff) + (2 * j + 1 < n && b >= cutoff);
    const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, c);
    if ((threadIdx.x & 31u) == 0) warp_sums[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x < 32) {
        const uint32_t t = __reduce_add_sync(0xFFFFFFFFu, threadIdx.x < (blockDim.x >> 5) ? warp_sums[threadIdx.x] : 0u);
        if (threadIdx.x == 0) tile_count[blockIdx.x] = t;
    }
}

__device__ __forceinline__ void retain_copy(const RetainCols& in, const RetainCols& out, uint32_t from, uint32_t to, int64_t ts) {
    out.ts[to] = ts;
#pragma unroll
    for (int c = 0; c < 6; ++c) out.i32[c][to] = __ldg(in.i32[c] + from);
    out.cost[to] = __ldg(in.cost + from);
}

// the survivors at the tile offsets k_list_scan made; places at or past n_keep are not stored
__global__ void __launch_bounds__(1024) k_retain_write(const RetainCols in, uint32_t n, int64_t cutoff, const uint32_t* __restrict__ tile_off,
                                                       uint32_t n_keep, const RetainCols out) {
    __shared__ uint32_t warp_sums[32];
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
    int64_t a, b;
    list_load_pair(in.ts, n, j, a, b);
    const bool ka = 2 * j < n && a >= cutoff, kb = 2 * j + 1 < n && b >= cutoff;
    const uint32_t ma = __ballot_sync(0xFFFFFFFFu, ka), mb = __ballot_sync(0xFFFFFFFFu, kb);
    if (lane == 0) warp_sums[warp] = __popc(ma) + __popc(mb);
    __syncthreads();
    uint32_t pos = tile_off[blockIdx.x] + __popc(ma & lt) + __popc(mb & lt);
    for (uint32_t w = 0; w < warp; ++w) pos += warp_sums[w];
    if (ka) { if (pos < n_keep) retain_copy(in, out, 2 * j, pos, a); ++pos; }
    if (kb && pos < n_keep) retain_copy(in, out, 2 * j + 1, pos, b);
}
#endif

}  // namespace lgw
