// Appending inserted usage records to the device-resident columns: `INSERT INTO tokens_usage` of
// llm_gateway_core/db/tokens_usage_db.py:119-162 (insert_usage), applied to the usage table's device copy at query time.
//
// One launch, k_usage_append, over two ranges of work items:
//  * [0, old): the n resident records, visited only when the call grows the columns (a copy of all eight fields into the
//    fresh columns) or remaps the model ranks (a new model name shifted the byte order of the names): the record's model_rank
//    r becomes map[r].  A rank at or past n_map is counted in *bad and left as it was; the host fails the call on a count > 0.
//  * [old, old + m): the m new records, read from the staging the host copied up in one transfer and written at n + j.
// old is n when growing or remapping, 0 otherwise.  Nothing is written outside [0, n + m) of the target columns.
// HBM bytes: 80 per new record (40 read from the staging, 40 written), + 8 per resident record for an in-place remap (its
// rank read and written), or + 80 for a growth copy (40 read, 40 written).
#pragma once
#include <stdint.h>

#include "retain.cuh"

namespace lgw {

#if defined(__CUDACC__)
struct AppendArgs {
    RetainCols src, dst;            // the resident columns; the target columns (src itself, or fresh ones with room for n + m)
    const int64_t* new_ts;          // staging: m timestamps, m costs, then the six int32 columns one after another
    const double* new_cost;
    const int32_t* new_i32;
    const int32_t* map;             // old rank -> new rank (n_map entries), or null
    uint32_t n_map, n, m, old;
    uint32_t* bad;                  // resident ranks at or past n_map
};

__global__ void __launch_bounds__(256) k_usage_append(const AppendArgs a) {
    const uint64_t total = (uint64_t)a.old + a.m, stride = (uint64_t)gridDim.x * blockDim.x;
    const bool grow = a.dst.ts != a.src.ts;
    uint32_t bad = 0;
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += stride) {
        const uint32_t i = (uint32_t)k;
        if (i < a.old) {
            int32_t r = a.src.i32[0][i];
            if (a.map) {
                if ((uint32_t)r < a.n_map) r = __ldg(a.map + r);
                else ++bad;
            }
            if (grow) {
                a.dst.ts[i] = __ldg(a.src.ts + i);
#pragma unroll
                for (int c = 1; c < 6; ++c) a.dst.i32[c][i] = __ldg(a.src.i32[c] + i);
                a.dst.cost[i] = __ldg(a.src.cost + i);
            }
            a.dst.i32[0][i] = r;
        } else {
            const uint32_t j = i - a.old, to = a.n + j;
            a.dst.ts[to] = __ldg(a.new_ts + j);
#pragma unroll
            for (int c = 0; c < 6; ++c) a.dst.i32[c][to] = __ldg(a.new_i32 + (size_t)c * a.m + j);
            a.dst.cost[to] = __ldg(a.new_cost + j);
        }
    }
    bad = __reduce_add_sync(0xFFFFFFFFu, bad);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(a.bad, bad);
}
#endif

}  // namespace lgw
