// Kernels for the request-body rewrite (SURVEY.md rows a1, a3, a4; config 2: 1024 bodies x 4 KiB).
//
//   k_body_rewrite  one warp per body.  Every lane runs the rendering machine of body_machine.cuh on
//                   the same bytes (no divergence, state in registers/local memory); string content --
//                   the bulk of a chat body -- moves 32 bytes per ballot (plain_run/copy_run), every
//                   other token goes through feed().  Output -> a fixed-stride slot, length + status.
//   k_body_offsets  exclusive prefix sum of the OK lengths -> packed offsets.
//   k_body_pack     slot -> packed output, one block per body, coalesced.
//   k_body_scan     chat.py:31-45 (validity, model text, stream flag), one warp per body.
//
// Algorithmic bytes per body: in + out (+ slot write and re-read by the pack pass).
#pragma once
#include <cuda_runtime.h>
#include "body_machine.cuh"
#include "body_fast.cuh"
#include "scan.cuh"

namespace lgw {

struct BodyPlan { uint32_t op_begin, op_end, mode, _pad; };
struct BodyResult { uint32_t status, out_len, matched, root_kind; };

#define LGW_BODY_WARPS 4

// ASCII-only bodies skip the sequential UTF-8 walk: 16 bytes per lane per round
__device__ __forceinline__ bool body_all_ascii(const uint8_t* in, uint32_t n) {
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t acc = 0;
    for (uint32_t i = lane; i < n; i += 32) acc |= in[i];
    return !__any_sync(0xffffffffu, (acc & 0x80u) != 0);
}

// data-parallel path: one block per body; bodies it calls irregular are queued for the exact machine
__global__ void __launch_bounds__(LGW_FAST_THREADS)
k_body_fast(const uint8_t* __restrict__ bodies, const uint64_t* __restrict__ body_off, uint32_t n,
            const uint32_t* __restrict__ plan_idx, const BodyPlan* __restrict__ plans, uint32_t n_plans,
            const BodyOp* __restrict__ ops, const uint8_t* __restrict__ blob,
            uint8_t* __restrict__ slots, uint32_t slot_cap, BodyResult* __restrict__ results,
            uint32_t* __restrict__ redo_count, uint32_t* __restrict__ redo_list) {
    __shared__ FastShared sh;
    const uint32_t b = blockIdx.x;
    if (b >= n) return;
    const uint8_t* in = bodies + body_off[b];
    const uint32_t len = (uint32_t)(body_off[b + 1] - body_off[b]);
    const uint32_t pi = plan_idx[b];
    if (pi >= n_plans) { if (threadIdx.x == 0) results[b] = BodyResult{BS_EXOTIC, 0, 0, 0}; return; }
    const BodyPlan pl = plans[pi];
    uint32_t out_len = 0, matched = 0;
    const uint32_t st = fast_rewrite(&sh, in, len, (int)pl.mode, ops + pl.op_begin, pl.op_end - pl.op_begin, blob,
                                     slots + (size_t)b * slot_cap, slot_cap, &out_len, &matched);
    if (threadIdx.x == 0) {
        if (st == LGW_FAST_IRREGULAR) redo_list[atomicAdd(redo_count, 1u)] = b;
        else results[b] = BodyResult{st, out_len, matched, KD_OBJ};       // the data-parallel path only accepts object roots
    }
}

// the exact sequential machine, one warp per queued body (every lane runs it redundantly; lane 0 writes)
__global__ void __launch_bounds__(32 * LGW_BODY_WARPS)
k_body_rewrite(const uint8_t* __restrict__ bodies, const uint64_t* __restrict__ body_off, uint32_t n,
               const uint32_t* __restrict__ plan_idx, const BodyPlan* __restrict__ plans, uint32_t n_plans,
               const BodyOp* __restrict__ ops, const uint8_t* __restrict__ blob,
               uint8_t* __restrict__ slots, uint32_t slot_cap, BodyResult* __restrict__ results,
               const uint32_t* __restrict__ redo_count, const uint32_t* __restrict__ redo_list) {
    const uint32_t todo = redo_list ? *redo_count : n;
    for (uint32_t w = blockIdx.x * LGW_BODY_WARPS + (threadIdx.x >> 5); w < todo; w += gridDim.x * LGW_BODY_WARPS) {
        const uint32_t b = redo_list ? redo_list[w] : w;
        const uint8_t* in = bodies + body_off[b];
        const uint32_t len = (uint32_t)(body_off[b + 1] - body_off[b]);
        const uint32_t pi = plan_idx[b];
        BodyResult res{BS_EXOTIC, 0, 0, 0};
        if (pi < n_plans) {
            const BodyPlan pl = plans[pi];
            BodyRewriter m;
            uint32_t out_len = 0;
            m.reset((int)pl.mode, ops + pl.op_begin, pl.op_end - pl.op_begin, blob, slots + (size_t)b * slot_cap, slot_cap);
            res.status = rewrite_body_checked(m, in, len, body_all_ascii(in, len), &out_len);
            res.out_len = out_len;
            res.matched = m.matched;
            res.root_kind = m.root_kind;
        }
        if ((threadIdx.x & 31u) == 0) results[b] = res;
    }
}

// exclusive scan over the OK lengths; one block, n is small (thousands) compared with the bodies
__global__ void __launch_bounds__(1024)
k_body_offsets(const BodyResult* __restrict__ results, uint32_t n, uint64_t out_cap, uint64_t* __restrict__ out_off) {
    __shared__ WarpSums<uint64_t> warp_sums;
    const uint64_t total = block_scan(n, threadIdx.x, blockDim.x, warp_sums,
                                      [&](uint32_t i) { const BodyResult r = results[i]; return r.status == BS_OK ? r.out_len : 0u; },
                                      [&](uint32_t i, uint64_t off) { out_off[i] = off; });
    if (threadIdx.x == 0) out_off[n] = total;
}

__global__ void __launch_bounds__(256)
k_body_pack(const uint8_t* __restrict__ slots, uint32_t slot_cap, BodyResult* __restrict__ results, uint32_t n,
            const uint64_t* __restrict__ out_off, uint8_t* __restrict__ out, uint64_t out_cap) {
    for (uint32_t b = blockIdx.x; b < n; b += gridDim.x) {
        const BodyResult r = results[b];
        if (r.status != BS_OK) continue;
        const uint64_t o = out_off[b];
        if (o + r.out_len > out_cap) { if (threadIdx.x == 0) results[b].status = BS_OVERFLOW; continue; }
        const uint8_t* src = slots + (size_t)b * slot_cap;
        uint8_t* dst = out + o;
        // align the destination to 16 B, then move 16 B per thread (source re-aligned with byte_perm funnel is not worth it: slots are L2-resident)
        const uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
        const uint32_t h = head < r.out_len ? head : r.out_len;
        if (threadIdx.x < h) dst[threadIdx.x] = src[threadIdx.x];
        const uint32_t body = (r.out_len - h) & ~15u;
        for (uint32_t j = threadIdx.x * 16; j < body; j += 256 * 16) {
            const uint8_t* s = src + h + j;
            uint4 v;
            if ((((uintptr_t)s) & 3) == 0) {
                const uint32_t* s4 = (const uint32_t*)s;
                v.x = s4[0]; v.y = s4[1]; v.z = s4[2]; v.w = s4[3];
            } else {
                uint32_t w[4];
                #pragma unroll
                for (int k = 0; k < 4; ++k) w[k] = (uint32_t)s[4 * k] | ((uint32_t)s[4 * k + 1] << 8) | ((uint32_t)s[4 * k + 2] << 16) | ((uint32_t)s[4 * k + 3] << 24);
                v.x = w[0]; v.y = w[1]; v.z = w[2]; v.w = w[3];
            }
            *(uint4*)(dst + h + j) = v;
        }
        for (uint32_t j = h + body + threadIdx.x; j < r.out_len; j += 256) dst[j] = src[j];
    }
}

__global__ void __launch_bounds__(32 * LGW_BODY_WARPS)
k_body_scan(const uint8_t* __restrict__ bodies, const uint64_t* __restrict__ body_off, uint32_t n,
            uint32_t model_cap, BodyScan* __restrict__ scans, uint8_t* __restrict__ models) {
    const uint32_t b = blockIdx.x * LGW_BODY_WARPS + (threadIdx.x >> 5);
    if (b >= n) return;
    const uint8_t* in = bodies + body_off[b];
    const uint32_t len = (uint32_t)(body_off[b + 1] - body_off[b]);
    BodyRewriter m;
    BodyScan sc;
    scan_body(m, in, len, &sc, models + (size_t)b * model_cap, model_cap);     // lanes write identical bytes
    if ((threadIdx.x & 31u) == 0) scans[b] = sc;
}

}  // namespace lgw
