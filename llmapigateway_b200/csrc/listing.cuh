// Newest-first record listing (/v1/api/usage-records): `ORDER BY timestamp DESC LIMIT ? OFFSET ?` of
// llm_gateway_core/db/tokens_usage_db.py:69-117 over the device-resident timestamp column of the usage table.
//
// Order: (ts_us DESC, record index ASC) -- equal timestamps in insertion order, as UsageTable's host path lists them.
// As an ascending unsigned key that is (kd, index) with kd = ts ^ 0x7FFF'FFFF'FFFF'FFFF: 96 bits, unique per record.
//
//  1. Radix select of the two boundary keys, at ranks `first` and `last = first + count - 1`, in the same passes: 12 passes of
//     one 8-bit digit each, most significant first (8 of kd, 4 of the index).  A pass histograms the digit of the elements
//     still under each boundary's prefix (k_list_hist, 16-byte loads, block-private shared histograms), and k_list_pick
//     fixes the digit whose cumulative count covers the rank.  Once the elements under the two prefixes are at most
//     n / LGW_LIST_CAND_DIV, k_list_cand copies them to scratch as (kd, index) pairs and the later passes read only those.
//  2. Ordered compaction (k_list_tile_count, k_list_scan, k_list_tile_write) of the keys between the two boundaries: exactly
//     `count` pairs, in index order.
//  3. Page sort: up to LGW_LIST_SMEM_SORT pairs in one block (bitonic in shared memory, k_list_sort_small); larger pages
//     (a full listing too) with a stable LSD radix sort of kd, 8 passes of k_lsd_hist / k_list_scan / k_lsd_scatter.
//     The pairs come in index order, so stability leaves equal timestamps in index order.
#pragma once
#include <stdint.h>

namespace lgw {

#define LGW_LIST_CAND_DIV 16u        /* compact the candidates once they are at most n / 16 */
#define LGW_LIST_SMEM_SORT 8192u     /* pages up to this many records sort in one block: 8192 x 12 B = 96 KiB of shared memory */
#define LGW_LIST_DIGITS 12           /* 8-bit digits of the 96-bit key */
#define LGW_LIST_CTILE 2048u         /* compaction tile: 1024 threads x one 16-byte load */
#define LGW_LIST_STILE 4096u         /* LSD tile: 256 threads x 16 rounds */

LGW_RHD uint64_t list_key(int64_t ts) { return (uint64_t)ts ^ 0x7FFFFFFFFFFFFFFFull; }

#if defined(__CUDACC__)
struct ListPair { uint64_t k; uint32_t i, pad; };

struct ListSel {
    uint64_t hi[2];                  // the boundary keys so far: digits fixed by the passes done, zero below
    uint32_t lo[2];
    uint64_t rank[2];                // rank of each boundary among the elements under its prefix
    uint32_t use_cand, compact;      // compact: k_list_cand copies the candidates after this pick; use_cand: passes read them
    unsigned long long n_cand;
    uint32_t hist[2][256];
};

__device__ __forceinline__ uint64_t list_mask_hi(int fixed) { return fixed <= 0 ? 0ull : fixed >= 8 ? ~0ull : ~0ull << (64 - 8 * fixed); }
__device__ __forceinline__ uint32_t list_mask_lo(int fixed) { return fixed <= 8 ? 0u : ~0u << (32 - 8 * (fixed - 8)); }
__device__ __forceinline__ uint32_t list_digit(uint64_t k, uint32_t i, int d) {
    return d < 8 ? (uint32_t)(k >> (56 - 8 * d)) & 255u : (i >> (24 - 8 * (d - 8))) & 255u;
}

__global__ void k_list_init(ListSel* s, uint64_t first, uint64_t last) {
    for (uint32_t k = threadIdx.x; k < 512; k += blockDim.x) (&s->hist[0][0])[k] = 0;
    if (threadIdx.x == 0) {
        s->hi[0] = s->hi[1] = 0; s->lo[0] = s->lo[1] = 0; s->rank[0] = first; s->rank[1] = last;
        s->use_cand = s->compact = 0; s->n_cand = 0;
    }
}

// one element into the block's histograms: lanes with the same digit add once (whole warp present)
__device__ __forceinline__ void list_count(uint32_t (*h)[256], uint64_t k, uint32_t i, bool valid, int d, const uint64_t hi[2], const uint32_t lo[2],
                                           uint64_t mh, uint32_t ml, uint32_t lane) {
    const uint32_t dig = list_digit(k, i, d);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
        const bool in = valid && ((k ^ hi[b]) & mh) == 0 && ((i ^ lo[b]) & ml) == 0;
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, in ? dig : 256u + lane);
        if (in && (peers & ((1u << lane) - 1u)) == 0) atomicAdd(&h[b][dig], (uint32_t)__popc(peers));
    }
}

// select pass d: histogram of digit d over the elements under each boundary's prefix (digits 0 .. d-1)
__global__ void __launch_bounds__(256) k_list_hist(const int64_t* __restrict__ ts, uint32_t n, const ListPair* __restrict__ cand, ListSel* s, int d) {
    __shared__ uint32_t h[2][256];
    for (uint32_t k = threadIdx.x; k < 512; k += blockDim.x) (&h[0][0])[k] = 0;
    const uint64_t hi[2] = {s->hi[0], s->hi[1]};
    const uint32_t lo[2] = {s->lo[0], s->lo[1]};
    const bool from_cand = s->use_cand | s->compact;
    const uint64_t mh = list_mask_hi(d);
    const uint32_t ml = list_mask_lo(d);
    const uint32_t lane = threadIdx.x & 31u, stride = gridDim.x * blockDim.x;
    __syncthreads();
    if (from_cand) {
        const uint32_t m = (uint32_t)s->n_cand;
        for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < m; base += stride) {    // (warp-uniform trips)
            const uint32_t j = base + lane;
            ListPair p{0, 0, 0};
            if (j < m) p = cand[j];
            list_count(h, p.k, p.i, j < m, d, hi, lo, mh, ml, lane);
        }
    } else {
        const uint32_t pairs = (uint32_t)(((uint64_t)n + 1) / 2);
        for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < pairs; base += stride) {
            const uint32_t j = base + lane;
            int64_t a = 0, b = 0;
            if (2 * j + 1 < n) { const longlong2 v = __ldg(reinterpret_cast<const longlong2*>(ts) + j); a = v.x; b = v.y; }
            else if (2 * j < n) a = __ldg(ts + 2 * j);
            list_count(h, list_key(a), 2 * j, 2 * j < n, d, hi, lo, mh, ml, lane);
            list_count(h, list_key(b), 2 * j + 1, 2 * j + 1 < n, d, hi, lo, mh, ml, lane);
        }
    }
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < 512; k += blockDim.x) if ((&h[0][0])[k]) atomicAdd(&s->hist[0][0] + k, (&h[0][0])[k]);
}

// fix digit d of both boundaries; zero the histograms; decide whether the candidates are few enough to compact
__global__ void k_list_pick(ListSel* s, int d, uint32_t cap) {
    __shared__ uint32_t grp[2];
    __shared__ uint32_t h[2][256];                    // (the serial walk below reads shared memory, not 256 dependent global loads)
    for (uint32_t k = threadIdx.x; k < 512; k += blockDim.x) (&h[0][0])[k] = (&s->hist[0][0])[k];
    __syncthreads();
    if (threadIdx.x < 2) {
        const int b = threadIdx.x;
        uint64_t r = s->rank[b];
        uint32_t dig = 0, cnt = 0;
        for (; dig < 255; ++dig) { cnt = h[b][dig]; if (r < cnt) break; r -= cnt; }
        if (dig == 255) cnt = h[b][255];
        s->rank[b] = r;
        if (d < 8) s->hi[b] |= (uint64_t)dig << (56 - 8 * d);
        else s->lo[b] |= dig << (24 - 8 * (d - 8));
        grp[b] = cnt;
    }
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < 512; k += blockDim.x) (&s->hist[0][0])[k] = 0;
    if (threadIdx.x == 0) {
        if (s->compact) { s->use_cand = 1; s->compact = 0; }
        else if (!s->use_cand && d + 1 < LGW_LIST_DIGITS) {
            const bool same = s->hi[0] == s->hi[1] && s->lo[0] == s->lo[1];
            const uint64_t under = same ? grp[0] : (uint64_t)grp[0] + grp[1];
            if (under <= cap) s->compact = 1;
        }
    }
}

// copy the elements under either prefix (`fixed` digits) to the candidate list, when k_list_pick asked for it
__global__ void __launch_bounds__(256) k_list_cand(const int64_t* __restrict__ ts, uint32_t n, ListPair* __restrict__ cand, ListSel* s, int fixed) {
    if (!s->compact) return;
    const uint64_t hi[2] = {s->hi[0], s->hi[1]};
    const uint32_t lo[2] = {s->lo[0], s->lo[1]};
    const uint64_t mh = list_mask_hi(fixed);
    const uint32_t ml = list_mask_lo(fixed);
    const uint32_t lane = threadIdx.x & 31u, lt = (1u << lane) - 1u, stride = gridDim.x * blockDim.x;
    const uint32_t pairs = (uint32_t)(((uint64_t)n + 1) / 2);
    for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < pairs; base += stride) {
        const uint32_t j = base + lane;
        int64_t v[2] = {0, 0};
        if (2 * j + 1 < n) { const longlong2 w = __ldg(reinterpret_cast<const longlong2*>(ts) + j); v[0] = w.x; v[1] = w.y; }
        else if (2 * j < n) v[0] = __ldg(ts + 2 * j);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const uint32_t i = 2 * j + u;
            const uint64_t k = list_key(v[u]);
            const bool in = i < n && ((((k ^ hi[0]) & mh) == 0 && ((i ^ lo[0]) & ml) == 0) || (((k ^ hi[1]) & mh) == 0 && ((i ^ lo[1]) & ml) == 0));
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, in);
            unsigned long long at = 0;
            if (lane == 0 && m) at = atomicAdd(&s->n_cand, (unsigned long long)__popc(m));
            at = __shfl_sync(0xFFFFFFFFu, at, 0);
            if (in) cand[at + __popc(m & lt)] = ListPair{k, i, 0};
        }
    }
}

__device__ __forceinline__ bool list_between(uint64_t k, uint32_t i, const ListSel& s) {
    return (k > s.hi[0] || (k == s.hi[0] && i >= s.lo[0])) && (k < s.hi[1] || (k == s.hi[1] && i <= s.lo[1]));
}

__device__ __forceinline__ void list_load_pair(const int64_t* __restrict__ ts, uint32_t n, uint32_t j, int64_t& a, int64_t& b) {
    a = b = 0;
    if (2 * j + 1 < n) { const longlong2 v = __ldg(reinterpret_cast<const longlong2*>(ts) + j); a = v.x; b = v.y; }
    else if (2 * j < n) a = __ldg(ts + 2 * j);
}

// records of each compaction tile between the two boundaries
__global__ void __launch_bounds__(1024) k_list_tile_count(const int64_t* __restrict__ ts, uint32_t n, const ListSel* __restrict__ sp, uint32_t* __restrict__ tile_count) {
    __shared__ uint32_t warp_sums[32];
    const ListSel s = *sp;
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    int64_t a, b;
    list_load_pair(ts, n, j, a, b);
    const uint32_t c = (2 * j < n && list_between(list_key(a), 2 * j, s)) + (2 * j + 1 < n && list_between(list_key(b), 2 * j + 1, s));
    const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, c);
    if ((threadIdx.x & 31u) == 0) warp_sums[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x < 32) {
        const uint32_t t = __reduce_add_sync(0xFFFFFFFFu, threadIdx.x < (blockDim.x >> 5) ? warp_sums[threadIdx.x] : 0u);
        if (threadIdx.x == 0) tile_count[blockIdx.x] = t;
    }
}

// exclusive scan in place of column blockIdx.x (len entries at v + blockIdx.x * len); the column's total to totals[blockIdx.x]
__global__ void __launch_bounds__(1024) k_list_scan(uint32_t* v, uint32_t len, uint32_t* totals) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t base;
    uint32_t* col = v + (size_t)blockIdx.x * len;
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (uint32_t start = 0; start < len; start += blockDim.x) {
        const uint32_t k = start + threadIdx.x;
        const uint32_t x0 = k < len ? col[k] : 0u;
        uint32_t x = x0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        uint32_t before = 0, all = 0;
        for (uint32_t w = 0; w < (blockDim.x >> 5); ++w) { const uint32_t t = warp_sums[w]; if (w < warp) before += t; all += t; }
        if (k < len) col[k] = base + before + x - x0;
        __syncthreads();
        if (threadIdx.x == 0) base += all;
        __syncthreads();
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = base;
}

// the keys between the two boundaries, in index order, at the tile offsets k_list_scan made.  Only the first `count` are stored:
// keys / idx hold `count` entries, and a selection that put more records between the boundaries is caught by the host's check
// of the total (k_list_scan's), not by writing past them into the rest of the scratch.
__global__ void __launch_bounds__(1024) k_list_tile_write(const int64_t* __restrict__ ts, uint32_t n, const ListSel* __restrict__ sp, const uint32_t* __restrict__ tile_off,
                                                          uint32_t count, uint64_t* __restrict__ keys, uint32_t* __restrict__ idx) {
    __shared__ uint32_t warp_sums[32];
    const ListSel s = *sp;
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
    int64_t a, b;
    list_load_pair(ts, n, j, a, b);
    const uint64_t ka = list_key(a), kb = list_key(b);
    const bool ia = 2 * j < n && list_between(ka, 2 * j, s), ib = 2 * j + 1 < n && list_between(kb, 2 * j + 1, s);
    const uint32_t ma = __ballot_sync(0xFFFFFFFFu, ia), mb = __ballot_sync(0xFFFFFFFFu, ib);
    if (lane == 0) warp_sums[warp] = __popc(ma) + __popc(mb);
    __syncthreads();
    uint32_t pos = tile_off[blockIdx.x] + __popc(ma & lt) + __popc(mb & lt);
    for (uint32_t w = 0; w < warp; ++w) pos += warp_sums[w];
    if (ia) { if (pos < count) { keys[pos] = ka; idx[pos] = 2 * j; } ++pos; }
    if (ib && pos < count) { keys[pos] = kb; idx[pos] = 2 * j + 1; }
}

// pages up to LGW_LIST_SMEM_SORT: bitonic sort of (kd, index) in shared memory by one block; indices out as uint64
__global__ void __launch_bounds__(1024) k_list_sort_small(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ idx, uint32_t m, uint64_t* __restrict__ out) {
    extern __shared__ uint64_t sk[];
    uint32_t p = 1;
    while (p < m) p <<= 1;
    uint32_t* si = reinterpret_cast<uint32_t*>(sk + p);
    for (uint32_t i = threadIdx.x; i < p; i += blockDim.x) { sk[i] = i < m ? keys[i] : ~0ull; si[i] = i < m ? idx[i] : ~0u; }   // (pads sort last)
    __syncthreads();
    for (uint32_t size = 2; size <= p; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < p / 2; t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const uint64_t ka = sk[lo], kb = sk[hi];
                const uint32_t ia = si[lo], ib = si[hi];
                const bool b_first = kb < ka || (kb == ka && ib < ia);
                if (b_first == up) { sk[lo] = kb; sk[hi] = ka; si[lo] = ib; si[hi] = ia; }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) out[i] = si[i];
}

// LSD pass, step 1: per-tile counts of the digit at `shift`, digit-major ([256][n_tiles]) so that one scan per digit column
// and a scan of the 256 column totals give every (digit, tile) its output offset
__global__ void __launch_bounds__(256) k_lsd_hist(const uint64_t* __restrict__ keys, uint32_t m, int shift, uint32_t* __restrict__ tile_hist, uint32_t n_tiles) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t r = 0; r < LGW_LIST_STILE / 256; ++r) {
        const uint32_t i = blockIdx.x * LGW_LIST_STILE + r * 256 + threadIdx.x;
        const bool v = i < m;
        const uint32_t dig = v ? (uint32_t)(keys[i] >> shift) & 255u : 0u;
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, v ? dig : 256u + lane);
        if (v && (peers & ((1u << lane) - 1u)) == 0) atomicAdd(&h[dig], (uint32_t)__popc(peers));
    }
    __syncthreads();
    tile_hist[(size_t)threadIdx.x * n_tiles + blockIdx.x] = h[threadIdx.x];
}

// LSD pass, step 3: stable scatter.  A tile goes in 16 rounds of 256 keys in index order; inside a round, a key's place is the
// digit's running offset + the same digit's keys of the warps before + its rank among the same digit's lanes of its warp.
__global__ void __launch_bounds__(256) k_lsd_scatter(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ idx, uint32_t m, int shift,
                                                     const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ totals, uint32_t n_tiles,
                                                     uint64_t* __restrict__ keys_out, uint32_t* __restrict__ idx_out) {
    __shared__ uint32_t run[256];
    __shared__ uint32_t wcnt[8][256];                 // (round + 1) << 8 | lanes of warp w with the digit, this round
    __shared__ uint32_t wpre[8][256];
    __shared__ uint32_t wsum[8];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
    for (uint32_t w = 0; w < 8; ++w) wcnt[w][threadIdx.x] = 0;
    {   // run[d] = keys of digits below d (exclusive scan of the totals) + this tile's offset within digit d
        const uint32_t t = totals[threadIdx.x];
        uint32_t x = t;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31) wsum[warp] = x;
        __syncthreads();
        uint32_t before = 0;
        for (uint32_t w = 0; w < warp; ++w) before += wsum[w];
        run[threadIdx.x] = before + x - t + tile_off[(size_t)threadIdx.x * n_tiles + blockIdx.x];
    }
    __syncthreads();
    for (uint32_t r = 0; r < LGW_LIST_STILE / 256; ++r) {
        const uint32_t i = blockIdx.x * LGW_LIST_STILE + r * 256 + threadIdx.x;
        const bool v = i < m;
        const uint64_t k = v ? keys[i] : 0ull;
        const uint32_t x = v ? idx[i] : 0u;
        const uint32_t dig = (uint32_t)(k >> shift) & 255u;
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, v ? dig : 256u + lane);
        const uint32_t rank = __popc(peers & lt);
        if (v && rank == 0) wcnt[warp][dig] = ((r + 1) << 8) | (uint32_t)__popc(peers);
        __syncthreads();
        uint32_t acc = run[threadIdx.x];               // thread d: the warps' offsets for digit d
        for (uint32_t w = 0; w < 8; ++w) {
            const uint32_t c = wcnt[w][threadIdx.x];
            wpre[w][threadIdx.x] = acc;
            acc += (c >> 8) == r + 1 ? (c & 255u) : 0u;
        }
        run[threadIdx.x] = acc;
        __syncthreads();
        if (v) { const uint32_t pos = wpre[warp][dig] + rank; keys_out[pos] = k; idx_out[pos] = x; }
    }
}

__global__ void __launch_bounds__(256) k_list_widen(const uint32_t* __restrict__ idx, uint32_t m, uint64_t* __restrict__ out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) out[i] = idx[i];
}
#endif

}  // namespace lgw
