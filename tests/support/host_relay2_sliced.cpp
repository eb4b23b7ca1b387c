// TEST AID ONLY: the emulated bulk kernels of host_relay2.cpp, plus a step cut into slices the way lgw_sse_step cuts a
// host-buffer step (step_slice_cuts in csrc/step_types.cuh), so that the CPU suite can run the kernels' slice edges.
// Never linked into the product library.
#include "host_relay2.cpp"

extern "C" {

// lgwt_bulk_step with n_slices: the three kernels run once per slice with the engine's launch arguments -- tile_base = the
// slice's first byte, n_bytes = its end, the segment arrays offset by its first segment; the row queue is emptied once for the
// whole step, and the tile table is shared by the slices of a step as it is on the device.  Mode 1 and a single slice: the
// ordinary step.
int lgwt_bulk_step_sliced(void* h, const uint8_t* data, uint32_t n_bytes, const uint32_t* chunk_off, uint32_t n_chunks,
                          const uint32_t* seg_chunk, const uint32_t* seg_slot, uint32_t n_segs, uint8_t* out, lgw_seg_result* seg_out,
                          lgw_row_event* rows_out, uint32_t rows_cap, uint32_t* n_rows, uint32_t tiles_per_warp, uint32_t n_slices) {
    HostEngine* e = (HostEngine*)h;
    uint32_t cut[18];
    if (n_slices < 1 || n_slices > 14 || e->mode == 1) n_slices = 1;
    n_slices = step_slice_cuts(n_bytes, chunk_off, seg_chunk, n_segs, n_slices, cut);
    if (n_slices == 1)
        return lgwt_bulk_step(h, data, n_bytes, chunk_off, n_chunks, seg_chunk, seg_slot, n_segs, out, seg_out, rows_out, rows_cap, n_rows, tiles_per_warp);
    const StepArgs a = make_args(e, data, n_bytes, chunk_off, n_chunks, seg_chunk, seg_slot, n_segs, out, seg_out);
    e->rowq_count = 0;
    for (uint32_t j = 0; j < n_slices; ++j) {
        const uint32_t s0 = cut[j], s1 = cut[j + 1];
        if (s1 <= s0) continue;
        const uint32_t c0 = seg_chunk[s0], c1 = seg_chunk[s1];
        const uint32_t b0 = chunk_off[c0], b1 = chunk_off[c1];
        StepArgs sa = a;
        sa.tile_base = b0; sa.n_bytes = b1; sa.chunk_lo = c0; sa.chunk_hi = c1;
        sa.seg_chunk = seg_chunk + s0; sa.seg_slot = seg_slot + s0; sa.n_segs = s1 - s0; sa.seg_out = a.seg_out + s0;
        sa.reset_rows = 0;
        simt::launch((sa.n_segs + 127) / 128, 128, [&] { k_prime2(sa); });
        const uint32_t base0 = b0 & ~15u;
        const uint32_t n_tiles = b1 > base0 ? (b1 - base0 + R2_TILE - 1) / R2_TILE : 0u;
        if (n_tiles) {
            const uint32_t max_warps = e->n_blocks * R2_WARPS;
            uint32_t tpw = tiles_per_warp ? tiles_per_warp : (n_tiles + max_warps - 1) / max_warps;
            uint32_t warps = (n_tiles + tpw - 1) / tpw;
            if (warps > max_warps) { tpw = (n_tiles + max_warps - 1) / max_warps; warps = (n_tiles + tpw - 1) / tpw; }
            const uint32_t blocks = (warps + R2_WARPS - 1) / R2_WARPS;
            simt::launch(blocks, R2_THREADS, [&] { k_relay2(sa, n_tiles, tpw, base0); });
        }
        simt::launch((sa.n_segs + R2_CWARPS - 1) / R2_CWARPS, R2_CWARPS * 32, [&] { k_commit2(sa); });
    }
    uint32_t cnt = e->rowq_count < e->rowq_cap ? e->rowq_count : e->rowq_cap;
    if (cnt > rows_cap) cnt = rows_cap;
    memcpy(rows_out, e->rowq.data(), (size_t)cnt * sizeof(RowEvent));
    *n_rows = cnt;
    return 0;
}

}  // extern "C"
