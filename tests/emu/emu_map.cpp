// emu_map.cpp -- TEST INFRASTRUCTURE: the pileup with a dirty-sector map (kdl_pileup_range_map) compiled for the host and
// run under tests/emu/cuda_emu.h, as emu_pileup.cpp does for the pileup without one.  The kernel sources are included
// as they are; nothing here is part of the product.
#define KDL_HOST_EMU 1
#include "cuda_emu.h"

#include "../../kindel_b200/csrc/kdl_common.cuh"
#include "../../kindel_b200/csrc/pileup_tile.cu"
#include "../../kindel_b200/csrc/pileup_general.cu"
#include "../../kindel_b200/csrc/pileup_simple.cu"

static char g_error[512];

#define EMU_RUN(grid, block, ...)                                                                   \
    do {                                                                                            \
        const char* e_ = emu::launch((unsigned)(grid), (unsigned)(block), [&] { __VA_ARGS__; });    \
        if (e_) { snprintf(g_error, sizeof g_error, "%s", e_); return 1; }                          \
    } while (0)

extern "C" {

const char* emu_map_last_error() { return g_error; }

// The kernels kdl_pileup_range_map launches for KDL_PILEUP_FRESH_WEIGHTS (| KDL_PILEUP_ZERO_REST when zero_rest) over the
// whole slot range, in its order and with its choices: the zeroing pass when K1 does not zero, K0 + K1 (F_STORE, or
// F_ATOMIC for split > 1; cx: the piece instantiation, else the lean one with K1e counting the bases), K1e, K1g -- or,
// for a batch the tile kernel cannot take, K1s + K1g.  Dense complex reads (>= 1 in 16) leave the map set instead of
// marking it.  All pointers are HOST pointers; dirty_map may be NULL (kdl_pileup_range).  Returns 0, or 1 with
// emu_map_last_error() set.
int emu_map_pileup(const kdl_batch* batch, int32_t* counts, long long n_slots, uint32_t* tile_index, uint32_t* dirty_map,
                   int zero_rest, int split, int cx, int32_t* ins_events, int32_t* err_flag, int grid) {
    g_error[0] = 0;
    const kdl_batch b = *batch;
    const bool tiled = b.n_reads > b.n_hard && n_slots % KDL_TILE == 0 && b.reads_sorted && tile_index &&
                       b.reach_right > 0 && b.reach_right <= KDL_FAST_MAXLEN + KDL_TILE_MAXREACH;
    const long long n_tiles = n_slots / KDL_TILE;
    const bool k1_stores = tiled && split == 1 && n_tiles > 0;
    const int zero_from = k1_stores ? 5 : 0;
    const int zero_to = zero_rest && !k1_stores ? KDL_NCOL : 5;
    const bool zero_pass = zero_to > zero_from;
    const bool saturate = dirty_map && b.n_complex > 0 && b.n_complex * 16 >= b.n_reads && (k1_stores || zero_pass);
    uint32_t* mark = saturate ? nullptr : dirty_map;
    if (zero_pass) {
        uint32_t* zmap = saturate || (zero_from <= 5 && zero_to == KDL_NCOL) ? dirty_map : nullptr;
        const uint32_t fill = saturate ? ~0u : 0u;
        EMU_RUN(grid, 256, kdl::zero_cols_kernel(counts, n_slots, zero_from, zero_to, 0, n_slots, zmap, fill));
    }
    if (b.n_reads == 0) return 0;
    if (tiled) {
        EMU_RUN((n_tiles * 32 + 255) / 256, 256, kdl::tile_index_kernel(b, 0, n_tiles, tile_index));
        const int zr = k1_stores && zero_rest ? 1 : 0;
        const uint32_t after = saturate && k1_stores ? ~0u : 0u;
        uint32_t* kmap = k1_stores ? dirty_map : nullptr;
#define KDL_EMU_TILE(M, X) kdl::pileup_tile_kernel<M, X>(b, counts, n_slots, tile_index, 0, n_tiles, split, zr, kmap, after)
        if (split == 1) {
            if (cx) EMU_RUN(grid, kdl::W_THREADS, KDL_EMU_TILE(kdl::F_STORE, true));
            else EMU_RUN(grid, kdl::W_THREADS, KDL_EMU_TILE(kdl::F_STORE, false));
        } else {
            if (cx) EMU_RUN(grid, kdl::W_THREADS, KDL_EMU_TILE(kdl::F_ATOMIC, true));
            else EMU_RUN(grid, kdl::W_THREADS, KDL_EMU_TILE(kdl::F_ATOMIC, false));
        }
#undef KDL_EMU_TILE
        if (b.n_complex > b.n_hard) {
            if (cx) EMU_RUN((b.n_complex + 255) / 256, 256, kdl::pileup_events_kernel<1>(b, counts, n_slots, ins_events, 0, mark));
            else EMU_RUN((b.n_complex + 31) / 32, 256, kdl::pileup_events_kernel<8>(b, counts, n_slots, ins_events, 1, mark));
        }
        if (b.n_hard > 0)
            EMU_RUN(grid, 256, kdl::pileup_general_kernel(b, b.hard_idx, b.n_hard, counts, n_slots, ins_events, err_flag, mark));
    } else {
        if (b.n_reads > b.n_complex) EMU_RUN(grid, 256, kdl::pileup_simple_atomic_kernel(b, counts, n_slots, err_flag));
        if (b.n_complex > 0)
            EMU_RUN(grid, 256, kdl::pileup_general_kernel(b, nullptr, b.n_reads, counts, n_slots, ins_events, err_flag, mark));
    }
    return 0;
}

}  // extern "C"
