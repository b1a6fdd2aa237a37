// api.cu -- the C ABI declared in include/kindel_b200.h (unity build of the kernel files).
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "kdl_common.cuh"
#include "pileup_general.cu"
#include "pileup_simple.cu"
#include "pileup_tile.cu"
#include "pileup_mask.cu"
#include "vote.cu"
#include "assemble.cu"
#include "variants.cu"
#include "select.cu"
#include "primers.cu"
#include "mates.cu"
#include "quality.cu"
#include "amplicons.cu"
#include "normalise.cu"
#include "dedup.cu"
#include "left_align.cu"

namespace {

std::atomic<long long> g_launches{0};

inline int grid_for(long long items, int per_block, int cap) {
    long long g = (items + per_block - 1) / per_block;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (int)g;
}

#ifndef KDL_HOST_EMU
constexpr int kMaxDevices = 64;

inline int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
    return dev;
}

// SM count of the CURRENT device (a process may drive several GPUs)
inline int sm_count() {
    static std::atomic<int> cache[kMaxDevices];
    const int dev = current_device();
    int n = cache[dev].load(std::memory_order_relaxed);
    if (n <= 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;  // H100 SXM
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

// opt-in to > 48 KB dynamic shared memory for the tile kernel's instantiations, once per device
template <int kFlush, bool kCx>
inline int ensure_tile_smem() {
    static std::atomic<int> done[kMaxDevices];
    const int dev = current_device();
    if (done[dev].load(std::memory_order_acquire)) return KDL_OK;
    if (cudaFuncSetAttribute(kdl::pileup_tile_kernel<kFlush, kCx>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)sizeof(kdl::TileSmem<kdl::TileCfg<kCx>>)) != cudaSuccess)
        return KDL_ERR_CUDA;
    done[dev].store(1, std::memory_order_release);
    return KDL_OK;
}

inline int check_launch() {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError() == cudaSuccess ? KDL_OK : KDL_ERR_CUDA;
}
#else
// the kernel emulator (tests/emu/cuda_emu.h): the SM count it is set to, no shared-memory limit, its launch error
inline int sm_count() { return emu::M().sm_count; }

template <int kFlush, bool kCx>
inline int ensure_tile_smem() { return KDL_OK; }

inline int check_launch() {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return emu::take_launch_error() ? KDL_ERR_CUDA : KDL_OK;
}
#endif

template <int kFlush, bool kCx>
inline int launch_tile(const kdl_batch& b, int32_t* counts, long long n_slots, long long tile_lo, long long n_tiles,
                       int split, int zero_rest, uint32_t* dirty_map, uint32_t map_after, cudaStream_t st) {
    int rc = ensure_tile_smem<kFlush, kCx>();
    if (rc != KDL_OK) return rc;
    const long long units = n_tiles * split, max_grid = (long long)sm_count() * 2;  // two CTAs per SM, persistent
    const long long grid = units < max_grid ? units : max_grid;
    KDL_LAUNCH((kdl::pileup_tile_kernel<kFlush, kCx>), (unsigned)grid, kdl::W_THREADS,
               sizeof(kdl::TileSmem<kdl::TileCfg<kCx>>), st,
               b, counts, n_slots, b.tile_index, tile_lo, n_tiles, split, zero_rest, dirty_map, map_after);
    return KDL_OK;
}

// CTAs per unit of work (a tile of K1, a window of K1w) when there are fewer units than `per_sm` CTAs per SM would
// fill, with at least ~256 reads per CTA; KDL_SPLIT overrides it
int depth_split(long long units, int per_sm, long long reads) {
    int split = 1;
    const long long slots = (long long)sm_count() * per_sm;
    if (units < slots) {
        long long want = (slots + units - 1) / units;
        const long long deep = reads / (units * 256);
        if (want > deep) want = deep;
        split = (int)(want < 1 ? 1 : (want > 32 ? 32 : want));
    }
    if (const char* ev = getenv("KDL_SPLIT")) { const int v = atoi(ev); if (v >= 1 && v <= 64) split = v; }
    return split;
}

int validate_batch(const kdl_batch* b) {
    if (!b || b->n_reads < 0 || b->n_contigs < 0 || b->n_hard < 0 || b->n_complex < b->n_hard)
        return KDL_ERR_INVALID_ARG;
    if (b->n_reads > 0 && (!b->ref_start || !b->seq_off || !b->l_seq || !b->seq4 ||
                           !b->contig_read_off || !b->contig_len || !b->contig_slot))
        return KDL_ERR_INVALID_ARG;
    if ((b->n_hard > 0 && !b->hard_idx) || (b->n_complex > 0 && !b->complex_idx)) return KDL_ERR_INVALID_ARG;
    if (b->reach_right < b->max_simple_len || b->reach_left < 0) return KDL_ERR_INVALID_ARG;
    return KDL_OK;
}

}  // namespace

extern "C" {

int kdl_abi_version(void) { return KDL_ABI_VERSION; }

const char* kdl_status_string(int status) {
    switch (status) {
        case KDL_OK: return "ok";
        case KDL_ERR_INVALID_ARG: return "invalid argument";
        case KDL_ERR_CUDA: return "CUDA error";
        case KDL_ERR_NO_DEVICE: return "no CUDA device";
        case KDL_ERR_INDEX: return "IndexError: read walks off the contig or off its SEQ";
        case KDL_ERR_KEY: return "KeyError: base outside A,C,G,T,N in an M or S op";
        default: return "unknown status";
    }
}

int64_t kdl_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int kdl_pileup(const kdl_batch* batch, int32_t* counts, int64_t n_slots, int32_t* ins_events,
               int32_t* err_flag, void* stream) {
    return kdl_pileup_range(batch, counts, n_slots, 0, n_slots, 0, ins_events, err_flag, stream);
}

int kdl_pileup_range(const kdl_batch* batch, int32_t* counts, int64_t n_slots, int64_t slot_lo,
                     int64_t slot_hi, int32_t flags, int32_t* ins_events, int32_t* err_flag, void* stream) {
    return kdl_pileup_range_map(batch, counts, n_slots, slot_lo, slot_hi, flags, nullptr, ins_events, err_flag, stream);
}

int kdl_pileup_range_map(const kdl_batch* batch, int32_t* counts, int64_t n_slots, int64_t slot_lo, int64_t slot_hi,
                         int32_t flags, uint32_t* dirty_map, int32_t* ins_events, int32_t* err_flag, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!counts || !err_flag || n_slots <= 0 || slot_lo < 0 || slot_hi > n_slots || slot_lo > slot_hi ||
        (reinterpret_cast<uintptr_t>(dirty_map) & 15))
        return KDL_ERR_INVALID_ARG;
    const bool tileable = (n_slots % KDL_TILE) == 0 && (slot_lo % KDL_TILE) == 0 && (slot_hi % KDL_TILE) == 0;
    if ((slot_lo & 3) || (slot_hi & 3)) return KDL_ERR_INVALID_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int cap = sm_count() * 8;
    const bool has_tile_reads = batch->n_reads > batch->n_hard;
    const bool tiled = has_tile_reads && tileable && batch->reads_sorted && batch->tile_index &&
                       batch->reach_right > 0 && batch->reach_right <= KDL_FAST_MAXLEN + KDL_TILE_MAXREACH;
    const bool fresh = (flags & KDL_PILEUP_FRESH_WEIGHTS) != 0;
    const long long tile_lo = slot_lo / KDL_TILE, n_tiles = (slot_hi - slot_lo) / KDL_TILE;
    // Depth split: a small reference piled deep has fewer tiles than the GPU has CTA slots (30 kb = 59 tiles for
    // 296 slots); `split` CTAs then share a tile by read range and flush with REDs into a zeroed table.
    const int split = tiled && n_tiles > 0 ? depth_split(n_tiles, 2, batch->n_reads) : 1;
    bool cx_by_atomics = (batch->n_complex - batch->n_hard) * 16 < batch->n_reads;
    if (const char* ev = getenv("KDL_CX")) cx_by_atomics = !strcmp(ev, "atomics") ? true : (!strcmp(ev, "pieces") ? false : cx_by_atomics);
    // zeroing that the chosen kernels will not do themselves: the tile kernel overwrites the weight columns of a
    // fresh table and, on request, zeroes columns 5..18 window by window in its flush (only the sectors the map marks)
    const int zero_in_k1 = (tiled && split == 1 && fresh && n_tiles > 0 && (flags & KDL_PILEUP_ZERO_REST)) ? 1 : 0;
    const int zero_from = (fresh && !(tiled && split == 1)) ? 0 : 5;
    const int zero_to = ((flags & KDL_PILEUP_ZERO_REST) && !zero_in_k1) ? KDL_NCOL : 5;
    const bool zero_pass = zero_to > zero_from && slot_hi > slot_lo;
    // The dirty-sector map.  Complex reads this dense (>= 1 in 16; a few per cent of sectors stay clean at 1 in 100)
    // dirty nearly every sector: instead of K1w / K1e / K1g marking what they write, the kernel that zeroes -- K1's
    // flush, or the zeroing pass -- leaves every record of the range set, and the next pileup zeroes all of it.  Where
    // neither runs, the writers mark.
    const bool k1_stores = tiled && split == 1 && fresh && n_tiles > 0;
    const bool saturate = dirty_map && batch->n_complex > 0 && batch->n_complex * 16 >= batch->n_reads &&
                          (k1_stores || zero_pass);
    uint32_t* mark_map = saturate ? nullptr : dirty_map;
    if (zero_pass) {
        uint32_t* zmap = saturate || (zero_from <= 5 && zero_to == KDL_NCOL) ? dirty_map : nullptr;
        KDL_LAUNCH(kdl::zero_cols_kernel, sm_count() * 4, 256, 0, st, counts, n_slots, zero_from, zero_to, slot_lo,
                   slot_hi, zmap, saturate ? ~0u : 0u);
        if ((rc = check_launch()) != KDL_OK) return rc;
    }
    const uint32_t map_after = saturate && k1_stores ? ~0u : 0u;
    if (batch->n_reads == 0) return KDL_OK;
    if (tiled) {
        if (n_tiles > 0) {
            // K0: read range per tile of the slot range (the linear index of a sorted BAM, built on device)
            KDL_LAUNCH(kdl::tile_index_kernel, (unsigned)((n_tiles * 32 + 255) / 256), 256, 0, st, *batch, tile_lo,
                       n_tiles, batch->tile_index);
            if ((rc = check_launch()) != KDL_OK) return rc;
            // K1: the tile-owner kernel.  Tile-eligible complex reads go through its piece machinery (kCx) when
            // they are a sizeable share of the batch; when they are rare (< 1/16 of the reads) the lean instantiation
            // runs and K1w counts their bases too
            const bool cx = batch->n_complex > batch->n_hard && !cx_by_atomics;
            if (split > 1) {
                rc = cx ? launch_tile<kdl::F_ATOMIC, true>(*batch, counts, n_slots, tile_lo, n_tiles, split, 0, nullptr, 0, st)
                        : launch_tile<kdl::F_ATOMIC, false>(*batch, counts, n_slots, tile_lo, n_tiles, split, 0, nullptr, 0, st);
            } else if (fresh) {
                rc = cx ? launch_tile<kdl::F_STORE, true>(*batch, counts, n_slots, tile_lo, n_tiles, 1, zero_in_k1, dirty_map,
                                                          map_after, st)
                        : launch_tile<kdl::F_STORE, false>(*batch, counts, n_slots, tile_lo, n_tiles, 1, zero_in_k1, dirty_map,
                                                           map_after, st);
            } else {
                rc = cx ? launch_tile<kdl::F_ADD, true>(*batch, counts, n_slots, tile_lo, n_tiles, 1, 0, nullptr, 0, st)
                        : launch_tile<kdl::F_ADD, false>(*batch, counts, n_slots, tile_lo, n_tiles, 1, 0, nullptr, 0, st);
            }
            if (rc != KDL_OK) return rc;
            if ((rc = check_launch()) != KDL_OK) return rc;
        }
        if (batch->n_complex > batch->n_hard && cx_by_atomics && n_tiles > 0) {
            // K1w: everything of the rare tile-eligible complex reads the lean K1 left out, window by window (the
            // windows' reads come from K0's index)
            const long long n_win = (slot_hi - slot_lo + kdl::CW_SLOTS - 1) / kdl::CW_SLOTS;
            const int wsplit = depth_split(n_win, 8, batch->n_complex - batch->n_hard);
            KDL_LAUNCH(kdl::pileup_window_kernel, (unsigned)(n_win * wsplit), kdl::CW_THREADS,
                       sizeof(int32_t) * kdl::CW_SMEM_COLS * kdl::CW_SLOTS, st, *batch, counts, n_slots, slot_lo,
                       slot_hi, wsplit, ins_events, mark_map);
            if ((rc = check_launch()) != KDL_OK) return rc;
        } else if (batch->n_complex > batch->n_hard && !cx_by_atomics) {
            // K1e: insertions / deletions / clips of the tile-eligible complex reads whose bases K1 counted as pieces
            KDL_LAUNCH(kdl::pileup_events_kernel, (unsigned)((batch->n_complex + 255) / 256), 256, 0, st, *batch, counts,
                       n_slots, ins_events, mark_map);
            if ((rc = check_launch()) != KDL_OK) return rc;
        }
        if (batch->n_hard > 0) {  // K1g: the reads that may wrap or raise, atomically, after the tile stores
            const int grid = grid_for(batch->n_hard, 8, cap);
            KDL_LAUNCH(kdl::pileup_general_kernel, grid, 256, 0, st, *batch, batch->hard_idx, batch->n_hard, counts,
                       n_slots, ins_events, err_flag, mark_map);
            if ((rc = check_launch()) != KDL_OK) return rc;
        }
    } else {
        // order-independent fallback (unsorted input): K1s for the simple reads, K1g for every complex read
        if (batch->n_reads > batch->n_complex) {
            const int grid = grid_for(batch->n_reads, 8, cap);  // 8 warps (reads) per 256-thread CTA
            KDL_LAUNCH(kdl::pileup_simple_atomic_kernel, grid, 256, 0, st, *batch, counts, n_slots, err_flag);
            if ((rc = check_launch()) != KDL_OK) return rc;
        }
        if (batch->n_complex > 0) {
            const int grid = grid_for(batch->n_reads, 8, cap);
            KDL_LAUNCH(kdl::pileup_general_kernel, grid, 256, 0, st, *batch, nullptr, batch->n_reads, counts, n_slots,
                       ins_events, err_flag, mark_map);
            if ((rc = check_launch()) != KDL_OK) return rc;
        }
    }
    return KDL_OK;
}

int kdl_unmask(const kdl_batch* batch, const kdl_qmask* qmask, int32_t* counts, int64_t n_slots, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!qmask || !counts || n_slots <= 0 || qmask->n_reads < 0 || qmask->n_bases < 0 || qmask->n_reads > batch->n_reads)
        return KDL_ERR_INVALID_ARG;
    if (qmask->n_reads == 0) return KDL_OK;
    if (!qmask->read_idx || !qmask->off || !qmask->qpos) return KDL_ERR_INVALID_ARG;
    const long long grid = (qmask->n_reads + kdl::kQThreads - 1) / kdl::kQThreads;
    KDL_LAUNCH(kdl::unmask_kernel, (unsigned)grid, kdl::kQThreads, 0, (cudaStream_t)stream, *batch, *qmask, counts,
               n_slots);
    return check_launch();
}

int kdl_diagnose(const kdl_batch* batch, kdl_diag* diag_dev, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!diag_dev) return KDL_ERR_INVALID_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    KDL_LAUNCH(kdl::diagnose_init_kernel, 1, 1, 0, st, diag_dev);
    if ((rc = check_launch()) != KDL_OK) return rc;
    if (batch->n_hard > 0) {
        const long long grid = (batch->n_hard + 255) / 256;
        KDL_LAUNCH(kdl::diagnose_kernel, (unsigned)grid, 256, 0, st, *batch, diag_dev);
        if ((rc = check_launch()) != KDL_OK) return rc;
    }
    KDL_LAUNCH(kdl::diagnose_final_kernel, 1, 1, 0, st, diag_dev);
    return check_launch();
}

int kdl_vote(const int32_t* counts, int64_t n_slots, int64_t min_depth_ceil, uint8_t* calls,
             void* stream) {
    if (!counts || !calls || n_slots <= 0 || (n_slots & 3)) return KDL_ERR_INVALID_ARG;
    kdl::Peers none;
    none.n = 0;
    const long long quads = n_slots / 4;
    const long long grid = (quads + 255) / 256;
    KDL_LAUNCH(kdl::vote_kernel<false>, (unsigned)grid, 256, 0, (cudaStream_t)stream,
               counts, none, n_slots, 0, n_slots, min_depth_ceil, calls, nullptr, kdl::MajorityVote{});
    return check_launch();
}

static bool valid_threshold(double t) { return t >= 0.0 && t <= 1.0; }  // false for NaN

int kdl_vote_iupac(const int32_t* counts, int64_t n_slots, int64_t min_depth_ceil, double threshold, uint8_t* calls,
                   void* stream) {
    if (!counts || !calls || n_slots <= 0 || (n_slots & 3) || !valid_threshold(threshold)) return KDL_ERR_INVALID_ARG;
    kdl::Peers none;
    none.n = 0;
    const long long quads = n_slots / 4;
    const long long grid = (quads + 255) / 256;
    KDL_LAUNCH((kdl::vote_kernel<false, kdl::IupacVote>), (unsigned)grid, 256, 0, (cudaStream_t)stream,
               counts, none, n_slots, 0, n_slots, min_depth_ceil, calls, nullptr, kdl::IupacVote{threshold});
    return check_launch();
}

int kdl_derive(const int32_t* counts, int64_t n_slots, int32_t* out, void* stream) {
    if (!counts || !out || n_slots <= 0) return KDL_ERR_INVALID_ARG;
    const long long grid = (n_slots + 255) / 256;
    KDL_LAUNCH(kdl::derive_kernel, (unsigned)grid, 256, 0, (cudaStream_t)stream, counts, n_slots, out);
    return check_launch();
}

int kdl_vote_peers(const int32_t* const* peer_counts, int32_t n_peers, int64_t n_slots,
                   int64_t slot_lo, int64_t slot_hi, int64_t min_depth_ceil, uint8_t* calls,
                   int32_t* reduced, void* stream) {
    return kdl_vote_peers_sparse(peer_counts, nullptr, nullptr, n_peers, n_slots, slot_lo, slot_hi,
                                 min_depth_ceil, calls, reduced, stream);
}

static int make_exchange(const kdl_exchange* x, kdl::Exchange* e, int64_t n_slots) {
    if (!x || x->n_ranks < 1 || x->n_ranks > 16 || x->rank < 0 || x->rank >= x->n_ranks || !x->counter)
        return KDL_ERR_INVALID_ARG;
    e->peers.n = x->n_ranks;
    e->rank = x->rank;
    e->counter = x->counter;
    for (int p = 0; p < x->n_ranks; ++p) {
        if (!x->tables[p] || !x->calls[p] || !x->ready[p] || !x->done[p]) return KDL_ERR_INVALID_ARG;
        e->peers.tab[p] = x->tables[p];
        e->peers.lo[p] = x->foot_lo[p];
        e->peers.hi[p] = n_slots > 0 && x->foot_hi[p] > n_slots ? n_slots : x->foot_hi[p];
        if ((e->peers.lo[p] & 3) || (e->peers.hi[p] & 3)) return KDL_ERR_INVALID_ARG;
        e->calls[p] = x->calls[p];
        e->ready[p] = x->ready[p];
        e->done[p] = x->done[p];
        e->slice_lo[p] = x->slice_lo[p];
        e->slice_hi[p] = x->slice_hi[p];
        if ((x->slice_lo[p] & 3) || (x->slice_hi[p] & 3) || x->slice_hi[p] < x->slice_lo[p]) return KDL_ERR_INVALID_ARG;
    }
    e->ready_local = x->ready[x->rank];
    e->done_local = x->done[x->rank];
    return KDL_OK;
}

int kdl_exchange_signal(const kdl_exchange* x, int32_t epoch, void* stream) {
    kdl::Exchange e;
    int rc = make_exchange(x, &e, 0);
    if (rc != KDL_OK) return rc;
    KDL_LAUNCH(kdl::exchange_signal_kernel, 1, 32, 0, (cudaStream_t)stream, e, epoch);
    return check_launch();
}

int kdl_exchange_wait(const kdl_exchange* x, int32_t epoch, void* stream) {
    kdl::Exchange e;
    int rc = make_exchange(x, &e, 0);
    if (rc != KDL_OK) return rc;
    dim3 grid((unsigned)(sm_count() * 2 / x->n_ranks + 1), (unsigned)x->n_ranks);
    KDL_LAUNCH(kdl::exchange_gather_kernel, grid, 256, 0, (cudaStream_t)stream, e, epoch);
    return check_launch();
}

extern "C++" template <class Vote>  // (a template cannot have C linkage)
int exchange_vote(const kdl_exchange* x, int64_t n_slots, int64_t min_depth_ceil, int32_t epoch, Vote vote,
                  void* stream) {
    if (n_slots <= 0 || (n_slots & 3)) return KDL_ERR_INVALID_ARG;
    kdl::Exchange e;
    int rc = make_exchange(x, &e, n_slots);
    if (rc != KDL_OK) return rc;
    if (x->slice_hi[x->rank] > n_slots) return KDL_ERR_INVALID_ARG;
    const long long quads = (x->slice_hi[x->rank] - x->slice_lo[x->rank]) / 4;
    long long grid = (quads + 255) / 256;
    const long long cap = (long long)sm_count() * 8;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;  // an empty slice still has to take part in the flag protocol
    KDL_LAUNCH(kdl::vote_exchange_kernel<Vote>, (unsigned)grid, 256, 0, (cudaStream_t)stream, e, n_slots,
               min_depth_ceil, epoch, vote);
    return check_launch();
}

int kdl_exchange_vote(const kdl_exchange* x, int64_t n_slots, int64_t min_depth_ceil, int32_t epoch,
                      void* stream) {
    return exchange_vote(x, n_slots, min_depth_ceil, epoch, kdl::MajorityVote{}, stream);
}

int kdl_exchange_vote_iupac(const kdl_exchange* x, int64_t n_slots, int64_t min_depth_ceil, double threshold,
                            int32_t epoch, void* stream) {
    if (!valid_threshold(threshold)) return KDL_ERR_INVALID_ARG;
    return exchange_vote(x, n_slots, min_depth_ceil, epoch, kdl::IupacVote{threshold}, stream);
}

int kdl_cdr_flags(const int32_t* counts, int64_t n_slots, int64_t slot_lo, int64_t slot_hi,
                  double clip_decay_threshold, uint8_t* flags, uint8_t* bases, void* stream) {
    if (!counts || !flags || !bases || n_slots <= 0 || slot_lo < 0 || slot_hi > n_slots || slot_lo > slot_hi)
        return KDL_ERR_INVALID_ARG;
    if (slot_hi == slot_lo) return KDL_OK;
    const long long grid = (slot_hi - slot_lo + 255) / 256;
    KDL_LAUNCH(kdl::cdr_flags_kernel, (unsigned)grid, 256, 0, (cudaStream_t)stream, counts, n_slots, slot_lo, slot_hi,
               clip_decay_threshold, flags, bases);
    return check_launch();
}

int64_t kdl_assemble_scratch_words(int64_t n_slots) {
    return n_slots < 0 ? 0 : (n_slots + 1 + kdl::A_BLOCK - 1) / kdl::A_BLOCK + 1;
}

int kdl_assemble(const uint8_t* calls, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                 int32_t n_contigs, const int64_t* ins_slot, const uint32_t* ins_off, const uint8_t* ins_bytes,
                 int64_t n_ins, uint32_t* block_sums, uint32_t* offsets, uint8_t* out, void* stream) {
    if (!calls || n_slots <= 0 || !contig_slot || !contig_len || n_contigs < 0 || n_ins < 0 || !block_sums || !offsets ||
        !out || (n_ins > 0 && (!ins_slot || !ins_off || !ins_bytes)))
        return KDL_ERR_INVALID_ARG;
    kdl::AssembleArgs a;
    a.calls = calls; a.n_slots = n_slots; a.contig_slot = contig_slot; a.contig_len = contig_len; a.n_contigs = n_contigs;
    a.ins_slot = ins_slot; a.ins_off = ins_off; a.ins_bytes = ins_bytes; a.n_ins = n_ins;
    const long long n_blocks = (n_slots + 1 + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    KDL_LAUNCH(kdl::assemble_sums_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, st, a, block_sums);
    if ((rc = check_launch()) != KDL_OK) return rc;
    KDL_LAUNCH(kdl::assemble_scan_sums_kernel, 1, kdl::A_THREADS, 0, st, block_sums, n_blocks);
    if ((rc = check_launch()) != KDL_OK) return rc;
    KDL_LAUNCH(kdl::assemble_scatter_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, st, a, block_sums, offsets, out);
    return check_launch();
}

int kdl_consensus_qual(const int32_t* counts, const uint8_t* calls, int64_t n_slots, uint8_t* qual, void* stream) {
    if (!counts || !calls || !qual || n_slots <= 0 || (n_slots & 3)) return KDL_ERR_INVALID_ARG;
    const long long grid = (n_slots / 4 + 255) / 256;
    KDL_LAUNCH(kdl::consensus_qual_kernel, (unsigned)grid, 256, 0, (cudaStream_t)stream, counts, calls, n_slots, qual);
    return check_launch();
}

int kdl_assemble_qual(const uint32_t* offsets, const uint8_t* qual, int64_t n_slots, const int64_t* ins_slot,
                      const uint8_t* ins_qual, int64_t n_ins, uint8_t* out, void* stream) {
    if (!offsets || !qual || !out || n_slots <= 0 || n_ins < 0 || (n_ins > 0 && (!ins_slot || !ins_qual)))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    KDL_LAUNCH(kdl::assemble_qual_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, (cudaStream_t)stream,
               offsets, qual, n_slots, ins_slot, ins_qual, n_ins, out);
    return check_launch();
}

int64_t kdl_variant_scratch_words(int64_t n_slots) {
    return n_slots < 0 ? 0 : (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK + 1;
}

static int variant_args(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                        int32_t n_contigs, int64_t abs_floor, double rel_threshold, kdl::VariantArgs* a) {
    // the scan counts sites in uint32; abs_floor outside [-1, 2^31] is a caller that skipped the clamp
    if (!counts || n_slots <= 0 || (n_slots & 3) || n_slots > (int64_t)UINT32_MAX || n_contigs < 0 ||
        (n_contigs > 0 && (!contig_slot || !contig_len)) || abs_floor < -1 || abs_floor > (1LL << 31))
        return KDL_ERR_INVALID_ARG;
    *a = kdl::VariantArgs{};
    a->counts = counts; a->n_slots = n_slots;
    a->layout.contig_slot = contig_slot; a->layout.contig_len = contig_len; a->layout.n_contigs = n_contigs;
    a->abs_floor = abs_floor; a->rel_threshold = rel_threshold;
    return KDL_OK;
}

int kdl_variant_count(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                      int32_t n_contigs, int64_t abs_floor, double rel_threshold, uint32_t* block_sums, void* stream) {
    kdl::VariantArgs a;
    int rc = variant_args(counts, n_slots, contig_slot, contig_len, n_contigs, abs_floor, rel_threshold, &a);
    if (rc != KDL_OK) return rc;
    if (!block_sums) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    cudaStream_t st = (cudaStream_t)stream;
    KDL_LAUNCH(kdl::variant_sums_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, st, a, block_sums);
    if ((rc = check_launch()) != KDL_OK) return rc;
    KDL_LAUNCH(kdl::assemble_scan_sums_kernel, 1, kdl::A_THREADS, 0, st, block_sums, n_blocks);
    return check_launch();
}

int kdl_variant_scatter(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                        int32_t n_contigs, int64_t abs_floor, double rel_threshold, const uint32_t* block_sums,
                        int64_t n_sites, int64_t* site_slot, int32_t* site_counts, uint8_t* site_mask, void* stream) {
    kdl::VariantArgs a;
    int rc = variant_args(counts, n_slots, contig_slot, contig_len, n_contigs, abs_floor, rel_threshold, &a);
    if (rc != KDL_OK) return rc;
    if (!block_sums || n_sites < 0 || n_sites > n_slots || (n_sites > 0 && (!site_slot || !site_counts || !site_mask)))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    KDL_LAUNCH(kdl::variant_scatter_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, (cudaStream_t)stream,
               a, block_sums, n_sites, site_slot, site_counts, site_mask);
    return check_launch();
}

static int variant_ref_args(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot,
                            const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                            double rel_threshold, kdl::RefVariantArgs* a) {
    kdl::VariantArgs v;
    int rc = variant_args(counts, n_slots, contig_slot, contig_len, n_contigs, abs_floor, rel_threshold, &v);
    if (rc != KDL_OK) return rc;
    if (!ref || (reinterpret_cast<uintptr_t>(ref) & 3)) return KDL_ERR_INVALID_ARG;
    *a = kdl::RefVariantArgs{};
    a->counts = counts; a->n_slots = n_slots; a->layout = v.layout; a->ref = ref;
    a->abs_floor = abs_floor; a->rel_threshold = rel_threshold;
    return KDL_OK;
}

int kdl_variant_ref_count(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                          int32_t n_contigs, const uint8_t* ref, int64_t abs_floor, double rel_threshold,
                          uint32_t* block_sums, void* stream) {
    kdl::RefVariantArgs a;
    int rc = variant_ref_args(counts, n_slots, contig_slot, contig_len, n_contigs, ref, abs_floor, rel_threshold, &a);
    if (rc != KDL_OK) return rc;
    if (!block_sums) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    cudaStream_t st = (cudaStream_t)stream;
    KDL_LAUNCH(kdl::variant_ref_sums_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, st, a, block_sums);
    if ((rc = check_launch()) != KDL_OK) return rc;
    KDL_LAUNCH(kdl::assemble_scan_sums_kernel, 1, kdl::A_THREADS, 0, st, block_sums, n_blocks);
    return check_launch();
}

int kdl_variant_ref_scatter(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot,
                            const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                            double rel_threshold, const uint32_t* block_sums, int64_t n_sites, int64_t* site_slot,
                            int32_t* site_counts, int64_t* site_dpa, uint8_t* site_mask, void* stream) {
    kdl::RefVariantArgs a;
    int rc = variant_ref_args(counts, n_slots, contig_slot, contig_len, n_contigs, ref, abs_floor, rel_threshold, &a);
    if (rc != KDL_OK) return rc;
    if (!block_sums || n_sites < 0 || n_sites > n_slots ||
        (n_sites > 0 && (!site_slot || !site_counts || !site_dpa || !site_mask)))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    KDL_LAUNCH(kdl::variant_ref_scatter_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, (cudaStream_t)stream,
               a, block_sums, n_sites, site_slot, site_counts, site_dpa, site_mask);
    return check_launch();
}

static int variant_multi_args(const int32_t* counts, int32_t n_samples, int64_t n_slots, const int64_t* contig_slot,
                              const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                              double rel_threshold, kdl::VariantArgs* v) {
    int rc = variant_args(counts, n_slots, contig_slot, contig_len, n_contigs, abs_floor, rel_threshold, v);
    if (rc != KDL_OK) return rc;
    if (n_samples < 1 || (ref && (reinterpret_cast<uintptr_t>(ref) & 3))) return KDL_ERR_INVALID_ARG;
    return KDL_OK;
}

int kdl_variant_multi_count(const int32_t* counts, int32_t n_samples, int64_t n_slots, const int64_t* contig_slot,
                            const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                            double rel_threshold, uint32_t* block_sums, void* stream) {
    kdl::VariantArgs v;
    int rc = variant_multi_args(counts, n_samples, n_slots, contig_slot, contig_len, n_contigs, ref, abs_floor,
                                rel_threshold, &v);
    if (rc != KDL_OK) return rc;
    if (!block_sums) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    cudaStream_t st = (cudaStream_t)stream;
    if (ref) {
        KDL_LAUNCH(kdl::variant_multi_sums_kernel<true>, (unsigned)n_blocks, kdl::A_THREADS, 0, st,
                   kdl::MultiVariantArgs<true>::make(v, n_samples, ref), block_sums);
    } else {
        KDL_LAUNCH(kdl::variant_multi_sums_kernel<false>, (unsigned)n_blocks, kdl::A_THREADS, 0, st,
                   kdl::MultiVariantArgs<false>::make(v, n_samples, ref), block_sums);
    }
    if ((rc = check_launch()) != KDL_OK) return rc;
    KDL_LAUNCH(kdl::assemble_scan_sums_kernel, 1, kdl::A_THREADS, 0, st, block_sums, n_blocks);
    return check_launch();
}

int kdl_variant_multi_scatter(const int32_t* counts, int32_t n_samples, int64_t n_slots, const int64_t* contig_slot,
                              const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                              double rel_threshold, const uint32_t* block_sums, int64_t n_sites, int64_t* site_slot,
                              uint8_t* site_mask, void* stream) {
    kdl::VariantArgs v;
    int rc = variant_multi_args(counts, n_samples, n_slots, contig_slot, contig_len, n_contigs, ref, abs_floor,
                                rel_threshold, &v);
    if (rc != KDL_OK) return rc;
    if (!block_sums || n_sites < 0 || n_sites > n_slots || (n_sites > 0 && (!site_slot || !site_mask)))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    cudaStream_t st = (cudaStream_t)stream;
    if (ref) {
        KDL_LAUNCH(kdl::variant_multi_scatter_kernel<true>, (unsigned)n_blocks, kdl::A_THREADS, 0, st,
                   kdl::MultiVariantArgs<true>::make(v, n_samples, ref), block_sums, n_sites, site_slot, site_mask);
    } else {
        KDL_LAUNCH(kdl::variant_multi_scatter_kernel<false>, (unsigned)n_blocks, kdl::A_THREADS, 0, st,
                   kdl::MultiVariantArgs<false>::make(v, n_samples, ref), block_sums, n_sites, site_slot, site_mask);
    }
    return check_launch();
}

int64_t kdl_deletion_scratch_words(int64_t n_reads) {
    return n_reads < 0 ? 0 : (n_reads + kdl::A_THREADS - 1) / kdl::A_THREADS + 1;
}

int kdl_deletion_count(const kdl_batch* batch, uint32_t* block_sums, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!block_sums || batch->n_reads > (int64_t)UINT32_MAX) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (batch->n_reads + kdl::A_THREADS - 1) / kdl::A_THREADS;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_blocks > 0) {
        KDL_LAUNCH(kdl::deletion_sums_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, st, *batch, block_sums);
        if ((rc = check_launch()) != KDL_OK) return rc;
    }
    KDL_LAUNCH(kdl::assemble_scan_sums_kernel, 1, kdl::A_THREADS, 0, st, block_sums, n_blocks);
    return check_launch();
}

int kdl_deletion_scatter(const kdl_batch* batch, const uint32_t* block_sums, int64_t n_events, int64_t* ev_slot,
                         int32_t* ev_len, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!block_sums || n_events < 0 || (n_events > 0 && (!ev_slot || !ev_len))) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (batch->n_reads + kdl::A_THREADS - 1) / kdl::A_THREADS;
    if (n_blocks == 0) return KDL_OK;
    KDL_LAUNCH(kdl::deletion_scatter_kernel, (unsigned)n_blocks, kdl::A_THREADS, 0, (cudaStream_t)stream,
               *batch, block_sums, n_events, ev_slot, ev_len);
    return check_launch();
}

int kdl_left_align_deletions(const int64_t* keys, int64_t n_keys, const int64_t* contig_slot, int32_t n_contigs,
                             const uint8_t* ref, int64_t* keys_out, void* stream) {
    if (n_keys < 0 || n_contigs < 0 || (n_keys > 0 && (!keys || !ref || !keys_out || (n_contigs > 0 && !contig_slot))))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_keys + kdl::LA_THREADS - 1) / kdl::LA_THREADS;
    if (n_blocks == 0) return KDL_OK;
    KDL_LAUNCH(kdl::left_align_deletions_kernel, (unsigned)n_blocks, kdl::LA_THREADS, 0, (cudaStream_t)stream,
               keys, n_keys, contig_slot, n_contigs, ref, keys_out);
    return check_launch();
}

int kdl_left_align_insertions(const kdl_batch* batch, const int32_t* ins_events, int64_t n_events, const uint8_t* dead,
                              const uint8_t* ref, int64_t* norm_slot, int32_t* rot, int32_t* hist, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (n_events < 0 || (n_events > 0 && (!ins_events || (reinterpret_cast<uintptr_t>(ins_events) & 15) || !ref ||
                                          !norm_slot || !rot || !hist)))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = (n_events + kdl::LA_THREADS - 1) / kdl::LA_THREADS;
    if (n_blocks == 0) return KDL_OK;
    KDL_LAUNCH(kdl::left_align_insertions_kernel, (unsigned)n_blocks, kdl::LA_THREADS, 0, (cudaStream_t)stream,
               *batch, ins_events, n_events, dead, ref, norm_slot, rot, hist);
    return check_launch();
}

static long long select_blocks(int64_t n_reads) { return (n_reads + kdl::S_THREADS) / kdl::S_THREADS; }

static int select_qmask(const kdl_qmask* qmask, kdl_qmask* q) {
    *q = kdl_qmask{};
    if (!qmask || qmask->n_reads == 0) return KDL_OK;
    if (qmask->n_reads < 0 || qmask->n_bases < 0 || !qmask->read_idx || !qmask->off || (qmask->n_bases > 0 && !qmask->qpos))
        return KDL_ERR_INVALID_ARG;
    *q = *qmask;
    return KDL_OK;
}

int64_t kdl_select_scratch_words(int64_t n_reads) {
    return n_reads < 0 ? 0 : (int64_t)kdl::S_REC * (select_blocks(n_reads) + 1);
}

int kdl_select_count(const kdl_batch* batch, const kdl_qmask* qmask, const uint8_t* keep, uint32_t* scratch,
                     void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    kdl_qmask q;
    if ((rc = select_qmask(qmask, &q)) != KDL_OK) return rc;
    if (!scratch || (batch->n_reads > 0 && !keep) || batch->n_reads >= (int64_t)UINT32_MAX) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = select_blocks(batch->n_reads);
    cudaStream_t st = (cudaStream_t)stream;
    KDL_LAUNCH(kdl::select_sums_kernel, (unsigned)n_blocks, kdl::S_THREADS, 0, st, *batch, q, keep, scratch);
    if ((rc = check_launch()) != KDL_OK) return rc;
    KDL_LAUNCH(kdl::select_combine_kernel, 1, kdl::S_THREADS, 0, st, scratch, n_blocks);
    return check_launch();
}

int kdl_select_scatter(const kdl_batch* batch, const kdl_qmask* qmask, const uint8_t* keep, const uint32_t* scratch,
                       const kdl_batch* out, const kdl_qmask* out_mask, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    kdl_qmask q, om;
    if ((rc = select_qmask(qmask, &q)) != KDL_OK || (rc = select_qmask(out_mask, &om)) != KDL_OK) return rc;
    if ((rc = validate_batch(out)) != KDL_OK) return rc;
    if (!scratch || (batch->n_reads > 0 && !keep) || batch->n_reads >= (int64_t)UINT32_MAX ||
        out->n_reads > batch->n_reads || out->n_contigs != batch->n_contigs || !out->contig_read_off ||
        (out->n_reads > 0 && out->seq4_words > 0 && !out->seq4))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = select_blocks(batch->n_reads);
    KDL_LAUNCH(kdl::select_scatter_kernel, (unsigned)n_blocks, kdl::S_THREADS, 0, (cudaStream_t)stream,
               *batch, q, keep, scratch, *out, const_cast<int64_t*>(out->contig_read_off), om);
    return check_launch();
}

static long long primer_blocks(int64_t n_reads) { return n_reads / kdl::P_BLOCK + 1; }

static int primer_args(const kdl_batch* batch, const kdl_qmask* qmask, const kdl_primers* primers, kdl_qmask* q) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if ((rc = select_qmask(qmask, q)) != KDL_OK) return rc;
    if (!primers || primers->n_contigs != batch->n_contigs || primers->n_intervals < 0 ||
        primers->n_intervals >= (int64_t)INT32_MAX || !primers->contig_off || batch->n_reads >= (int64_t)UINT32_MAX ||
        (primers->n_intervals > 0 && (!primers->start_sorted || !primers->end_max || !primers->end_sorted ||
                                      !primers->start_min)))
        return KDL_ERR_INVALID_ARG;
    return KDL_OK;
}

int64_t kdl_primers_scratch_words(int64_t n_reads) {
    return n_reads < 0 ? 0 : (int64_t)kdl::P_NROW * (primer_blocks(n_reads) + 1) + kdl::P_TOTALS;
}

int kdl_primers_count(const kdl_batch* batch, const kdl_qmask* qmask, const kdl_primers* primers, uint32_t* scratch,
                      void* stream) {
    kdl_qmask q;
    int rc = primer_args(batch, qmask, primers, &q);
    if (rc != KDL_OK) return rc;
    if (!scratch) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = primer_blocks(batch->n_reads);
    cudaStream_t st = (cudaStream_t)stream;
    KDL_LAUNCH(kdl::primers_sums_kernel, (unsigned)n_blocks, kdl::P_THREADS, 0, st, *batch, q, *primers, scratch,
               n_blocks);
    if ((rc = check_launch()) != KDL_OK) return rc;
    for (int k = kdl::P_MBASES; k <= kdl::P_MREADS; ++k) {
        KDL_LAUNCH(kdl::assemble_scan_sums_kernel, 1, kdl::A_THREADS, 0, st, scratch + (size_t)k * (n_blocks + 1),
                   n_blocks);
        if ((rc = check_launch()) != KDL_OK) return rc;
    }
    KDL_LAUNCH(kdl::primers_totals_kernel, 1, kdl::P_THREADS, 0, st, scratch, n_blocks);
    return check_launch();
}

int kdl_primers_apply(const kdl_batch* batch, const kdl_qmask* qmask, const kdl_primers* primers,
                      const uint32_t* scratch, uint32_t* seq4, const kdl_qmask* out_mask, void* stream) {
    kdl_qmask q, om;
    int rc = primer_args(batch, qmask, primers, &q);
    if (rc != KDL_OK) return rc;
    if ((rc = select_qmask(out_mask, &om)) != KDL_OK) return rc;
    if (!scratch || (batch->n_reads > 0 && !seq4) || (om.n_reads > 0 && om.n_bases > 0 && !om.qpos))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = primer_blocks(batch->n_reads);
    KDL_LAUNCH(kdl::primers_scatter_kernel, (unsigned)n_blocks, kdl::P_THREADS, 0, (cudaStream_t)stream, *batch, q,
               *primers, scratch, n_blocks, seq4, om);
    return check_launch();
}

static long long overlap_blocks(int64_t n_reads) { return n_reads / kdl::M_THREADS + 1; }

int kdl_mates_pair(const kdl_batch* batch, const uint64_t* name_hash, const int32_t* mate_start,
                   const uint8_t* pair_role, const int32_t* order, int64_t n_order, int32_t* mate, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (n_order < 0 || n_order > batch->n_reads || batch->n_reads >= (int64_t)INT32_MAX ||
        (batch->n_reads > 0 && !mate) || (n_order > 0 && (!name_hash || !mate_start || !pair_role || !order)))
        return KDL_ERR_INVALID_ARG;
    if (batch->n_reads == 0) return KDL_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const long long n = batch->n_reads;
    const long long grid = (n + kdl::M_THREADS - 1) / kdl::M_THREADS;
    KDL_LAUNCH(kdl::mates_clear_kernel, (unsigned)(grid < 4096 ? grid : 4096), kdl::M_THREADS, 0, st, mate, n);
    if ((rc = check_launch()) != KDL_OK || n_order < 2) return rc;
    KDL_LAUNCH(kdl::mates_pair_kernel, (unsigned)((n_order + kdl::M_THREADS - 1) / kdl::M_THREADS), kdl::M_THREADS, 0,
               st, *batch, name_hash, mate_start, pair_role, order, n_order, mate);
    return check_launch();
}

static int overlap_args(const kdl_batch* batch, const kdl_qmask* qmask, const int32_t* mate, kdl_qmask* q) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if ((rc = select_qmask(qmask, q)) != KDL_OK) return rc;
    if ((batch->n_reads > 0 && !mate) || batch->n_reads >= (int64_t)INT32_MAX) return KDL_ERR_INVALID_ARG;
    return KDL_OK;
}

int64_t kdl_overlap_scratch_words(int64_t n_reads) {
    return n_reads < 0 ? 0 : (int64_t)kdl::M_NROW * (overlap_blocks(n_reads) + 1) + kdl::M_TOTALS;
}

int kdl_overlap_count(const kdl_batch* batch, const kdl_qmask* qmask, const int32_t* mate, uint32_t* scratch,
                      void* stream) {
    kdl_qmask q;
    int rc = overlap_args(batch, qmask, mate, &q);
    if (rc != KDL_OK) return rc;
    if (!scratch) return KDL_ERR_INVALID_ARG;
    const long long n_blocks = overlap_blocks(batch->n_reads);
    cudaStream_t st = (cudaStream_t)stream;
    KDL_LAUNCH(kdl::overlap_sums_kernel, (unsigned)n_blocks, kdl::M_THREADS, 0, st, *batch, q, mate, scratch, n_blocks);
    if ((rc = check_launch()) != KDL_OK) return rc;
    for (int k = 0; k < kdl::M_NSCAN; ++k) {
        KDL_LAUNCH(kdl::assemble_scan_sums_kernel, 1, kdl::A_THREADS, 0, st, scratch + (size_t)k * (n_blocks + 1),
                   n_blocks);
        if ((rc = check_launch()) != KDL_OK) return rc;
    }
    KDL_LAUNCH(kdl::overlap_totals_kernel, 1, kdl::M_THREADS, 0, st, scratch, n_blocks);
    return check_launch();
}

int kdl_overlap_apply(const kdl_batch* batch, const kdl_qmask* qmask, const int32_t* mate, const uint32_t* scratch,
                      uint32_t* seq4, const kdl_qmask* out_mask, int32_t* drops, int64_t n_drops, void* stream) {
    kdl_qmask q, om;
    int rc = overlap_args(batch, qmask, mate, &q);
    if (rc != KDL_OK) return rc;
    if ((rc = select_qmask(out_mask, &om)) != KDL_OK) return rc;
    if (!scratch || (batch->n_reads > 0 && !seq4) || (om.n_reads > 0 && om.n_bases > 0 && !om.qpos) || n_drops < 0 ||
        (n_drops > 0 && !drops))
        return KDL_ERR_INVALID_ARG;
    const long long n_blocks = overlap_blocks(batch->n_reads);
    KDL_LAUNCH(kdl::overlap_scatter_kernel, (unsigned)n_blocks, kdl::M_THREADS, 0, (cudaStream_t)stream, *batch, q,
               mate, scratch, n_blocks, seq4, om, drops, n_drops);
    return check_launch();
}

int kdl_overlap_untake(const int32_t* drops, int64_t n_drops, int32_t* counts, int64_t n_slots, void* stream) {
    if (n_drops < 0 || n_slots <= 0 || !counts || (n_drops > 0 && !drops)) return KDL_ERR_INVALID_ARG;
    if (n_drops == 0) return KDL_OK;
    KDL_LAUNCH(kdl::overlap_untake_kernel, (unsigned)((n_drops + kdl::M_THREADS - 1) / kdl::M_THREADS),
               kdl::M_THREADS, 0, (cudaStream_t)stream, drops, n_drops, counts, n_slots);
    return check_launch();
}

static bool amplicons_ok(const kdl_amplicons* a, int32_t n_contigs) {
    return a && a->n_contigs == n_contigs && a->n_amplicons >= 0 && a->left_off && a->right_off &&
           (a->n_amplicons == 0 || (a->left_at && a->left_label && a->right_at && a->right_label && a->amp_contig &&
                                    a->insert_start && a->insert_end));
}

int kdl_amplicons_assign(const kdl_batch* batch, const kdl_amplicons* amplicons, int32_t* label, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!amplicons_ok(amplicons, batch->n_contigs) || (batch->n_reads > 0 && !label)) return KDL_ERR_INVALID_ARG;
    if (batch->n_reads == 0) return KDL_OK;
    KDL_LAUNCH(kdl::amplicons_assign_kernel, (unsigned)((batch->n_reads + kdl::AM_THREADS - 1) / kdl::AM_THREADS),
               kdl::AM_THREADS, 0, (cudaStream_t)stream, *batch, *amplicons, label);
    return check_launch();
}

int kdl_amplicons_depth(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                        int32_t n_contigs, const kdl_amplicons* amplicons, int64_t min_depth, int64_t* stats,
                        void* stream) {
    if (!counts || n_slots <= 0 || n_contigs < 0 || !amplicons_ok(amplicons, n_contigs)) return KDL_ERR_INVALID_ARG;
    if (amplicons->n_amplicons == 0) return KDL_OK;
    if (!stats || !contig_slot || !contig_len) return KDL_ERR_INVALID_ARG;
    const long long n = amplicons->n_amplicons;
    KDL_LAUNCH(kdl::amplicons_depth_kernel, (unsigned)((n + kdl::AM_WARPS - 1) / kdl::AM_WARPS), kdl::AM_THREADS, 0,
               (cudaStream_t)stream, counts, n_slots, contig_slot, contig_len, n_contigs, *amplicons, min_depth,
               reinterpret_cast<long long*>(stats));
    return check_launch();
}

// K13's grid: G CTAs of `per` tiles each over the batch's ceil(n / NM_THREADS) tiles -- two per SM as the persistent
// grids, no more than there are tiles, and so few that H (G * K int32) stays within KDL_NORMALISE_MAX_WORDS (one CTA
// when K alone exceeds it)
static int normalise_grid(long long n_reads, long long n_keys, long long* per) {
    const long long tiles = n_reads > 0 ? (n_reads + kdl::NM_THREADS - 1) / kdl::NM_THREADS : 1;
    long long g = (long long)sm_count() * 2;
    if (g > tiles) g = tiles;
    if (n_keys > 0 && g > KDL_NORMALISE_MAX_WORDS / n_keys) g = KDL_NORMALISE_MAX_WORDS / n_keys;
    if (g < 1) g = 1;
    *per = (tiles + g - 1) / g;
    return (int)((tiles + *per - 1) / *per);
}

int64_t kdl_normalise_scratch_words(int64_t n_reads, int32_t n_amplicons) {
    if (n_reads < 0 || n_amplicons < 0 || n_amplicons > (1 << 30)) return -1;
    long long per;
    return (int64_t)normalise_grid(n_reads, 2ll * n_amplicons, &per) * 2ll * n_amplicons;
}

int kdl_normalise(const int32_t* label, const uint8_t* reverse, int64_t n_reads, int32_t n_amplicons, int64_t cap,
                  int32_t* scratch, int64_t scratch_words, uint8_t* keep, int32_t* total, int64_t* dropped,
                  void* stream) {
    if (n_reads < 0 || n_amplicons < 0 || n_amplicons > (1 << 30) || cap < 1 || !dropped) return KDL_ERR_INVALID_ARG;
    if (n_reads > 0 && (!label || !reverse || !keep)) return KDL_ERR_INVALID_ARG;
    const long long K = 2ll * n_amplicons;
    long long per;
    const int grid = normalise_grid(n_reads, K, &per);
    if (K > 0 && (!total || !scratch || scratch_words < (long long)grid * K)) return KDL_ERR_INVALID_ARG;
    const cudaStream_t st = (cudaStream_t)stream;
    long long* drop = reinterpret_cast<long long*>(dropped);
    KDL_LAUNCH(kdl::normalise_count_kernel, (unsigned)grid, kdl::NM_THREADS, 0, st, label, reverse, n_reads,
               n_amplicons, per, scratch, drop);
    int rc = check_launch();
    if (rc != KDL_OK) return rc;
    if (K > 0) {
        KDL_LAUNCH(kdl::normalise_scan_kernel, (unsigned)((K + kdl::NM_THREADS - 1) / kdl::NM_THREADS),
                   kdl::NM_THREADS, 0, st, scratch, grid, n_amplicons, cap, total, drop);
        rc = check_launch();
        if (rc != KDL_OK) return rc;
    }
    if (n_reads == 0) return KDL_OK;
    KDL_LAUNCH(kdl::normalise_mark_kernel, (unsigned)grid, kdl::NM_THREADS, 0, st, label, reverse, n_reads, n_amplicons,
               per, cap, scratch, keep);
    return check_launch();
}

// K14's grids: one thread per read (K14k) or per sorted entry (K14s), at least one CTA
static long long dedup_ctas(long long items) { return items > 0 ? (items + kdl::DD_THREADS - 1) / kdl::DD_THREADS : 1; }

static bool dedup_lists_ok(const kdl_dedup_lists* l) {
    return l && l->pair_contig && l->pair_e1 && l->pair_e2 && l->pair_rank && l->pair_r1 && l->pair_r2 &&
           l->single_contig && l->single_key && l->single_rank && l->single_read && l->end && l->paired;
}

int kdl_dedup_entries(const kdl_batch* batch, const uint8_t* reverse, const int32_t* dup_score, const int32_t* mate,
                      const kdl_dedup_lists* lists, uint8_t* keep, int64_t* totals, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!totals || (batch->n_reads > 0 && (!reverse || !dup_score || !keep || !dedup_lists_ok(lists))))
        return KDL_ERR_INVALID_ARG;
    const cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)dedup_ctas(batch->n_reads);
    unsigned long long* tot = reinterpret_cast<unsigned long long*>(totals);
    kdl_dedup_lists l = {};
    if (lists) l = *lists;
    KDL_LAUNCH(kdl::dedup_ends_kernel, grid, kdl::DD_THREADS, 0, st, *batch, reverse, dup_score, l.end, l.paired, keep,
               tot);
    if ((rc = check_launch()) != KDL_OK || batch->n_reads == 0) return rc;
    if (mate) {
        KDL_LAUNCH(kdl::dedup_pairs_kernel, grid, kdl::DD_THREADS, 0, st, *batch, dup_score, mate, l, l.end, l.paired,
                   tot);
        if ((rc = check_launch()) != KDL_OK) return rc;
    }
    KDL_LAUNCH(kdl::dedup_singles_kernel, grid, kdl::DD_THREADS, 0, st, *batch, dup_score, l, l.end, l.paired, tot);
    return check_launch();
}

int64_t kdl_dedup_scratch_words(int64_t n_entries) {
    if (n_entries < 0 || n_entries >= (1ll << 31)) return -1;
    return 3 * n_entries + 2 * dedup_ctas(n_entries);
}

int kdl_dedup_select(const kdl_dedup_lists* lists, const int64_t* pair_order, int64_t n_pairs,
                     const int64_t* single_order, int64_t n_singles, int32_t* scratch, int64_t scratch_words,
                     uint8_t* keep, int64_t* totals, void* stream) {
    if (n_pairs < 0 || n_singles < 0 || n_pairs >= (1ll << 31) || n_singles >= (1ll << 31) || !totals)
        return KDL_ERR_INVALID_ARG;
    if (n_pairs + n_singles == 0) return KDL_OK;
    const long long need = kdl_dedup_scratch_words(n_pairs > n_singles ? n_pairs : n_singles);
    if (!dedup_lists_ok(lists) || !keep || !scratch || scratch_words < need || (n_pairs > 0 && !pair_order) ||
        (n_singles > 0 && !single_order))
        return KDL_ERR_INVALID_ARG;
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* tot = reinterpret_cast<unsigned long long*>(totals);
    const kdl_dedup_lists& l = *lists;
    const kdl::DedupList pairs = {pair_order, n_pairs, l.pair_contig, l.pair_e1, l.pair_e2,
                                  reinterpret_cast<const unsigned long long*>(l.pair_rank), l.pair_r1, l.pair_r2};
    const kdl::DedupList singles = {single_order, n_singles, l.single_contig, l.single_key, nullptr,
                                    reinterpret_cast<const unsigned long long*>(l.single_rank), l.single_read, nullptr};
    int rc = KDL_OK;
    for (const kdl::DedupList& L : {pairs, singles}) {  // (one after the other on the stream: the scratch is reused)
        if (L.m == 0) continue;
        const long long ctas = dedup_ctas(L.m);
        unsigned long long* best = reinterpret_cast<unsigned long long*>(scratch);
        int32_t* run = scratch + 2 * L.m;
        int32_t* cta_head = run + L.m;
        int32_t* carry = cta_head + ctas;
        KDL_LAUNCH(kdl::dedup_heads_kernel, (unsigned)ctas, kdl::DD_THREADS, 0, st, L, best, cta_head);
        if ((rc = check_launch()) != KDL_OK) return rc;
        KDL_LAUNCH(kdl::dedup_carry_kernel, 1, kdl::DD_THREADS, 0, st, cta_head, carry, ctas);
        if ((rc = check_launch()) != KDL_OK) return rc;
        KDL_LAUNCH(kdl::dedup_best_kernel, (unsigned)ctas, kdl::DD_THREADS, 0, st, L, carry, run, best);
        if ((rc = check_launch()) != KDL_OK) return rc;
        KDL_LAUNCH(kdl::dedup_mark_kernel, (unsigned)ctas, kdl::DD_THREADS, 0, st, L, run, best, keep, tot);
        if ((rc = check_launch()) != KDL_OK) return rc;
    }
    return rc;
}

// K0 + K11 + K11g of one sum policy (kdl::PhredSums or kdl::WeightSums, quality.cu), arguments checked
extern "C++" template <class Sums>
int quality_launch(const kdl_batch* batch, const uint8_t* qual8, Sums sums, int64_t n_slots, cudaStream_t st) {
    int rc;
    const int cap = sm_count() * 8;
    // the tile-owner path under the conditions of kdl_pileup_range's
    const bool tiled = batch->n_reads > batch->n_hard && (n_slots % KDL_TILE) == 0 && batch->reads_sorted &&
                       batch->tile_index && batch->reach_right > 0 &&
                       batch->reach_right <= KDL_FAST_MAXLEN + KDL_TILE_MAXREACH;
    if (tiled) {
        const long long n_tiles = n_slots / KDL_TILE;
        KDL_LAUNCH(kdl::tile_index_kernel, (unsigned)((n_tiles * 32 + 255) / 256), 256, 0, st, *batch, 0ll, n_tiles,
                   batch->tile_index);  // K0, into the caller's scratch: no ordering dependency on kdl_pileup
        if ((rc = check_launch()) != KDL_OK) return rc;
        KDL_LAUNCH(kdl::quality_tile_kernel<Sums>, (unsigned)n_tiles, kdl::kQtThreads, 0, st, *batch, qual8, sums,
                   n_slots, batch->tile_index);
        if ((rc = check_launch()) != KDL_OK) return rc;
        if (batch->n_hard == 0) return KDL_OK;
        KDL_LAUNCH(kdl::quality_general_kernel<Sums>, grid_for(batch->n_hard, 8, cap), 256, 0, st, *batch, qual8,
                   batch->hard_idx, batch->n_hard, sums, n_slots);
        return check_launch();
    }
    KDL_LAUNCH(kdl::quality_zero_kernel<Sums>, sm_count() * 4, 256, 0, st, sums, n_slots);
    if ((rc = check_launch()) != KDL_OK) return rc;
    if (batch->n_reads == 0) return KDL_OK;
    KDL_LAUNCH(kdl::quality_general_kernel<Sums>, grid_for(batch->n_reads, 8, cap), 256, 0, st, *batch, qual8, nullptr,
               batch->n_reads, sums, n_slots);
    return check_launch();
}

int kdl_quality_pileup(const kdl_batch* batch, const uint8_t* qual8, uint32_t* qsum, uint64_t* emass, int64_t n_slots,
                       void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!qsum || !emass || n_slots <= 0 || (n_slots & 3) || (batch->n_reads > 0 && !qual8) ||
        (reinterpret_cast<uintptr_t>(qual8) & 7) || (reinterpret_cast<uintptr_t>(qsum) & 15) ||
        (reinterpret_cast<uintptr_t>(emass) & 15))
        return KDL_ERR_INVALID_ARG;
    unsigned long long* em = reinterpret_cast<unsigned long long*>(emass);
    return quality_launch(batch, qual8, kdl::PhredSums{qsum, em}, n_slots, (cudaStream_t)stream);
}

int kdl_quality_weights(const kdl_batch* batch, const uint8_t* qual8, uint64_t* wsum, int64_t n_slots, void* stream) {
    int rc = validate_batch(batch);
    if (rc != KDL_OK) return rc;
    if (!wsum || n_slots <= 0 || (n_slots & 3) || (batch->n_reads > 0 && !qual8) ||
        (reinterpret_cast<uintptr_t>(qual8) & 7) || (reinterpret_cast<uintptr_t>(wsum) & 15))
        return KDL_ERR_INVALID_ARG;
    return quality_launch(batch, qual8, kdl::WeightSums{reinterpret_cast<unsigned long long*>(wsum)}, n_slots,
                          (cudaStream_t)stream);
}

int kdl_vote_quality(const int32_t* counts, const uint64_t* wsum, int64_t n_slots, int64_t min_depth_ceil,
                     uint8_t* calls, uint8_t* qual, void* stream) {
    if (!counts || !wsum || !calls || n_slots <= 0 || (n_slots & 3)) return KDL_ERR_INVALID_ARG;
    kdl::Peers none;
    none.n = 0;
    const long long quads = n_slots / 4;
    const long long grid = (quads + 255) / 256;
    KDL_LAUNCH((kdl::vote_kernel<false, kdl::QualityVote>), (unsigned)grid, 256, 0, (cudaStream_t)stream,
               counts, none, n_slots, 0, n_slots, min_depth_ceil, calls, nullptr,
               kdl::QualityVote{reinterpret_cast<const unsigned long long*>(wsum), n_slots, qual});
    return check_launch();
}

#ifndef KDL_HOST_EMU  // device memory and IPC handles: nothing the kernel emulator can stand in for
int kdl_table_alloc(int64_t bytes, void** dev_ptr) {
    if (!dev_ptr || bytes <= 0) return KDL_ERR_INVALID_ARG;
    *dev_ptr = nullptr;
    if (cudaMalloc(dev_ptr, (size_t)bytes) != cudaSuccess) return KDL_ERR_CUDA;
    if (cudaMemset(*dev_ptr, 0, (size_t)bytes) != cudaSuccess) return KDL_ERR_CUDA;
    return KDL_OK;
}
int kdl_table_free(void* dev_ptr) { return cudaFree(dev_ptr) == cudaSuccess ? KDL_OK : KDL_ERR_CUDA; }
int kdl_ipc_export(void* dev_ptr, uint8_t handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    if (!dev_ptr || !handle) return KDL_ERR_INVALID_ARG;
    cudaIpcMemHandle_t h;
    if (cudaIpcGetMemHandle(&h, dev_ptr) != cudaSuccess) return KDL_ERR_CUDA;
    std::memcpy(handle, &h, 64);
    return KDL_OK;
}
int kdl_ipc_open(const uint8_t handle[64], void** dev_ptr) {
    if (!dev_ptr || !handle) return KDL_ERR_INVALID_ARG;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle, 64);
    return cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess ? KDL_OK : KDL_ERR_CUDA;
}
int kdl_ipc_close(void* dev_ptr) { return cudaIpcCloseMemHandle(dev_ptr) == cudaSuccess ? KDL_OK : KDL_ERR_CUDA; }
#endif

int kdl_vote_peers_sparse(const int32_t* const* peer_counts, const int64_t* foot_lo, const int64_t* foot_hi,
                          int32_t n_peers, int64_t n_slots, int64_t slot_lo, int64_t slot_hi,
                          int64_t min_depth_ceil, uint8_t* calls, int32_t* reduced, void* stream) {
    if (!peer_counts || n_peers < 1 || n_peers > 16 || !calls || n_slots <= 0 || (n_slots & 3) ||
        slot_lo < 0 || slot_hi > n_slots || (slot_lo & 3) || (slot_hi & 3))
        return KDL_ERR_INVALID_ARG;
    if (slot_hi <= slot_lo) return KDL_OK;
    kdl::Peers peers;
    peers.n = n_peers;
    for (int p = 0; p < n_peers; ++p) {
        if (!peer_counts[p]) return KDL_ERR_INVALID_ARG;
        peers.tab[p] = peer_counts[p];
        peers.lo[p] = foot_lo ? foot_lo[p] : 0;
        peers.hi[p] = foot_hi ? foot_hi[p] : n_slots;
        if ((peers.lo[p] & 3) || (peers.hi[p] & 3)) return KDL_ERR_INVALID_ARG;
    }
    const long long quads = (slot_hi - slot_lo) / 4;
    const long long grid = (quads + 255) / 256;
    KDL_LAUNCH(kdl::vote_kernel<true>, (unsigned)grid, 256, 0, (cudaStream_t)stream,
               nullptr, peers, n_slots, slot_lo, slot_hi, min_depth_ceil, calls, reduced, kdl::MajorityVote{});
    return check_launch();
}

}  // extern "C"

#ifndef KDL_HOST_EMU
#include "host_ctx.inl"
#endif
