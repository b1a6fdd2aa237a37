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
    int split = 1;
    if (tiled && n_tiles > 0) {
        const long long slots = (long long)sm_count() * 2;
        if (n_tiles < slots) {
            long long want = (slots + n_tiles - 1) / n_tiles;
            const long long deep = batch->n_reads / (n_tiles * 256);  // at least ~256 reads per unit
            if (want > deep) want = deep;
            split = (int)(want < 1 ? 1 : (want > 32 ? 32 : want));
        }
        if (const char* ev = getenv("KDL_SPLIT")) { const int v = atoi(ev); if (v >= 1 && v <= 64) split = v; }
    }
    bool cx_by_atomics = (batch->n_complex - batch->n_hard) * 16 < batch->n_reads;
    if (const char* ev = getenv("KDL_CX")) cx_by_atomics = !strcmp(ev, "atomics") ? true : (!strcmp(ev, "pieces") ? false : cx_by_atomics);
    // zeroing that the chosen kernels will not do themselves: the tile kernel overwrites the weight columns of a
    // fresh table and, on request, zeroes columns 5..18 window by window in its flush (only the sectors the map marks)
    const int zero_in_k1 = (tiled && split == 1 && fresh && n_tiles > 0 && (flags & KDL_PILEUP_ZERO_REST)) ? 1 : 0;
    const int zero_from = (fresh && !(tiled && split == 1)) ? 0 : 5;
    const int zero_to = ((flags & KDL_PILEUP_ZERO_REST) && !zero_in_k1) ? KDL_NCOL : 5;
    const bool zero_pass = zero_to > zero_from && slot_hi > slot_lo;
    // The dirty-sector map.  Complex reads this dense (>= 1 in 16; a few per cent of sectors stay clean at 1 in 100)
    // dirty nearly every sector: instead of K1e / K1g marking op by op, the kernel that zeroes -- K1's flush, or the
    // zeroing pass -- leaves every record of the range set, and the next pileup zeroes all of it.  Where neither runs,
    // the writers mark.
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
            // runs and K1e counts their bases too, with REDs
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
        if (batch->n_complex > batch->n_hard) {  // K1e: insertions / deletions / clips of the tile-eligible complex reads
            if (cx_by_atomics)  // their bases too: 8 lanes per read
                KDL_LAUNCH(kdl::pileup_events_kernel<8>, (unsigned)((batch->n_complex + 31) / 32), 256, 0, st,
                           *batch, counts, n_slots, ins_events, 1, mark_map);
            else                // a few scattered REDs per read: one thread per read
                KDL_LAUNCH(kdl::pileup_events_kernel<1>, (unsigned)((batch->n_complex + 255) / 256), 256, 0, st,
                           *batch, counts, n_slots, ins_events, 0, mark_map);
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
