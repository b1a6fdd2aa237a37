// emu_iupac.cpp -- TEST INFRASTRUCTURE: the IUPAC vote (K2 and K2x with IupacVote, kindel_b200/csrc/vote.cu), K4 and K5
// (assemble.cu) compiled for the host and run under tests/emu/cuda_emu.h, as emu_pileup.cpp does for the other
// kernels.  The kernel sources are included as they are; nothing here is part of the product.
#define KDL_HOST_EMU 1
#include "cuda_emu.h"

#include <vector>

#include "../../kindel_b200/csrc/kdl_common.cuh"
#include "../../kindel_b200/csrc/vote.cu"
#include "../../kindel_b200/csrc/assemble.cu"

static char g_error[512];

#define EMU_RUN(grid, block, ...)                                              \
    do {                                                                        \
        const char* e_ = emu::launch((unsigned)(grid), (unsigned)(block), [&] { __VA_ARGS__; }); \
        if (e_) { snprintf(g_error, sizeof g_error, "%s", e_); return 1; }      \
    } while (0)

extern "C" {

const char* emu_iupac_last_error() { return g_error; }

// 0: threads in order (default), 1: reverse order, 2: a fresh pseudo-random order every scheduler round
void emu_iupac_set_schedule(int mode, unsigned long long seed) {
    emu::M().schedule = mode;
    emu::M().rng = seed * 0x9E3779B97F4A7C15ull + 1;
}

// K2 with the IUPAC vote, as kdl_vote_iupac launches it.  HOST pointers.
int emu_vote_iupac(const int32_t* counts, long long n_slots, long long min_depth_ceil, double threshold, uint8_t* calls) {
    g_error[0] = 0;
    kdl::Peers none;
    none.n = 0;
    const kdl::IupacVote vote{threshold};
    EMU_RUN((n_slots / 4 + 255) / 256, 256,
            kdl::vote_kernel<false, kdl::IupacVote>(counts, none, n_slots, 0, n_slots, min_depth_ceil, calls, nullptr, vote));
    return 0;
}

// One epoch of the fused exchange with the IUPAC vote for ALL ranks on one machine (as emu_exchange_epoch in
// emu_pileup.cpp): the ready flags first, every rank's K2x (kdl_exchange_vote_iupac), then every rank's K2g.
int emu_exchange_epoch_iupac(const kdl_exchange* xs, int n_ranks, long long n_slots, long long min_depth_ceil,
                             double threshold, int epoch, int grid) {
    g_error[0] = 0;
    const kdl::IupacVote vote{threshold};
    std::vector<kdl::Exchange> ex(n_ranks);
    for (int r = 0; r < n_ranks; ++r) {
        const kdl_exchange& x = xs[r];
        kdl::Exchange& e = ex[r];
        e.peers.n = x.n_ranks;
        e.rank = x.rank;
        e.counter = x.counter;
        for (int p = 0; p < x.n_ranks; ++p) {
            e.peers.tab[p] = x.tables[p];
            e.peers.lo[p] = x.foot_lo[p];
            e.peers.hi[p] = x.foot_hi[p] > n_slots ? n_slots : x.foot_hi[p];
            e.calls[p] = x.calls[p];
            e.ready[p] = x.ready[p];
            e.done[p] = x.done[p];
            e.slice_lo[p] = x.slice_lo[p];
            e.slice_hi[p] = x.slice_hi[p];
        }
        e.ready_local = x.ready[x.rank];
        e.done_local = x.done[x.rank];
    }
    for (int r = 0; r < n_ranks; ++r) EMU_RUN(1, 32, kdl::exchange_signal_kernel(ex[r], epoch));
    for (int r = 0; r < n_ranks; ++r)
        EMU_RUN(grid, 256, kdl::vote_exchange_kernel<kdl::IupacVote>(ex[r], n_slots, min_depth_ceil, epoch, vote));
    for (int r = 0; r < n_ranks; ++r) {
        for (int p = 0; p < n_ranks; ++p) {  // blockIdx.y = peer: the emulator's grid is one-dimensional
            const char* e_ = emu::launch_y((unsigned)grid, (unsigned)p, (unsigned)n_ranks, 256,
                                           [&] { kdl::exchange_gather_kernel(ex[r], epoch); });
            if (e_) { snprintf(g_error, sizeof g_error, "%s", e_); return 1; }
        }
    }
    return 0;
}

// K4 as kdl_cdr_flags launches it: flags and bases of slots [slot_lo, slot_hi).  HOST pointers.
int emu_cdr_flags(const int32_t* counts, long long n_slots, long long slot_lo, long long slot_hi, double decay,
                  uint8_t* flags, uint8_t* bases) {
    g_error[0] = 0;
    if (slot_hi <= slot_lo) return 0;
    EMU_RUN((slot_hi - slot_lo + 255) / 256, 256, kdl::cdr_flags_kernel(counts, n_slots, slot_lo, slot_hi, decay, flags, bases));
    return 0;
}

// K5 as kdl_assemble launches it (sums, scan of the block sums, scatter).  HOST pointers.
int emu_assemble(const uint8_t* calls, long long n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                 int n_contigs, const int64_t* ins_slot, const uint32_t* ins_off, const uint8_t* ins_bytes, long long n_ins,
                 uint32_t* block_sums, uint32_t* offsets, uint8_t* out) {
    g_error[0] = 0;
    kdl::AssembleArgs a;
    a.calls = calls; a.n_slots = n_slots; a.contig_slot = contig_slot; a.contig_len = contig_len; a.n_contigs = n_contigs;
    a.ins_slot = ins_slot; a.ins_off = ins_off; a.ins_bytes = ins_bytes; a.n_ins = n_ins;
    const long long n_blocks = (n_slots + 1 + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    EMU_RUN(n_blocks, kdl::A_THREADS, kdl::assemble_sums_kernel(a, block_sums));
    EMU_RUN(1, kdl::A_THREADS, kdl::assemble_scan_sums_kernel(block_sums, n_blocks));
    EMU_RUN(n_blocks, kdl::A_THREADS, kdl::assemble_scatter_kernel(a, block_sums, offsets, out));
    return 0;
}

}  // extern "C"
