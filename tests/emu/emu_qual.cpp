// emu_qual.cpp -- TEST INFRASTRUCTURE: the consensus-quality kernels K2q and K5q (kindel_b200/csrc/assemble.cu), with
// K5 in front of K5q, compiled for the host and run under tests/emu/cuda_emu.h, as emu_iupac.cpp does for the vote.
// The kernel sources are included as they are; nothing here is part of the product.
#define KDL_HOST_EMU 1
#include "cuda_emu.h"

#include "../../kindel_b200/csrc/kdl_common.cuh"
#include "../../kindel_b200/csrc/assemble.cu"

static char g_error[512];

#define EMU_RUN(grid, block, ...)                                              \
    do {                                                                        \
        const char* e_ = emu::launch((unsigned)(grid), (unsigned)(block), [&] { __VA_ARGS__; }); \
        if (e_) { snprintf(g_error, sizeof g_error, "%s", e_); return 1; }      \
    } while (0)

extern "C" {

const char* emu_qual_last_error() { return g_error; }

// 0: threads in order (default), 1: reverse order, 2: a fresh pseudo-random order every scheduler round
void emu_qual_set_schedule(int mode, unsigned long long seed) {
    emu::M().schedule = mode;
    emu::M().rng = seed * 0x9E3779B97F4A7C15ull + 1;
}

// K2q as kdl_consensus_qual launches it.  HOST pointers.
int emu_consensus_qual(const int32_t* counts, const uint8_t* calls, long long n_slots, uint8_t* qual) {
    g_error[0] = 0;
    EMU_RUN((n_slots / 4 + 255) / 256, 256, kdl::consensus_qual_kernel(counts, calls, n_slots, qual));
    return 0;
}

// K5 (as kdl_assemble) and then K5q (as kdl_assemble_qual) on its offsets.  HOST pointers.
int emu_assemble_qual(const uint8_t* calls, const uint8_t* qual, long long n_slots, const int64_t* contig_slot,
                      const int32_t* contig_len, int n_contigs, const int64_t* ins_slot, const uint32_t* ins_off,
                      const uint8_t* ins_bytes, const uint8_t* ins_qual, long long n_ins, uint32_t* block_sums,
                      uint32_t* offsets, uint8_t* out, uint8_t* qout) {
    g_error[0] = 0;
    kdl::AssembleArgs a;
    a.calls = calls; a.n_slots = n_slots; a.contig_slot = contig_slot; a.contig_len = contig_len; a.n_contigs = n_contigs;
    a.ins_slot = ins_slot; a.ins_off = ins_off; a.ins_bytes = ins_bytes; a.n_ins = n_ins;
    const long long n_blocks = (n_slots + 1 + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    EMU_RUN(n_blocks, kdl::A_THREADS, kdl::assemble_sums_kernel(a, block_sums));
    EMU_RUN(1, kdl::A_THREADS, kdl::assemble_scan_sums_kernel(block_sums, n_blocks));
    EMU_RUN(n_blocks, kdl::A_THREADS, kdl::assemble_scatter_kernel(a, block_sums, offsets, out));
    const long long q_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    EMU_RUN(q_blocks, kdl::A_THREADS,
            kdl::assemble_qual_kernel(offsets, qual, n_slots, ins_slot, ins_qual, n_ins, qout));
    return 0;
}

}  // extern "C"
