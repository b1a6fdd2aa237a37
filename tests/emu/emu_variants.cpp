// emu_variants.cpp -- TEST INFRASTRUCTURE: the variant-site kernels K6 (kindel_b200/csrc/variants.cu), with K5's scan
// kernel between them, compiled for the host and run under tests/emu/cuda_emu.h, as emu_qual.cpp does for K2q / K5q.
// The kernel sources are included as they are; nothing here is part of the product.
#define KDL_HOST_EMU 1
#include "cuda_emu.h"

#include "../../kindel_b200/csrc/kdl_common.cuh"
#include "../../kindel_b200/csrc/assemble.cu"
#include "../../kindel_b200/csrc/variants.cu"

static char g_error[512];

#define EMU_RUN(grid, block, ...)                                              \
    do {                                                                        \
        const char* e_ = emu::launch((unsigned)(grid), (unsigned)(block), [&] { __VA_ARGS__; }); \
        if (e_) { snprintf(g_error, sizeof g_error, "%s", e_); return 1; }      \
    } while (0)

static kdl::VariantArgs args(const int32_t* counts, long long n_slots, const int64_t* contig_slot,
                             const int32_t* contig_len, int n_contigs, long long abs_floor, double rel) {
    kdl::VariantArgs a{};
    a.counts = counts; a.n_slots = n_slots;
    a.layout.contig_slot = contig_slot; a.layout.contig_len = contig_len; a.layout.n_contigs = n_contigs;
    a.abs_floor = abs_floor; a.rel_threshold = rel;
    return a;
}

extern "C" {

const char* emu_variants_last_error() { return g_error; }

// 0: threads in order (default), 1: reverse order, 2: a fresh pseudo-random order every scheduler round
void emu_variants_set_schedule(int mode, unsigned long long seed) {
    emu::M().schedule = mode;
    emu::M().rng = seed * 0x9E3779B97F4A7C15ull + 1;
}

// sums + scan as kdl_variant_count launches them; the number of sites is block_sums[n_blocks].  HOST pointers.
int emu_variant_count(const int32_t* counts, long long n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                      int n_contigs, long long abs_floor, double rel, uint32_t* block_sums) {
    g_error[0] = 0;
    const kdl::VariantArgs a = args(counts, n_slots, contig_slot, contig_len, n_contigs, abs_floor, rel);
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    EMU_RUN(n_blocks, kdl::A_THREADS, kdl::variant_sums_kernel(a, block_sums));
    EMU_RUN(1, kdl::A_THREADS, kdl::assemble_scan_sums_kernel(block_sums, n_blocks));
    return 0;
}

// the scatter as kdl_variant_scatter launches it.  HOST pointers.
int emu_variant_scatter(const int32_t* counts, long long n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                        int n_contigs, long long abs_floor, double rel, const uint32_t* block_sums, long long n_sites,
                        int64_t* site_slot, int32_t* site_counts, uint8_t* site_mask) {
    g_error[0] = 0;
    const kdl::VariantArgs a = args(counts, n_slots, contig_slot, contig_len, n_contigs, abs_floor, rel);
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    EMU_RUN(n_blocks, kdl::A_THREADS,
            kdl::variant_scatter_kernel(a, block_sums, n_sites, site_slot, site_counts, site_mask));
    return 0;
}

}  // extern "C"
