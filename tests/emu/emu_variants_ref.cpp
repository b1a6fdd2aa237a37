// emu_variants_ref.cpp -- TEST INFRASTRUCTURE: K6r (the site passes against reference codes) and K7 (the deletion
// events) of kindel_b200/csrc/variants.cu, with K5's scan kernel between their passes, compiled for the host and run
// under tests/emu/cuda_emu.h, as emu_variants.cpp does for K6.  The kernel sources are included as they are; nothing
// here is part of the product.
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

static kdl::RefVariantArgs args(const int32_t* counts, long long n_slots, const int64_t* contig_slot,
                                const int32_t* contig_len, int n_contigs, const uint8_t* ref, long long abs_floor,
                                double rel) {
    kdl::RefVariantArgs a{};
    a.counts = counts; a.n_slots = n_slots; a.ref = ref;
    a.layout.contig_slot = contig_slot; a.layout.contig_len = contig_len; a.layout.n_contigs = n_contigs;
    a.abs_floor = abs_floor; a.rel_threshold = rel;
    return a;
}

extern "C" {

const char* emu_variants_ref_last_error() { return g_error; }

// 0: threads in order (default), 1: reverse order, 2: a fresh pseudo-random order every scheduler round
void emu_variants_ref_set_schedule(int mode, unsigned long long seed) {
    emu::M().schedule = mode;
    emu::M().rng = seed * 0x9E3779B97F4A7C15ull + 1;
}

// sums + scan as kdl_variant_ref_count launches them; the number of sites is block_sums[n_blocks].  HOST pointers.
int emu_variant_ref_count(const int32_t* counts, long long n_slots, const int64_t* contig_slot,
                          const int32_t* contig_len, int n_contigs, const uint8_t* ref, long long abs_floor, double rel,
                          uint32_t* block_sums) {
    g_error[0] = 0;
    const kdl::RefVariantArgs a = args(counts, n_slots, contig_slot, contig_len, n_contigs, ref, abs_floor, rel);
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    EMU_RUN(n_blocks, kdl::A_THREADS, kdl::variant_ref_sums_kernel(a, block_sums));
    EMU_RUN(1, kdl::A_THREADS, kdl::assemble_scan_sums_kernel(block_sums, n_blocks));
    return 0;
}

// the scatter as kdl_variant_ref_scatter launches it.  HOST pointers.
int emu_variant_ref_scatter(const int32_t* counts, long long n_slots, const int64_t* contig_slot,
                            const int32_t* contig_len, int n_contigs, const uint8_t* ref, long long abs_floor,
                            double rel, const uint32_t* block_sums, long long n_sites, int64_t* site_slot,
                            int32_t* site_counts, int64_t* site_dpa, uint8_t* site_mask) {
    g_error[0] = 0;
    const kdl::RefVariantArgs a = args(counts, n_slots, contig_slot, contig_len, n_contigs, ref, abs_floor, rel);
    const long long n_blocks = (n_slots + kdl::A_BLOCK - 1) / kdl::A_BLOCK;
    EMU_RUN(n_blocks, kdl::A_THREADS,
            kdl::variant_ref_scatter_kernel(a, block_sums, n_sites, site_slot, site_counts, site_dpa, site_mask));
    return 0;
}

// K7's count + scan as kdl_deletion_count launches them (a kdl_batch over HOST pointers)
int emu_deletion_count(const kdl_batch* b, uint32_t* block_sums) {
    g_error[0] = 0;
    const long long n_blocks = (b->n_reads + kdl::A_THREADS - 1) / kdl::A_THREADS;
    if (n_blocks > 0) EMU_RUN(n_blocks, kdl::A_THREADS, kdl::deletion_sums_kernel(*b, block_sums));
    EMU_RUN(1, kdl::A_THREADS, kdl::assemble_scan_sums_kernel(block_sums, n_blocks));
    return 0;
}

int emu_deletion_scatter(const kdl_batch* b, const uint32_t* block_sums, long long n_events, int64_t* ev_slot,
                         int32_t* ev_len) {
    g_error[0] = 0;
    const long long n_blocks = (b->n_reads + kdl::A_THREADS - 1) / kdl::A_THREADS;
    if (n_blocks > 0)
        EMU_RUN(n_blocks, kdl::A_THREADS, kdl::deletion_scatter_kernel(*b, block_sums, n_events, ev_slot, ev_len));
    return 0;
}

}  // extern "C"
