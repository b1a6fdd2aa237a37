// emu_select.cpp -- TEST INFRASTRUCTURE: K8 (the device read selection of kindel_b200/csrc/select.cu) compiled for the
// host and run under tests/emu/cuda_emu.h, launched as kdl_select_count / kdl_select_scatter launch it.  The kernel
// source is included as it is; nothing here is part of the product.
#define KDL_HOST_EMU 1
#include "cuda_emu.h"

#include "../../kindel_b200/csrc/kdl_common.cuh"
#include "../../kindel_b200/csrc/select.cu"

static char g_error[512];

#define EMU_RUN(grid, block, ...)                                              \
    do {                                                                        \
        const char* e_ = emu::launch((unsigned)(grid), (unsigned)(block), [&] { __VA_ARGS__; }); \
        if (e_) { snprintf(g_error, sizeof g_error, "%s", e_); return 1; }      \
    } while (0)

static kdl_qmask or_empty(const kdl_qmask* q) { return q ? *q : kdl_qmask{}; }

extern "C" {

const char* emu_select_last_error() { return g_error; }

// 0: threads in order (default), 1: reverse order, 2: a fresh pseudo-random order every scheduler round
void emu_select_set_schedule(int mode, unsigned long long seed) {
    emu::M().schedule = mode;
    emu::M().rng = seed * 0x9E3779B97F4A7C15ull + 1;
}

long long emu_select_scratch_words(long long n_reads) {
    return (long long)kdl::S_REC * ((n_reads + kdl::S_THREADS) / kdl::S_THREADS + 1);
}

// the counts + combine as kdl_select_count launches them.  HOST pointers.
int emu_select_count(const kdl_batch* b, const kdl_qmask* q, const uint8_t* keep, uint32_t* scratch) {
    g_error[0] = 0;
    const long long n_blocks = (b->n_reads + kdl::S_THREADS) / kdl::S_THREADS;
    const kdl_qmask qm = or_empty(q);
    EMU_RUN(n_blocks, kdl::S_THREADS, kdl::select_sums_kernel(*b, qm, keep, scratch));
    EMU_RUN(1, kdl::S_THREADS, kdl::select_combine_kernel(scratch, n_blocks));
    return 0;
}

// the scatter as kdl_select_scatter launches it.  HOST pointers.
int emu_select_scatter(const kdl_batch* b, const kdl_qmask* q, const uint8_t* keep, const uint32_t* scratch,
                       const kdl_batch* out, const kdl_qmask* out_mask) {
    g_error[0] = 0;
    const long long n_blocks = (b->n_reads + kdl::S_THREADS) / kdl::S_THREADS;
    const kdl_qmask qm = or_empty(q), om = or_empty(out_mask);
    EMU_RUN(n_blocks, kdl::S_THREADS,
            kdl::select_scatter_kernel(*b, qm, keep, scratch, *out, const_cast<int64_t*>(out->contig_read_off), om));
    return 0;
}

}  // extern "C"
