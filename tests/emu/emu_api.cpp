// emu_api.cpp -- TEST INFRASTRUCTURE: the C ABI of kindel_b200/csrc/api.cu, launch code and kernels, compiled for the
// host and run under tests/emu/cuda_emu.h.  api.cu is included whole: KDL_HOST_EMU turns its KDL_LAUNCH sites into
// emulated launches and leaves out what needs a real device (table allocation, IPC handles, kdl_ctx_*).  The kdl_*
// entry points take HOST pointers here; the stream is ignored.  Nothing here is part of the product.
#define KDL_HOST_EMU 1
#include "cuda_emu.h"

#include "../../kindel_b200/csrc/api.cu"

extern "C" {

// the text of the launch failure behind the last KDL_ERR_CUDA
const char* emu_last_error() { return emu::M().last_error; }

// 0: threads in order (default), 1: reverse order, 2: a fresh pseudo-random order every scheduler round
void emu_set_schedule(int mode, unsigned long long seed) {
    emu::M().schedule = mode;
    emu::M().rng = seed * 0x9E3779B97F4A7C15ull + 1;
}

// what api.cu's sm_count() returns: it sizes the persistent and grid-stride grids and the depth split
void emu_set_sm_count(int n) { emu::M().sm_count = n; }

// K0 + K1's kCx instantiation over every tile of a batch without tile-eligible complex reads, flushing as
// kdl_pileup_range would for `fresh` / `split`.  No kdl_* entry point runs kCx on such a batch (it takes the lean
// instantiation); this keeps the piece instantiation's own stages and item cuts checked on simple reads.
int emu_pileup_tile_cx(const kdl_batch* batch, int32_t* counts, int64_t n_slots, int fresh, int split, int zero_rest) {
    const long long n_tiles = n_slots / KDL_TILE;
    KDL_LAUNCH(kdl::tile_index_kernel, (unsigned)((n_tiles * 32 + 255) / 256), 256, 0, nullptr, *batch, 0, n_tiles,
               batch->tile_index);
    int rc = check_launch();
    if (rc != KDL_OK) return rc;
    const kdl_batch& b = *batch;
    if (split > 1) rc = launch_tile<kdl::F_ATOMIC, true>(b, counts, n_slots, 0, n_tiles, split, 0, nullptr, 0, nullptr);
    else if (fresh)
        rc = launch_tile<kdl::F_STORE, true>(b, counts, n_slots, 0, n_tiles, 1, zero_rest, nullptr, 0, nullptr);
    else rc = launch_tile<kdl::F_ADD, true>(b, counts, n_slots, 0, n_tiles, 1, 0, nullptr, 0, nullptr);
    return rc != KDL_OK ? rc : check_launch();
}

// ---- self-test of the emulator: a bulk copy must not be visible before its mbarrier completes -----------
namespace {
struct alignas(16) SelfSmem {
    uint32_t data[64];
    uint64_t bar;
};
int selftest(bool wait) {
    static uint32_t src[64] __attribute__((aligned(16)));
    static int mismatches;
    for (int i = 0; i < 64; ++i) src[i] = 0x1000u + (uint32_t)i;
    mismatches = 0;
    const char* err = emu::launch(1, 64, [&] {
        SelfSmem& sm = *reinterpret_cast<SelfSmem*>(kdl::smem_raw);
        const int tid = (int)threadIdx.x;
        if (tid == 0) kdl::mbar_init(&sm.bar, 1);
        __syncthreads();
        if (tid == 0) {
            kdl::mbar_expect_tx(&sm.bar, sizeof sm.data);
            kdl::bulk_g2s(sm.data, src, sizeof sm.data, &sm.bar);
        }
        if (wait) kdl::mbar_wait(&sm.bar, 0);
        if (sm.data[tid] != src[tid]) atomicAdd(&mismatches, 1);
        __syncthreads();
    });
    if (err) return -1;
    return mismatches ? 1 : 0;
}
}  // namespace

int emu_selftest_missing_wait() { return selftest(false); }
int emu_selftest_missing_wait_fixed() { return selftest(true); }

}  // extern "C"
