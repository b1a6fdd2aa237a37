// normalise.cu -- K13 (extension: `--normalise N` with a named `--primers` scheme): keep the first N reads of each
// (amplicon, strand) group in batch order, the rest are dropped before the pileup.  No sort: an order-preserving rank
// within each group from per-CTA counts (include/kindel_b200.h, kdl_normalise).
//
// Key of read r: 2 * label[r] + (reverse[r] != 0) for a label in [0, n_amplicons) (K12's amplicon), else -1 (never
// capped).  The grid is G CTAs; CTA j owns the reads of tiles [j * per, (j + 1) * per), a tile being NM_THREADS reads,
// so every CTA's reads are one contiguous run of the batch and the CTAs are in batch order.  H is int32 [G][K],
// K = 2 * n_amplicons, row j private to CTA j.
//   K13c  count: CTA j zeroes row j and counts its keys into it, one atomic add per warp peer group (warp_peers:
//         the lanes holding one key add their number once).
//   K13s  scan: one thread per key; H[j][key] becomes the count of the key in CTAs before j (exclusive prefix over
//         j), total[key] its count in the batch, and *dropped gains max(total[key] - cap, 0).
//   K13m  mark: CTA j walks its tiles in order.  A read's rank in its group is H[j][key] (the key's reads before this
//         tile) + the reads of its key in earlier warps of the tile (a shared list of (key, count) per warp, one entry
//         per peer group) + its rank among its warp's peers.  keep = key < 0 or rank < cap.  The key's last read in
//         the tile then stores rank + 1 into H[j][key] for the next tile.
// Every lane of a warp runs every collective (the tail of the batch takes key -1), so the full-mask collectives are
// exact.  The peer groups are built from one shuffle and one ballot per distinct key of the warp (warp_peers), so the
// same source runs under the kernel emulator (tests/emu/), which models those collectives.
#include "kdl_common.cuh"

namespace kdl {

constexpr int NM_THREADS = 256;
constexpr int NM_WARPS = NM_THREADS / 32;

__device__ __forceinline__ int normalise_key(const int32_t* __restrict__ label, const uint8_t* __restrict__ reverse,
                                             long long r, long long n, int n_amplicons) {
    if (r >= n) return -1;
    const int l = label[r];
    return (l >= 0 && l < n_amplicons) ? 2 * l + (reverse[r] != 0) : -1;
}

// The lanes of the warp whose key equals this lane's (what __match_any_sync returns), one shuffle and one ballot per
// distinct key: the lowest lane not yet matched broadcasts its key and every lane holding it answers.  The loop is
// warp-uniform; amplicon reads in file order put one to a few keys in a warp.
__device__ __forceinline__ unsigned warp_peers(int key) {
    unsigned todo = 0xffffffffu, peers = 0u;
    while (todo) {
        const int k = __shfl_sync(0xffffffffu, key, __ffs(todo) - 1);
        const unsigned same = __ballot_sync(0xffffffffu, key == k);
        if (key == k) peers = same;
        todo &= ~same;
    }
    return peers;
}

// K13c
__global__ void __launch_bounds__(NM_THREADS)
normalise_count_kernel(const int32_t* __restrict__ label, const uint8_t* __restrict__ reverse, long long n,
                       int n_amplicons, long long per, int32_t* __restrict__ hist, long long* __restrict__ dropped) {
    const long long K = 2ll * n_amplicons;
    int32_t* __restrict__ row = hist + (long long)blockIdx.x * K;
    for (long long k = threadIdx.x; k < K; k += NM_THREADS) row[k] = 0;
    if (blockIdx.x == 0 && threadIdx.x == 0) *dropped = 0;
    __syncthreads();
    const long long lo = (long long)blockIdx.x * per * NM_THREADS;
    const long long hi = lo + per * NM_THREADS < n ? lo + per * NM_THREADS : n;
    const int lane = threadIdx.x & 31;
    for (long long base = lo; base < hi; base += NM_THREADS) {  // (uniform trip count: every lane meets the match)
        const int key = normalise_key(label, reverse, base + threadIdx.x, hi, n_amplicons);
        const unsigned peers = warp_peers(key);
        if (key >= 0 && lane == __ffs(peers) - 1) atomicAdd(row + key, __popc(peers));
    }
}

// K13s
__global__ void __launch_bounds__(NM_THREADS)
normalise_scan_kernel(int32_t* __restrict__ hist, int grid, int n_amplicons, long long cap,
                      int32_t* __restrict__ total, long long* __restrict__ dropped) {
    const long long K = 2ll * n_amplicons;
    const long long key = (long long)blockIdx.x * NM_THREADS + threadIdx.x;
    if (key >= K) return;
    int32_t s = 0;
    for (int j = 0; j < grid; ++j) {
        const int32_t c = hist[(long long)j * K + key];
        hist[(long long)j * K + key] = s;
        s += c;
    }
    total[key] = s;
    if ((long long)s > cap) atomicAdd(reinterpret_cast<unsigned long long*>(dropped), (unsigned long long)(s - cap));
}

// K13m
__global__ void __launch_bounds__(NM_THREADS)
normalise_mark_kernel(const int32_t* __restrict__ label, const uint8_t* __restrict__ reverse, long long n,
                      int n_amplicons, long long per, long long cap, int32_t* __restrict__ hist,
                      uint8_t* __restrict__ keep) {
    __shared__ int s_key[NM_WARPS][32];
    __shared__ int s_cnt[NM_WARPS][32];
    __shared__ int s_len[NM_WARPS];
    const long long K = 2ll * n_amplicons;
    int32_t* __restrict__ row = hist + (long long)blockIdx.x * K;
    const long long lo = (long long)blockIdx.x * per * NM_THREADS;
    const long long hi = lo + per * NM_THREADS < n ? lo + per * NM_THREADS : n;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned below = (1u << lane) - 1u;  // %lanemask_lt
    for (long long base = lo; base < hi; base += NM_THREADS) {
        const long long r = base + threadIdx.x;
        const int key = normalise_key(label, reverse, r, hi, n_amplicons);
        const unsigned peers = warp_peers(key);
        const bool leader = lane == __ffs(peers) - 1;
        const unsigned leaders = __ballot_sync(0xffffffffu, leader && key >= 0);
        if (leader && key >= 0) {  // this warp's list: one (key, count) per peer group, in lane order
            const int at = __popc(leaders & below);
            s_key[warp][at] = key;
            s_cnt[warp][at] = __popc(peers);
        }
        if (lane == 0) s_len[warp] = __popc(leaders);
        __syncthreads();
        int before = 0;
        bool later = false;
        if (key >= 0) {
            for (int w = 0; w < NM_WARPS; ++w) {
                if (w == warp) continue;
                const int m = s_len[w];
                for (int k = 0; k < m; ++k)
                    if (s_key[w][k] == key) {
                        if (w < warp) before += s_cnt[w][k];
                        else later = true;
                    }
            }
        }
        const int rank = key >= 0 ? row[key] + before + __popc(peers & below) : 0;
        if (r < hi) keep[r] = (key < 0 || (long long)rank < cap) ? 1 : 0;
        __syncthreads();  // every read of row[] and of the lists is done
        if (key >= 0 && !later && (peers >> lane) == 1u) row[key] = rank + 1;  // the key's last read in the tile
    }
}

}  // namespace kdl
