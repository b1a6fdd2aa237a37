// dedup.cu -- K14k `dedup_*_kernel` entry lists and K14s selection (extension: `--dedup`): duplicate reads and read
// pairs removed before the pileup, by fragment ends and a base-quality score, as samtools markdup -r and Picard
// MarkDuplicates do (include/kindel_b200.h K14 and DESIGN.md section 1 have the rule).
//
// End of a read: e = 2 u + strand, u its unclipped 5' position (forward: POS0 minus the S / H ops before the first
// M/D/N/=/X op; reverse: POS0 + the M/D/N/=/X lengths - 1 + the S / H ops after the last one).  A simple read is one
// M op, so its u is its start or start + len - 1; a complex or KDL_HARD read's ops are its seq4 trailer.
//   K14k-e  one thread per read: keep = 1, end[r] (KDL_DEDUP_ALONE for a read left alone: dup_score < 0, or no
//           M/D/N/=/X op), paired[r] = 0; the first thread zeroes the totals record.
//   K14k-p  one thread per read: an R2 (mate[r] >= 0) whose R1 is not left alone marks both mates paired and appends
//           one pair entry (contig, E1 <= E2, score rank, R1, R2) and two marker entries (contig, 2 E + 0).
//   K14k-s  one thread per read: a read neither left alone nor paired appends one single entry (contig, 2 E + 1).
//           The appends are warp-aggregated atomics on the totals record, so the lists are compacted in any order.
// The host sorts both lists by key (stable passes of torch.sort); markers sort before the singles of their end.
//   K14s-h  one thread per sorted entry: run heads (an entry whose key differs from the one before), each CTA's last
//           head, best[i] = ~0.
//   K14s-c  one CTA: each CTA's carry, the last head before it (an exclusive max-scan over the CTAs).
//   K14s-b  one thread per sorted entry: its run head H (a CTA max-scan of the heads and the carry), stored; the
//           candidates' ranks reduced per run within the warp (the lanes of a run are contiguous: a segmented
//           shuffle-down min), one 64-bit atomicMin per run and warp into best[H].  No thread walks a run.
//   K14s-m  one thread per sorted entry: a candidate whose rank is not best[H] is removed (keep 0 for its read, or
//           both mates), counted into the totals record.
// rank = (0xffffffff - score) << 32 | index: the smallest rank is the largest score, then the smallest index
// (R1 + R2's int64 sum and the smaller mate index for a pair), and ranks are unique, so one entry wins each run.
// Every lane of a warp runs every collective (the tail takes a null entry); the collectives are the shuffles and
// ballots the kernel emulator (tests/emu/) models.
#include "kdl_common.cuh"

namespace kdl {

constexpr int DD_THREADS = 256;
constexpr int DD_WARPS = DD_THREADS / 32;
constexpr unsigned long long DD_NONE = ~0ull;

__device__ __forceinline__ bool ref_op(uint32_t op) { return op == 0u || op == 2u || op == 3u || op == 7u || op == 8u; }
__device__ __forceinline__ bool clip_op(uint32_t op) { return op == 4u || op == 5u; }

// K14k-e
__global__ void __launch_bounds__(DD_THREADS)
dedup_ends_kernel(kdl_batch b, const uint8_t* __restrict__ reverse, const int32_t* __restrict__ score,
                  int64_t* __restrict__ end, uint8_t* __restrict__ paired, uint8_t* __restrict__ keep,
                  unsigned long long* __restrict__ totals) {
    const long long r = (long long)blockIdx.x * DD_THREADS + threadIdx.x;
    if (r == 0)
        for (int k = 0; k < KDL_DEDUP_TOTALS; ++k) totals[k] = 0ull;
    if (r >= b.n_reads) return;
    keep[r] = 1;
    paired[r] = 0;
    const uint32_t lraw = (uint32_t)b.l_seq[r];
    const long long pos = b.ref_start[r];
    long long lead = 0, span = 0, trail = 0;
    bool any = false;
    if (!(lraw & KDL_COMPLEX)) {
        span = (long long)lraw;
        any = true;
    } else {
        const uint32_t* blk = b.seq4 + (size_t)b.seq_off[r] + ((complex_len(lraw) + 7) >> 3);
        const uint32_t n_ops = blk[0];
        for (uint32_t k = 0; k < n_ops; ++k) {
            const uint32_t w = blk[2 + k], op = w & 15u;
            const long long len = (long long)(w >> 4);
            if (ref_op(op)) {
                span += len;
                any = true;
                trail = 0;
            } else if (clip_op(op)) {
                if (any) trail += len;
                else lead += len;
            }
        }
    }
    if (score[r] < 0 || !any) {
        end[r] = KDL_DEDUP_ALONE;
        return;
    }
    const int strand = reverse[r] != 0;
    const long long u = strand ? pos + span - 1 + trail : pos - lead;
    end[r] = 2 * u + strand;
}

// lane's slot among the warp's appending lanes; the warp's leader takes them all from *counter at once
__device__ __forceinline__ long long warp_append(bool has, unsigned long long* counter, unsigned per) {
    const unsigned want = __ballot_sync(0xffffffffu, has);
    const int lane = threadIdx.x & 31;
    unsigned long long base = 0ull;
    if (want && lane == __ffs(want) - 1) base = atomicAdd(counter, (unsigned long long)(__popc(want) * per));
    base = __shfl_sync(0xffffffffu, base, want ? __ffs(want) - 1 : 0);
    return (long long)base + (long long)__popc(want & ((1u << lane) - 1u)) * per;
}

__device__ __forceinline__ unsigned long long dedup_rank(long long score, long long index) {
    return ((0xffffffffull - (unsigned long long)score) << 32) | (unsigned long long)index;
}

// K14k-p
__global__ void __launch_bounds__(DD_THREADS)
dedup_pairs_kernel(kdl_batch b, const int32_t* __restrict__ score, const int32_t* __restrict__ mate,
                   kdl_dedup_lists L, const int64_t* __restrict__ end, uint8_t* __restrict__ paired,
                   unsigned long long* __restrict__ totals) {
    const long long r = (long long)blockIdx.x * DD_THREADS + threadIdx.x;  // (whole warps: every lane meets the ballot)
    long long r1 = -1;
    if (r < b.n_reads) {
        const int32_t m = mate[r];
        if (m >= 0 && m < b.n_reads && m != r && end[r] != KDL_DEDUP_ALONE && end[m] != KDL_DEDUP_ALONE) r1 = m;
    }
    const long long at = warp_append(r1 >= 0, totals + 0, 1u);
    const long long mk = warp_append(r1 >= 0, totals + 1, 2u);
    if (r1 < 0) return;
    paired[r] = 1;
    paired[r1] = 1;
    const int c = find_contig(b.contig_read_off, b.n_contigs, r);
    const long long e1 = end[r1], e2 = end[r];
    L.pair_contig[at] = c;
    L.pair_e1[at] = e1 < e2 ? e1 : e2;
    L.pair_e2[at] = e1 < e2 ? e2 : e1;
    L.pair_rank[at] = dedup_rank((long long)score[r1] + score[r], r1 < r ? r1 : r);
    L.pair_r1[at] = (int32_t)r1;
    L.pair_r2[at] = (int32_t)r;
    L.single_contig[mk] = c;
    L.single_key[mk] = 2 * e1;
    L.single_read[mk] = -1;
    L.single_rank[mk] = DD_NONE;
    L.single_contig[mk + 1] = c;
    L.single_key[mk + 1] = 2 * e2;
    L.single_read[mk + 1] = -1;
    L.single_rank[mk + 1] = DD_NONE;
}

// K14k-s
__global__ void __launch_bounds__(DD_THREADS)
dedup_singles_kernel(kdl_batch b, const int32_t* __restrict__ score, kdl_dedup_lists L,
                     const int64_t* __restrict__ end, const uint8_t* __restrict__ paired,
                     unsigned long long* __restrict__ totals) {
    const long long r = (long long)blockIdx.x * DD_THREADS + threadIdx.x;
    const bool single = r < b.n_reads && end[r] != KDL_DEDUP_ALONE && !paired[r];
    const long long at = warp_append(single, totals + 1, 1u);
    if (!single) return;
    L.single_contig[at] = find_contig(b.contig_read_off, b.n_contigs, r);
    L.single_key[at] = 2 * end[r] + 1;
    L.single_read[at] = (int32_t)r;
    L.single_rank[at] = dedup_rank(score[r], r);
}

// One sorted list as K14s sees it: the pair list (e2 != nullptr, key (contig, e1, e2)) or the single list (key
// (contig, key >> 1), the low bit the domain: 0 a pair's marker, 1 a single)
struct DedupList {
    const int64_t* order;
    long long m;
    const int32_t* contig;
    const int64_t* e1;
    const int64_t* e2;
    const unsigned long long* rank;
    const int32_t* r1;  // pair: R1; single list: the read (-1 for a marker)
    const int32_t* r2;  // pair: R2; single list: nullptr
    __device__ __forceinline__ bool same(long long a, long long c) const {
        if (contig[a] != contig[c]) return false;
        if (e2) return e1[a] == e1[c] && e2[a] == e2[c];
        return (e1[a] >> 1) == (e1[c] >> 1);
    }
    __device__ __forceinline__ bool head(long long i) const { return i == 0 || !same(order[i], order[i - 1]); }
};

__device__ __forceinline__ long long warp_max_scan(long long v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d && o > v) v = o;
    }
    return v;
}

// inclusive max-scan of v over the CTA (every thread calls it)
__device__ __forceinline__ long long cta_max_scan(long long v) {
    __shared__ long long s_warp[DD_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_max_scan(v);
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    long long before = -1;
    for (int w = 0; w < warp; ++w) before = s_warp[w] > before ? s_warp[w] : before;
    __syncthreads();  // (s_warp is reused by the next call)
    return v > before ? v : before;
}

// K14s-h
__global__ void __launch_bounds__(DD_THREADS)
dedup_heads_kernel(DedupList L, unsigned long long* __restrict__ best, int32_t* __restrict__ cta_head) {
    const long long i = (long long)blockIdx.x * DD_THREADS + threadIdx.x;
    const bool h = i < L.m && L.head(i);
    if (i < L.m) best[i] = DD_NONE;
    const long long last = cta_max_scan(h ? i : -1);
    if (threadIdx.x == DD_THREADS - 1) cta_head[blockIdx.x] = (int32_t)last;
}

// K14s-c: carry[j] = the last head in CTAs before j (-1 for none), one CTA in chunks of DD_THREADS
__global__ void __launch_bounds__(DD_THREADS)
dedup_carry_kernel(const int32_t* __restrict__ cta_head, int32_t* __restrict__ carry, long long n_cta) {
    __shared__ long long s_incl[DD_THREADS];
    long long run = -1;  // the last head of the chunks before
    for (long long base = 0; base < n_cta; base += DD_THREADS) {
        const long long j = base + threadIdx.x;
        s_incl[threadIdx.x] = cta_max_scan(j < n_cta ? cta_head[j] : -1);
        __syncthreads();
        long long excl = threadIdx.x ? s_incl[threadIdx.x - 1] : -1;
        if (run > excl) excl = run;
        if (j < n_cta) carry[j] = (int32_t)excl;
        if (s_incl[DD_THREADS - 1] > run) run = s_incl[DD_THREADS - 1];
        __syncthreads();
    }
}

// K14s-b
__global__ void __launch_bounds__(DD_THREADS)
dedup_best_kernel(DedupList L, const int32_t* __restrict__ carry, int32_t* __restrict__ run,
                  unsigned long long* __restrict__ best) {
    const long long i = (long long)blockIdx.x * DD_THREADS + threadIdx.x;
    const bool in = i < L.m;
    const bool h = in && L.head(i);
    long long H = cta_max_scan(h ? i : -1);
    if (carry[blockIdx.x] > H) H = carry[blockIdx.x];
    unsigned long long v = DD_NONE;
    if (in) {
        run[i] = (int32_t)H;
        const long long e = L.order[i];
        // a candidate: every pair; a single whose run starts with a single, i.e. no pair end shares it
        if (L.e2 || ((L.e1[e] & 1) && (L.e1[L.order[H]] & 1))) v = L.rank[e];
    }
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {  // segmented min toward the run's first lane in the warp
        const unsigned long long o = __shfl_down_sync(0xffffffffu, v, d);
        const long long oh = __shfl_down_sync(0xffffffffu, H, d);
        if (lane + d < 32 && oh == H && o < v) v = o;
    }
    const long long prev = __shfl_up_sync(0xffffffffu, H, 1);
    if (in && (lane == 0 || prev != H) && v != DD_NONE) atomicMin(best + H, v);
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

// K14s-m
__global__ void __launch_bounds__(DD_THREADS)
dedup_mark_kernel(DedupList L, const int32_t* __restrict__ run, const unsigned long long* __restrict__ best,
                  uint8_t* __restrict__ keep, unsigned long long* __restrict__ totals) {
    const long long i = (long long)blockIdx.x * DD_THREADS + threadIdx.x;
    unsigned long long removed = 0ull, shadowed = 0ull;
    if (i < L.m) {
        const long long e = L.order[i], H = run[i];
        if (L.e2) {
            if (L.rank[e] != best[H]) {
                keep[L.r1[e]] = 0;
                keep[L.r2[e]] = 0;
                removed = 1ull;
            }
        } else if (L.e1[e] & 1) {
            const bool shadow = !(L.e1[L.order[H]] & 1);
            if (shadow || L.rank[e] != best[H]) {
                keep[L.r1[e]] = 0;
                removed = 1ull;
                shadowed = shadow ? 1ull : 0ull;
            }
        }
    }
    removed = warp_sum(removed);
    shadowed = warp_sum(shadowed);
    if ((threadIdx.x & 31) == 0) {
        if (removed) atomicAdd(totals + (L.e2 ? 2 : 3), removed);
        if (shadowed) atomicAdd(totals + 4, shadowed);
    }
}

}  // namespace kdl
