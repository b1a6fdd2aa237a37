// amplicons.cu -- K12 `amplicons_assign_kernel` and K12d `amplicons_depth_kernel` (extension: `kindel amplicons
// --primers scheme.bed`): which amplicon of a tiled scheme each read comes from, and how deep each amplicon's insert is.
//
// K12, per read on contig c (include/kindel_b200.h, kdl_amplicons_assign):
//   s, e     the walk cursors of its first and its last M/=/X base, as K9 takes them (complex_ends, primers.cu)
//   left     the label of s among c's LEFT-primer segments, right the label of e among its RIGHT-primer segments: one
//            binary search each over the breakpoints the host built (kindel_b200/primers.py amplicon_arrays)
//   label    -1 when neither end is in a primer, -3 when either end is in primers of several amplicons, -2 when the
//            ends name two different amplicons, else the amplicon one or both ends name
// One thread per read: a simple read costs its three words of metadata, the contig search and two binary searches; a
// complex read walks its CIGAR once.
//
// K12d, per amplicon: A+C+G+T of the count table over its insert's slots contig_slot + [insert_start, insert_end),
// reduced by one warp -- the sum (int64), the minimum and the number of positions at or above min_depth.  Inserts of a
// tiled scheme overlap their neighbours' primers, so every amplicon reads its own range.
#include "kdl_common.cuh"

namespace kdl {

constexpr int AM_THREADS = 256;
constexpr int AM_WARPS = AM_THREADS / 32;  // K12d: amplicons per CTA

enum { AMP_UNPRIMED = -1, AMP_MISPAIRED = -2, AMP_AMBIGUOUS = -3 };

// the label of cursor x among one side's segments of contig c: [off[c], off[c + 1]) of at / label
__device__ __forceinline__ int segment_label(const int64_t* __restrict__ off, const int32_t* __restrict__ at,
                                             const int32_t* __restrict__ label, int c, long long x, long long L) {
    if (x < 0 || x >= L) return AMP_UNPRIMED;
    const long long lo = off[c], hi = off[c + 1];
    const long long k = upper_bound_i32(at, lo, hi, x) - 1;  // the last breakpoint <= x
    return k >= lo ? label[k] : AMP_UNPRIMED;
}

__device__ __forceinline__ int amplicon_of(const kdl_batch& b, const kdl_amplicons& a, long long r) {
    const uint32_t lraw = (uint32_t)b.l_seq[r];
    const int c = find_contig(b.contig_read_off, b.n_contigs, r);
    const long long start = b.ref_start[r];
    const long long L = b.contig_len[c];
    long long s, e;
    if (!(lraw & KDL_COMPLEX)) {  // simple: one M op of l_seq bases at the start
        if ((long long)lraw <= 0) return AMP_UNPRIMED;
        s = start;
        e = start + (long long)lraw - 1;
    } else {
        const long long lseq = complex_len(lraw);
        const uint32_t* __restrict__ blk = b.seq4 + (size_t)b.seq_off[r] + ((lseq + 7) >> 3);
        if (!complex_ends(blk + 2, blk[0], start, L, &s, &e)) return AMP_UNPRIMED;
    }
    const int l = segment_label(a.left_off, a.left_at, a.left_label, c, s, L);
    const int rt = segment_label(a.right_off, a.right_at, a.right_label, c, e, L);
    if (l == AMP_AMBIGUOUS || rt == AMP_AMBIGUOUS) return AMP_AMBIGUOUS;
    if (l >= 0 && rt >= 0 && l != rt) return AMP_MISPAIRED;
    return l >= 0 ? l : rt;  // (-1 when both are -1)
}

__global__ void __launch_bounds__(AM_THREADS)
amplicons_assign_kernel(kdl_batch b, kdl_amplicons a, int32_t* __restrict__ label) {
    const long long r = (long long)blockIdx.x * AM_THREADS + threadIdx.x;
    if (r < b.n_reads) label[r] = amplicon_of(b, a, r);
}

// stats[3 * j + 0] = the sum of A+C+G+T over amplicon j's insert, [1] its minimum, [2] the positions with
// A+C+G+T >= min_depth.  An amplicon whose insert does not lie in its contig gets zeros.
__global__ void __launch_bounds__(AM_THREADS)
amplicons_depth_kernel(const int32_t* __restrict__ counts, long long n_slots, const int64_t* __restrict__ contig_slot,
                       const int32_t* __restrict__ contig_len, int n_contigs, kdl_amplicons a, long long min_depth,
                       long long* __restrict__ stats) {
    const int lane = threadIdx.x & 31;
    const long long j = (long long)blockIdx.x * AM_WARPS + (threadIdx.x >> 5);
    if (j >= a.n_amplicons) return;
    const int c = a.amp_contig[j];
    const long long i0 = a.insert_start[j], i1 = a.insert_end[j];
    long long sum = 0, covered = 0, lowest = 0x7fffffffffffffffLL;
    if (c >= 0 && c < n_contigs && 0 <= i0 && i0 < i1 && i1 <= (long long)contig_len[c]) {
        const long long base = contig_slot[c];
        for (long long p = base + i0 + lane; p < base + i1; p += 32) {
            const long long d = (long long)counts[p] + counts[n_slots + p] + counts[2 * n_slots + p] +
                                counts[3 * n_slots + p];
            sum += d;
            covered += d >= min_depth;
            lowest = d < lowest ? d : lowest;
        }
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, k);
        covered += __shfl_xor_sync(0xffffffffu, covered, k);
        const long long o = __shfl_xor_sync(0xffffffffu, lowest, k);
        lowest = o < lowest ? o : lowest;
    }
    if (lane == 0) {
        stats[3 * j] = sum;
        stats[3 * j + 1] = lowest == 0x7fffffffffffffffLL ? 0 : lowest;
        stats[3 * j + 2] = covered;
    }
}

}  // namespace kdl
