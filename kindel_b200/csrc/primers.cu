// primers.cu -- K9 `primers_*_kernel` (extension: `--primers scheme.bed`): masks the bases of every read that copy an
// amplicon primer, on the device, before the pileup.  A masked base is what min_base_quality makes of a low-quality
// base: an N nibble in seq4, listed in the batch's mask list so that K1q takes back its column-4 count.
//
// The rule (DESIGN.md section 1, include/kindel_b200.h K9), per read on contig c with at least one M/=/X base:
//   s, e     the walk cursors (kindel.py:40-81, before the Python index wrap) of its first and its last M/=/X base
//   left     B = the largest end of the primers [a, b) of c with a <= s < b; the M/=/X bases with cursor in [s, B)
//   right    A = the smallest start of the primers with a <= e < b; the M/=/X bases with cursor in [A, e]
// Cursors of a read's M/=/X bases strictly increase along the read, so each side is a run of them: per M op the
// masked bases are at most two query ranges, ascending over the read.  Nothing else of a read is touched.
//
// Per contig the host builds two sorted views of its primers (include/kindel_b200.h, kdl_primers): by start with the
// running maximum of the end -- the last start <= s gives B when that maximum is > s -- and by end with the suffix
// minimum of the start -- the first end > e gives A when that minimum is <= e.  One binary search per end of a read.
//
// The new mask list is the sorted union of the batch's own list (min_base_quality) and the primer bases, per read:
//   count    one thread per P_PER consecutive reads: each read's share (merged bases, 1 when it has any, 1 when it has
//            primer bases, primer bases), summed per CTA into four rows of the scratch
//   scan     assemble_scan_sums_kernel over the first two rows (exclusive prefixes), and one CTA that sums the other
//            two and writes the totals record the host reads back to size the outputs
//   scatter  the count again, the CTA's prefix added: read_idx / off / qpos of the merged list, and the primer bases'
//            nibbles set to N.  A read owns whole words of seq4, so its thread writes them without atomics.
#include "kdl_common.cuh"

namespace kdl {

constexpr int P_THREADS = 256;
constexpr int P_PER = 4;                       // consecutive reads per thread
constexpr int P_BLOCK = P_THREADS * P_PER;     // reads per CTA
enum { P_MBASES = 0, P_MREADS, P_PREADS, P_PBASES, P_NROW };  // rows of the scratch (n_blocks + 1 words each)
constexpr int P_TOTALS = 8;                    // words of the totals record behind the rows

// B and A of a read's two ends (no primer there: B = s, A = e + 1)
struct PrimerWindow {
    long long B, A;
};

// index of the first element of v[lo, hi) that is > x
__device__ __forceinline__ long long upper_bound_i32(const int32_t* __restrict__ v, long long lo, long long hi,
                                                     long long x) {
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if ((long long)v[mid] <= x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ PrimerWindow primer_window(const kdl_primers& p, int c, long long s, long long e) {
    PrimerWindow w{s, e + 1};
    const long long lo = p.contig_off[c], hi = p.contig_off[c + 1];
    if (lo == hi) return w;
    const long long kl = upper_bound_i32(p.start_sorted, lo, hi, s);  // primers lo .. kl - 1 start at or before s
    if (kl > lo && (long long)p.end_max[kl - 1] > s) w.B = p.end_max[kl - 1];
    const long long kr = upper_bound_i32(p.end_sorted, lo, hi, e);    // primers kr .. hi - 1 end after e
    if (kr < hi && (long long)p.start_min[kr] <= e) w.A = p.start_min[kr];
    return w;
}

// The walk cursors *s, *e of the first and the last M/=/X base of a complex read (CIGAR words cig[0, n_ops), walk
// from `start` on a contig of length L), before the Python index wrap: M/=/X and D advance the cursor, a first S does
// not, a later S advances it while it is below L.  False when the read has no M/=/X base.  Shared by K9 and K12.
__device__ __forceinline__ bool complex_ends(const uint32_t* __restrict__ cig, uint32_t n_ops, long long start,
                                             long long L, long long* s, long long* e) {
    long long r_pos = start;
    bool any = false;
    *s = 0;
    *e = -1;
    for (uint32_t i = 0; i < n_ops; ++i) {
        const uint32_t cg = cig[i];
        const long long len = cg >> 4;
        const int op = cg & 0xF;
        if (op == 0 || op == 7 || op == 8) {
            if (len > 0) {
                if (!any) *s = r_pos;
                any = true;
                *e = r_pos + len - 1;
            }
            r_pos += len;
        } else if (op == 2) {
            r_pos += len;
        } else if (op == 4 && i != 0) {
            long long n_adv = L - r_pos;
            r_pos += n_adv < 0 ? 0 : (n_adv > len ? len : n_adv);
        }
    }
    return any;
}

// Calls emit(q0, q1) for the query ranges [q0, q1) of read r's primer bases, ascending and disjoint (clipped to its
// SEQ: a hard read whose walk runs past it raises in the pileup).  The walk is K1g's (pileup_general.cu): M/=/X and
// D advance the cursor, a first S does not, a later S advances both cursors while the cursor is below L.
template <class F>
__device__ void primer_ranges(const kdl_batch& b, const kdl_primers& p, long long r, F&& emit) {
    const uint32_t lraw = (uint32_t)b.l_seq[r];
    const int c = find_contig(b.contig_read_off, b.n_contigs, r);
    const long long start = b.ref_start[r];
    auto part = [&](long long r_pos, long long q_pos, long long len, long long lseq, const PrimerWindow& w) {
        // the op's bases [0, l1) have cursor < B, [r0, len) cursor >= A; one range when they meet
        const long long l1 = w.B - r_pos < len ? (w.B - r_pos > 0 ? w.B - r_pos : 0) : len;
        const long long r0 = w.A - r_pos > 0 ? (w.A - r_pos < len ? w.A - r_pos : len) : 0;
        const long long qmax = lseq - q_pos;  // bases of the op that lie inside SEQ
        auto put = [&](long long k0, long long k1) {
            k1 = k1 < qmax ? k1 : qmax;
            if (k1 > k0) emit(q_pos + k0, q_pos + k1);
        };
        if (l1 >= r0) {  // (len > 0: then [0, l1) and [r0, len) together are all of the op)
            put(0, len);
        } else {
            put(0, l1);
            put(r0, len);
        }
    };
    if (!(lraw & KDL_COMPLEX)) {  // simple: one M op of l_seq bases at the start
        const long long len = lraw;
        if (len <= 0) return;
        const PrimerWindow w = primer_window(p, c, start, start + len - 1);
        if (w.B > start || w.A <= start + len - 1) part(start, 0, len, len, w);
        return;
    }
    const long long L = b.contig_len[c];
    const long long lseq = complex_len(lraw);
    const uint32_t* __restrict__ blk = b.seq4 + (size_t)b.seq_off[r] + ((lseq + 7) >> 3);
    const uint32_t n_ops = blk[0];
    const uint32_t* __restrict__ cig = blk + 2;
    // pass 1: the cursors of the first and the last M/=/X base
    long long s, e;
    if (!complex_ends(cig, n_ops, start, L, &s, &e)) return;
    const PrimerWindow w = primer_window(p, c, s, e);
    if (w.B <= s && w.A > e) return;
    // pass 2: the ranges, op by op
    long long r_pos = start;
    long long q_pos = 0;
    for (uint32_t i = 0; i < n_ops; ++i) {
        const uint32_t cg = cig[i];
        const long long len = cg >> 4;
        const int op = cg & 0xF;
        if (op == 0 || op == 7 || op == 8) {
            if (len > 0 && (r_pos < w.B || r_pos + len > w.A)) part(r_pos, q_pos, len, lseq, w);
            r_pos += len;
            q_pos += len;
        } else if (op == 1) {
            q_pos += len;
        } else if (op == 2) {
            r_pos += len;
        } else if (op == 4) {
            if (i == 0) {
                q_pos += len;
            } else {
                long long n_adv = L - r_pos;
                n_adv = n_adv < 0 ? 0 : (n_adv > len ? len : n_adv);
                r_pos += n_adv;
                q_pos += n_adv;
            }
        }
    }
}

// the read's run in the batch's own mask list: [*b0, *b1) of q.qpos (empty when it has none)
__device__ __forceinline__ void own_mask(const kdl_qmask& q, long long r, uint32_t* b0, uint32_t* b1) {
    *b0 = *b1 = 0;
    if (q.n_reads <= 0) return;
    long long lo = 0, hi = q.n_reads;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if ((long long)q.read_idx[mid] < r) lo = mid + 1; else hi = mid;
    }
    if (lo < q.n_reads && (long long)q.read_idx[lo] == r) {
        *b0 = q.off[lo];
        *b1 = q.off[lo + 1];
    }
}

// The merge of a read's run [m0, m1) of the batch's own mask list with new bases given as ascending, disjoint query
// ranges -- the sorted union, each base once.  Shared by K9 (primer bases) and K10 (mates.cu: overlap bases).
// MergeCount sizes it: after the ranges, merged() = the bases of the union.
struct MergeCount {
    const uint32_t* __restrict__ own;
    uint32_t m0, k, m1, added, same;

    __device__ __forceinline__ MergeCount(const kdl_qmask& q, uint32_t b0, uint32_t b1)
        : own(q.qpos), m0(b0), k(b0), m1(b1), added(0), same(0) {}
    __device__ __forceinline__ void add(long long q0, long long q1) {
        added += (uint32_t)(q1 - q0);
        while (k < m1 && (long long)own[k] < q0) ++k;
        while (k < m1 && (long long)own[k] < q1) { ++same; ++k; }
    }
    __device__ __forceinline__ uint32_t merged() const { return added + (m1 - m0) - same; }
};

// MergeWrite writes it from qpos[o] on (writes bounded by cap) and sets the new bases' nibbles to N in `words`, the
// read's own words of seq4; finish() after the last range.
struct MergeWrite {
    const uint32_t* __restrict__ own;
    uint32_t k, m1;
    uint32_t* __restrict__ qpos;
    long long o, cap;

    __device__ __forceinline__ MergeWrite(const kdl_qmask& q, uint32_t b0, uint32_t b1, uint32_t* out, long long at,
                                          long long n_out)
        : own(q.qpos), k(b0), m1(b1), qpos(out), o(at), cap(n_out) {}
    __device__ __forceinline__ void put(long long qq) {
        if (o < cap) qpos[o] = (uint32_t)qq;
        ++o;
    }
    __device__ __forceinline__ void add(long long q0, long long q1, uint32_t* words) {
        while (k < m1 && (long long)own[k] < q0) put(own[k++]);
        for (long long qq = q0; qq < q1; ++qq) {
            put(qq);
            words[qq >> 3] |= 0xFu << (28 - 4 * (int)(qq & 7));  // N
        }
        while (k < m1 && (long long)own[k] < q1) ++k;  // already listed
    }
    __device__ __forceinline__ void finish() {
        while (k < m1) put(own[k++]);
    }
};

// read r's entry orr of the merged list `om`, its bases from ob on: read_idx / off written, the writer returned.
// Writes are bounded by om's counts (the totals), so a wrong count stays in bounds.
__device__ __forceinline__ MergeWrite merged_list_entry(const kdl_qmask& q, const kdl_qmask& om, long long r,
                                                        long long orr, long long ob) {
    if (orr < om.n_reads) {
        const_cast<uint32_t*>(om.read_idx)[orr] = (uint32_t)r;
        const_cast<uint32_t*>(om.off)[orr] = (uint32_t)ob;
    }
    uint32_t m0, m1;
    own_mask(q, r, &m0, &m1);
    return MergeWrite(q, m0, m1, const_cast<uint32_t*>(om.qpos), ob, om.n_bases);
}

// read r's share of the four rows
__device__ __forceinline__ void primer_item(const kdl_batch& b, const kdl_qmask& q, const kdl_primers& p, long long r,
                                            uint32_t (&v)[P_NROW]) {
#pragma unroll
    for (int k = 0; k < P_NROW; ++k) v[k] = 0;
    if (r >= b.n_reads) return;
    uint32_t m0, m1;
    own_mask(q, r, &m0, &m1);
    MergeCount mc(q, m0, m1);
    primer_ranges(b, p, r, [&](long long q0, long long q1) { mc.add(q0, q1); });
    const uint32_t n_p = mc.added;
    v[P_MBASES] = mc.merged();
    v[P_MREADS] = v[P_MBASES] ? 1u : 0u;
    v[P_PREADS] = n_p ? 1u : 0u;
    v[P_PBASES] = n_p;
}

// row k of the scratch: scratch + k * (n_blocks + 1); the totals record behind the last row
__global__ void __launch_bounds__(P_THREADS)
primers_sums_kernel(kdl_batch b, kdl_qmask q, kdl_primers p, uint32_t* __restrict__ scratch, long long n_blocks) {
    const long long r0 = (long long)blockIdx.x * P_BLOCK + (long long)P_PER * threadIdx.x;
    uint32_t t[P_NROW] = {0, 0, 0, 0};
    for (int j = 0; j < P_PER; ++j) {
        uint32_t v[P_NROW];
        primer_item(b, q, p, r0 + j, v);
#pragma unroll
        for (int k = 0; k < P_NROW; ++k) t[k] += v[k];
    }
    uint32_t tot[P_NROW];
    cta_scan_vec(t, tot);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < P_NROW; ++k) scratch[(size_t)k * (n_blocks + 1) + blockIdx.x] = tot[k];
    }
}

// one CTA, after the scans of rows 0 and 1: the totals record = [0] reads in the merged list, [1] bases in it,
// [2] reads with primer bases, [3] primer bases, [4..7] 0
__global__ void __launch_bounds__(P_THREADS)
primers_totals_kernel(uint32_t* __restrict__ scratch, long long n_blocks) {
    const uint32_t* rp = scratch + (size_t)P_PREADS * (n_blocks + 1);
    const uint32_t* bp = scratch + (size_t)P_PBASES * (n_blocks + 1);
    uint32_t v[2] = {0, 0};
    for (long long i = threadIdx.x; i < n_blocks; i += P_THREADS) {
        v[0] += rp[i];
        v[1] += bp[i];
    }
    uint32_t tot[2];
    cta_scan_vec(v, tot);
    if (threadIdx.x == 0) {
        uint32_t* rec = scratch + (size_t)P_NROW * (n_blocks + 1);
        rec[0] = scratch[(size_t)P_MREADS * (n_blocks + 1) + n_blocks];
        rec[1] = scratch[(size_t)P_MBASES * (n_blocks + 1) + n_blocks];
        rec[2] = tot[0];
        rec[3] = tot[1];
        for (int k = 4; k < P_TOTALS; ++k) rec[k] = 0;
    }
}

// `om` carries the caller's output arrays (const in the struct, written here) and the totals as its counts; every
// write is bounded by them, so a wrong count stays in bounds.
__global__ void __launch_bounds__(P_THREADS)
primers_scatter_kernel(kdl_batch b, kdl_qmask q, kdl_primers p, const uint32_t* __restrict__ scratch,
                       long long n_blocks, uint32_t* seq4, kdl_qmask om) {
    const long long r0 = (long long)blockIdx.x * P_BLOCK + (long long)P_PER * threadIdx.x;
    uint32_t n[P_PER], t[2] = {0, 0};
#pragma unroll
    for (int j = 0; j < P_PER; ++j) {
        uint32_t v[P_NROW];
        primer_item(b, q, p, r0 + j, v);
        n[j] = v[P_MBASES];
        t[0] += v[P_MBASES];
        t[1] += v[P_MREADS];
    }
    uint32_t tot[2];
    cta_scan_vec(t, tot);
    long long ob = (long long)t[0] + scratch[(size_t)P_MBASES * (n_blocks + 1) + blockIdx.x];
    long long orr = (long long)t[1] + scratch[(size_t)P_MREADS * (n_blocks + 1) + blockIdx.x];
    if (blockIdx.x == 0 && threadIdx.x == 0 && om.n_reads > 0) const_cast<uint32_t*>(om.off)[om.n_reads] = (uint32_t)om.n_bases;
#pragma unroll
    for (int j = 0; j < P_PER; ++j) {
        if (!n[j]) continue;
        const long long r = r0 + j;
        MergeWrite mw = merged_list_entry(q, om, r, orr, ob);
        uint32_t* words = seq4 + (size_t)b.seq_off[r];  // (may be b.seq4 itself: the CIGAR words are only read)
        primer_ranges(b, p, r, [&](long long q0, long long q1) { mw.add(q0, q1, words); });
        mw.finish();
        ob += n[j];
        ++orr;
    }
}

}  // namespace kdl
