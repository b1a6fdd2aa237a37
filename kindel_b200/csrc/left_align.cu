// left_align.cu -- K15d / K15i (extension: `variants --vcf --reference --left-align`): every deletion and insertion
// event moved to the leftmost place that gives the same haplotype against the reference, before the events are grouped
// and tested, so that one indel an aligner placed at several offsets of a repeat is one allele.
//
// g = the reference codes of the slots (0-3 = A, C, G, T; 4 = anything else, and every slot that is not a position),
// s0 the first slot of the event's contig.
//   K15d, a deletion key (r << 28 | n), r an absolute slot: while r > s0, g[r-1] < 4 and g[r-1] == g[r+n-1]: r -= 1.
//   K15i, an insertion event row (slot p, read, q_off, len) whose string t has m = min(q_off + len, SEQ) - q_off bases:
//     with k = 0, while m > 0, p > s0, g[p-1] < 4 and the code of t[(m-1-k) mod m] == g[p-1]: p -= 1, k += 1.  The
//     normalised string is t rotated right by k mod m; a base of t that is not A, C, G or T stops the shift.
// The shifts depend on nothing but the event and g, so one thread per key or row is the whole algorithm; a loop runs
// at most the repeat's length.  K15i reads the string's nibbles from seq4 as it goes (one cached load per step): most
// rows stop at the first step, and a row in a long repeat walks its own few words.

namespace kdl {

constexpr int LA_THREADS = 256;

// the contig whose slots [contig_slot, contig_slot + L] hold slot s: the last one with contig_slot <= s, or -1
__device__ __forceinline__ int contig_of_slot(const int64_t* __restrict__ contig_slot, int n_contigs, long long s) {
    int lo = 0, hi = n_contigs;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (contig_slot[mid] <= s) lo = mid + 1; else hi = mid;
    }
    return lo - 1;
}

// BAM nibble -> reference code: A, C, G, T = 0-3, every other nibble 4 (it matches no reference base)
__device__ __forceinline__ unsigned nib2code(int nib) {
    // nib:   0 1 2 3 4 5 6 7 8 9 a b c d e f
    // code:  4 0 1 4 2 4 4 4 3 4 4 4 4 4 4 4
    return (unsigned)((0x4444444344424104ULL >> (nib * 4)) & 0xFu);
}

__global__ void __launch_bounds__(LA_THREADS)
left_align_deletions_kernel(const int64_t* __restrict__ keys, long long n_keys, const int64_t* __restrict__ contig_slot,
                            int n_contigs, const uint8_t* __restrict__ ref, int64_t* __restrict__ out) {
    const long long i = (long long)blockIdx.x * LA_THREADS + threadIdx.x;
    if (i >= n_keys) return;
    const long long key = keys[i];
    const long long n = key & ((1LL << 28) - 1);
    long long r = key >> 28;
    const int c = contig_of_slot(contig_slot, n_contigs, r);
    if (c >= 0 && n > 0) {
        const long long s0 = contig_slot[c];
        while (r > s0) {
            const unsigned a = __ldg(ref + r - 1);
            if (a > 3u || a != __ldg(ref + r + n - 1)) break;
            --r;
        }
    }
    out[i] = (r << 28) | n;
}

// rows with dead[i] != 0 (the insertions K10 dropped) get norm_slot -1 and count nowhere
__global__ void __launch_bounds__(LA_THREADS)
left_align_insertions_kernel(kdl_batch b, const int32_t* __restrict__ events, long long n_events,
                             const uint8_t* __restrict__ dead, const uint8_t* __restrict__ ref,
                             int64_t* __restrict__ norm_slot, int32_t* __restrict__ rot, int32_t* __restrict__ hist) {
    const long long i = (long long)blockIdx.x * LA_THREADS + threadIdx.x;
    if (i >= n_events) return;
    if (dead && dead[i]) {
        norm_slot[i] = -1;
        rot[i] = 0;
        return;
    }
    const int4 ev = __ldg(reinterpret_cast<const int4*>(events) + i);  // (slot, read, q_off, len)
    long long p = ev.x;
    const long long read = ev.y, q0 = ev.z;
    const uint32_t lraw = (uint32_t)b.l_seq[read];
    const long long lseq = (lraw & KDL_COMPLEX) ? complex_len(lraw) : (long long)lraw;
    long long q1 = q0 + ev.w;
    q1 = q1 < lseq ? q1 : lseq;
    const long long m = q1 > q0 ? q1 - q0 : 0;  // the string as Python slicing clips it at the end of SEQ
    long long k = 0;
    const int c = contig_of_slot(b.contig_slot, b.n_contigs, p);
    if (m > 0 && c >= 0) {
        const long long s0 = b.contig_slot[c];
        const uint32_t* __restrict__ seq = b.seq4 + (size_t)b.seq_off[read];
        long long j = m - 1;  // the string's last base, moving left with the shift
        while (p > s0) {
            const unsigned g = __ldg(ref + p - 1);
            if (g > 3u || nib2code(nibble_at(seq, q0 + j)) != g) break;
            --p;
            ++k;
            j = j == 0 ? m - 1 : j - 1;
        }
    }
    norm_slot[i] = p;
    rot[i] = (int32_t)(m > 0 ? k % m : 0);
    atomicAdd(hist + p, 1);
}

}  // namespace kdl
