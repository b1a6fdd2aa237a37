// kdl_common.cuh -- shared device helpers for the kindel_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/kindel_b200.h"

// The CTA's dynamic shared memory.  (KDL_HOST_EMU: tests/emu/ compiles the kernels for the host, where the
// array is an ordinary global and `__shared__` variables are statics; the device build never defines it.)
#ifndef KDL_HOST_EMU
#define KDL_DYNAMIC_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#else
#define KDL_DYNAMIC_SMEM(name) extern unsigned char name[]
#endif

// Every kernel launch of api.cu.  Under KDL_HOST_EMU the emulator runs the grid on the host, row by row of a
// two-dimensional grid, and keeps a failure for check_launch() as the runtime keeps a launch error.  A kernel name
// with a comma in its template arguments goes in parentheses.
#ifndef KDL_HOST_EMU
#define KDL_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#else
#define KDL_LAUNCH(kernel, grid, block, smem, stream, ...) \
    emu::launch_grid(dim3(grid), dim3(block), [&] { kernel(__VA_ARGS__); })
#endif

namespace kdl {

// BAM nibble ("=ACMGRSVTWYHKDBN") -> weight column 0..4 (A,C,G,T,N) or -1.  Only the five keys
// of the reference's per-position dicts exist (kindel/kindel.py:29); anything else is a KeyError
// when it is used by an M or S op (kindel.py:52,72,79).  Packed 4 bits per entry: 0xF = invalid.
__device__ __forceinline__ int nib2col(int nib) {
    // nib:            0 1 2 3 4 5 6 7 8 9 a b c d e f
    // col (F = bad):  F 0 1 F 2 F F F 3 F F F F F F 4
    const unsigned long long lut = 0x4FFFFFF3FFF2F10FULL;
    int v = (int)((lut >> (nib * 4)) & 0xF);
    return v == 0xF ? -1 : v;
}

// 8 bases per 32-bit word, first base in the most significant nibble
__device__ __forceinline__ int nibble_at(const uint32_t* __restrict__ seq, long long q) {
    return (int)((seq[q >> 3] >> (28 - 4 * (int)(q & 7))) & 0xFu);
}

// SEQ length of a complex read's l_seq word: tile-eligible reads keep it in bits 0..15 (bits 16..22 hold their
// M-op count), KDL_HARD reads in bits 0..29
__device__ __forceinline__ long long complex_len(uint32_t lraw) {
    return (lraw & KDL_HARD) ? (long long)(lraw & 0x3fffffffu) : (long long)(lraw & KDL_LEN_MASK);
}

// Python list indexing (list length n): negative indices wrap once, otherwise IndexError (-1).
__device__ __forceinline__ long long pyindex(long long i, long long n) {
    if (i < 0) i += n;
    return (i < 0 || i >= n) ? -1 : i;
}

// contig c with contig_read_off[c] <= r < contig_read_off[c+1] (empty contigs skipped naturally)
__device__ __forceinline__ int find_contig(const int64_t* __restrict__ off, int n_contigs, long long r) {
    int lo = 0, hi = n_contigs;  // first index in (lo, hi] with off[idx] > r
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (off[mid + 1] > r) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// ---- dirty-sector map of columns 5..18 (kdl_pileup_range_map, include/kindel_b200.h) --------------------------
// uint32 map[4 * ceil(n_slots / 64)]: one 16-byte record per 64-slot window w; byte b (0..13) of the record is column
// 5 + b, bit s of that byte stands for slots [64 w + 8 s, 64 w + 8 s + 8) -- one 32-byte sector of the column.  A slot
// of columns 5..18 is non-zero only if its bit is set; a set bit over a zero sector is always allowed.
// mark_dirty sets the bits of columns [col, col + n_col) over slots [s0, s1): one atomicOr per record word touched,
// a handful per CIGAR op (the map is small enough to stay in L2).
__device__ __forceinline__ void mark_dirty(uint32_t* __restrict__ map, int col, int n_col, long long s0, long long s1) {
    if (s0 >= s1) return;
    const uint32_t bytes = ((1u << n_col) - 1u) << (col - KDL_DEL);  // bytes of the record the columns own
    uint32_t* rec = map + 4 * (s0 >> 6);
    int lo = (int)(s0 & 63), left = (int)(s1 - s0);  // (one CIGAR op: fewer than 2^28 slots)
    do {                                              // the windows [s0, s1) meets, from slot lo of the first
        const int hi = left < 64 - lo ? lo + left : 64;
        const uint32_t sec = ((2u << ((hi - 1) >> 3)) - 1u) & ~((1u << (lo >> 3)) - 1u);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t nib = (bytes >> (4 * k)) & 0xFu;
            const uint32_t v = sec * ((nib & 1u) | ((nib & 2u) << 7) | ((nib & 4u) << 14) | ((nib & 8u) << 21));
            if (v) atomicOr(rec + k, v);
        }
        left -= hi - lo;
        lo = 0;
        rec += 4;
    } while (left > 0);
}

// mark_dirty of the slots base + pyindex(i, n) for i in [lo, hi) that exist: the negative part wraps by n
__device__ __forceinline__ void mark_dirty_py(uint32_t* __restrict__ map, int col, int n_col, long long base,
                                              long long lo, long long hi, long long n) {
    const long long a = lo > -n ? lo : -n, e = hi < 0 ? hi : 0;
    if (a < e) mark_dirty(map, col, n_col, base + a + n, base + e + n);
    mark_dirty(map, col, n_col, base + (lo > 0 ? lo : 0), base + (hi < n ? hi : n));
}

// consensus() over the five base counts (kindel/kindel.py:369-381): first maximum in dict order
// A,T,G,C,N; all-zero -> N with no tie; tie = another key holds the same non-zero maximum.
// Returns the emitted code (tie -> 4 = N) and the consensus key's count through *freq.
__device__ __forceinline__ int base_vote(int a, int c, int g, int t, int n, int* freq, int* raw_base) {
    int best = a, code = 0;
    if (t > best) { best = t; code = 3; }
    if (g > best) { best = g; code = 2; }
    if (c > best) { best = c; code = 1; }
    if (n > best) { best = n; code = 4; }
    const int ties = (a == best) + (c == best) + (g == best) + (t == best) + (n == best);
    if (best == 0) code = 4;  // ("N", 0): sum == 0 (counts are non-negative)
    *freq = best;
    *raw_base = code;
    return (best != 0 && ties > 1) ? 4 : code;
}

// The D / N / I decisions of one slot of consensus_sequence (kindel/kindel.py:402-424) in integer arithmetic:
//   del > 0.5*depth            <=> 2*del > depth
//   depth < min_depth          <=> depth < ceil(min_depth)
//   ins > min(0.5*d, 0.5*dn)   <=> 2*ins > min(d, dn)
// Every vote makes them in this order.  Returns true with the whole call byte in *call for a 'D' or an 'N' slot; false
// with the change code (0 or 3 for 'I') in bits 4-5 of *call and the base left to the vote.
__device__ __forceinline__ bool vote_decided(int a, int c, int g, int t, int del, int ins, long long depth_next,
                                             long long min_depth_ceil, unsigned* call) {
    const long long depth = (long long)a + c + g + t;  // N excluded (kindel.py:404)
    if (2ll * del > depth) { *call = (1u << 4) | 4u; return true; }
    if (depth < min_depth_ceil) { *call = (2u << 4) | 4u; return true; }
    const long long thr = depth < depth_next ? depth : depth_next;
    *call = (2ll * ins > thr) ? (3u << 4) : 0u;
    return false;
}

// One slot of consensus_sequence with consensus()'s base
__device__ __forceinline__ unsigned vote_slot(int a, int c, int g, int t, int n, int del, int ins,
                                              long long depth_next, long long min_depth_ceil) {
    unsigned call;
    if (vote_decided(a, c, g, t, del, ins, depth_next, min_depth_ceil, &call)) return call;
    int freq, raw;
    return call | (unsigned)base_vote(a, c, g, t, n, &freq, &raw);
}

// descending compare-exchange: x keeps the larger value
__device__ __forceinline__ void cx_desc(int& x, int& y) {
    const int hi = x > y ? x : y, lo = x > y ? y : x;
    x = hi;
    y = lo;
}

// The emitted base of the IUPAC vote (extension: `iupac_threshold` t in [0, 1]).  D = A + C + G + T (N is not an
// allele, as in kindel.py:404).  L(b) = sum of the counts of every base with count >= count(b); v = the largest
// count(b) > 0 with L(b) >= t * D; the call is the set S = {b : count(b) >= v}, so tied bases enter together.
// The comparison is ONE correctly rounded double multiply and a compare (no add: nothing can be contracted).
// The four counts are sorted by a fixed compare-exchange network; the prefix sums p_k of the sorted counts never
// decrease, so the first p_k >= t * D names v (p_k <= L(x_k), and every larger count's tie group ends before k).
// Returns the base code 0..3 when |S| = 1, 4 (N) when D = 0, else 0x80 | mask with mask A=1 C=2 G=4 T=8 (the BAM
// nibble: the letter is "=ACMGRSVTWYHKDBN"[mask]).  No data-dependent branch.
__device__ __forceinline__ unsigned iupac_base(int a, int c, int g, int t, double threshold) {
    int x0 = a, x1 = c, x2 = g, x3 = t;
    cx_desc(x0, x1);
    cx_desc(x2, x3);
    cx_desc(x0, x2);
    cx_desc(x1, x3);
    cx_desc(x1, x2);
    const long long p0 = x0, p1 = p0 + x1, p2 = p1 + x2, d = p2 + x3;  // counts < 2^31: the sums need 64 bits
    const double need = threshold * (double)d;
    const int v = (double)p0 >= need ? x0 : (double)p1 >= need ? x1 : (double)p2 >= need ? x2 : x3;
    const unsigned mask = (unsigned)(a >= v) | ((unsigned)(c >= v) << 1) | ((unsigned)(g >= v) << 2) |
                          ((unsigned)(t >= v) << 3);
    const unsigned single = (mask >> 1) - (mask >> 3);  // 1, 2, 4, 8 -> 0, 1, 2, 3
    const unsigned code = (mask & (mask - 1u)) ? (0x80u | mask) : single;
    return d == 0 ? 4u : code;
}

// vote_slot with the IUPAC base: the D / N / I decisions and their order are vote_slot's; only the base differs
__device__ __forceinline__ unsigned vote_slot_iupac(int a, int c, int g, int t, int del, int ins, long long depth_next,
                                                    long long min_depth_ceil, double threshold) {
    unsigned call;
    if (vote_decided(a, c, g, t, del, ins, depth_next, min_depth_ceil, &call)) return call;
    return call | iupac_base(a, c, g, t, threshold);
}

// The emitted base of the quality vote (extension: `quality_vote`): b* = the base with the largest summed weight
// (wsum, WeightSums in quality.cu); N when that sum is 0 or two bases share it.  *q = min(60, (wsum[b*] - the
// runner-up's) >> 16), the Phred-scaled likelihood ratio of the call over the runner-up; 0 for N.  Integer only.
__device__ __forceinline__ unsigned weight_base(unsigned long long wa, unsigned long long wc, unsigned long long wg,
                                                unsigned long long wt, unsigned* q) {
    unsigned long long best = wa, second = 0ull;
    unsigned code = 0u;
    const unsigned long long w[3] = {wc, wg, wt};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (w[k] > best) { second = best; best = w[k]; code = (unsigned)k + 1u; }
        else if (w[k] > second) second = w[k];
    }
    if (best == 0ull || best == second) { *q = 0u; return 4u; }
    const unsigned long long d = (best - second) >> 16;
    *q = d < 60ull ? (unsigned)d : 60u;
    return code;
}

// Vote policies of K2 / K2x (template arguments of vote_kernel and vote_exchange_kernel); `s` is the slot
struct MajorityVote {  // the reference's vote
    __device__ __forceinline__ unsigned operator()(long long, int a, int c, int g, int t, int n, int del, int ins,
                                                   long long depth_next, long long min_depth_ceil) const {
        return vote_slot(a, c, g, t, n, del, ins, depth_next, min_depth_ceil);
    }
};
struct IupacVote {  // ambiguity codes below a frequency threshold
    double threshold;
    __device__ __forceinline__ unsigned operator()(long long, int a, int c, int g, int t, int, int del, int ins,
                                                   long long depth_next, long long min_depth_ceil) const {
        return vote_slot_iupac(a, c, g, t, del, ins, depth_next, min_depth_ceil, threshold);
    }
};
struct QualityVote {  // the base by summed base-quality weights; qual (may be NULL): the Q of each slot, 0 unless a base
    const unsigned long long* __restrict__ wsum;  // [4][n_slots]
    long long n_slots;
    uint8_t* __restrict__ qual;
    __device__ __forceinline__ unsigned operator()(long long s, int a, int c, int g, int t, int, int del, int ins,
                                                   long long depth_next, long long min_depth_ceil) const {
        unsigned call, q = 0u;
        if (!vote_decided(a, c, g, t, del, ins, depth_next, min_depth_ceil, &call))
            call |= weight_base(__ldg(wsum + s), __ldg(wsum + n_slots + s), __ldg(wsum + 2 * n_slots + s),
                                __ldg(wsum + 3 * n_slots + s), &q);
        if (qual) qual[s] = (uint8_t)q;
        return call;
    }
};

}  // namespace kdl
