// assemble.cu -- what follows the vote on the device instead of in Python loops over the reference length:
//
//   K4 `cdr_flags_kernel`   the per-position predicates of the --realign path (reference kindel/kindel.py:182-185,
//                           202, 243-246, 256): is a position clip-dominant, does a clip consensus extend through it,
//                           and which base the clip consensus has there -- for the right-clipped (->) and the
//                           left-clipped (<-) reads.  2 bytes per slot leave the device instead of the 76-byte table
//                           row; pairing, LCS merge and patching stay on the host (sequential, tiny).
//   K5 `assemble_*_kernel`  the consensus text itself (kindel.py:413-424): emitted length per position (0 for a
//                           deletion call, 1 for a base or an N, 1 + len for an insertion), an exclusive scan over the
//                           whole slot space, and a scatter of the base letters (or IUPAC codes) and the insertion
//                           strings.  One pass
//                           serves every contig: contig c's sequence is out[off[slot_c] .. off[slot_c + L_c]).
//
// The float compares of the reference are restated exactly: `clip / (depth + del + 1) > 0.5` is 2 clip > depth + del + 1
// in integers; `clip > (depth + del) * threshold` is ONE correctly rounded double multiply and a compare -- the same
// IEEE operation numpy performs.
#include "kdl_common.cuh"

namespace kdl {

// flags: bit 0 dominant(->) 1 extend(->) 2 dominant(<-) 3 extend(<-).  bases: low nibble -> base code, high nibble <-.
__global__ void __launch_bounds__(256)
cdr_flags_kernel(const int32_t* __restrict__ counts, long long n_slots, long long slot_lo, long long slot_hi,
                 double decay, uint8_t* __restrict__ flags, uint8_t* __restrict__ bases) {
    const long long s = slot_lo + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slot_hi) return;
    long long depth = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) depth += __ldg(counts + (long long)k * n_slots + s);  // all five keys (kindel.py:182)
    const long long tot = depth + __ldg(counts + (long long)KDL_DEL * n_slots + s);
    unsigned f = 0, b = 0;
#pragma unroll
    for (int dir = 0; dir < 2; ++dir) {
        const int c0 = dir ? KDL_CEW_A : KDL_CSW_A;
        int w[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) w[k] = __ldg(counts + (long long)(c0 + k) * n_slots + s);
        const long long cd = (long long)w[0] + w[1] + w[2] + w[3];  // clip depth: A,C,G,T (kindel.py:90-95)
        if (2 * cd > tot + 1) f |= 1u << (2 * dir);
        if ((double)cd > (double)tot * decay) f |= 2u << (2 * dir);
        int freq, raw;
        base_vote(w[0], w[1], w[2], w[3], w[4], &freq, &raw);  // first maximum in A,T,G,C,N order; empty -> N
        b |= (unsigned)raw << (4 * dir);
    }
    flags[s] = (uint8_t)f;
    bases[s] = (uint8_t)b;
}

// ---- K5 ---------------------------------------------------------------------------------------------------
constexpr int A_THREADS = 256;
constexpr int A_PER = 4;
constexpr int A_BLOCK = A_THREADS * A_PER;  // slots per CTA

struct AssembleArgs {
    const uint8_t* calls;
    long long n_slots;
    const int64_t* contig_slot;
    const int32_t* contig_len;
    int n_contigs;
    const int64_t* ins_slot;   // ascending slots whose call carries change 'I'
    const uint32_t* ins_off;   // [n_ins + 1] byte offsets into ins_bytes
    const uint8_t* ins_bytes;  // the chosen insertion strings, as they are to be printed
    long long n_ins;
};

// is slot s a reference position (not the extra slot behind a contig, not padding)?
__device__ __forceinline__ bool is_position(const AssembleArgs& a, long long s) {
    int lo = 0, hi = a.n_contigs;  // last contig with contig_slot <= s
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a.contig_slot[mid] <= s) lo = mid + 1; else hi = mid;
    }
    if (lo == 0) return false;
    const int c = lo - 1;
    return s < a.contig_slot[c] + a.contig_len[c];
}

__device__ __forceinline__ long long find_ins(const AssembleArgs& a, long long s) {
    long long lo = 0, hi = a.n_ins;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (a.ins_slot[mid] < s) lo = mid + 1; else hi = mid;
    }
    return (lo < a.n_ins && a.ins_slot[lo] == s) ? lo : -1;
}

__device__ __forceinline__ uint32_t emit_len(const AssembleArgs& a, long long s) {
    if (s >= a.n_slots || !is_position(a, s)) return 0u;
    const unsigned c = a.calls[s];
    const unsigned change = (c >> 4) & 3u;
    if (change == 1u) return 0u;  // 'D': nothing is emitted (kindel.py:413-414)
    uint32_t n = 1u;
    if (change == 3u) {
        const long long k = find_ins(a, s);
        if (k >= 0) n += a.ins_off[k + 1] - a.ins_off[k];
    }
    return n;
}

__device__ __forceinline__ uint32_t cta_exclusive_scan(uint32_t v, uint32_t* total) {
    __shared__ uint32_t warp_sum[A_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    __syncthreads();  // warp_sum may still be read by a previous call
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int k = 0; k < A_THREADS / 32; ++k) {
        const uint32_t t = warp_sum[k];
        if (k < warp) before += t;
        all += t;
    }
    *total = all;
    return before + incl - v;
}

__global__ void __launch_bounds__(A_THREADS)
assemble_sums_kernel(AssembleArgs a, uint32_t* __restrict__ block_sums) {
    const long long base = (long long)blockIdx.x * A_BLOCK + (long long)A_PER * threadIdx.x;
    uint32_t t = 0;
#pragma unroll
    for (int k = 0; k < A_PER; ++k) t += emit_len(a, base + k);
    uint32_t total;
    cta_exclusive_scan(t, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// one CTA: block_sums -> exclusive prefix in place, grand total behind the last one
__global__ void __launch_bounds__(A_THREADS)
assemble_scan_sums_kernel(uint32_t* __restrict__ block_sums, long long n_blocks) {
    uint32_t carry = 0;
    for (long long b0 = 0; b0 < n_blocks; b0 += A_THREADS) {
        const long long i = b0 + threadIdx.x;
        const uint32_t v = i < n_blocks ? block_sums[i] : 0u;
        uint32_t total;
        const uint32_t ex = cta_exclusive_scan(v, &total);
        if (i < n_blocks) block_sums[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) block_sums[n_blocks] = carry;
}

// offsets[s] = where slot s's text starts (offsets[n_slots] = total length); the text itself into out
__global__ void __launch_bounds__(A_THREADS)
assemble_scatter_kernel(AssembleArgs a, const uint32_t* __restrict__ block_sums, uint32_t* __restrict__ offsets,
                        uint8_t* __restrict__ out) {
    const long long base = (long long)blockIdx.x * A_BLOCK + (long long)A_PER * threadIdx.x;
    uint32_t n[A_PER], t = 0;
#pragma unroll
    for (int k = 0; k < A_PER; ++k) { n[k] = emit_len(a, base + k); t += n[k]; }
    uint32_t total;
    uint32_t off = block_sums[blockIdx.x] + cta_exclusive_scan(t, &total);
#pragma unroll
    for (int k = 0; k < A_PER; ++k) {
        const long long s = base + k;
        if (s <= a.n_slots) offsets[s] = off;  // (s == n_slots: the grand total)
        if (n[k]) {
            const unsigned c = a.calls[s];
            uint32_t p = off;
            if (n[k] > 1u) {  // insertion string first (kindel.py:419-422)
                const long long j = find_ins(a, s);
                const uint32_t b0 = a.ins_off[j];
                for (uint32_t q = 0; q + 1u < n[k]; ++q) out[p++] = a.ins_bytes[b0 + q];
            }
            // bit 7: a multi-base IUPAC call, bits 0-3 its base set as a BAM nibble (kdl_vote_iupac)
            out[p] = (c & 0x80u) ? (uint8_t)("=ACMGRSVTWYHKDBN"[c & 15u])
                                 : (uint8_t)("ACGTN"[(c & 7u) > 4u ? 4u : (c & 7u)]);
        }
        off += n[k];
    }
}

}  // namespace kdl
