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
//   K2q / K5q               (extension) the Phred quality of every emitted character: one byte per slot from the call
//                           byte and the four base counts, then a scatter beside K5's text through K5's offsets.
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

// ---- K2q / K5q: per-base consensus qualities (extension, `qualities=True`) ------------------------------------
// Q of an emitted base: D = A + C + G + T (N excluded, as in the vote), k = the call's support (the called base's
// count; the summed counts of a multi-base IUPAC set; 0 for every call that emits N).  Q = 0 when k = 0, else the
// largest q in 0..60 with (double)(D - k + 1) * TEN[q] <= (double)(D + 2) -- the rule of succession's disagreement
// rate (D - k + 1) / (D + 2) against 10^(-q/10), as ONE correctly rounded multiply and a compare (no add: nothing
// can be contracted), so CUDA, C and Python agree bit for bit.  TEN[q] = the correctly rounded double of 10^(q/10).
__constant__ double kQualTen[61] = {
    0x1.0000000000000p+0, 0x1.4248ef8fc2604p+0, 0x1.95bb8f6d46052p+0, 0x1.fec982d5bb8afp+0,
    0x1.41857e9d4cc5fp+1, 0x1.94c583ada5b53p+1, 0x1.fd93c1f526de0p+1, 0x1.40c28430012e7p+2,
    0x1.93d00d2348996p+2, 0x1.fc5ebcec13541p+2, 0x1.4000000000000p+3, 0x1.92db2b73b2f85p+3,
    0x1.fb2a734897867p+3, 0x1.3f3df1c59536ep+4, 0x1.91e6de449ff77p+4, 0x1.f9f6e4990f227p+4,
    0x1.3e7c5939384acp+5, 0x1.90f3253c017a1p+5, 0x1.f8c4106c1abfbp+5, 0x1.3dbb36138c149p+6,
    0x1.9000000000000p+6, 0x1.f791f6509fb66p+6, 0x1.3cfa880d5eb40p+7, 0x1.8f0d6e36fa849p+7,
    0x1.f66095d5c7f54p+7, 0x1.3c3a4edfa9759p+8, 0x1.8e1b6f87865d7p+8, 0x1.f52fee8b01d89p+8,
    0x1.3b7a8a4390b7dp+9, 0x1.8d2a03986f19bp+9, 0x1.f400000000000p+9, 0x1.3abb39f263d20p+10,
    0x1.8c392a10b6611p+10, 0x1.f2d0c9c4b925bp+10, 0x1.39fc5da59cf95p+11, 0x1.8b48e29793d2fp+11,
    0x1.f1a24b6967f4cp+11, 0x1.393df516e1276p+12, 0x1.8a592cd474e5cp+12, 0x1.f074847e8ae02p+12,
    0x1.3880000000000p+13, 0x1.896a086efcc67p+13, 0x1.ef477494e3f95p+13, 0x1.37c27e1af3b79p+14,
    0x1.887b750f0437ap+14, 0x1.ee1b1b3d78c7ap+14, 0x1.37056f21e0f90p+15, 0x1.878d725c99713p+15,
    0x1.ecef7809921f4p+15, 0x1.3648d2cf16cc1p+16, 0x1.86a0000000000p+16, 0x1.ebc48a8abbf81p+16,
    0x1.358ca8dd0e7bdp+17, 0x1.85b31da1b0a57p+17, 0x1.ea9a5252c5458p+17, 0x1.34d0f1066b7ccp+18,
    0x1.84c6caea59374p+18, 0x1.e970cef3bfcd8p+18, 0x1.3415ab05fb538p+19, 0x1.83db0782dc7f1p+19,
    0x1.e848000000000p+19,
};
constexpr int kQualMax = 60;

// the condition is monotone in q and holds at q = 0 (D - k + 1 <= D + 2): a 6-step binary search finds the largest q
__device__ __forceinline__ unsigned phred_q(long long d, long long k, const double* ten) {
    if (k <= 0) return 0u;
    const double e = (double)(d - k + 1), lim = (double)(d + 2);
    unsigned q = 0;
#pragma unroll
    for (unsigned step = 32; step; step >>= 1)
        if (q + step <= (unsigned)kQualMax && e * ten[q + step] <= lim) q += step;
    return q;
}

// Q of one slot from its call byte and A, C, G, T counts (a 'D' or 'N' call has base code 4: k = 0)
__device__ __forceinline__ unsigned slot_q(int a, int c, int g, int t, unsigned call, const double* ten) {
    const long long d = (long long)a + c + g + t;
    long long k;
    if (call & 0x80u) {  // multi-base IUPAC set; all four bases is the letter N
        const unsigned m = call & 15u;
        k = m == 15u ? 0 : (long long)((m & 1u) ? a : 0) + ((m & 2u) ? c : 0) + ((m & 4u) ? g : 0) + ((m & 8u) ? t : 0);
    } else {
        const unsigned code = call & 7u;
        k = code == 0u ? a : code == 1u ? c : code == 2u ? g : code == 3u ? t : 0;
    }
    return phred_q(d, k, ten);
}

// K2q: n_slots % 4 == 0.  One thread = 4 slots: 128-bit loads of the four base columns and 4 call bytes in, 4 Q
// bytes (0..60) out -- 18 B per slot.  Runs after any vote (K2, K2 IUPAC, K2x + K2g): the call bytes say what was
// emitted.
__global__ void __launch_bounds__(256)
consensus_qual_kernel(const int32_t* __restrict__ counts, const uint8_t* __restrict__ calls, long long n_slots,
                      uint8_t* __restrict__ qual) {
    __shared__ double ten[64];
    if (threadIdx.x <= (unsigned)kQualMax) ten[threadIdx.x] = kQualTen[threadIdx.x];
    __syncthreads();
    const long long s = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (s >= n_slots) return;
    int4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = __ldg(reinterpret_cast<const int4*>(counts + (long long)k * n_slots + s));
    const uint32_t c = __ldg(reinterpret_cast<const uint32_t*>(calls + s));
    const unsigned q0 = slot_q(v[0].x, v[1].x, v[2].x, v[3].x, c & 0xffu, ten);
    const unsigned q1 = slot_q(v[0].y, v[1].y, v[2].y, v[3].y, (c >> 8) & 0xffu, ten);
    const unsigned q2 = slot_q(v[0].z, v[1].z, v[2].z, v[3].z, (c >> 16) & 0xffu, ten);
    const unsigned q3 = slot_q(v[0].w, v[1].w, v[2].w, v[3].w, c >> 24, ten);
    *reinterpret_cast<uint32_t*>(qual + s) = q0 | (q1 << 8) | (q2 << 16) | (q3 << 24);
}

// K5q: the quality text beside K5's consensus text, from the offsets K5 wrote: slot s owns
// out[offsets[s] .. offsets[s + 1]); its first n - 1 bytes are the inserted string's (ins_qual of that 'I' slot), the
// last one the slot's own Q.  Every byte is '!' + Q (Phred+33).
__global__ void __launch_bounds__(A_THREADS)
assemble_qual_kernel(const uint32_t* __restrict__ offsets, const uint8_t* __restrict__ qual, long long n_slots,
                     const int64_t* __restrict__ ins_slot, const uint8_t* __restrict__ ins_qual, long long n_ins,
                     uint8_t* __restrict__ out) {
    AssembleArgs a{};
    a.ins_slot = ins_slot;
    a.n_ins = n_ins;
    const long long base = (long long)blockIdx.x * A_BLOCK + (long long)A_PER * threadIdx.x;
#pragma unroll
    for (int k = 0; k < A_PER; ++k) {
        const long long s = base + k;
        if (s >= n_slots) return;
        const uint32_t o = offsets[s], n = offsets[s + 1] - o;
        if (!n) continue;
        if (n > 1u) {
            const long long j = find_ins(a, s);
            const uint8_t b = (uint8_t)(33u + (j >= 0 ? ins_qual[j] : 0u));
            for (uint32_t p = 0; p + 1u < n; ++p) out[o + p] = b;
        }
        out[o + n - 1u] = (uint8_t)(33u + qual[s]);
    }
}

}  // namespace kdl
