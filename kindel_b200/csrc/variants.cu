// variants.cu -- K6 `variant_*_kernel` (extension): the sites of `variants --only-variants` and of the VCF, selected
// on the device so that only the selected sites leave it instead of the 76-byte table row of every position.
//
// The rule (kindel_b200/kindel.py `variant_alleles`): per position, t = columns 0-5 (A, C, G, T, N, deletions),
// depth = their sum, top = the first maximum in that order, share_k = t_k / depth (0 at depth 0); allele k is a variant
// when t_k > abs_threshold and share_k > rel_threshold and k != top.  A site is a position with a variant allele.
// `abs_floor` is floor(abs_threshold) clamped to [-1, 2^31] by the caller (for an integer count t > x == t > floor(x);
// NaN is passed as 2^31, which no int32 count exceeds).  share_k is ONE correctly rounded double division of two
// integers below 2^53 -- the value numpy's true division gives -- and a compare against rel_threshold (NaN: false).
//
// Same three launches as K5: per-CTA site counts, the one-CTA scan of those counts (K5's own scan kernel), then a
// scatter that re-evaluates the rule and writes the records in ascending slot order: the order is the slot order, no
// atomic decides it.  The extra slot behind a contig and the padding are never sites (K5's `is_position`).
// n_slots % 4 == 0: one thread = 4 slots, six 128-bit loads; 24 B per slot are read by each of the two passes.

namespace kdl {

struct VariantArgs {
    const int32_t* counts;  // [19][n_slots]; columns 0-5 are read
    long long n_slots;
    AssembleArgs layout;    // contig_slot / contig_len / n_contigs, for is_position
    long long abs_floor;
    double rel_threshold;
};

// bit k set: allele k is a variant at this slot (not yet restricted to positions)
__device__ __forceinline__ unsigned variant_bits(const int (&t)[6], long long abs_floor, double rel) {
    long long depth = 0;
    int top = 0, best = t[0];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        depth += t[k];
        if (t[k] > best) { best = t[k]; top = k; }  // first maximum
    }
    unsigned bits = 0;
    const double d = (double)depth;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        // the division only for the alleles the count test leaves (most of them fail it): it dominates the cost
        if (k != top && (long long)t[k] > abs_floor) {
            const double share = depth > 0 ? (double)t[k] / d : 0.0;
            if (share > rel) bits |= 1u << k;
        }
    }
    return bits;
}

// the counts and variant bits of the 4 slots from s (s % 4 == 0, s < n_slots); bits are 0 at every slot that is not a
// position
__device__ __forceinline__ void variant_quad(const VariantArgs& a, long long s, int (&t)[4][6], unsigned (&bits)[4]) {
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const int4 v = __ldg(reinterpret_cast<const int4*>(a.counts + (long long)k * a.n_slots + s));
        t[0][k] = v.x; t[1][k] = v.y; t[2][k] = v.z; t[3][k] = v.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        bits[j] = variant_bits(t[j], a.abs_floor, a.rel_threshold);
        if (bits[j] && !is_position(a.layout, s + j)) bits[j] = 0;  // slot L behind a contig, padding
    }
}

__global__ void __launch_bounds__(A_THREADS)
variant_sums_kernel(VariantArgs a, uint32_t* __restrict__ block_sums) {
    const long long s = (long long)blockIdx.x * A_BLOCK + (long long)A_PER * threadIdx.x;
    uint32_t n = 0;
    if (s < a.n_slots) {
        int t[4][6];
        unsigned bits[4];
        variant_quad(a, s, t, bits);
        n = (bits[0] != 0) + (bits[1] != 0) + (bits[2] != 0) + (bits[3] != 0);
    }
    uint32_t total;
    cta_exclusive_scan(n, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// block_sums: the exclusive prefix assemble_scan_sums_kernel left.  Records: site_slot[i], site_counts[k * n_sites + i]
// (k = 0..5, column-major like the table), site_mask[i] (bits 0-5 = the variant alleles).
__global__ void __launch_bounds__(A_THREADS)
variant_scatter_kernel(VariantArgs a, const uint32_t* __restrict__ block_sums, long long n_sites,
                       int64_t* __restrict__ site_slot, int32_t* __restrict__ site_counts,
                       uint8_t* __restrict__ site_mask) {
    const long long s = (long long)blockIdx.x * A_BLOCK + (long long)A_PER * threadIdx.x;
    int t[4][6];
    unsigned bits[4] = {0u, 0u, 0u, 0u};
    uint32_t n = 0;
    if (s < a.n_slots) {
        variant_quad(a, s, t, bits);
        n = (bits[0] != 0) + (bits[1] != 0) + (bits[2] != 0) + (bits[3] != 0);
    }
    uint32_t total;
    long long o = (long long)block_sums[blockIdx.x] + cta_exclusive_scan(n, &total);
    if (!n) return;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (!bits[j]) continue;
        if (o < n_sites) {  // (n_sites is the count the first pass found; the guard only keeps a wrong one in bounds)
            site_slot[o] = s + j;
#pragma unroll
            for (int k = 0; k < 6; ++k) site_counts[(long long)k * n_sites + o] = t[j][k];
            site_mask[o] = (uint8_t)bits[j];
        }
        ++o;
    }
}

}  // namespace kdl
