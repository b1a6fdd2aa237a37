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
//
// The two passes are templates over a site policy (`variant_sums` / `variant_scatter`), the way the IUPAC vote is a
// policy of K2: VariantArgs is K6's, RefVariantArgs (K6r, below) compares against reference bases.
//
// K7 `deletion_*_kernel` (extension, at the end): the deletion events (slot, length) of the complex reads' CIGARs,
// in read order and then op order, with the same count / scan / scatter shape over reads instead of slots.

namespace kdl {

struct VariantArgs {
    const int32_t* counts;  // [19][n_slots]; columns 0-5 are read
    long long n_slots;
    AssembleArgs layout;    // contig_slot / contig_len / n_contigs, for is_position
    long long abs_floor;
    double rel_threshold;

    // the site policy of the two passes
    struct Quad { int t[4][6]; };                                  // what one thread keeps of its 4 slots
    struct Out { int64_t* slot; int32_t* counts; uint8_t* mask; };  // the records
    __device__ __forceinline__ void load(long long, Quad&) const {}  // (every thread; nothing to share)
    __device__ __forceinline__ void eval(long long s, Quad& q, unsigned (&bits)[4]) const;
    __device__ __forceinline__ void write(const Out& out, const Quad& q, int j, long long o, long long n_sites,
                                          long long slot, unsigned bits) const;
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

__device__ __forceinline__ void VariantArgs::eval(long long s, Quad& q, unsigned (&bits)[4]) const {
    variant_quad(*this, s, q.t, bits);
}

__device__ __forceinline__ void VariantArgs::write(const Out& out, const Quad& q, int j, long long o, long long n_sites,
                                                   long long slot, unsigned bits) const {
    out.slot[o] = slot;
#pragma unroll
    for (int k = 0; k < 6; ++k) out.counts[(long long)k * n_sites + o] = q.t[j][k];
    out.mask[o] = (uint8_t)bits;
}

// ---- the two passes, over any site policy P ------------------------------------------------------------------
// P::load runs on every thread of the CTA (s may lie past the table: it may hold warp collectives); P::eval only for
// s < n_slots, and sets bits[j] != 0 for each of the 4 slots that is a site; P::write stores site j as record o.
template <class P>
__device__ __forceinline__ void variant_sums(const P& a, uint32_t* __restrict__ block_sums) {
    const long long s = (long long)blockIdx.x * A_BLOCK + (long long)A_PER * threadIdx.x;
    uint32_t n = 0;
    typename P::Quad q;
    a.load(s, q);
    if (s < a.n_slots) {
        unsigned bits[4];
        a.eval(s, q, bits);
        n = (bits[0] != 0) + (bits[1] != 0) + (bits[2] != 0) + (bits[3] != 0);
    }
    uint32_t total;
    cta_exclusive_scan(n, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

template <class P>
__device__ __forceinline__ void variant_scatter(const P& a, const uint32_t* __restrict__ block_sums, long long n_sites,
                                                const typename P::Out& out) {
    const long long s = (long long)blockIdx.x * A_BLOCK + (long long)A_PER * threadIdx.x;
    typename P::Quad q;
    unsigned bits[4] = {0u, 0u, 0u, 0u};
    uint32_t n = 0;
    a.load(s, q);
    if (s < a.n_slots) {
        a.eval(s, q, bits);
        n = (bits[0] != 0) + (bits[1] != 0) + (bits[2] != 0) + (bits[3] != 0);
    }
    uint32_t total;
    long long o = (long long)block_sums[blockIdx.x] + cta_exclusive_scan(n, &total);
    if (!n) return;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (!bits[j]) continue;
        // (n_sites is the count the first pass found; the guard only keeps a wrong one in bounds)
        if (o < n_sites) a.write(out, q, j, o, n_sites, s + j, bits[j]);
        ++o;
    }
}

__global__ void __launch_bounds__(A_THREADS)
variant_sums_kernel(VariantArgs a, uint32_t* __restrict__ block_sums) {
    variant_sums(a, block_sums);
}

// block_sums: the exclusive prefix assemble_scan_sums_kernel left.  Records: site_slot[i], site_counts[k * n_sites + i]
// (k = 0..5, column-major like the table), site_mask[i] (bits 0-5 = the variant alleles).
__global__ void __launch_bounds__(A_THREADS)
variant_scatter_kernel(VariantArgs a, const uint32_t* __restrict__ block_sums, long long n_sites,
                       int64_t* __restrict__ site_slot, int32_t* __restrict__ site_counts,
                       uint8_t* __restrict__ site_mask) {
    variant_scatter(a, block_sums, n_sites, VariantArgs::Out{site_slot, site_counts, site_mask});
}

// ---- K6r: sites against reference bases (`variants --vcf --reference`) ---------------------------------------
// Per slot s of contig c: p = s - contig_slot[c], g = ref[s] (0-3 = A, C, G, T; 4 = anything else, and every slot
// that is not a position), t = columns 0-6, depth(s) = t0 + ... + t5.
//   SNV bit k (k = 0..3), only at 0 <= p < L: k != g, t_k > abs_floor, t_k / depth(s) > rel (0 at depth 0).
//   insertion-candidate bit 6, at 0 <= p <= L (slot L holds the insertions behind the last base): t6 > abs_floor and
//   t6 / DPa > rel, DPa = depth(s - 1) for p >= 1 and depth(s) for p = 0.  Every inserted string's count is <= t6,
//   so the bit is necessary for any string to pass; the host tests the strings.
// depth(s - 1) of a thread's first slot comes from the lane that owns it (a shuffle); lane 0 loads it.  28 B of
// counts and 1 B of reference per slot are read by each pass.
struct RefVariantArgs {
    const int32_t* counts;  // [19][n_slots]; columns 0-6 are read
    long long n_slots;
    AssembleArgs layout;    // contig_slot / contig_len / n_contigs
    const uint8_t* ref;     // [n_slots] codes, 4-byte aligned
    long long abs_floor;
    double rel_threshold;

    struct Quad {
        int t[4][7];
        long long depth[4];
        long long prev;      // depth(s - 1) (0 at s = 0)
        long long dpa[4];    // DPa of each slot (set by eval where a bit is set)
        uint32_t g;          // the 4 reference codes, slot s in the low byte
    };
    struct Out { int64_t* slot; int32_t* counts; int64_t* dpa; uint8_t* mask; };
    __device__ __forceinline__ void load(long long s, Quad& q) const;
    __device__ __forceinline__ void eval(long long s, Quad& q, unsigned (&bits)[4]) const;
    __device__ __forceinline__ void write(const Out& out, const Quad& q, int j, long long o, long long n_sites,
                                          long long slot, unsigned bits) const;
};

__device__ __forceinline__ void RefVariantArgs::load(long long s, Quad& q) const {
    long long last = 0;
    if (s < n_slots) {
#pragma unroll
        for (int k = 0; k < 7; ++k) {
            const int4 v = __ldg(reinterpret_cast<const int4*>(counts + (long long)k * n_slots + s));
            q.t[0][k] = v.x; q.t[1][k] = v.y; q.t[2][k] = v.z; q.t[3][k] = v.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            long long d = 0;
#pragma unroll
            for (int k = 0; k < 6; ++k) d += q.t[j][k];
            q.depth[j] = d;
        }
        q.g = __ldg(reinterpret_cast<const uint32_t*>(ref + s));
        last = q.depth[3];
    }
    long long prev = __shfl_up_sync(0xffffffffu, last, 1);  // every lane: the whole warp takes part
    if ((threadIdx.x & 31) == 0) {                              // slot s - 1 belongs to the warp before
        prev = 0;
        if (s > 0 && s < n_slots) {
#pragma unroll
            for (int k = 0; k < 6; ++k) prev += __ldg(counts + (long long)k * n_slots + s - 1);
        }
    }
    q.prev = prev;
}

__device__ __forceinline__ unsigned ref_site_bits(const RefVariantArgs& a, long long s, const int (&t)[7], unsigned g,
                                                  long long depth, long long prev, long long* dpa) {
    unsigned bits = 0;
    const double d = (double)depth;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if ((unsigned)k != g && (long long)t[k] > a.abs_floor) {
            const double share = depth > 0 ? (double)t[k] / d : 0.0;
            if (share > a.rel_threshold) bits |= 1u << k;
        }
    }
    const bool ins = (long long)t[6] > a.abs_floor;
    if (!bits && !ins) return 0u;
    int lo = 0, hi = a.layout.n_contigs;  // the last contig with contig_slot <= s
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a.layout.contig_slot[mid] <= s) lo = mid + 1; else hi = mid;
    }
    if (lo == 0) return 0u;
    const long long p = s - a.layout.contig_slot[lo - 1], L = a.layout.contig_len[lo - 1];
    if (p >= L) bits = 0u;  // SNVs at positions only
    const long long da = p == 0 ? depth : prev;
    if (ins && p <= L) {
        const double share = da > 0 ? (double)t[6] / (double)da : 0.0;
        if (share > a.rel_threshold) bits |= 1u << 6;
    }
    *dpa = da;
    return bits;
}

__device__ __forceinline__ void RefVariantArgs::eval(long long s, Quad& q, unsigned (&bits)[4]) const {
#pragma unroll
    for (int j = 0; j < 4; ++j)
        bits[j] = ref_site_bits(*this, s + j, q.t[j], (q.g >> (8 * j)) & 0xFFu, q.depth[j],
                                j == 0 ? q.prev : q.depth[j - 1], &q.dpa[j]);
}

__device__ __forceinline__ void RefVariantArgs::write(const Out& out, const Quad& q, int j, long long o,
                                                      long long n_sites, long long slot, unsigned bits) const {
    out.slot[o] = slot;
#pragma unroll
    for (int k = 0; k < 7; ++k) out.counts[(long long)k * n_sites + o] = q.t[j][k];
    out.dpa[o] = q.dpa[j];
    out.mask[o] = (uint8_t)bits;
}

__global__ void __launch_bounds__(A_THREADS)
variant_ref_sums_kernel(RefVariantArgs a, uint32_t* __restrict__ block_sums) {
    variant_sums(a, block_sums);
}

// Records: site_slot[i], site_counts[k * n_sites + i] (k = 0..6), site_dpa[i], site_mask[i] (bits 0-3 SNV alleles
// A, C, G, T; bit 6 the insertion candidate).
__global__ void __launch_bounds__(A_THREADS)
variant_ref_scatter_kernel(RefVariantArgs a, const uint32_t* __restrict__ block_sums, long long n_sites,
                           int64_t* __restrict__ site_slot, int32_t* __restrict__ site_counts,
                           int64_t* __restrict__ site_dpa, uint8_t* __restrict__ site_mask) {
    variant_scatter(a, block_sums, n_sites, RefVariantArgs::Out{site_slot, site_counts, site_dpa, site_mask});
}

// ---- K6m: the sites of several samples at once (`variants --vcf a.bam b.bam ...`) ----------------------------
// counts = T, the samples' tables stacked over one shared layout: int32 [n_samples][7][n_slots].  Per slot, with t^i
// sample i's columns and depth^i = t0^i + ... + t5^i:
//   pooled (ref == NULL): P = sum_i t^i over columns 0-5 in int64, top = the first maximum of P; bit k (k = 0..5,
//     k != top) when some sample has t_k^i > abs_floor and t_k^i / depth^i > rel (0 at depth 0); positions only.
//   reference: bits 0-3 are K6r's SNV test of each sample against g, bit 6 K6r's insertion test with each sample's
//     own DPa; both ORed over the samples, at K6r's positions.
// The test of each sample does not depend on top, so one read of every sample's columns serves both halves of the
// pooled rule: the per-sample bits are ORed, P is summed beside them, and top's bit is cleared at the end.  The
// whole rule runs in `load` (every thread of the CTA), because the loop over samples holds DPa's shuffle: lanes past
// n_slots join it with zeros.  Only (slot, OR-ed mask) is written; the host gathers the samples' rows at the sites.
// Each pass reads 24 B (pooled) or 28 B + 1 B of reference (reference mode) per slot and sample.
template <bool kRef>
struct MultiVariantArgs {
    const int32_t* counts;  // [n_samples][7][n_slots]
    long long n_slots;
    int n_samples;
    AssembleArgs layout;    // contig_slot / contig_len / n_contigs of the shared layout
    const uint8_t* ref;     // [n_slots] codes (reference mode)
    long long abs_floor;
    double rel_threshold;

    static constexpr int kCols = kRef ? 7 : 6;
    static MultiVariantArgs make(const VariantArgs& v, int n_samples, const uint8_t* ref) {
        MultiVariantArgs a{};
        a.counts = v.counts; a.n_slots = v.n_slots; a.n_samples = n_samples; a.layout = v.layout; a.ref = ref;
        a.abs_floor = v.abs_floor; a.rel_threshold = v.rel_threshold;
        return a;
    }
    struct Quad { unsigned bits[4]; };
    struct Out { int64_t* slot; uint8_t* mask; };
    __device__ __forceinline__ void load(long long s, Quad& q) const;
    __device__ __forceinline__ void eval(long long, Quad& q, unsigned (&bits)[4]) const {
#pragma unroll
        for (int j = 0; j < 4; ++j) bits[j] = q.bits[j];
    }
    __device__ __forceinline__ void write(const Out& out, const Quad& q, int j, long long o, long long,
                                          long long slot, unsigned bits) const {
        out.slot[o] = slot;
        out.mask[o] = (uint8_t)bits;
    }
};

// where each of the 4 slots from s lies: bit 0 = a position (0 <= p < L), bit 1 = an insertion slot (0 <= p <= L),
// bit 2 = the first slot of its contig (p = 0); 3 bits per slot, slot s + j at bit 3j
__device__ __forceinline__ unsigned quad_places(const AssembleArgs& l, long long s) {
    int lo = 0, hi = l.n_contigs;  // the last contig with contig_slot <= s
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (l.contig_slot[mid] <= s) lo = mid + 1; else hi = mid;
    }
    int c = lo - 1;
    unsigned w = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        while (c + 1 < l.n_contigs && l.contig_slot[c + 1] <= s + j) ++c;  // (contigs of length 0 own one slot)
        if (c < 0) continue;
        const long long p = s + j - l.contig_slot[c], L = l.contig_len[c];
        w |= ((p < L ? 1u : 0u) | (p <= L ? 2u : 0u) | (p == 0 ? 4u : 0u)) << (3 * j);
    }
    return w;
}

template <bool kRef>
__device__ __forceinline__ void MultiVariantArgs<kRef>::load(long long s, Quad& q) const {
    const bool in = s < n_slots;
    const unsigned places = in ? quad_places(layout, s) : 0u;
    const uint32_t g = (kRef && in) ? __ldg(reinterpret_cast<const uint32_t*>(ref + s)) : 0u;
    unsigned acc[4] = {0u, 0u, 0u, 0u};
    long long pool[4][6];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int k = 0; k < 6; ++k) pool[j][k] = 0;
    const double rel = rel_threshold;
#pragma unroll 1
    for (int i = 0; i < n_samples; ++i) {  // uniform over the warp: every lane runs every sample
        const int32_t* __restrict__ tab = counts + (long long)i * 7 * n_slots;
        int t[4][kCols];
        long long depth[4] = {0, 0, 0, 0};
        if (in) {
#pragma unroll
            for (int k = 0; k < kCols; ++k) {
                const int4 v = __ldg(reinterpret_cast<const int4*>(tab + (long long)k * n_slots + s));
                t[0][k] = v.x; t[1][k] = v.y; t[2][k] = v.z; t[3][k] = v.w;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int k = 0; k < 6; ++k) depth[j] += t[j][k];
        }
        if (kRef) {
            long long prev = __shfl_up_sync(0xffffffffu, depth[3], 1);  // depth(s - 1) of this sample
            if ((threadIdx.x & 31) == 0) {
                prev = 0;
                if (s > 0 && in) {
#pragma unroll
                    for (int k = 0; k < 6; ++k) prev += __ldg(tab + (long long)k * n_slots + s - 1);
                }
            }
            if (!in) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const unsigned gj = (g >> (8 * j)) & 0xFFu;
                const double d = (double)depth[j];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if ((unsigned)k != gj && (long long)t[j][k] > abs_floor) {
                        const double share = depth[j] > 0 ? (double)t[j][k] / d : 0.0;
                        if (share > rel) acc[j] |= 1u << k;
                    }
                }
                if ((long long)t[j][6] > abs_floor) {
                    const long long da = (places >> (3 * j)) & 4u ? depth[j] : (j == 0 ? prev : depth[j - 1]);
                    const double share = da > 0 ? (double)t[j][6] / (double)da : 0.0;
                    if (share > rel) acc[j] |= 1u << 6;
                }
            }
        } else if (in) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const double d = (double)depth[j];
#pragma unroll
                for (int k = 0; k < 6; ++k) {
                    pool[j][k] += t[j][k];
                    if ((long long)t[j][k] > abs_floor) {
                        const double share = depth[j] > 0 ? (double)t[j][k] / d : 0.0;
                        if (share > rel) acc[j] |= 1u << k;
                    }
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const unsigned pl = (places >> (3 * j)) & 7u;
        unsigned b = acc[j];
        if (kRef) {
            b = (pl & 1u ? (b & 15u) : 0u) | (pl & 2u ? (b & 64u) : 0u);
        } else {
            int top = 0;
            long long best = pool[j][0];
#pragma unroll
            for (int k = 1; k < 6; ++k)
                if (pool[j][k] > best) { best = pool[j][k]; top = k; }  // first maximum
            b = pl & 1u ? b & ~(1u << top) : 0u;
        }
        q.bits[j] = b;
    }
}

template <bool kRef>
__global__ void __launch_bounds__(A_THREADS, 2)
variant_multi_sums_kernel(MultiVariantArgs<kRef> a, uint32_t* __restrict__ block_sums) {
    variant_sums(a, block_sums);
}

// Records: site_slot[i], site_mask[i] (pooled: bits 0-5 = alleles A, C, G, T, N, deletions; reference: bits 0-3 SNV
// alleles, bit 6 the insertion candidate), in ascending slot order.
template <bool kRef>
__global__ void __launch_bounds__(A_THREADS, 2)
variant_multi_scatter_kernel(MultiVariantArgs<kRef> a, const uint32_t* __restrict__ block_sums, long long n_sites,
                             int64_t* __restrict__ site_slot, uint8_t* __restrict__ site_mask) {
    variant_scatter(a, block_sums, n_sites, typename MultiVariantArgs<kRef>::Out{site_slot, site_mask});
}

// ---- K7: deletion events -------------------------------------------------------------------------------------
// One thread per read.  Simple reads (l_seq bit 31 clear) have no D op.  A complex read's CIGAR block sits behind its
// bases in seq4: [n_ops][evt_off][ops...].  The reference cursor moves as in kindel.py:40-81 (K1g restates it): M / = /
// X and D advance it; an S that is op #0 does not; any other S advances it while r_pos < L; I, N, H, P do not.  Each D
// of length n >= 1 at cursor r with 0 <= r and r + n <= L is the event (contig_slot + r, n); one that wraps (POS 0)
// or runs past the contig end is still in the table's deletion column but is no event.
template <class Emit>
__device__ __forceinline__ void walk_deletions(const kdl_batch& b, long long r, Emit&& emit) {
    const uint32_t lraw = (uint32_t)b.l_seq[r];
    if (!(lraw & KDL_COMPLEX)) return;
    const int c = find_contig(b.contig_read_off, b.n_contigs, r);
    const long long L = b.contig_len[c];
    const long long base = b.contig_slot[c];
    const uint32_t* __restrict__ blk = b.seq4 + (size_t)b.seq_off[r] + ((complex_len(lraw) + 7) >> 3);
    const uint32_t n_ops = blk[0];
    const uint32_t* __restrict__ ops = blk + 2;
    long long r_pos = b.ref_start[r];
    for (uint32_t i = 0; i < n_ops; ++i) {
        const uint32_t cg = ops[i];
        const long long len = cg >> 4;
        const int op = cg & 0xF;
        if (op == 0 || op == 7 || op == 8) {  // M = X
            r_pos += len;
        } else if (op == 2) {                 // D
            if (len > 0 && r_pos >= 0 && r_pos + len <= L) emit(base + r_pos, len);
            r_pos += len;
        } else if (op == 4 && i != 0) {       // right clip: advances while r_pos < L
            long long n_adv = L - r_pos;
            n_adv = n_adv < 0 ? 0 : (n_adv > len ? len : n_adv);
            r_pos += n_adv;
        }
    }
}

__global__ void __launch_bounds__(A_THREADS)
deletion_sums_kernel(kdl_batch b, uint32_t* __restrict__ block_sums) {
    const long long r = (long long)blockIdx.x * A_THREADS + threadIdx.x;
    uint32_t n = 0;
    if (r < b.n_reads) walk_deletions(b, r, [&](long long, long long) { ++n; });
    uint32_t total;
    cta_exclusive_scan(n, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// block_sums: the exclusive prefix of the per-CTA counts.  Events: ev_slot[i], ev_len[i], in read order, then op order.
__global__ void __launch_bounds__(A_THREADS)
deletion_scatter_kernel(kdl_batch b, const uint32_t* __restrict__ block_sums, long long n_events,
                        int64_t* __restrict__ ev_slot, int32_t* __restrict__ ev_len) {
    const long long r = (long long)blockIdx.x * A_THREADS + threadIdx.x;
    uint32_t n = 0;
    if (r < b.n_reads) walk_deletions(b, r, [&](long long, long long) { ++n; });
    uint32_t total;
    long long o = (long long)block_sums[blockIdx.x] + cta_exclusive_scan(n, &total);
    if (!n) return;
    walk_deletions(b, r, [&](long long slot, long long len) {
        if (o < n_events) {  // (as in K6: the guard only keeps a wrong count in bounds)
            ev_slot[o] = slot;
            ev_len[o] = (int32_t)len;
        }
        ++o;
    });
}

}  // namespace kdl
