// quality.cu -- K11 / K11g: the reads' base qualities summed per position and base (extension: `variants --vcf --qual`).
//
// The counted bases are exactly those the pileup counts in columns 0-3: M/=/X bases whose nibble is A, C, G or T after
// every mask (a base masked by quality, primer or mate overlap is an N nibble and adds nothing; clipped and inserted
// bases, N and deletions add nothing).  Per slot s:
//   qsum[k * n_slots + s]  uint32  the summed Phred of the counted bases of allele k (k = 0..3: A, C, G, T)
//   emass[s]               uint64  the summed EPS[min(q, 93)] over the slot's counted bases, EPS[q] the integer nearest
//                                  to 2^32 * 10^(-q / 10): the expected number of sequencing errors, in units of 2^-32
// Both are integer sums, so the result does not depend on the order the bases are added in.
//
// K11 (quality_tile_kernel) is the tile-owner kernel of a coordinate-sorted batch: one CTA per 512-slot tile takes the
// reads [lo, hi) of K0's index, stages their starts and words in chunks of 1024 reads, and counts them without a global
// atomic.  Each of its 8 warps owns a 64-slot window and finds the chunk's reads that can reach it with two warp
// searches; a lane owns 8 consecutive slots, and the four quarter-warps walk different reads (as K1's consumers do).
// For a simple read, the 8 bases a lane needs are ONE funnel shift of two seq4 words and their qualities one funnel
// shift of two 8-byte qual8 words (qual8 rides beside seq4: base k of read r is byte 8 * seq_off[r] + k).  The sums stay
// in registers; the quarters are added by shuffles at the end.  Tile-eligible complex reads (~1 % of a short-read BAM)
// are walked through the CIGAR behind their bases by one warp each (its lanes over an op's bases), with shared-memory
// atomics into the tile; by the flatten contract they never wrap.  The tile is then written with plain stores: no zeroing pass.
//
// K11g (quality_general_kernel) walks what K11 leaves out: the KDL_HARD reads after K11 (K1g's walk, its Python index
// wrap and right-clip stall included), or every read of a batch K11 cannot take (unsorted, or no tile_index) after a
// zeroing pass -- one warp per read, global atomics (a native 64-bit RED for emass; in shared memory the 64-bit add is a
// CAS loop, which only K11's complex reads take).
//
// K11w / K11g-w (extension: `consensus --quality-vote`) are the same kernels with the WeightSums policy: per slot
//   wsum[k * n_slots + s]  uint64  the summed W[min(q, 93)] of the counted bases of allele k (the table below)
// A lane sums a chunk in uint32 registers, and the four quarters fold them into uint64 at the chunk's end.
#include "tile_common.cuh"

namespace kdl {

constexpr int kQtThreads = 256;  // 8 warps x 64 slots = one tile
constexpr int kQtChunk = 1024;   // reads staged per round (lower_bound_warp searches at most 1024)
constexpr int kEpsMax = 93;

// EPS[q] = round(2^32 * 10^(-q / 10)), q = 0..93 (tests/test_variant_qual.py pins it against an exact computation)
__constant__ unsigned long long kQualEps[kEpsMax + 1] = {
    4294967296ull, 3411613790ull, 2709941160ull, 2152582778ull, 1709857278ull, 1358187913ull,
    1078847007ull, 856958639ull, 680706443ull, 540704347ull, 429496730ull, 341161379ull,
    270994116ull, 215258278ull, 170985728ull, 135818791ull, 107884701ull, 85695864ull,
    68070644ull, 54070435ull, 42949673ull, 34116138ull, 27099412ull, 21525828ull,
    17098573ull, 13581879ull, 10788470ull, 8569586ull, 6807064ull, 5407043ull,
    4294967ull, 3411614ull, 2709941ull, 2152583ull, 1709857ull, 1358188ull,
    1078847ull, 856959ull, 680706ull, 540704ull, 429497ull, 341161ull,
    270994ull, 215258ull, 170986ull, 135819ull, 107885ull, 85696ull,
    68071ull, 54070ull, 42950ull, 34116ull, 27099ull, 21526ull,
    17099ull, 13582ull, 10788ull, 8570ull, 6807ull, 5407ull,
    4295ull, 3412ull, 2710ull, 2153ull, 1710ull, 1358ull,
    1079ull, 857ull, 681ull, 541ull, 429ull, 341ull,
    271ull, 215ull, 171ull, 136ull, 108ull, 86ull,
    68ull, 54ull, 43ull, 34ull, 27ull, 22ull,
    17ull, 14ull, 11ull, 9ull, 7ull, 5ull,
    4ull, 3ull, 3ull, 2ull,
};

// W[q] = the integer nearest to 2^16 * 10 log10(3 (1 - e) / e), e = min(10^(-q / 10), 3/4), q = 0..93: the log-likelihood
// ratio, in 1/65536 Phred, of "the true base is the one read" against "it is one particular other base", the error
// spread evenly over the other three (tests/test_quality_vote.py pins it against an exact computation)
__constant__ uint32_t kQualWeight[kEpsMax + 1] = {
    0u, 0u, 160037u, 311335u, 430336u, 532174u, 623571u, 708096u,
    787861u, 864214u, 938059u, 1010026u, 1080568u, 1150020u, 1218628u, 1286580u,
    1354022u, 1421062u, 1487787u, 1554264u, 1620546u, 1686672u, 1752677u, 1818584u,
    1884415u, 1950185u, 2015906u, 2081590u, 2147243u, 2212872u, 2278481u, 2344076u,
    2409659u, 2475232u, 2540797u, 2606356u, 2671911u, 2737461u, 2803009u, 2868554u,
    2934098u, 2999640u, 3065180u, 3130720u, 3196259u, 3261797u, 3327335u, 3392873u,
    3458410u, 3523947u, 3589483u, 3655020u, 3720556u, 3786093u, 3851629u, 3917165u,
    3982701u, 4048238u, 4113774u, 4179310u, 4244846u, 4310382u, 4375918u, 4441454u,
    4506990u, 4572526u, 4638062u, 4703598u, 4769134u, 4834670u, 4900206u, 4965742u,
    5031278u, 5096814u, 5162350u, 5227886u, 5293422u, 5358958u, 5424494u, 5490030u,
    5555566u, 5621102u, 5686638u, 5752174u, 5817710u, 5883246u, 5948782u, 6014318u,
    6079854u, 6145390u, 6210926u, 6276462u, 6341998u, 6407534u,
};

// column 0..3 of a one-hot nibble (A=1 C=2 G=4 T=8), -1 for anything else (N, padding, exotic bases)
__device__ __forceinline__ int acgt_col(uint32_t nib) {
    return (nib == 1u) ? 0 : (nib == 2u) ? 1 : (nib == 4u) ? 2 : (nib == 8u) ? 3 : -1;
}

__device__ __forceinline__ uint32_t clamp_q(uint32_t q) { return q < kEpsMax ? q : kEpsMax; }

template <class Sums>
__device__ __forceinline__ void load_table(typename Sums::Entry* tab) {
    for (int i = threadIdx.x; i <= kEpsMax; i += blockDim.x) tab[i] = Sums::entry(i);
}

// Sum policies of K11 / K11g (template arguments): what a counted base of quality q adds to its slot and where the sums
// live.  In K11 a lane keeps the sums of its 8 slots in registers (Regs), the tile's complex reads add into shared
// memory (Smem), and store() writes the tile; K11g adds to the tables with global atomics.
struct PhredSums {  // `variants --vcf --qual`: qsum[4][n_slots] uint32 and emass[n_slots] uint64
    uint32_t* qsum;
    unsigned long long* emass;
    using Entry = unsigned long long;
    static constexpr int kMinBlocks = 0;  // (0: no minimum, the launch bounds K11 always had)
    __device__ static Entry entry(int q) { return kQualEps[q]; }
    struct Smem {
        uint32_t q[4][KDL_TILE];
        unsigned long long e[KDL_TILE];
    };
    struct Regs {
        uint32_t s[4][8];
        unsigned long long e[8];
    };
    __device__ static void zero(Smem& sm, int i) {
        sm.q[0][i] = 0u; sm.q[1][i] = 0u; sm.q[2][i] = 0u; sm.q[3][i] = 0u;
        sm.e[i] = 0ull;
    }
    __device__ static void zero(Regs& r) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { r.s[0][j] = r.s[1][j] = r.s[2][j] = r.s[3][j] = 0u; r.e[j] = 0ull; }
    }
    __device__ static void add(Regs& r, int j, uint32_t nib, uint32_t q, const Entry* tab) {
        r.s[0][j] += nib == 1u ? q : 0u;
        r.s[1][j] += nib == 2u ? q : 0u;
        r.s[2][j] += nib == 4u ? q : 0u;
        r.s[3][j] += nib == 8u ? q : 0u;
        r.e[j] += (nib && !(nib & (nib - 1u))) ? tab[clamp_q(q)] : 0ull;
    }
    __device__ static void end_chunk(Regs&, int) {}
    __device__ static void add(Smem& sm, int col, int slot, uint32_t q, const Entry* tab) {
        atomicAdd(&sm.q[col][slot], q);
        atomicAdd(&sm.e[slot], tab[clamp_q(q)]);
    }
    __device__ void add(long long slot, long long n_slots, int col, uint32_t q, const Entry* tab) const {
        atomicAdd(qsum + (long long)col * n_slots + slot, q);
        atomicAdd(emass + slot, tab[clamp_q(q)]);
    }
    // the four quarters hold partial sums of the same 8 slots: add them, then quarter q writes column q, quarter 0 emass
    __device__ void store(Regs& r, const Smem& sm, int quarter, int a0, long long t0, long long n_slots) const {
        uint32_t out[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            uint32_t x = r.s[0][j], y = r.s[1][j], z = r.s[2][j], w = r.s[3][j];
            unsigned long long m = r.e[j];
            x += __shfl_xor_sync(0xffffffffu, x, 8);  x += __shfl_xor_sync(0xffffffffu, x, 16);
            y += __shfl_xor_sync(0xffffffffu, y, 8);  y += __shfl_xor_sync(0xffffffffu, y, 16);
            z += __shfl_xor_sync(0xffffffffu, z, 8);  z += __shfl_xor_sync(0xffffffffu, z, 16);
            w += __shfl_xor_sync(0xffffffffu, w, 8);  w += __shfl_xor_sync(0xffffffffu, w, 16);
            m += __shfl_xor_sync(0xffffffffu, m, 8);  m += __shfl_xor_sync(0xffffffffu, m, 16);
            out[j] = (quarter == 0 ? x : quarter == 1 ? y : quarter == 2 ? z : w) + sm.q[quarter][a0 + j];
            r.e[j] = m + sm.e[a0 + j];
        }
        uint4* dq = reinterpret_cast<uint4*>(qsum + (long long)quarter * n_slots + t0 + a0);
        dq[0] = make_uint4(out[0], out[1], out[2], out[3]);
        dq[1] = make_uint4(out[4], out[5], out[6], out[7]);
        if (quarter == 0) {
            ulonglong2* de = reinterpret_cast<ulonglong2*>(emass + t0 + a0);
#pragma unroll
            for (int j = 0; j < 4; ++j) de[j] = make_ulonglong2(r.e[2 * j], r.e[2 * j + 1]);
        }
    }
    __device__ void zero_tables(long long gtid, long long stride, long long n_slots) const {
        for (long long s = gtid; s < 4 * n_slots; s += stride) qsum[s] = 0u;
        for (long long s = gtid; s < n_slots; s += stride) emass[s] = 0ull;
    }
};

struct WeightSums {  // `consensus --quality-vote`: wsum[4][n_slots] uint64, the summed W[min(q, 93)] per base
    unsigned long long* wsum;
    using Entry = uint32_t;
    static constexpr int kMinBlocks = 1;  // (without it ptxas caps K11w at 64 registers and spills)
    __device__ static Entry entry(int q) { return kQualWeight[q]; }
    struct Smem {
        unsigned long long w[4][KDL_TILE];
    };
    // s: the chunk's partial sums -- a quarter-warp adds at most kQtChunk / 4 = 256 reads to a slot per chunk, and
    // 256 * W[93] < 2^32, so uint32 is exact; w: the folded sums of column `quarter` of the lane's 8 slots
    struct Regs {
        uint32_t s[4][8];
        unsigned long long w[8];
    };
    __device__ static void zero(Smem& sm, int i) { sm.w[0][i] = 0ull; sm.w[1][i] = 0ull; sm.w[2][i] = 0ull; sm.w[3][i] = 0ull; }
    __device__ static void zero(Regs& r) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { r.s[0][j] = r.s[1][j] = r.s[2][j] = r.s[3][j] = 0u; r.w[j] = 0ull; }
    }
    __device__ static void add(Regs& r, int j, uint32_t nib, uint32_t q, const Entry* tab) {
        const uint32_t w = tab[clamp_q(q)];
        r.s[0][j] += nib == 1u ? w : 0u;
        r.s[1][j] += nib == 2u ? w : 0u;
        r.s[2][j] += nib == 4u ? w : 0u;
        r.s[3][j] += nib == 8u ? w : 0u;
    }
    // the chunk's partials of the four quarters, added in 64 bits; quarter q keeps column q (whole warp, converged)
    __device__ static void end_chunk(Regs& r, int quarter) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                unsigned long long x = r.s[k][j];
                x += __shfl_xor_sync(0xffffffffu, x, 8);
                x += __shfl_xor_sync(0xffffffffu, x, 16);
                r.w[j] += quarter == k ? x : 0ull;
                r.s[k][j] = 0u;
            }
        }
    }
    __device__ static void add(Smem& sm, int col, int slot, uint32_t q, const Entry* tab) {
        atomicAdd(&sm.w[col][slot], (unsigned long long)tab[clamp_q(q)]);
    }
    __device__ void add(long long slot, long long n_slots, int col, uint32_t q, const Entry* tab) const {
        atomicAdd(wsum + (long long)col * n_slots + slot, (unsigned long long)tab[clamp_q(q)]);
    }
    __device__ void store(Regs& r, const Smem& sm, int quarter, int a0, long long t0, long long n_slots) const {
        ulonglong2* dw = reinterpret_cast<ulonglong2*>(wsum + (long long)quarter * n_slots + t0 + a0);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            dw[j] = make_ulonglong2(r.w[2 * j] + sm.w[quarter][a0 + 2 * j], r.w[2 * j + 1] + sm.w[quarter][a0 + 2 * j + 1]);
    }
    __device__ void zero_tables(long long gtid, long long stride, long long n_slots) const {
        for (long long s = gtid; s < 4 * n_slots; s += stride) wsum[s] = 0ull;
    }
};

template <class Sums>
__global__ void __launch_bounds__(kQtThreads, Sums::kMinBlocks)
quality_tile_kernel(kdl_batch b, const uint8_t* __restrict__ qual8, Sums sums, long long n_slots,
                    const uint32_t* __restrict__ index) {
    __shared__ typename Sums::Smem s_sum;            // the complex reads' sums
    __shared__ typename Sums::Entry s_tab[kEpsMax + 1];
    __shared__ int s_start[kQtChunk];                // read start slot relative to the tile (clamped)
    __shared__ uint32_t s_off[kQtChunk];
    __shared__ uint32_t s_lw[kQtChunk];
    __shared__ int s_cx[kQtChunk];                   // the chunk's tile-eligible complex reads
    __shared__ int s_ncx;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long t0 = (long long)blockIdx.x * KDL_TILE;
    const uint32_t* e = index + F_IDX * blockIdx.x;
    const long long lo = e[0], hi = e[1];
    for (int i = threadIdx.x; i < KDL_TILE; i += blockDim.x) Sums::zero(s_sum, i);
    load_table<Sums>(s_tab);
    const uint64_t* __restrict__ qw = reinterpret_cast<const uint64_t*>(qual8);  // 8 qualities per seq4 word

    const int quarter = lane >> 3;
    const int a0 = warp * 64 + 8 * (lane & 7);  // the lane's first slot, relative to the tile
    typename Sums::Regs acc;
    Sums::zero(acc);

    for (long long base = lo; base < hi; base += kQtChunk) {
        const int n = (int)(hi - base < kQtChunk ? hi - base : kQtChunk);
        __syncthreads();  // (the previous chunk's readers are done; the first time: the zeroing and the table)
        if (threadIdx.x == 0) s_ncx = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const long long r = base + i;
            const int c = find_contig(b.contig_read_off, b.n_contigs, r);
            long long g = b.contig_slot[c] + b.ref_start[r] - t0;
            g = g < -(1ll << 30) ? -(1ll << 30) : (g > (1ll << 30) ? (1ll << 30) : g);
            const uint32_t lw = (uint32_t)b.l_seq[r];
            s_start[i] = (int)g;
            s_off[i] = b.seq_off[r];
            s_lw[i] = lw;
            if ((lw & (KDL_COMPLEX | KDL_HARD)) == KDL_COMPLEX && g < KDL_TILE && g > -KDL_TILE_MAXREACH - KDL_FAST_MAXLEN)
                s_cx[atomicAdd(&s_ncx, 1)] = i;  // a tile-eligible complex read: a warp walks it below
        }
        __syncthreads();
        int ra, re;
        lower_bound_warp2(s_start, n, warp * 64 - b.reach_right + 1, warp * 64 + 64, lane, ra, re);
        for (int i = ra + quarter; i < re; i += 4) {
            const uint32_t lw = s_lw[i];
            if (lw & KDL_COMPLEX) continue;  // (the warp walks below, or K11g)
            const int len = (int)lw;
            const int d = a0 - s_start[i];  // the lane's first slot as a query offset of the read
            if (d + 8 <= 0 || d >= len) continue;
            const int k = d >> 3, sh = d & 7, nw = (len + 7) >> 3;
            const uint32_t off = s_off[i];
            const bool in0 = k >= 0, in1 = k + 1 < nw;  // (k < nw always holds, k + 1 >= 0 too)
            const uint32_t w0 = in0 ? b.seq4[off + k] : 0u, w1 = in1 ? b.seq4[off + k + 1] : 0u;
            const uint64_t q0 = in0 ? qw[off + k] : 0ull, q1 = in1 ? qw[off + k + 1] : 0ull;
            const uint32_t word = __funnelshift_l(w1, w0, 4 * sh);  // nibbles d .. d + 7, outside the read 0
            const uint64_t qv = sh ? (q0 >> (8 * sh)) | (q1 << (64 - 8 * sh)) : q0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint32_t nib = (word >> (28 - 4 * j)) & 0xFu;
                const uint32_t q = (uint32_t)(qv >> (8 * j)) & 0xFFu;
                Sums::add(acc, j, nib, q, s_tab);
            }
        }
        Sums::end_chunk(acc, quarter);
        // the complex reads: one warp per read walks its CIGAR (warp-uniform), the lanes stride over an op's bases that
        // land in this tile, shared-memory atomics
        for (int j = warp; j < s_ncx; j += kQtThreads / 32) {
            const int i = s_cx[j];
            const uint32_t* __restrict__ seq = b.seq4 + s_off[i];
            const uint32_t* __restrict__ blk = seq + (((s_lw[i] & KDL_LEN_MASK) + 7) >> 3);
            const int n_ops = (int)blk[0];
            const uint8_t* __restrict__ qr = qual8 + 8ull * s_off[i];
            int r_pos = s_start[i], q_pos = 0;
            for (int o = 0; o < n_ops && r_pos < KDL_TILE; ++o) {
                const uint32_t cg = blk[2 + o];
                const int len = (int)(cg >> 4), op = (int)(cg & 0xF);
                if (op == 0 || op == 7 || op == 8) {  // M = X
                    const int d0 = r_pos < 0 ? -r_pos : 0;
                    const int d1 = r_pos + len > KDL_TILE ? KDL_TILE - r_pos : len;
                    for (int d = d0 + lane; d < d1; d += 32) {
                        const int col = acgt_col((uint32_t)nibble_at(seq, q_pos + d));
                        if (col < 0) continue;
                        Sums::add(s_sum, col, r_pos + d, (uint32_t)qr[q_pos + d], s_tab);
                    }
                    r_pos += len;
                    q_pos += len;
                } else if (op == 1) {  // I
                    q_pos += len;
                } else if (op == 2) {  // D
                    r_pos += len;
                } else if (op == 4) {  // S: a left clip advances the query only, a right clip both cursors
                    if (o > 0) r_pos += len;
                    q_pos += len;
                }
            }
        }
    }
    __syncthreads();  // the complex reads' shared sums are complete (also when the tile has no read)
    sums.store(acc, s_sum, quarter, a0, t0, n_slots);
}

// K11g: one warp per read of `list` (NULL: every read), K1g's walk (kindel.py:40-81 with the Python index wrap and the
// right-clip stall); a simple read is one M op.  Bases that would raise in K1g are skipped (the pileup raises then).
template <class Sums>
__global__ void __launch_bounds__(256)
quality_general_kernel(kdl_batch b, const uint8_t* __restrict__ qual8, const uint32_t* __restrict__ list, long long n_list,
                       Sums sums, long long n_slots) {
    __shared__ typename Sums::Entry s_tab[kEpsMax + 1];
    load_table<Sums>(s_tab);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long j = warp0; j < n_list; j += n_warps) {
        const long long r = list ? (long long)list[j] : j;
        const uint32_t lraw = (uint32_t)b.l_seq[r];
        const int c = find_contig(b.contig_read_off, b.n_contigs, r);
        const long long L = b.contig_len[c], slot0 = b.contig_slot[c];
        const uint32_t* __restrict__ seq = b.seq4 + (size_t)b.seq_off[r];
        const uint8_t* __restrict__ qr = qual8 + 8ull * b.seq_off[r];
        const bool cx = (lraw & KDL_COMPLEX) != 0;
        const long long lseq = cx ? complex_len(lraw) : (long long)lraw;
        const uint32_t* __restrict__ blk = seq + ((lseq + 7) >> 3);
        const uint32_t n_ops = cx ? blk[0] : 1u;
        long long r_pos = b.ref_start[r], q_pos = 0;
        for (uint32_t i = 0; i < n_ops; ++i) {
            const uint32_t cg = cx ? blk[2 + i] : (uint32_t)(lseq << 4);
            const long long len = cg >> 4;
            const int op = cg & 0xF;
            if (op == 0 || op == 7 || op == 8) {  // M = X
                for (long long k = lane; k < len; k += 32) {
                    const long long q = q_pos + k, idx = pyindex(r_pos + k, L);
                    if (q >= lseq || idx < 0) continue;
                    const int col = acgt_col((uint32_t)nibble_at(seq, q));
                    if (col < 0) continue;
                    sums.add(slot0 + idx, n_slots, col, (uint32_t)qr[q], s_tab);
                }
                r_pos += len;
                q_pos += len;
            } else if (op == 1) {  // I
                q_pos += len;
            } else if (op == 2) {  // D
                r_pos += len;
            } else if (op == 4) {  // S
                if (i == 0) {
                    q_pos += len;
                } else {  // a right clip advances while r_pos < L (kindel.py:78-81)
                    long long n_adv = L - r_pos;
                    n_adv = n_adv < 0 ? 0 : (n_adv > len ? len : n_adv);
                    r_pos += n_adv;
                    q_pos += n_adv;
                }
            }
        }
    }
}

template <class Sums>
__global__ void __launch_bounds__(256) quality_zero_kernel(Sums sums, long long n_slots) {
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    sums.zero_tables(gtid, stride, n_slots);
}

}  // namespace kdl
