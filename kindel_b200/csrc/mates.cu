// mates.cu -- K10p `mates_pair_kernel`, K10 `overlap_*_kernel` and K10u `overlap_untake_kernel` (extension:
// `--mask-overlaps`): where the two mates of one read pair cover the same reference positions, only the first mate
// (R1) is counted.  The second mate (R2) is masked there before the pileup, as min_base_quality masks a base (an N
// nibble in seq4, listed in the mask list so that K1q takes back its column-4 count), and its deletions and
// insertions there are taken back after the pileup (K10u).
//
// The rule (DESIGN.md section 1, include/kindel_b200.h K10):
//   pair      two reads of the batch with pair_role 1 and 2 that are the only ones with pair_role != 0 and their name
//             hash, on one contig, each starting where the other's mate_start says, neither KDL_HARD
//   covers    R1 covers cursor x (the walk of kindel.py:40-81) when it has an M/=/X base there, inside its SEQ, whose
//             nibble is not N (after the quality and the primer masks), or a D op over x
//   R2        its M/=/X bases at covered cursors are masked; a D op at [r, r + n) is dropped whole when R1 covers r;
//             an I op at slot p is dropped when R1 covers p - 1 and p
// Neither read of a pair is KDL_HARD, so every slot either touches lies inside [1, L - 1] of its contig: the slot of
// cursor x is contig_slot + x, with no Python index wrap, and a right clip advances the cursor by its whole length.
//
// K10p: the host compacts the reads with pair_role != 0 and sorts them by name hash (a torch sort, as K7's
// grouping); one thread per sorted entry then finds the groups of exactly two and checks the rest.
// K10 has K9's shape (primers.cu): a count pass, assemble_scan_sums_kernel over the rows that need prefixes, one CTA
// for the totals record, and a scatter that writes the merged mask list -- per read the sorted union of its own
// entries and its overlap bases --, R2's N nibbles in place, and one row per dropped D or I op.  R1 is only read and
// no read is both an R1 and an R2, so nothing races.  One thread per read: R1's coverage comes from walking both
// CIGARs together (a simple R1 is one M op: a range test and a nibble read).
// K10u: one thread per drop row, after K1q on the same stream, subtracts what K1w / K1e / K1g added for the dropped op
// (they also marked its sectors in the dirty map already).
#include "kdl_common.cuh"

namespace kdl {

constexpr int M_THREADS = 256;  // one read per thread; cta_scan_vec's CTA size (select.cu)
// rows of the scratch (n_blocks + 1 words each): the first M_NSCAN get exclusive prefixes, the others are summed
enum { M_MBASES = 0, M_MREADS, M_DROPS, M_PAIRS, M_OBASES, M_ODEL, M_OINS, M_NROW };
constexpr int M_NSCAN = 3;
constexpr int M_TOTALS = 8;  // words of the totals record behind the rows

// ---- K10p ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(M_THREADS) mates_clear_kernel(int32_t* __restrict__ mate, long long n) {
    for (long long i = (long long)blockIdx.x * M_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * M_THREADS)
        mate[i] = -1;
}

// order[0 .. m): the reads with pair_role != 0, sorted by name hash.  The first entry of every group of exactly two
// pairs them when the rule holds: mate[R2] = R1.
__global__ void __launch_bounds__(M_THREADS)
mates_pair_kernel(kdl_batch b, const uint64_t* __restrict__ hash, const int32_t* __restrict__ mate_start,
                  const uint8_t* __restrict__ role, const int32_t* __restrict__ order, long long m,
                  int32_t* __restrict__ mate) {
    const long long i = (long long)blockIdx.x * M_THREADS + threadIdx.x;
    if (i + 1 >= m) return;
    const long long a = order[i], c = order[i + 1];
    if (a < 0 || a >= b.n_reads || c < 0 || c >= b.n_reads) return;
    const uint64_t h = hash[a];
    if (hash[c] != h) return;                                     // a group of one
    auto at = [&](long long j) { return order[j] >= 0 && order[j] < b.n_reads && hash[order[j]] == h; };
    if (i > 0 && at(i - 1)) return;                                // not the group's first entry (or three or more)
    if (i + 2 < m && at(i + 2)) return;                            // three or more
    const int ra = role[a], rc = role[c];
    if (!((ra == 1 && rc == 2) || (ra == 2 && rc == 1))) return;
    if (((uint32_t)b.l_seq[a] | (uint32_t)b.l_seq[c]) & KDL_HARD) return;
    if (find_contig(b.contig_read_off, b.n_contigs, a) != find_contig(b.contig_read_off, b.n_contigs, c)) return;
    if (b.ref_start[a] != mate_start[c] || b.ref_start[c] != mate_start[a]) return;
    if (ra == 1) mate[c] = (int32_t)a; else mate[a] = (int32_t)c;
}

// ---- K10: R1's coverage -------------------------------------------------------------------------------------------
// covers(x) for non-decreasing x, walking R1's ops once.  lo / hi: the cursors R1's ops span.
struct Cover {
    const uint32_t* seq;
    const uint32_t* ops;
    int n_ops, o;
    int r_pos, q_pos, lseq, lo, hi;  // (neither mate is KDL_HARD: cursors and lengths fit 32 bits)
    bool simple;

    __device__ __forceinline__ void init(const kdl_batch& b, long long r) {
        const uint32_t lraw = (uint32_t)b.l_seq[r];
        seq = b.seq4 + (size_t)b.seq_off[r];
        lo = r_pos = b.ref_start[r];
        q_pos = 0;
        o = 0;
        simple = !(lraw & KDL_COMPLEX);
        if (simple) {
            lseq = (int)lraw;
            hi = lo + lseq;
            ops = nullptr;
            n_ops = 0;
            return;
        }
        lseq = (int)complex_len(lraw);
        const uint32_t* blk = seq + ((lseq + 7) >> 3);
        n_ops = (int)blk[0];
        ops = blk + 2;
        hi = lo;
        for (int k = 0; k < n_ops; ++k) {
            const int op = (int)(ops[k] & 0xF);
            if (op == 0 || op == 7 || op == 8 || op == 2 || (op == 4 && k != 0)) hi += (int)(ops[k] >> 4);
        }
    }

    __device__ __forceinline__ bool at(int x) {
        if (x < lo || x >= hi) return false;
        if (simple) return nibble_at(seq, x - lo) != 15;
        for (; o < n_ops; ++o) {  // step past the ops that end at or before x
            const int len = (int)(ops[o] >> 4);
            const int op = (int)(ops[o] & 0xF);
            const bool m = op == 0 || op == 7 || op == 8;
            if ((m || op == 2 || (op == 4 && o != 0)) && x < r_pos + len) break;
            if (m || (op == 4 && o != 0)) { r_pos += len; q_pos += len; }
            else if (op == 1 || op == 4) q_pos += len;
            else if (op == 2) r_pos += len;
        }
        if (o >= n_ops || x < r_pos) return false;
        const int op = (int)(ops[o] & 0xF);
        if (op == 2) return true;
        if (op == 0 || op == 7 || op == 8) {
            const int q = q_pos + (x - r_pos);
            return q < lseq && nibble_at(seq, q) != 15;
        }
        return false;  // a right clip
    }
};

// the M/=/X op [x0, x0 + len) of R2 at query q0: base(q0, q1) for the runs of its bases at covered cursors
template <class FB>
__device__ __forceinline__ void covered_runs(Cover& cv, int x0, int q0, int len, FB& base) {
    const int a = x0 > cv.lo ? x0 : cv.lo, e = x0 + len < cv.hi ? x0 + len : cv.hi;
    int run = -1;
    for (int x = a; x < e; ++x) {
        if (cv.at(x)) {
            if (run < 0) run = q0 + (x - x0);
        } else if (run >= 0) {
            base(run, q0 + (x - x0));
            run = -1;
        }
    }
    if (run >= 0) base(run, q0 + (e - x0));
}

// R2's overlap with R1: base(q0, q1) for the query ranges of its masked bases (ascending, disjoint), drop(slot, len,
// evt) for every dropped op (evt = its insertion-event row, -1 for a D), in op order.
template <class FB, class FD>
__device__ __forceinline__ void overlap_walk(const kdl_batch& b, long long r2, long long r1, FB&& base, FD&& drop) {
    Cover cv;
    cv.init(b, r1);
    const uint32_t lraw = (uint32_t)b.l_seq[r2];
    const int start = b.ref_start[r2];
    if (!(lraw & KDL_COMPLEX)) {
        covered_runs(cv, start, 0, (int)lraw, base);
        return;
    }
    const int c = find_contig(b.contig_read_off, b.n_contigs, r2);
    const long long slot0 = b.contig_slot[c];
    const int lseq = (int)complex_len(lraw);
    const uint32_t* blk = b.seq4 + (size_t)b.seq_off[r2] + ((lseq + 7) >> 3);
    const int n_ops = (int)blk[0];
    uint32_t evt = blk[1];
    const uint32_t* ops = blk + 2;
    int r_pos = start, q_pos = 0, ins_p = -1;
    bool ins_cov = false;
    for (int o = 0; o < n_ops; ++o) {
        const int len = (int)(ops[o] >> 4);
        const int op = (int)(ops[o] & 0xF);
        if (op == 0 || op == 7 || op == 8) {
            covered_runs(cv, r_pos, q_pos, len, base);
            r_pos += len;
            q_pos += len;
        } else if (op == 1) {
            if (r_pos != ins_p) {  // (a second I at the same slot asks what the first one asked)
                ins_p = r_pos;
                ins_cov = cv.at(r_pos - 1) && cv.at(r_pos);
            }
            if (ins_cov) drop(slot0 + r_pos, len, (long long)evt);
            ++evt;
            q_pos += len;
        } else if (op == 2) {
            if (cv.at(r_pos)) drop(slot0 + r_pos, len, -1ll);
            r_pos += len;
        } else if (op == 4) {
            if (o != 0) r_pos += len;
            q_pos += len;
        }
    }
}

// read r's share of the rows
__device__ __forceinline__ void overlap_item(const kdl_batch& b, const kdl_qmask& q, const int32_t* __restrict__ mate,
                                             long long r, uint32_t (&v)[M_NROW]) {
#pragma unroll
    for (int k = 0; k < M_NROW; ++k) v[k] = 0;
    if (r >= b.n_reads) return;
    uint32_t m0, m1;
    own_mask(q, r, &m0, &m1);
    const long long r1 = mate[r];
    MergeCount mc(q, m0, m1);  // (primers.cu: K9's merge of the own list with new bases)
    uint32_t nd = 0, ni = 0;
    if (r1 >= 0) {
        overlap_walk(
            b, r, r1, [&](long long q0, long long q1) { mc.add(q0, q1); },
            [&](long long, long long, long long evt) { if (evt < 0) ++nd; else ++ni; });
        v[M_PAIRS] = 1;
    }
    const uint32_t n_o = mc.added;
    v[M_MBASES] = mc.merged();
    v[M_MREADS] = v[M_MBASES] ? 1u : 0u;
    v[M_DROPS] = nd + ni;
    v[M_OBASES] = n_o;
    v[M_ODEL] = nd;
    v[M_OINS] = ni;
}

// row k of the scratch: scratch + k * (n_blocks + 1); the totals record behind the last row.  (The minimum of one CTA
// per SM lets ptxas keep the walk's state in registers: without it the kernel spills.)
__global__ void __launch_bounds__(M_THREADS, 1)
overlap_sums_kernel(kdl_batch b, kdl_qmask q, const int32_t* __restrict__ mate, uint32_t* __restrict__ scratch,
                    long long n_blocks) {
    uint32_t v[M_NROW], tot[M_NROW];
    overlap_item(b, q, mate, (long long)blockIdx.x * M_THREADS + threadIdx.x, v);
    cta_scan_vec(v, tot);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < M_NROW; ++k) scratch[(size_t)k * (n_blocks + 1) + blockIdx.x] = tot[k];
    }
}

// one CTA, after the scans of the first M_NSCAN rows: the totals record = [0] reads in the merged list, [1] bases in
// it, [2] drop rows, [3] pairs, [4] overlap bases, [5] dropped deletions, [6] dropped insertions, [7] 0
__global__ void __launch_bounds__(M_THREADS) overlap_totals_kernel(uint32_t* __restrict__ scratch, long long n_blocks) {
    uint32_t v[M_NROW - M_NSCAN], tot[M_NROW - M_NSCAN];
#pragma unroll
    for (int k = 0; k < M_NROW - M_NSCAN; ++k) v[k] = 0;
    for (long long i = threadIdx.x; i < n_blocks; i += M_THREADS) {
#pragma unroll
        for (int k = 0; k < M_NROW - M_NSCAN; ++k) v[k] += scratch[(size_t)(M_NSCAN + k) * (n_blocks + 1) + i];
    }
    cta_scan_vec(v, tot);
    if (threadIdx.x == 0) {
        uint32_t* rec = scratch + (size_t)M_NROW * (n_blocks + 1);
        rec[0] = scratch[(size_t)M_MREADS * (n_blocks + 1) + n_blocks];
        rec[1] = scratch[(size_t)M_MBASES * (n_blocks + 1) + n_blocks];
        rec[2] = scratch[(size_t)M_DROPS * (n_blocks + 1) + n_blocks];
#pragma unroll
        for (int k = 0; k < M_NROW - M_NSCAN; ++k) rec[M_NSCAN + k] = tot[k];
        rec[7] = 0;
    }
}

// `om` carries the caller's output arrays and the totals as its counts, `n_drops` the rows `drops` holds; every
// write is bounded by them.  drops[j] = (slot, len, read, evt), evt = -1 for a D.
__global__ void __launch_bounds__(M_THREADS)
overlap_scatter_kernel(kdl_batch b, kdl_qmask q, const int32_t* __restrict__ mate, const uint32_t* __restrict__ scratch,
                       long long n_blocks, uint32_t* seq4, kdl_qmask om, int32_t* __restrict__ drops, long long n_drops) {
    const long long r = (long long)blockIdx.x * M_THREADS + threadIdx.x;
    uint32_t v[M_NROW];
    overlap_item(b, q, mate, r, v);
    uint32_t p[M_NSCAN] = {v[M_MBASES], v[M_MREADS], v[M_DROPS]}, tot[M_NSCAN];
    cta_scan_vec(p, tot);
    const long long ob = (long long)p[0] + scratch[(size_t)M_MBASES * (n_blocks + 1) + blockIdx.x];
    const long long orr = (long long)p[1] + scratch[(size_t)M_MREADS * (n_blocks + 1) + blockIdx.x];
    long long od = (long long)p[2] + scratch[(size_t)M_DROPS * (n_blocks + 1) + blockIdx.x];
    if (blockIdx.x == 0 && threadIdx.x == 0 && om.n_reads > 0) const_cast<uint32_t*>(om.off)[om.n_reads] = (uint32_t)om.n_bases;
    if (!v[M_MBASES] && !v[M_DROPS]) return;
    // (a read with drop rows but no merged base gets no list entry: its writer's writes are all bounded away)
    MergeWrite mw = v[M_MBASES] ? merged_list_entry(q, om, r, orr, ob) : MergeWrite(q, 0, 0, nullptr, 0, 0);
    const long long r1 = mate[r];
    if (r1 >= 0) {
        uint32_t* words = seq4 + (size_t)b.seq_off[r];  // R2's own words; R1's are only read, from b.seq4
        overlap_walk(
            b, r, r1, [&](long long q0, long long q1) { mw.add(q0, q1, words); },
            [&](long long slot, long long len, long long evt) {
                if (od < n_drops)
                    reinterpret_cast<int4*>(drops)[od] = make_int4((int)slot, (int)len, (int)r, (int)evt);
                ++od;
            });
    }
    mw.finish();
}

// ---- K10u ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(M_THREADS)
overlap_untake_kernel(const int32_t* __restrict__ drops, long long n_drops, int32_t* __restrict__ counts,
                      long long n_slots) {
    const long long j = (long long)blockIdx.x * M_THREADS + threadIdx.x;
    if (j >= n_drops) return;
    const int4 d = reinterpret_cast<const int4*>(drops)[j];
    if (d.x < 0 || d.y < 0 || (long long)d.x + (d.w >= 0 ? 1 : d.y) > n_slots) return;  // (not a row K10 writes)
    if (d.w >= 0) {
        atomicAdd(counts + (long long)KDL_INS * n_slots + d.x, -1);
    } else {
        for (int k = 0; k < d.y; ++k) atomicAdd(counts + (long long)KDL_DEL * n_slots + d.x + k, -1);
    }
}

}  // namespace kdl
