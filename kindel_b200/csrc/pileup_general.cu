// pileup_general.cu -- K1g: the general CIGAR walk (any op mix), one warp per read, global atomics.
//
// Walks the reads the tile kernel leaves out: the KDL_HARD ones of a coordinate-sorted batch (they may wrap a
// Python index or raise, or are too long for a tile) -- listed in batch.hard_idx -- or, for batches the tile
// kernel cannot take at all (unsorted input), every complex read (list == NULL: all reads are scanned and the
// simple ones skipped).  A complex read's CIGAR sits behind its bases in seq4: [n_ops][evt_off][ops...].
//
// Restates the per-read loop of the reference, kindel/kindel.py:40-81 (M/=/X :49-54, I :55-58,
// D :59-62, left clip :64-73, right clip :74-81; N/H/P fall through), including its edge
// behaviour (SURVEY.md Appendix A): Python negative-index wrap for POS==0 and clip_starts[r_pos-1],
// any non-first S treated as a right clip that advances both cursors while r_pos < ref_len, q_pos
// stalling once the clip overhangs the contig end.
//
// The warp reads each CIGAR op once (uniform load), then its 32 lanes stride over the op's bases
// so the count updates of one op go to 32 consecutive slots of a column (coalesced REDs).  Reads
// handled here are the minority that carry indels / clips; plain nM reads take K1s/K1f
// (pileup_simple.cu).  Any data error only raises err_flag; kdl_diagnose finds the exact one.
#include "tile_common.cuh"  // (K1w reads K0's tile index)

namespace kdl {

__global__ void __launch_bounds__(256)
pileup_general_kernel(kdl_batch b, const uint32_t* __restrict__ list, long long n_list, int32_t* __restrict__ counts,
                      long long n_slots, int32_t* __restrict__ ins_events, int32_t* __restrict__ err_flag,
                      uint32_t* __restrict__ dirty_map = nullptr) {
    const int lane = threadIdx.x & 31;
    const bool marks = dirty_map != nullptr && lane == 0;  // (the ops are warp-uniform: lane 0 marks their sectors)
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    bool bad = false;

    for (long long j = warp0; j < n_list; j += n_warps) {
        const long long r = list ? (long long)list[j] : j;
        const uint32_t lraw = (uint32_t)b.l_seq[r];
        if (!(lraw & KDL_COMPLEX)) continue;  // simple read: K1 / K1s count it
        const int c = find_contig(b.contig_read_off, b.n_contigs, r);
        const long long L = b.contig_len[c];
        const long long base = b.contig_slot[c];
        const long long lseq = complex_len(lraw);
        const uint32_t* __restrict__ seq = b.seq4 + (size_t)b.seq_off[r];
        const uint32_t* __restrict__ blk = seq + ((lseq + 7) >> 3);  // [n_ops][evt_off][ops...]
        const uint32_t c0 = 0, c1 = blk[0];
        const uint32_t* __restrict__ cig = blk + 2;
        long long r_pos = b.ref_start[r];
        long long q_pos = 0;
        uint32_t evt = blk[1];

        for (uint32_t i = c0; i < c1; ++i) {
            const uint32_t cg = cig[i];
            const long long len = cg >> 4;
            const int op = cg & 0xF;
            if (op == 0 || op == 7 || op == 8) {  // M = X
                for (long long k = lane; k < len; k += 32) {
                    const long long q = q_pos + k;
                    const long long idx = pyindex(r_pos + k, L);
                    if (q >= lseq || idx < 0) { bad = true; continue; }
                    const int col = nib2col(nibble_at(seq, q));
                    if (col < 0) { bad = true; continue; }
                    atomicAdd(counts + (long long)(KDL_W_A + col) * n_slots + base + idx, 1);
                }
                r_pos += len;
                q_pos += len;
            } else if (op == 1) {  // I
                if (marks) mark_dirty_py(dirty_map, KDL_INS, 1, base, r_pos, r_pos + 1, L + 1);
                if (lane == 0) {
                    const long long idx = pyindex(r_pos, L + 1);
                    if (idx < 0) {
                        bad = true;
                    } else {
                        atomicAdd(counts + (long long)KDL_INS * n_slots + base + idx, 1);
                        if (ins_events) {
                            int4 e = make_int4((int)(base + idx), (int)r, (int)q_pos, (int)len);
                            reinterpret_cast<int4*>(ins_events)[evt] = e;
                        }
                    }
                }
                evt += 1;
                q_pos += len;
            } else if (op == 2) {  // D
                if (marks) mark_dirty_py(dirty_map, KDL_DEL, 1, base, r_pos, r_pos + len, L + 1);
                for (long long k = lane; k < len; k += 32) {
                    const long long idx = pyindex(r_pos + k, L + 1);
                    if (idx < 0) { bad = true; continue; }
                    atomicAdd(counts + (long long)KDL_DEL * n_slots + base + idx, 1);
                }
                r_pos += len;
            } else if (op == 4) {  // S
                if (i == c0) {     // left clip: only when it is op #0 (kindel.py:64)
                    if (marks) {
                        mark_dirty_py(dirty_map, KDL_CLIP_ENDS, 1, base, r_pos, r_pos + 1, L + 1);
                        mark_dirty(dirty_map, KDL_CEW_A, 5, base + (r_pos - len > 0 ? r_pos - len : 0),
                                   base + (r_pos < L ? r_pos : L));  // (bases left of the contig are skipped, not wrapped)
                    }
                    if (lane == 0) {
                        const long long idx = pyindex(r_pos, L + 1);
                        if (idx < 0) bad = true;
                        else atomicAdd(counts + (long long)KDL_CLIP_ENDS * n_slots + base + idx, 1);
                    }
                    for (long long g = lane; g < len; g += 32) {
                        if (g >= lseq) { bad = true; continue; }
                        const long long rel = r_pos - len + g;
                        if (rel < 0) continue;
                        if (rel >= L) { bad = true; continue; }
                        const int col = nib2col(nibble_at(seq, g));
                        if (col < 0) { bad = true; continue; }
                        atomicAdd(counts + (long long)(KDL_CEW_A + col) * n_slots + base + rel, 1);
                    }
                    q_pos += len;
                } else {  // right clip
                    if (lane == 0) {
                        const long long idx = pyindex(r_pos - 1, L + 1);
                        if (idx < 0) bad = true;
                        else atomicAdd(counts + (long long)KDL_CLIP_STARTS * n_slots + base + idx, 1);
                    }
                    // iterations that advance: while r_pos < L (kindel.py:78-81)
                    long long n_adv = L - r_pos;
                    n_adv = n_adv < 0 ? 0 : (n_adv > len ? len : n_adv);
                    if (marks) {
                        mark_dirty_py(dirty_map, KDL_CLIP_STARTS, 1, base, r_pos - 1, r_pos, L + 1);
                        mark_dirty_py(dirty_map, KDL_CSW_A, 5, base, r_pos, r_pos + n_adv, L);
                    }
                    for (long long k = lane; k < n_adv; k += 32) {
                        const long long q = q_pos + k;
                        const long long idx = pyindex(r_pos + k, L);
                        if (q >= lseq || idx < 0) { bad = true; continue; }
                        const int col = nib2col(nibble_at(seq, q));
                        if (col < 0) { bad = true; continue; }
                        atomicAdd(counts + (long long)(KDL_CSW_A + col) * n_slots + base + idx, 1);
                    }
                    // the stalled iterations still evaluate record.seq[q_pos] (kindel.py:77)
                    if (n_adv < len && q_pos + n_adv >= lseq) bad = true;
                    r_pos += n_adv;
                    q_pos += n_adv;
                }
            }
            // N, H, P, anything else: no-op (kindel.py:49-63 has no branch for them)
        }
    }
    if (bad) atomicOr(err_flag, 1);
}

// ---- K1e: the sparse updates of the TILE-ELIGIBLE complex reads when K1 counted their bases ---------------------
// With its piece instantiation the tile kernel counts these reads' M/=/X bases (pileup_tile.cu); what is left of the
// reference's loop -- insertions (kindel.py:55-58), deletions (:59-62), clip counts and clip bases (:64-81) -- is a
// handful of increments per read, done here once per read with REDs, one thread per read (these batches have many
// complex reads: a million threads hide the dependent loads).  By the flatten contract such a read cannot wrap an
// index or raise: no checks.  Insertion events go to their deterministic rows.
// dirty_map (may be NULL): the sectors of columns 5..18 these updates touch are marked there, once per op range.
__global__ void __launch_bounds__(256)
pileup_events_kernel(kdl_batch b, int32_t* __restrict__ counts, long long n_slots, int32_t* __restrict__ ins_events,
                     uint32_t* __restrict__ dirty_map) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= b.n_complex) return;
    const long long r = (long long)b.complex_idx[j];
    const uint32_t lraw = (uint32_t)b.l_seq[r];
    if ((lraw & (KDL_COMPLEX | KDL_HARD)) != KDL_COMPLEX) return;  // hard reads: K1g walks all of their ops
    const int c = find_contig(b.contig_read_off, b.n_contigs, r);
    const long long slot0 = b.contig_slot[c];
    int32_t* __restrict__ tab = counts + slot0;  // column 0 at this contig's first slot
    const uint32_t* __restrict__ seq = b.seq4 + (size_t)b.seq_off[r];
    const uint32_t* __restrict__ blk = seq + (((lraw & KDL_LEN_MASK) + 7) >> 3);  // [n_ops][evt_off][ops...]
    const int n_ops = (int)blk[0];
    uint32_t evt = blk[1];
    const uint32_t* __restrict__ ops = blk + 2;
    long long r_pos = b.ref_start[r];
    int q_pos = 0;
    for (int o = 0; o < n_ops; ++o) {
        const uint32_t cg = ops[o];
        const int len = (int)(cg >> 4);
        const int op = (int)(cg & 0xF);
        if (op == 0 || op == 7 || op == 8) {  // M = X: the tile kernel's
            r_pos += len;
            q_pos += len;
        } else if (op == 1) {  // I
            if (dirty_map) mark_dirty(dirty_map, KDL_INS, 1, slot0 + r_pos, slot0 + r_pos + 1);
            atomicAdd(tab + (long long)KDL_INS * n_slots + r_pos, 1);
            if (ins_events)
                reinterpret_cast<int4*>(ins_events)[evt] = make_int4((int)(slot0 + r_pos), (int)r, q_pos, len);
            evt += 1;
            q_pos += len;
        } else if (op == 2) {  // D
            if (dirty_map) mark_dirty(dirty_map, KDL_DEL, 1, slot0 + r_pos, slot0 + r_pos + len);
            for (int d = 0; d < len; ++d) atomicAdd(tab + (long long)KDL_DEL * n_slots + r_pos + d, 1);
            r_pos += len;
        } else if (op == 4) {  // S
            if (o == 0) {      // left clip: its bases end where the read starts
                if (dirty_map) {
                    mark_dirty(dirty_map, KDL_CLIP_ENDS, 1, slot0 + r_pos, slot0 + r_pos + 1);
                    mark_dirty(dirty_map, KDL_CEW_A, 5, slot0 + (r_pos - len > 0 ? r_pos - len : 0), slot0 + r_pos);
                }
                atomicAdd(tab + (long long)KDL_CLIP_ENDS * n_slots + r_pos, 1);
                for (int g = 0; g < len; ++g) {
                    const long long rel = r_pos - len + g;
                    if (rel >= 0) atomicAdd(tab + (long long)(KDL_CEW_A + nib2col(nibble_at(seq, g))) * n_slots + rel, 1);
                }
                q_pos += len;
            } else {           // right clip (never reaches the contig end for these reads)
                if (dirty_map) {
                    mark_dirty(dirty_map, KDL_CLIP_STARTS, 1, slot0 + r_pos - 1, slot0 + r_pos);
                    mark_dirty(dirty_map, KDL_CSW_A, 5, slot0 + r_pos, slot0 + r_pos + len);
                }
                atomicAdd(tab + (long long)KDL_CLIP_STARTS * n_slots + r_pos - 1, 1);
                for (int d = 0; d < len; ++d)
                    atomicAdd(tab + (long long)(KDL_CSW_A + nib2col(nibble_at(seq, q_pos + d))) * n_slots + r_pos + d, 1);
                r_pos += len;
                q_pos += len;
            }
        }
        // N, H, P: no-op
    }
}

// ---- K1w: the TILE-ELIGIBLE complex reads when they are rare, one CTA per window of slots --------------------------
// When tile-eligible complex reads are rare (a few per cent of a short-read BAM) the tile kernel runs its lean
// instantiation and treats them as inert: their ~130 bases each cost less here than the piece machinery costs every
// item.  K1w counts the reference's whole loop for them: M/=/X bases (kindel.py:49-54), insertions (:55-58),
// deletions (:59-62), clip counts and clip bases (:64-81).  By the flatten contract such a read cannot wrap an index
// or raise: no checks.
//
// The slot range is cut into windows of CW_SLOTS slots; a window is owned by one CTA (or, for a small reference piled
// deep, by `split` CTAs that share its reads).  The reads that can touch a window are one range of complex_idx: the
// reads are sorted by global start slot, K0's index gives the first and last read index of the window's tiles, and
// complex_idx is ascending.  The CTA walks each of them once, a group of lanes per read, and counts every update that
// falls inside the window: columns 0..6 into shared memory, the clip columns 7..18 (a few updates per read) with
// REDs.  (Those in shared memory too would take 76 instead of 28 KB per window and leave fewer CTAs per SM to hide
// the dependent loads of the walk.)  The flush then adds the shared counts to the table, only the 32-byte sectors
// they changed: plain 128-bit read-modify-writes when the CTA owns the window (K1 is done in stream order, K1g comes
// after), REDs when `split` CTAs share it.  Insertion events go to their deterministic rows, written by the CTA whose window holds
// the insertion's slot.
//
// dirty_map (may be NULL): the flush marks the sectors of columns 5 and 6 it changed; the clip updates mark their op
// ranges, clipped to the window.
constexpr int CW_SLOTS = 1024;   // slots per window
constexpr int CW_THREADS = 256;
constexpr int CW_SMEM_COLS = 7;  // columns 0..6 are counted in shared memory
static_assert(CW_SLOTS % KDL_TILE == 0 && CW_SLOTS % 256 == 0, "windows of whole tiles, whole map records per warp");

// first index of the ascending a[0, n) whose element is >= key, for two keys at once; whole warp, 32-ary (each
// round the 32 lanes probe the last element of 32 buckets of the remaining range in one memory round trip)
__device__ __forceinline__ void lower_bound2_u32(const uint32_t* __restrict__ a, long long n, uint32_t key1,
                                                 uint32_t key2, int lane, long long& r1, long long& r2) {
    long long lo[2] = {0, 0}, hi[2] = {n, n};  // the answer lies in [lo, hi]; a[hi] >= key or hi == n
    const uint32_t key[2] = {key1, key2};
    while (lo[0] < hi[0] || lo[1] < hi[1]) {  // warp-uniform
        long long step[2];
        bool ge[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            step[k] = (hi[k] - lo[k] + 31) >> 5;
            const long long i = lo[k] + (long long)(lane + 1) * step[k] - 1;
            ge[k] = lo[k] >= hi[k] || i >= hi[k] || a[i] >= key[k];
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const unsigned m = __ballot_sync(0xffffffffu, ge[k]);
            if (lo[k] >= hi[k]) continue;
            if (m == 0u) { lo[k] = hi[k]; continue; }  // even the last element of the range is < key
            const int b = __ffs(m) - 1;                 // first bucket whose last element is >= key
            const long long nl = lo[k] + (long long)b * step[k], nh = nl + step[k] - 1;
            hi[k] = nh < hi[k] ? nh : hi[k];
            lo[k] = step[k] == 1 ? hi[k] : nl;
        }
    }
    r1 = lo[0];
    r2 = lo[1];
}

__global__ void __launch_bounds__(CW_THREADS)
pileup_window_kernel(kdl_batch b, int32_t* __restrict__ counts, long long n_slots, long long slot_lo, long long slot_hi,
                     int split, int32_t* __restrict__ ins_events, uint32_t* __restrict__ dirty_map) {
    KDL_DYNAMIC_SMEM(smem_raw);
    int* acc = reinterpret_cast<int*>(smem_raw);  // [CW_SMEM_COLS][CW_SLOTS]: the window's counts
    __shared__ long long range[2];
    const int tid = threadIdx.x, lane = tid & 31;
    constexpr int n_sec = CW_SMEM_COLS * (CW_SLOTS / 8);  // 32-byte sectors of the shared counts
    const long long g0 = slot_lo + (long long)(blockIdx.x / split) * CW_SLOTS;
    const long long g1 = g0 + CW_SLOTS < slot_hi ? g0 + CW_SLOTS : slot_hi;
    for (int k = tid; k < 2 * n_sec; k += CW_THREADS) reinterpret_cast<int4*>(acc)[k] = make_int4(0, 0, 0, 0);
    if (tid < 32) {
        const uint32_t lo = b.tile_index[F_IDX * (g0 / KDL_TILE)], hi = b.tile_index[F_IDX * ((g1 - 1) / KDL_TILE) + 1];
        long long ja, je;
        lower_bound2_u32(b.complex_idx, b.n_complex, lo, hi, lane, ja, je);
        if (lane == 0) {
            const int part = (int)(blockIdx.x % split);
            range[0] = ja + (je - ja) * part / split;
            range[1] = ja + (je - ja) * (part + 1) / split;
        }
    }
    __syncthreads();
    const long long j0 = range[0], j1 = range[1];
    int lg = 0;  // 2^lg lanes per read: as many as keep the CTA busy, at most 32
    while (lg < 5 && ((j1 - j0) << (lg + 1)) <= CW_THREADS) ++lg;
    const int gl = tid & ((1 << lg) - 1), step = 1 << lg;
    for (long long j = j0 + (tid >> lg); j < j1; j += CW_THREADS >> lg) {
        const long long r = (long long)b.complex_idx[j];
        const uint32_t lraw = (uint32_t)b.l_seq[r];
        if ((lraw & (KDL_COMPLEX | KDL_HARD)) != KDL_COMPLEX) continue;  // hard reads: K1g walks all of their ops
        const int c = find_contig(b.contig_read_off, b.n_contigs, r);
        const long long slot0 = b.contig_slot[c];
        const long long wl = g0 - slot0, wh = g1 - slot0;  // the window in the contig's positions
        int32_t* __restrict__ tab = counts + slot0;  // column 0 at this contig's first slot
        const uint32_t* __restrict__ seq = b.seq4 + (size_t)b.seq_off[r];
        const uint32_t* __restrict__ blk = seq + (((lraw & KDL_LEN_MASK) + 7) >> 3);  // [n_ops][evt_off][ops...]
        const int n_ops = (int)blk[0];
        uint32_t evt = blk[1];
        const uint32_t* __restrict__ ops = blk + 2;
        long long r_pos = b.ref_start[r];
        int q_pos = 0;
        const bool marks = dirty_map != nullptr && gl == 0;
        for (int o = 0; o < n_ops; ++o) {
            const uint32_t cg = ops[o];
            const int len = (int)(cg >> 4);
            const int op = (int)(cg & 0xF);
            // the op's slots [r_pos, r_pos + len) inside the window (right clips and D; M/=/X too)
            const long long s0 = r_pos > wl ? r_pos : wl, s1 = r_pos + len < wh ? r_pos + len : wh;
            if (op == 0 || op == 7 || op == 8) {  // M = X
#pragma unroll 4
                for (long long s = s0 + gl; s < s1; s += step)
                    atomicAdd(acc + (KDL_W_A + nib2col(nibble_at(seq, q_pos + (s - r_pos)))) * CW_SLOTS + (s - wl), 1);
                r_pos += len;
                q_pos += len;
            } else if (op == 1) {  // I
                if (gl == 0 && r_pos >= wl && r_pos < wh) {
                    atomicAdd(acc + KDL_INS * CW_SLOTS + (r_pos - wl), 1);
                    if (ins_events)
                        reinterpret_cast<int4*>(ins_events)[evt] = make_int4((int)(slot0 + r_pos), (int)r, q_pos, len);
                }
                evt += 1;
                q_pos += len;
            } else if (op == 2) {  // D
                for (long long s = s0 + gl; s < s1; s += step) atomicAdd(acc + KDL_DEL * CW_SLOTS + (s - wl), 1);
                r_pos += len;
            } else if (op == 4) {  // S
                if (o == 0) {  // left clip: its bases end where the read starts (left of the contig: skipped)
                    const long long e0 = r_pos - len, c1 = r_pos < wh ? r_pos : wh;
                    long long c0 = e0 > 0 ? e0 : 0;
                    if (c0 < wl) c0 = wl;
                    if (gl == 0 && r_pos >= wl && r_pos < wh) {
                        if (marks) mark_dirty(dirty_map, KDL_CLIP_ENDS, 1, slot0 + r_pos, slot0 + r_pos + 1);
                        atomicAdd(tab + (long long)KDL_CLIP_ENDS * n_slots + r_pos, 1);
                    }
                    if (marks) mark_dirty(dirty_map, KDL_CEW_A, 5, slot0 + c0, slot0 + c1);
                    for (long long s = c0 + gl; s < c1; s += step)
                        atomicAdd(tab + (long long)(KDL_CEW_A + nib2col(nibble_at(seq, s - e0))) * n_slots + s, 1);
                    q_pos += len;
                } else {           // right clip (never reaches the contig end for these reads)
                    if (gl == 0 && r_pos - 1 >= wl && r_pos - 1 < wh) {
                        if (marks) mark_dirty(dirty_map, KDL_CLIP_STARTS, 1, slot0 + r_pos - 1, slot0 + r_pos);
                        atomicAdd(tab + (long long)KDL_CLIP_STARTS * n_slots + r_pos - 1, 1);
                    }
                    if (marks) mark_dirty(dirty_map, KDL_CSW_A, 5, slot0 + s0, slot0 + s1);
                    for (long long s = s0 + gl; s < s1; s += step)
                        atomicAdd(tab + (long long)(KDL_CSW_A + nib2col(nibble_at(seq, q_pos + (s - r_pos)))) * n_slots + s,
                                  1);
                    r_pos += len;
                    q_pos += len;
                }
            }
            // N, H, P: no-op
        }
    }
    __syncthreads();
    // flush: thread tid takes sectors tid, tid + CW_THREADS, ...; a warp's 32 sectors are 256 slots of one column
    for (int sec = tid; sec < n_sec; sec += CW_THREADS) {  // (n_sec is a multiple of 32: whole warps)
        const int col = sec / (CW_SLOTS / 8), off = 8 * (sec % (CW_SLOTS / 8));
        const int4* sp = reinterpret_cast<const int4*>(acc) + 2 * sec;
        const int4 d0 = sp[0], d1 = sp[1];
        const bool dirty = (d0.x | d0.y | d0.z | d0.w | d1.x | d1.y | d1.z | d1.w) != 0;
        int32_t* dst = counts + (long long)col * n_slots + g0 + off;
        if (dirty && split == 1) {
            int4* p = reinterpret_cast<int4*>(dst);
            int4 v0 = p[0], v1 = p[1];
            v0.x += d0.x; v0.y += d0.y; v0.z += d0.z; v0.w += d0.w;
            v1.x += d1.x; v1.y += d1.y; v1.z += d1.z; v1.w += d1.w;
            p[0] = v0;
            p[1] = v1;
        } else if (dirty) {
            const int d[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (d[k]) atomicAdd(dst + k, d[k]);
        }
        if (dirty_map && col >= KDL_DEL) {  // byte col - 5 of the 4 map records the warp's sectors make up
            const unsigned m = __ballot_sync(0xffffffffu, dirty);
            const unsigned bits = lane < 4 ? (m >> (8 * lane)) & 0xFFu : 0u;
            if (bits)
                atomicOr(dirty_map + 4 * ((g0 + off - 8 * lane) / 64 + lane) + (col - KDL_DEL) / 4,
                         bits << (8 * ((col - KDL_DEL) % 4)));
        }
    }
}

// ---- exact first error, reference iteration order (error path only) -------------------------
// One thread per read walks sequentially and stops at the first exception the reference would
// raise; the minimum over reads of (read << 24 | kind << 20 | nibble << 16 | op) is the error of
// the first offending record.
__device__ unsigned long long diagnose_read(const kdl_batch& b, long long j) {
    const long long r = (long long)b.hard_idx[j];  // only KDL_HARD reads can raise (flatten contract)
    const int c = find_contig(b.contig_read_off, b.n_contigs, r);
    const long long L = b.contig_len[c];
    const long long lseq = complex_len((uint32_t)b.l_seq[r]);
    const uint32_t* __restrict__ seq = b.seq4 + (size_t)b.seq_off[r];
    const uint32_t* __restrict__ blk = seq + ((lseq + 7) >> 3);
    const uint32_t c0 = 0, c1 = blk[0];
    const uint32_t* __restrict__ cig = blk + 2;
    long long r_pos = b.ref_start[r], q_pos = 0;
#define KDL_FAIL(kind, nib)                                                                     \
    return ((unsigned long long)r << 24) | ((unsigned long long)(kind) << 20) |                 \
           ((unsigned long long)(nib) << 16) | (unsigned long long)((i - c0) > 0xFFFF ? 0xFFFF : (i - c0))
    for (uint32_t i = c0; i < c1; ++i) {
        const uint32_t cg = cig[i];
        const long long len = cg >> 4;
        const int op = cg & 0xF;
        if (op == 0 || op == 7 || op == 8) {
            for (long long k = 0; k < len; ++k) {
                if (q_pos >= lseq) KDL_FAIL(0, 0);
                if (pyindex(r_pos, L) < 0) KDL_FAIL(0, 0);
                const int nib = nibble_at(seq, q_pos);
                if (nib2col(nib) < 0) KDL_FAIL(1, nib);
                ++r_pos; ++q_pos;
            }
        } else if (op == 1) {
            if (pyindex(r_pos, L + 1) < 0) KDL_FAIL(0, 0);
            q_pos += len;
        } else if (op == 2) {
            for (long long k = 0; k < len; ++k)
                if (pyindex(r_pos + k, L + 1) < 0) KDL_FAIL(0, 0);
            r_pos += len;
        } else if (op == 4) {
            if (i == c0) {
                if (pyindex(r_pos, L + 1) < 0) KDL_FAIL(0, 0);
                for (long long g = 0; g < len; ++g) {
                    if (g >= lseq) KDL_FAIL(0, 0);
                    const long long rel = r_pos - len + g;
                    if (rel >= 0) {
                        if (rel >= L) KDL_FAIL(0, 0);
                        const int nib = nibble_at(seq, g);
                        if (nib2col(nib) < 0) KDL_FAIL(1, nib);
                    }
                }
                q_pos += len;
            } else {
                if (pyindex(r_pos - 1, L + 1) < 0) KDL_FAIL(0, 0);
                for (long long k = 0; k < len; ++k) {
                    if (q_pos >= lseq) KDL_FAIL(0, 0);
                    if (r_pos < L) {
                        if (pyindex(r_pos, L) < 0) KDL_FAIL(0, 0);
                        const int nib = nibble_at(seq, q_pos);
                        if (nib2col(nib) < 0) KDL_FAIL(1, nib);
                        ++r_pos; ++q_pos;
                    }
                }
            }
        }
    }
#undef KDL_FAIL
    return ~0ull;
}

__global__ void diagnose_init_kernel(kdl_diag* d) {
    d->status = 0; d->reserved = 0; d->read = -1; d->nibble = 0; d->op_index = 0;
    *reinterpret_cast<unsigned long long*>(&d->read) = ~0ull;
}

__global__ void __launch_bounds__(256) diagnose_kernel(kdl_batch b, kdl_diag* d) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= b.n_hard) return;
    const unsigned long long key = diagnose_read(b, j);
    if (key != ~0ull) atomicMin(reinterpret_cast<unsigned long long*>(&d->read), key);
}

__global__ void diagnose_final_kernel(kdl_diag* d) {
    const unsigned long long key = *reinterpret_cast<unsigned long long*>(&d->read);
    if (key == ~0ull) { d->status = KDL_OK; d->read = -1; return; }
    d->status = ((key >> 20) & 0xF) ? KDL_ERR_KEY : KDL_ERR_INDEX;
    d->nibble = (int)((key >> 16) & 0xF);
    d->op_index = (int)(key & 0xFFFF);
    d->read = (long long)(key >> 24);
}

}  // namespace kdl
