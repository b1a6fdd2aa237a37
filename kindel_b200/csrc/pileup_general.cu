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
#include "kdl_common.cuh"

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

// ---- K1e: the sparse updates of the TILE-ELIGIBLE complex reads ------------------------------------------
// The tile kernel counts these reads' M/=/X bases (pileup_tile.cu); what is left of the reference's loop --
// insertions (kindel.py:55-58), deletions (:59-62), clip counts and clip bases (:64-81) -- is a handful of
// increments per read, done here once per read with REDs.  By the flatten contract such a read cannot wrap an index
// or raise: no checks.  Insertion events go to their deterministic rows.
//
// dirty_map (may be NULL): the sectors of columns 5..18 these updates touch are marked there, once per op range.
// with_m: also count the reads' M/=/X bases here, with REDs into the weight columns -- what kdl_pileup_range asks
// for when tile-eligible complex reads are RARE (a few per cent of a short-read BAM): the tile kernel then runs its
// lean instantiation and treats them as inert, and their ~130 bases each cost less as atomics than the piece
// machinery costs every item.  (Stream order puts these REDs behind the tile kernel's plain stores.)
// kLanes threads per read, striding over an op's bases.  1: 32 reads per warp instruction -- the cheapest way through
// the op loops when the updates are a few scattered REDs per read (a million threads hide the dependent loads).
// 8: what with_m (130 bases per read, few reads) wants -- 8 consecutive slots per RED, four reads' load chains in
// flight per warp.
template <int kLanes>
__global__ void __launch_bounds__(256)
pileup_events_kernel(kdl_batch b, int32_t* __restrict__ counts, long long n_slots, int32_t* __restrict__ ins_events,
                     int with_m, uint32_t* __restrict__ dirty_map = nullptr) {
    const int lane = (int)(threadIdx.x % kLanes);
    constexpr int kStep = kLanes;
    const long long gtid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long j = gtid / kLanes;
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
    const bool marks = dirty_map != nullptr && lane == 0;
    for (int o = 0; o < n_ops; ++o) {
        const uint32_t cg = ops[o];
        const int len = (int)(cg >> 4);
        const int op = (int)(cg & 0xF);
        if (op == 0 || op == 7 || op == 8) {  // M = X: the tile kernel's, unless with_m
            if (with_m)
                for (int d = lane; d < len; d += kStep)
                    atomicAdd(tab + (long long)(KDL_W_A + nib2col(nibble_at(seq, q_pos + d))) * n_slots + r_pos + d, 1);
            r_pos += len;
            q_pos += len;
        } else if (op == 1) {  // I
            if (lane == 0) {
                if (marks) mark_dirty(dirty_map, KDL_INS, 1, slot0 + r_pos, slot0 + r_pos + 1);
                atomicAdd(tab + (long long)KDL_INS * n_slots + r_pos, 1);
                if (ins_events)
                    reinterpret_cast<int4*>(ins_events)[evt] = make_int4((int)(slot0 + r_pos), (int)r, q_pos, len);
            }
            evt += 1;
            q_pos += len;
        } else if (op == 2) {  // D
            if (marks) mark_dirty(dirty_map, KDL_DEL, 1, slot0 + r_pos, slot0 + r_pos + len);
            for (int d = lane; d < len; d += kStep) atomicAdd(tab + (long long)KDL_DEL * n_slots + r_pos + d, 1);
            r_pos += len;
        } else if (op == 4) {  // S
            if (o == 0) {      // left clip: its bases end where the read starts
                if (marks) {
                    mark_dirty(dirty_map, KDL_CLIP_ENDS, 1, slot0 + r_pos, slot0 + r_pos + 1);
                    mark_dirty(dirty_map, KDL_CEW_A, 5, slot0 + (r_pos - len > 0 ? r_pos - len : 0), slot0 + r_pos);
                }
                if (lane == 0) atomicAdd(tab + (long long)KDL_CLIP_ENDS * n_slots + r_pos, 1);
                for (int g = lane; g < len; g += kStep) {
                    const long long rel = r_pos - len + g;
                    if (rel >= 0) atomicAdd(tab + (long long)(KDL_CEW_A + nib2col(nibble_at(seq, g))) * n_slots + rel, 1);
                }
                q_pos += len;
            } else {           // right clip (never reaches the contig end for these reads)
                if (marks) {
                    mark_dirty(dirty_map, KDL_CLIP_STARTS, 1, slot0 + r_pos - 1, slot0 + r_pos);
                    mark_dirty(dirty_map, KDL_CSW_A, 5, slot0 + r_pos, slot0 + r_pos + len);
                }
                if (lane == 0) atomicAdd(tab + (long long)KDL_CLIP_STARTS * n_slots + r_pos - 1, 1);
                for (int d = lane; d < len; d += kStep)
                    atomicAdd(tab + (long long)(KDL_CSW_A + nib2col(nibble_at(seq, q_pos + d))) * n_slots + r_pos + d, 1);
                r_pos += len;
                q_pos += len;
            }
        }
        // N, H, P: no-op
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
