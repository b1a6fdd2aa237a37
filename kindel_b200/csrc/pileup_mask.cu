// pileup_mask.cu -- K1q: takes back what masked bases added to the base-count columns (extension).
//
// A base below min_base_quality is masked at decode: its nibble is N (15) in seq4, so every pileup kernel (K1's
// bit-sliced count: A+C+G+T raw = coverage + 3N; K1w, K1e, K1g, K1s: nib2col(15) = 4) counts it as an N wherever the
// reference's walk (kindel/kindel.py:40-81) would count that base, and the insertion strings read it as N.  The
// masking rule is "read as N, then not counted": K1q runs after the pileup kernels in stream order and subtracts 1
// at the (column, slot) each listed base went to:
//   M/=/X           column 4 (weights N)              slot r_pos + (q - q_pos)
//   left clip       column 18 (clip_end_weights N)    slot r_pos - len + q, when >= 0
//   right clip      column 13 (clip_start_weights N)  slot r_pos + (q - q_pos), only the iterations that advance
//   I, D, N, H, P   nothing
// A simple read is one M op: slot = contig_slot + ref_start + q.  A complex read's CIGAR rides behind its bases in
// seq4; the walk is K1g's (pileup_general.cu), with its Python index wrap and right-clip stall, and skips exactly the
// updates K1g skips when a hard read raises (the host raises then and the table is not used).  Tile-eligible reads
// take the same walk: by the flatten contract it never wraps or stalls for them.
//
// One thread per read with masked bases, its query offsets ascending.  Reads are coordinate-sorted, so the masked
// bases of a CTA's 256 consecutive reads fall on a few hundred slots of column 4: they are summed in a shared-memory
// window first and flushed with one RED per touched slot; whatever falls outside the window (clips, unsorted input,
// a CTA spanning two contigs) goes straight to global memory.
#include "kdl_common.cuh"

namespace kdl {

constexpr int kQThreads = 256;
constexpr int kQWindow = 2048;  // column-4 slots summed in shared memory per CTA

__global__ void __launch_bounds__(kQThreads)
unmask_kernel(kdl_batch b, kdl_qmask m, int32_t* __restrict__ counts, long long n_slots) {
    __shared__ int win[kQWindow];
    for (int i = threadIdx.x; i < kQWindow; i += blockDim.x) win[i] = 0;
    const long long j0 = (long long)blockIdx.x * blockDim.x;
    const long long r0 = m.read_idx[j0];
    const long long win_lo = b.contig_slot[find_contig(b.contig_read_off, b.n_contigs, r0)] + b.ref_start[r0];
    int32_t* __restrict__ col_n = counts + (long long)KDL_W_N * n_slots;
    __syncthreads();

    const long long j = j0 + threadIdx.x;
    if (j < m.n_reads) {
        const long long r = m.read_idx[j];
        const uint32_t* __restrict__ qp = m.qpos + m.off[j];
        const int n_q = (int)(m.off[j + 1] - m.off[j]);
        const uint32_t lraw = (uint32_t)b.l_seq[r];
        const int c = find_contig(b.contig_read_off, b.n_contigs, r);
        const long long base = b.contig_slot[c];
        auto weight_n = [&](long long slot) {  // column 4, through the window when it is there
            const long long w = slot - win_lo;
            if (w >= 0 && w < kQWindow) atomicAdd(&win[w], -1);
            else atomicAdd(col_n + slot, -1);
        };
        if (!(lraw & KDL_COMPLEX)) {
            const long long s0 = base + b.ref_start[r];
            for (int k = 0; k < n_q; ++k) weight_n(s0 + qp[k]);
        } else {
            const long long L = b.contig_len[c];
            const long long lseq = complex_len(lraw);
            const uint32_t* __restrict__ blk = b.seq4 + (size_t)b.seq_off[r] + ((lseq + 7) >> 3);
            const uint32_t n_ops = blk[0];
            const uint32_t* __restrict__ cig = blk + 2;
            long long r_pos = b.ref_start[r], q_pos = 0;
            int k = 0;
            for (uint32_t i = 0; i < n_ops && k < n_q; ++i) {
                const uint32_t cg = cig[i];
                const long long len = cg >> 4;
                const int op = cg & 0xF;
                if (op == 0 || op == 7 || op == 8) {  // M = X
                    for (; k < n_q && qp[k] < q_pos + len; ++k) {
                        const long long idx = pyindex(r_pos + (qp[k] - q_pos), L);
                        if (idx >= 0) weight_n(base + idx);
                    }
                    r_pos += len;
                    q_pos += len;
                } else if (op == 1) {  // I
                    q_pos += len;
                } else if (op == 2) {  // D
                    r_pos += len;
                } else if (op == 4) {  // S
                    if (i == 0) {      // left clip (kindel.py:64-73)
                        for (; k < n_q && qp[k] < len; ++k) {
                            const long long rel = r_pos - len + qp[k];
                            if (rel >= 0 && rel < L) atomicAdd(counts + (long long)(KDL_CEW_A + 4) * n_slots + base + rel, -1);
                        }
                        q_pos += len;
                    } else {           // right clip: only the iterations that advance (kindel.py:78-81)
                        long long n_adv = L - r_pos;
                        n_adv = n_adv < 0 ? 0 : (n_adv > len ? len : n_adv);
                        for (; k < n_q && qp[k] < q_pos + n_adv; ++k) {
                            const long long idx = pyindex(r_pos + (qp[k] - q_pos), L);
                            if (idx >= 0) atomicAdd(counts + (long long)(KDL_CSW_A + 4) * n_slots + base + idx, -1);
                        }
                        r_pos += n_adv;
                        q_pos += n_adv;
                    }
                }
                // N, H, P: no-op.  Offsets the walk has passed without counting them (I, stalled clips) are done.
                while (k < n_q && qp[k] < q_pos) ++k;
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kQWindow; i += blockDim.x)
        if (win[i]) atomicAdd(col_n + win_lo + i, win[i]);
}

}  // namespace kdl
