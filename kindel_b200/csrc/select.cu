// select.cu -- K8 `select_*_kernel` (extension: `variants --vcf --strand`): the sub-batch of the reads a keep byte
// selects, built on the device from a resident batch, so that a second pileup can run over part of the reads without
// a host round trip for the read data.
//
// The result equals bamio.select_reads(batch, np.flatnonzero(keep)) field for field (include/kindel_b200.h, K8).
// Classification is per read, so every kept read keeps its l_seq word; what changes is where things are:
//   per read r: kept = keep[r] != 0, and when kept its share of each output --
//     1 read, its words in seq4 (bases, plus [n_ops][evt_off][ops] for a complex read), 1 complex / 1 hard read, its
//     I-op count (insertion events), 1 masked read and its masked bases
//   each output offset is the exclusive prefix of those shares over the reads before r; contig_read_off[c] is the
//   read prefix at the parent's contig_read_off[c]; evt_off of a kept complex read is the event prefix.
// The scalars: max_simple_len = max op length of the kept simple reads, reach_right = max of that and r_span + 1 of the
// kept tile-eligible reads, reach_left = max lead + 1 of those (the CIGAR walk of bamio.finalize); reads_sorted holds
// when no kept read starts (contig_slot + ref_start) before the largest start of the kept reads in front of it.
//
// Three launches: per-CTA shares, maxima and order facts (one thread per read), one CTA that turns them into
// exclusive prefixes and writes the totals record the host reads back to size the outputs, and the scatter, which
// recomputes the shares, adds its CTA's prefix, writes the per-read fields and then copies the kept reads' words as
// one coalesced range per CTA (the masked query offsets one warp per read).  Only the kept reads' words of seq4 and
// runs of qpos are read.

namespace kdl {

constexpr int S_THREADS = 256;  // reads per CTA, one thread each
constexpr int S_REC = 16;       // uint32 words per CTA record of the scratch (and of the totals record behind them)
enum { S_READS = 0, S_WORDS, S_CX, S_HARD, S_EVT, S_MREADS, S_MBASES, S_NSUM };
constexpr long long S_NONE = -0x7fffffffffffffffLL - 1;  // identity of the max scans

struct SelectItem {
    uint32_t v[S_NSUM];   // the read's share of each output; all 0 when it is not kept
    long long mx[3];      // its max_simple_len, reach_right and reach_left candidates
    long long g;          // global start slot (kept reads)
    uint32_t base_words;  // words of its bases
    uint32_t mask_src;    // start of its run in the parent's qpos
    bool kept;
};

__device__ __forceinline__ void select_item(const kdl_batch& b, const kdl_qmask& q, const uint8_t* __restrict__ keep,
                                            long long r, SelectItem& it) {
#pragma unroll
    for (int k = 0; k < S_NSUM; ++k) it.v[k] = 0;
    it.mx[0] = it.mx[1] = it.mx[2] = 0;
    it.g = 0;
    it.base_words = 0;
    it.mask_src = 0;
    it.kept = r < b.n_reads && keep[r] != 0;
    if (!it.kept) return;
    const uint32_t lraw = (uint32_t)b.l_seq[r];
    const int c = find_contig(b.contig_read_off, b.n_contigs, r);
    it.g = b.contig_slot[c] + (long long)b.ref_start[r];
    it.v[S_READS] = 1;
    if (!(lraw & KDL_COMPLEX)) {  // simple: l_seq is the length of its one M op
        it.base_words = (lraw + 7u) >> 3;
        it.v[S_WORDS] = it.base_words;
        it.mx[0] = it.mx[1] = lraw;
    } else {
        const bool hard = (lraw & KDL_HARD) != 0;
        it.base_words = (uint32_t)((complex_len(lraw) + 7) >> 3);
        const uint32_t* __restrict__ blk = b.seq4 + (size_t)b.seq_off[r] + it.base_words;
        const uint32_t n_ops = blk[0];
        it.v[S_WORDS] = it.base_words + 2u + n_ops;
        it.v[S_CX] = 1;
        it.v[S_HARD] = hard ? 1u : 0u;
        uint32_t n_ins = 0;
        long long r_span = 0, lead = 0;
        for (uint32_t i = 0; i < n_ops; ++i) {
            const uint32_t cg = blk[2 + i];
            const int op = cg & 0xF;
            const long long len = cg >> 4;
            n_ins += op == 1;
            if (op == 0 || op == 7 || op == 8 || op == 2 || (op == 4 && i != 0)) r_span += len;
            if (op == 4 && i == 0) lead = len;
        }
        it.v[S_EVT] = n_ins;
        if (!hard) {
            it.mx[1] = r_span + 1;
            it.mx[2] = lead + 1;
        }
    }
    if (q.n_reads > 0) {  // the read's entry in the ascending mask list, if it has one
        long long lo = 0, hi = q.n_reads;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if ((long long)q.read_idx[mid] < r) lo = mid + 1; else hi = mid;
        }
        if (lo < q.n_reads && (long long)q.read_idx[lo] == r) {
            it.v[S_MREADS] = 1;
            it.v[S_MBASES] = q.off[lo + 1] - q.off[lo];
            it.mask_src = q.off[lo];
        }
    }
}

// v -> its exclusive prefix over the CTA, element-wise; total = the CTA's sums
template <int N>
__device__ __forceinline__ void cta_scan_vec(uint32_t (&v)[N], uint32_t (&total)[N]) {
    __shared__ uint32_t warp_sum[S_THREADS / 32][N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl[N];
#pragma unroll
    for (int k = 0; k < N; ++k) incl[k] = v[k];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
#pragma unroll
        for (int k = 0; k < N; ++k) {
            const uint32_t o = __shfl_up_sync(0xffffffffu, incl[k], d);
            if (lane >= d) incl[k] += o;
        }
    }
    __syncthreads();  // warp_sum may still be read by a previous call
    if (lane == 31) {
#pragma unroll
        for (int k = 0; k < N; ++k) warp_sum[warp][k] = incl[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) {
        uint32_t before = 0, all = 0;
        for (int w = 0; w < S_THREADS / 32; ++w) {
            const uint32_t t = warp_sum[w][k];
            if (w < warp) before += t;
            all += t;
        }
        total[k] = all;
        v[k] = before + incl[k] - v[k];
    }
}

// the largest v of the threads before this one (S_NONE for thread 0); *total = the CTA's largest v
__device__ __forceinline__ long long cta_exclusive_max(long long v, long long* total) {
    __shared__ long long warp_max[S_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d && o > incl) incl = o;
    }
    long long ex = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) ex = S_NONE;
    __syncthreads();
    if (lane == 31) warp_max[warp] = incl;
    __syncthreads();
    long long all = S_NONE;
    for (int w = 0; w < S_THREADS / 32; ++w) {
        const long long t = warp_max[w];
        if (w < warp && t > ex) ex = t;
        if (t > all) all = t;
    }
    *total = all;
    return ex;
}

// every thread gets the CTA's maximum of each v[k]
template <int N>
__device__ __forceinline__ void cta_max_vec(long long (&v)[N]) {
    __shared__ long long warp_max[S_THREADS / 32][N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
#pragma unroll
        for (int k = 0; k < N; ++k) {
            const long long o = __shfl_xor_sync(0xffffffffu, v[k], d);
            if (o > v[k]) v[k] = o;
        }
    }
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) warp_max[warp][k] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) {
        long long m = S_NONE;
        for (int w = 0; w < S_THREADS / 32; ++w) m = warp_max[w][k] > m ? warp_max[w][k] : m;
        v[k] = m;
    }
}

// Record of CTA b (scratch + S_REC * b): [0..6] the shares' sums (the combine turns them into exclusive prefixes),
// [7] bit 0 = the CTA keeps a read, bit 1 = a kept read of it starts before a kept read in front of it in the CTA,
// [8..10] the maxima, [12..13] the smallest and [14..15] the largest start slot of its kept reads (int64).
__global__ void __launch_bounds__(S_THREADS)
select_sums_kernel(kdl_batch b, kdl_qmask q, const uint8_t* __restrict__ keep, uint32_t* __restrict__ scratch) {
    const long long r = (long long)blockIdx.x * S_THREADS + threadIdx.x;
    SelectItem it;
    select_item(b, q, keep, r, it);
    uint32_t tot[S_NSUM];
    cta_scan_vec(it.v, tot);
    long long g_max;
    const long long before = cta_exclusive_max(it.kept ? it.g : S_NONE, &g_max);
    long long red[5] = {it.mx[0], it.mx[1], it.mx[2], it.kept ? -it.g : S_NONE, (it.kept && it.g < before) ? 1 : 0};
    cta_max_vec(red);
    if (threadIdx.x == 0) {
        uint32_t* rec = scratch + (size_t)S_REC * blockIdx.x;
#pragma unroll
        for (int k = 0; k < S_NSUM; ++k) rec[k] = tot[k];
        rec[7] = (tot[S_READS] ? 1u : 0u) | (red[4] ? 2u : 0u);
        rec[8] = (uint32_t)red[0];
        rec[9] = (uint32_t)red[1];
        rec[10] = (uint32_t)red[2];
        rec[11] = 0;
        long long* g = reinterpret_cast<long long*>(rec + 12);
        g[0] = tot[S_READS] ? -red[3] : 0;  // (red[3] is S_NONE when nothing is kept)
        g[1] = g_max;
    }
}

// one CTA: the records' sums -> exclusive prefixes in place; the totals record behind the last one:
// [0..6] the totals, [7] reads_sorted, [8..10] max_simple_len, reach_right, reach_left.
// Each thread takes S_PER consecutive records per round into registers (independent loads, one memory latency): its
// sums and largest start, the CTA scans, then a serial pass that writes the prefixes and checks the order against the
// starts before it.
constexpr int S_PER = 4;

__global__ void __launch_bounds__(S_THREADS)
select_combine_kernel(uint32_t* __restrict__ scratch, long long n_blocks) {
    uint32_t carry[S_NSUM];
#pragma unroll
    for (int k = 0; k < S_NSUM; ++k) carry[k] = 0;
    long long carry_g = S_NONE;
    long long red[4] = {0, 0, 0, 0};  // the three maxima, "unsorted"
    for (long long b0 = 0; b0 < n_blocks; b0 += (long long)S_THREADS * S_PER) {
        const long long i0 = b0 + (long long)threadIdx.x * S_PER;
        uint32_t w[S_PER][S_REC];  // the records, as 16-byte loads (a record is 64-byte aligned)
#pragma unroll
        for (int j = 0; j < S_PER; ++j) {
#pragma unroll
            for (int k = 0; k < S_REC / 4; ++k) {
                uint4 x = make_uint4(0u, 0u, 0u, 0u);
                if (i0 + j < n_blocks) x = reinterpret_cast<const uint4*>(scratch + (size_t)S_REC * (size_t)(i0 + j))[k];
                w[j][4 * k] = x.x; w[j][4 * k + 1] = x.y; w[j][4 * k + 2] = x.z; w[j][4 * k + 3] = x.w;
            }
        }
        uint32_t v[S_NSUM];
#pragma unroll
        for (int k = 0; k < S_NSUM; ++k) v[k] = 0;
        long long last = S_NONE;
#pragma unroll
        for (int j = 0; j < S_PER; ++j) {
#pragma unroll
            for (int k = 0; k < S_NSUM; ++k) v[k] += w[j][k];
            const long long g_last = (long long)(((unsigned long long)w[j][15] << 32) | w[j][14]);
            if ((w[j][7] & 1u) && g_last > last) last = g_last;
#pragma unroll
            for (int k = 0; k < 3; ++k) red[k] = (long long)w[j][8 + k] > red[k] ? (long long)w[j][8 + k] : red[k];
        }
        uint32_t tot[S_NSUM];
        cta_scan_vec(v, tot);
        long long chunk_max;
        long long running = cta_exclusive_max(last, &chunk_max);
        running = carry_g > running ? carry_g : running;
#pragma unroll
        for (int j = 0; j < S_PER; ++j) {
            if (i0 + j >= n_blocks) break;
            uint32_t* rec = scratch + (size_t)S_REC * (size_t)(i0 + j);
#pragma unroll
            for (int k = 0; k < S_NSUM; ++k) {
                rec[k] = carry[k] + v[k];
                v[k] += w[j][k];
            }
            if (w[j][7] & 1u) {
                const long long g_first = (long long)(((unsigned long long)w[j][13] << 32) | w[j][12]);
                const long long g_last = (long long)(((unsigned long long)w[j][15] << 32) | w[j][14]);
                if ((w[j][7] & 2u) || g_first < running) red[3] = 1;
                running = g_last > running ? g_last : running;
            }
        }
#pragma unroll
        for (int k = 0; k < S_NSUM; ++k) carry[k] += tot[k];
        carry_g = chunk_max > carry_g ? chunk_max : carry_g;
    }
    cta_max_vec(red);
    if (threadIdx.x == 0) {
        uint32_t* tot = scratch + (size_t)S_REC * (size_t)n_blocks;
#pragma unroll
        for (int k = 0; k < S_NSUM; ++k) tot[k] = carry[k];
        tot[7] = red[3] ? 0u : 1u;
        tot[8] = (uint32_t)red[0];
        tot[9] = (uint32_t)red[1];
        tot[10] = (uint32_t)red[2];
        for (int k = 11; k < S_REC; ++k) tot[k] = 0;
    }
}

// The grid covers reads 0 .. n_reads (one item more: the end of contig_read_off and of the mask offsets).  `out` and
// `om` carry the caller's output arrays (const in the structs, written here) and the totals as their counts; every
// write is bounded by them, so a wrong count stays in bounds.
__global__ void __launch_bounds__(S_THREADS)
select_scatter_kernel(kdl_batch b, kdl_qmask q, const uint8_t* __restrict__ keep, const uint32_t* __restrict__ scratch,
                      kdl_batch out, int64_t* __restrict__ out_read_off, kdl_qmask om) {
    __shared__ uint32_t s_src[S_THREADS], s_dst[S_THREADS], s_n[S_THREADS], s_evt_at[S_THREADS], s_evt[S_THREADS];
    __shared__ uint32_t s_msrc[S_THREADS], s_mdst[S_THREADS], s_mn[S_THREADS];
    const long long r = (long long)blockIdx.x * S_THREADS + threadIdx.x;
    SelectItem it;
    select_item(b, q, keep, r, it);
    uint32_t o[S_NSUM], tot[S_NSUM];
#pragma unroll
    for (int k = 0; k < S_NSUM; ++k) o[k] = it.v[k];
    cta_scan_vec(o, tot);
    const uint32_t* rec = scratch + (size_t)S_REC * blockIdx.x;
#pragma unroll
    for (int k = 0; k < S_NSUM; ++k) o[k] += rec[k];

    const bool put = it.kept && (long long)o[S_READS] < out.n_reads;
    if (put) {
        const uint32_t k = o[S_READS];
        const_cast<int32_t*>(out.ref_start)[k] = b.ref_start[r];
        const_cast<uint32_t*>(out.seq_off)[k] = o[S_WORDS];
        const_cast<int32_t*>(out.l_seq)[k] = b.l_seq[r];
        if (it.v[S_CX] && (long long)o[S_CX] < out.n_complex) const_cast<uint32_t*>(out.complex_idx)[o[S_CX]] = k;
        if (it.v[S_HARD] && (long long)o[S_HARD] < out.n_hard) const_cast<uint32_t*>(out.hard_idx)[o[S_HARD]] = k;
        if (it.v[S_MREADS] && (long long)o[S_MREADS] < om.n_reads) {
            const_cast<uint32_t*>(om.read_idx)[o[S_MREADS]] = k;
            const_cast<uint32_t*>(om.off)[o[S_MREADS]] = o[S_MBASES];
        }
    }
    if (r <= b.n_reads) {  // the contigs whose reads begin at r (r == n_reads: the end, and the empty contigs there)
        int c = r < b.n_reads ? find_contig(b.contig_read_off, b.n_contigs, r) : b.n_contigs;
        for (; c >= 0 && b.contig_read_off[c] == r; --c) out_read_off[c] = o[S_READS];
        if (r == b.n_reads && om.n_reads > 0) const_cast<uint32_t*>(om.off)[om.n_reads] = (uint32_t)om.n_bases;
    }

    // the blocks: staged per read, then copied
    const bool fits = put && (long long)o[S_WORDS] + it.v[S_WORDS] <= out.seq4_words;
    const bool mfits = put && it.v[S_MREADS] && (long long)o[S_MBASES] + it.v[S_MBASES] <= om.n_bases;
    s_src[threadIdx.x] = it.kept ? b.seq_off[r] : 0u;
    s_dst[threadIdx.x] = o[S_WORDS] - rec[S_WORDS];  // from the CTA's first output word
    s_n[threadIdx.x] = fits ? it.v[S_WORDS] : 0u;
    s_evt_at[threadIdx.x] = it.v[S_CX] ? it.base_words + 1u : 0xffffffffu;  // the evt_off word of the trailer
    s_evt[threadIdx.x] = o[S_EVT];
    s_msrc[threadIdx.x] = it.mask_src;
    s_mdst[threadIdx.x] = o[S_MBASES];
    s_mn[threadIdx.x] = mfits ? it.v[S_MBASES] : 0u;
    __syncthreads();
    // the kept reads' words are one contiguous output range of tot[S_WORDS] words: the CTA copies it word by word,
    // each word's read found by a binary search over the staged destinations (every kept read has a word, so the last
    // read starting at or before a word is its owner)
    // (S_UNROLL words per thread per round: their loads are all issued before their stores)
    uint32_t* __restrict__ seq4 = const_cast<uint32_t*>(out.seq4);
    const long long base = rec[S_WORDS];
    constexpr int S_UNROLL = 4;
    for (uint32_t w0 = threadIdx.x; w0 < tot[S_WORDS]; w0 += S_UNROLL * S_THREADS) {
        uint32_t val[S_UNROLL];
        long long at[S_UNROLL];
#pragma unroll
        for (int u = 0; u < S_UNROLL; ++u) {
            const uint32_t w = w0 + (uint32_t)u * S_THREADS;
            at[u] = -1;
            val[u] = 0;
            if (w >= tot[S_WORDS]) continue;
            int lo = 0, hi = S_THREADS - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (s_dst[mid] <= w) lo = mid; else hi = mid - 1;
            }
            const uint32_t q = w - s_dst[lo];
            if (q < s_n[lo] && base + w < out.seq4_words) {
                at[u] = base + w;
                val[u] = q == s_evt_at[lo] ? s_evt[lo] : __ldg(b.seq4 + s_src[lo] + q);
            }
        }
#pragma unroll
        for (int u = 0; u < S_UNROLL; ++u)
            if (at[u] >= 0) seq4[at[u]] = val[u];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = warp * 32; j < warp * 32 + 32; ++j) {
        const uint32_t mn = s_mn[j];
        if (mn) {
            const uint32_t* __restrict__ src = q.qpos + s_msrc[j];
            uint32_t* __restrict__ dst = const_cast<uint32_t*>(om.qpos) + s_mdst[j];
            for (uint32_t w = lane; w < mn; w += 32) dst[w] = src[w];
        }
    }
}

}  // namespace kdl
