/* kindel_b200.h -- C ABI of the H100-native pileup/consensus engine (libkindel_b200.so).
 *
 * The reference (bede/kindel v1.2.1) is pure Python and has no FFI of its own; its seam for this
 * path is three Python callables (SURVEY.md section 8b):
 *     parse_records(ref_id, ref_len, records)          reference kindel/kindel.py:21-128
 *     consensus(weight)                                reference kindel/kindel.py:369-381
 *     consensus_sequence(weights, insertions, ...)     reference kindel/kindel.py:384-430
 * The entry points below are what a ctypes/cffi binding inside the reference's
 * `kindel/kindel.py` would call in place of those loops (the stub is shown in INTEGRATION.md;
 * the shipped host side that does exactly that is kindel_b200/kindel.py).
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / C++ types.  `stream` is a cudaStream_t passed as void*.
 *   - every function returns a kdl_status (0 = ok).  Nothing here allocates device memory except
 *     the kdl_ctx_* host-buffer path, which owns a growable workspace inside its context.
 *   - "device" entry points take DEVICE pointers and only enqueue work on `stream` (asynchronous;
 *     the caller synchronises).  "host" entry points (kdl_ctx_*) take HOST pointers, do the
 *     host->device copies, the kernels and the device->host copies themselves and return when the
 *     results are in the caller's buffers.
 *   - re-entrant per stream, no global mutable state.
 *
 * Data layout (all little-endian, see DESIGN.md section 3)
 *   reads, in the reference's iteration order (grouped by contig in first-seen order, file order
 *   inside a contig; records failing `mapped and len(seq) > 1`, kindel.py:43-46, already dropped):
 *     ref_start[n]   int32   0-based reference cursor at walk start (= SAM POS - 1; -1 if POS == 0)
 *     seq_off[n]     uint32  offset of the read's block in `seq4`, in 4-byte words (non-decreasing)
 *     l_seq[n]       int32   bits 0..29: SEQ length.  bit 31 (KDL_COMPLEX) clear = "simple" read: exactly
 *                            one M/=/X op whose length equals the SEQ length, fully inside the contig
 *                            (ref_start >= 0, ref_start + len <= L), every base one of A,C,G,T,N (nibbles
 *                            1,2,4,8,15), at most KDL_FAST_MAXLEN bases.  Its CIGAR is implied and never
 *                            travels.  bit 31 set = complex read: its CIGAR follows its bases in `seq4`
 *                            (below).  bit 30 (KDL_HARD) set as well = the general, atomic kernel K1g must
 *                            walk it (it may wrap a Python negative index, raise like the reference, or is
 *                            too long for a tile: SURVEY.md A-7..A-10); bit 30 clear = "tile-eligible": every
 *                            slot it touches lies in [1, L - 1] of its contig, its query span fits its SEQ,
 *                            it has at most KDL_TILE_MAXOPS ops and reaches at most KDL_TILE_MAXREACH slots
 *                            to either side of its start, and all its bases are A,C,G,T,N -- K1, K1w and K1e
 *                            walk it without bounds or error logic.  A tile-eligible read keeps its SEQ
 *                            length (<= KDL_FAST_MAXLEN) in bits 0..15 and its number of M/=/X ops in bits
 *                            16..22, so a tile can be sized before its bases are staged; a hard read keeps
 *                            its length in bits 0..29.
 *                            The flatten step classifies (kindel_b200/bamio.py).
 *     seq4[n_words]  uint32  one block per read, in read order.  Bases: BAM nibble codes
 *                            "=ACMGRSVTWYHKDBN", 8 per 32-bit word, FIRST base in the MOST significant
 *                            nibble (base k of a read sits at bits [28-4*(k%8), 32-4*(k%8)) of word k/8),
 *                            unused trailing nibbles of the last word zero.  A COMPLEX read's block goes on
 *                            with  [n_ops] [evt_off] [n_ops x CIGAR word]  -- BAM encoding len << 4 | op,
 *                            op index into "MIDNSHP=X"; evt_off = number of I ops of all reads before this
 *                            one (row of its first insertion event).  A tile's reads are one contiguous
 *                            byte range of this array, CIGARs included: one bulk copy stages them.
 *   contigs:
 *     contig_read_off[n_contigs+1] int64  reads of contig c are [off[c], off[c+1])
 *     contig_len[n_contigs]        int32  reference length L_c
 *     contig_slot[n_contigs]       int64  first table slot of contig c; it owns L_c + 1 slots
 *   count table: counts[KDL_NCOL][n_slots] int32, column-major (one contiguous array per column):
 *     0-4  weights A,C,G,T,N          (kindel.py:29,49-54)
 *     5    deletions                  (kindel.py:39,59-62)
 *     6    insertion events (total)   (kindel.py:38,55-58; the string-keyed dict is rebuilt from
 *                                      the event list below)
 *     7    clip_starts   8 clip_ends  (kindel.py:36-37,66,75)
 *     9-13 clip_start_weights A,C,G,T,N   14-18 clip_end_weights A,C,G,T,N (kindel.py:30-35,67-81)
 *   insertion events: ins_events[n_events][4] int32 = (slot, read, q_off, len), event k of the j-th
 *     listed read stored at row evt_off[j] + k  (deterministic, reference iteration order).
 *   masked bases (extension, kdl_qmask below): bases below a Phred quality threshold are N (nibble 15) in seq4 and
 *     listed per read; kdl_unmask takes back the count each of them added to a base-count column.
 */
#ifndef KINDEL_B200_H
#define KINDEL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KDL_ABI_VERSION 2
#define KDL_NCOL 19
#define KDL_NVOTE_COL 7 /* columns 0..6 are all the vote needs */
#define KDL_COMPLEX 0x80000000u
#define KDL_HARD 0x40000000u
#define KDL_LEN_MASK 0x0000ffffu   /* SEQ length of a complex read lives in bits 0..15 (longer reads are KDL_HARD
                                      and keep their length in bits 0..29 with the op count field zero) */
#define KDL_NM_SHIFT 16            /* bits 16..22: M/=/X op count of a complex read */
#define KDL_NM_MASK 0x7fu
#define KDL_TILE 512          /* slots per tile of the owner-computes pileup; n_slots % KDL_TILE == 0 */
#define KDL_FAST_MAXLEN 8192  /* longest read the flatten step may mark simple */
#define KDL_TILE_MAXOPS 64    /* most CIGAR ops of a tile-eligible complex read */
#define KDL_TILE_MAXREACH 1024 /* furthest slot, relative to its start, a tile-eligible complex read touches */

enum kdl_col {
    KDL_W_A = 0, KDL_W_C, KDL_W_G, KDL_W_T, KDL_W_N,
    KDL_DEL = 5, KDL_INS = 6, KDL_CLIP_STARTS = 7, KDL_CLIP_ENDS = 8,
    KDL_CSW_A = 9, KDL_CEW_A = 14
};

typedef enum kdl_status {
    KDL_OK = 0,
    KDL_ERR_INVALID_ARG = 1,
    KDL_ERR_CUDA = 2,
    KDL_ERR_NO_DEVICE = 3,
    /* data errors, mirroring the exceptions the reference raises (SURVEY.md App. A-10): */
    KDL_ERR_INDEX = 10, /* IndexError: walk ran off the contig / off SEQ (kindel.py:51,52,61) */
    KDL_ERR_KEY = 11    /* KeyError: base outside A,C,G,T,N used in an M or S op (kindel.py:52,72,79) */
} kdl_status;

/* Flattened read batch.  Pointers are device pointers for the device entry points and host
 * pointers for the kdl_ctx_* entry points. */
typedef struct kdl_batch {
    int64_t n_reads;
    int64_t seq4_words;  /* 32-bit words in seq4 */
    const int32_t* ref_start;
    const uint32_t* seq_off;
    const int32_t* l_seq;
    const uint32_t* seq4;
    int32_t n_contigs;
    int32_t reads_sorted;   /* 1 = contig_slot + ref_start and seq_off are non-decreasing over all reads */
    int32_t max_simple_len; /* longest simple read (bases); 0 if there is none */
    int32_t reach_right;    /* max over simple and tile-eligible reads of (last touched slot - start + 1) */
    int32_t reach_left;     /* max over tile-eligible reads of (start - first touched slot) */
    int32_t reserved0;
    const int64_t* contig_read_off;
    const int32_t* contig_len;
    const int64_t* contig_slot;
    /* complex reads: how many there are (tile-eligible + hard; columns 5..18 are only ever written when
     * this is non-zero) and the ascending indices of the KDL_HARD ones, which K1g walks */
    int64_t n_complex;
    int64_t n_hard;
    const uint32_t* complex_idx; /* [n_complex] ascending indices of ALL complex reads; may be NULL when n_complex == 0 */
    const uint32_t* hard_idx;    /* [n_hard] ascending indices of the KDL_HARD ones; may be NULL when n_hard == 0 */
    /* scratch for the tile index kdl_pileup builds (K0): uint32[8 * n_slots / KDL_TILE], device
     * memory owned by the caller.  NULL, or reads_sorted == 0, selects the order-independent
     * atomic kernels instead of the tile-owner kernel. */
    uint32_t* tile_index;
} kdl_batch;

/* Masked bases (extension; min_base_quality): a base masked at decode is an N nibble in seq4 -- the pileup counts
 * it as an N, the insertion strings read it as N -- and is listed here so that kdl_unmask can take back its count
 * from the base-count column it went to (weights N, clip_start_weights N, clip_end_weights N).  Pointers are device
 * pointers for kdl_unmask and host pointers for kdl_ctx_consensus_masked.
 *   read_idx[n_reads]   ascending indices of the reads with masked bases
 *   off[n_reads + 1]    read_idx[j]'s entries are qpos[off[j] .. off[j + 1])
 *   qpos[n_bases]       query offsets (0-based into SEQ), ascending per read */
typedef struct kdl_qmask {
    int64_t n_reads;
    int64_t n_bases;
    const uint32_t* read_idx;
    const uint32_t* off;
    const uint32_t* qpos;
} kdl_qmask;

/* Error report written by the pileup (device memory, 4 x int32, zero it before the call):
 *   [0] != 0 : some read hit a data error; call kdl_diagnose for the exact first one. */
typedef struct kdl_diag {
    int32_t status;    /* KDL_OK, KDL_ERR_INDEX or KDL_ERR_KEY */
    int32_t reserved;
    int64_t read;      /* index of the first offending read in iteration order */
    int32_t nibble;    /* for KDL_ERR_KEY: BAM nibble code of the offending base */
    int32_t op_index;  /* CIGAR op at which the walk failed */
} kdl_diag;

int kdl_abi_version(void);
const char* kdl_status_string(int status);
/* number of CUDA kernels this library has launched in this process (bench.py: gpu_launches) */
int64_t kdl_launch_count(void);

/* K1 -- pileup.  Replaces the loop at kindel/kindel.py:40-81.
 * Adds every read's contribution to `counts` (caller zeroes it first, so several batches -- or
 * several read shards -- can accumulate into one table) and writes the insertion event rows.
 * err_flag: device int32[4], caller-zeroed; [0] becomes non-zero if any read raised.
 * Coordinate-sorted batches (reads_sorted, tile_index scratch given) take K0 (tile index) + the tile-owner
 * kernel K1 (simple reads and the M/=/X bases of tile-eligible complex reads: no atomics), K1w (all of those
 * complex reads' updates when they are rare, window by window) or K1e (their insertion / deletion / clip updates, once
 * per read) and K1g (KDL_HARD reads, atomics);
 * anything else the order-independent atomic kernels K1s + K1g. */
int kdl_pileup(const kdl_batch* batch, int32_t* counts, int64_t n_slots, int32_t* ins_events,
               int32_t* err_flag, void* stream);

/* Same as kdl_pileup, restricted to the slot range [slot_lo, slot_hi) (multiples of KDL_TILE) that
 * contains everything the batch can touch (a shard's footprint), with control over zeroing:
 *   KDL_PILEUP_FRESH_WEIGHTS  columns 0..4 of the range hold stale data: the tile-owner kernel
 *                             OVERWRITES them (plain stores, no prior memset, no read-modify-write)
 *   KDL_PILEUP_ZERO_REST      columns 5..18 of the range are zeroed first (needed only when an
 *                             earlier pileup with complex reads dirtied them; with FRESH_WEIGHTS the tile-owner
 *                             kernel does it window by window in its flush, no separate pass) */
#define KDL_PILEUP_FRESH_WEIGHTS 1
#define KDL_PILEUP_ZERO_REST 2
int kdl_pileup_range(const kdl_batch* batch, int32_t* counts, int64_t n_slots, int64_t slot_lo,
                     int64_t slot_hi, int32_t flags, int32_t* ins_events, int32_t* err_flag, void* stream);

/* kdl_pileup_range with the table's dirty-sector map, so that KDL_PILEUP_ZERO_REST zeroes only what an earlier pileup
 * wrote instead of all of columns 5..18 (complex reads dirty a few per cent of their 32-byte sectors).
 *   dirty_map  device uint32[4 * ceil(n_slots / 64)], 16-byte aligned, owned by the caller with the table: one
 *              16-byte record per 64-slot window w; byte b (0..13) of the record is column 5 + b, bit s of that byte
 *              covers slots [64 w + 8 s, 64 w + 8 s + 8).
 *   invariant  a slot of columns 5..18 is non-zero only if its bit is set (a set bit over zeros is always allowed).
 *              A new table's map is zero with the table; a caller that writes columns 5..18 by other means sets every
 *              bit (0xFF bytes), and the next pileup with KDL_PILEUP_ZERO_REST zeroes everything.
 * The pileup keeps the invariant: every kernel that writes columns 5..18 marks what it writes, and the zeroing clears
 * the records of the windows it has zeroed whole.  A batch with complex reads as dense as 1 in 16 or more dirties nearly
 * every sector: where the pileup zeroes, it then sets every record of [slot_lo, slot_hi) instead of marking op by op.
 * NULL = kdl_pileup_range (zeroing of everything, no marking). */
int kdl_pileup_range_map(const kdl_batch* batch, int32_t* counts, int64_t n_slots, int64_t slot_lo, int64_t slot_hi,
                         int32_t flags, uint32_t* dirty_map, int32_t* ins_events, int32_t* err_flag, void* stream);

/* K1q -- after kdl_pileup / kdl_pileup_range of the same batch on the same stream: subtracts 1 at the (column, slot)
 * where the pileup counted each masked base (column 4 for M/=/X, 18 for a left clip, 13 for a right clip; nothing for
 * an inserted base).  Launches nothing when qmask->n_reads == 0. */
int kdl_unmask(const kdl_batch* batch, const kdl_qmask* qmask, int32_t* counts, int64_t n_slots, void* stream);

/* Exact first error in reference iteration order (only needed when err_flag[0] != 0).
 * `diag_dev`: device kdl_diag, written asynchronously. */
int kdl_diagnose(const kdl_batch* batch, kdl_diag* diag_dev, void* stream);

/* K2 -- per-position vote.  Replaces kindel/kindel.py:402-424 + 369-381 for every slot.
 * calls[s] : bits 0-2 = emitted base (0..4 = A,C,G,T,N; a tie emits N), bits 4-5 = change code
 *            (0 none, 1 'D' -> nothing emitted, 2 'N' -> 'N' emitted, 3 'I' -> insertion string
 *            precedes the base), bit 7 = 0 (kdl_vote_iupac sets it for a multi-base call, below).
 *            min_depth_ceil = ceil(min_depth). */
int kdl_vote(const int32_t* counts, int64_t n_slots, int64_t min_depth_ceil, uint8_t* calls,
             void* stream);

/* K2 with IUPAC ambiguity codes (extension; the reference has no such option), 0 <= threshold <= 1, else (or NaN)
 * KDL_ERR_INVALID_ARG.  The D, N and I decisions are kdl_vote's and so is every 'D' / 'N' call byte; only the base
 * of a slot that emits one differs.  With D = A + C + G + T (N excluded): D == 0 emits N; otherwise
 * L(b) = sum of the counts of all bases with count >= count(b), v = the largest count(b) > 0 with
 * (double)L(b) >= threshold * (double)D (one correctly rounded multiply), and the call is the set
 * S = {b : count(b) >= v}.  |S| = 1: the base code, as kdl_vote writes it.  |S| >= 2:
 * calls[s] = 0x80 | change << 4 | mask, mask A=1 C=2 G=4 T=8 (the BAM nibble, letter "=ACMGRSVTWYHKDBN"[mask]);
 * bit 7 is never set by kdl_vote. */
int kdl_vote_iupac(const int32_t* counts, int64_t n_slots, int64_t min_depth_ceil, double threshold, uint8_t* calls,
                   void* stream);

/* Derived per-position columns of the `alignment` tuple (kindel/kindel.py:83-96) + the ACGT depth
 * used by build_report (kindel.py:450).  out[5][n_slots] int32: consensus_depth, clip_start_depth,
 * clip_end_depth, clip_depth, acgt_depth. */
int kdl_derive(const int32_t* counts, int64_t n_slots, int32_t* out, void* stream);

/* K4 -- the per-position predicates of the --realign path (reference kindel/kindel.py:182-185,202,243-246,256) for
 * slots [slot_lo, slot_hi):  flags[s] bit 0 = clip-dominant for right-clipped reads: clip_start_depth /
 * (sum(weights) + deletions + 1) > 0.5; bit 1 = their clip consensus extends through s: clip_start_depth >
 * (sum(weights) + deletions) * clip_decay_threshold; bits 2, 3 = the same for left-clipped reads (clip_end_*).
 * bases[s]: low nibble = consensus()[0] of clip_start_weights[s] (0..4 = A,C,G,T,N), high nibble = of
 * clip_end_weights[s].  Masking of the contig ends, pairing and the LCS merge stay with the caller. */
int kdl_cdr_flags(const int32_t* counts, int64_t n_slots, int64_t slot_lo, int64_t slot_hi,
                  double clip_decay_threshold, uint8_t* flags, uint8_t* bases, void* stream);

/* K5 -- the consensus text of every contig from the call bytes (reference kindel/kindel.py:413-424): nothing for a
 * 'D' call, the base letter (N for an 'N' call or a tie; the IUPAC letter of a bit-7 call) otherwise, preceded by the
 * insertion string for an 'I' call.  The strings of the 'I' slots come from the caller (ins_slot ascending, bytes ins_bytes[ins_off[k] ..
 * ins_off[k+1]) as they are to be printed: the modal inserted string in lower case, or "N" for a tie).
 * offsets: device uint32[n_slots + 1], out: offsets[s] = where slot s's text starts in `out`, offsets[n_slots] = total;
 * contig c's sequence is out[offsets[contig_slot[c]] .. offsets[contig_slot[c] + contig_len[c]]).
 * block_sums: device scratch of kdl_assemble_scratch_words(n_slots) uint32.  out: device bytes, at least
 * (number of positions + total insertion bytes).  All pointers are device pointers. */
int64_t kdl_assemble_scratch_words(int64_t n_slots);
int kdl_assemble(const uint8_t* calls, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                 int32_t n_contigs, const int64_t* ins_slot, const uint32_t* ins_off, const uint8_t* ins_bytes,
                 int64_t n_ins, uint32_t* block_sums, uint32_t* offsets, uint8_t* out, void* stream);

/* K2q -- per-base consensus qualities (extension; the reference has no such output), after any vote of the same
 * table (kdl_vote, kdl_vote_iupac, or the exchange's reduced table and gathered calls).  n_slots % 4 == 0; only
 * columns 0-3 of counts are read.  qual[s] = Q in 0..60 of the base slot s emits: with D = A + C + G + T and k = the
 * call's support -- the count of the called base, the summed counts of a multi-base IUPAC set, 0 for every call that
 * emits N (min depth, tie, zero depth, N winning, the IUPAC set of all four bases) and for a 'D' call -- Q = 0 when
 * k = 0, else the largest q <= 60 with (double)(D - k + 1) * TEN[q] <= (double)(D + 2), TEN[q] the correctly rounded
 * double of 10^(q/10) (kindel_b200/csrc/assemble.cu). */
int kdl_consensus_qual(const int32_t* counts, const uint8_t* calls, int64_t n_slots, uint8_t* qual, void* stream);

/* K5q -- the quality text beside kdl_assemble's text, on the same stream after it: `offsets` is what kdl_assemble
 * wrote.  Slot s owns out[offsets[s] .. offsets[s + 1]): every byte of an inserted string gets '!' + ins_qual[k] of
 * its slot (ins_slot ascending, as given to kdl_assemble), the slot's last byte '!' + qual[s].  out: device bytes, as
 * many as kdl_assemble's text.  All pointers are device pointers. */
int kdl_assemble_qual(const uint32_t* offsets, const uint8_t* qual, int64_t n_slots, const int64_t* ins_slot,
                      const uint8_t* ins_qual, int64_t n_ins, uint8_t* out, void* stream);

/* K6 -- the variant sites of `variants --only-variants` and of the VCF (extension), selected on the device.  At each
 * position (slots [contig_slot[c], contig_slot[c] + contig_len[c]); never the extra slot behind a contig or the
 * padding), with t = columns 0-5 of counts (A, C, G, T, N, deletions), depth = their sum and top = the first maximum,
 * allele k is a variant when t[k] > abs_floor and (double)t[k] / (double)depth > rel_threshold (0 at depth 0) and
 * k != top; a site is a position with a variant allele.  abs_floor: floor of the absolute threshold clamped to
 * [-1, 2^31] (2^31 for NaN); rel_threshold: NaN selects nothing.  n_slots % 4 == 0, counts 16-byte aligned.
 *
 * kdl_variant_count runs the per-CTA counts and their scan; the number of sites is then block_sums[words - 1], with
 * block_sums device scratch of words = kdl_variant_scratch_words(n_slots) uint32.  kdl_variant_scatter, on the same
 * stream after it with the same arguments and n_sites = that number, writes the sites in ascending slot order:
 * site_slot[i], site_counts[k * n_sites + i] (k = 0..5) and site_mask[i] (bit k: allele k is a variant).  All pointers
 * are device pointers. */
int64_t kdl_variant_scratch_words(int64_t n_slots);
int kdl_variant_count(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                      int32_t n_contigs, int64_t abs_floor, double rel_threshold, uint32_t* block_sums, void* stream);
int kdl_variant_scatter(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                        int32_t n_contigs, int64_t abs_floor, double rel_threshold, const uint32_t* block_sums,
                        int64_t n_sites, int64_t* site_slot, int32_t* site_counts, uint8_t* site_mask, void* stream);

/* K6r -- the candidate sites of `variants --vcf --reference` (extension): K6's passes against reference bases.
 * ref[n_slots]: one code per slot, 0-3 = A, C, G, T, 4 = anything else (and every slot that is not a position),
 * 4-byte aligned.  Per slot s of contig c, p = s - contig_slot[c], g = ref[s], t = columns 0-6 of counts and
 * depth(s) = t[0] + ... + t[5]:
 *   bit k (k = 0..3, SNV allele A, C, G, T), only at 0 <= p < L: k != g, t[k] > abs_floor and
 *     (double)t[k] / (double)depth(s) > rel_threshold (0 at depth 0);
 *   bit 6 (insertion candidate), at 0 <= p <= L: t[6] > abs_floor and t[6] / DPa > rel_threshold, DPa = depth(s - 1)
 *     for p >= 1 and depth(s) for p = 0 (0 at DPa 0).
 * abs_floor / rel_threshold as for K6.  Counting, scratch (kdl_variant_scratch_words) and the site total as for
 * kdl_variant_count.  kdl_variant_ref_scatter writes, in ascending slot order, site_slot[i], site_counts[k * n_sites
 * + i] (k = 0..6), site_dpa[i] (DPa) and site_mask[i].  All pointers are device pointers. */
int kdl_variant_ref_count(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                          int32_t n_contigs, const uint8_t* ref, int64_t abs_floor, double rel_threshold,
                          uint32_t* block_sums, void* stream);
int kdl_variant_ref_scatter(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot,
                            const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                            double rel_threshold, const uint32_t* block_sums, int64_t n_sites, int64_t* site_slot,
                            int32_t* site_counts, int64_t* site_dpa, uint8_t* site_mask, void* stream);

/* K6m -- the sites of several samples at once (`variants --vcf a.bam b.bam ...`, extension): K6's passes over the
 * samples' tables stacked on one shared layout.  counts: int32 [n_samples][7][n_slots] (sample i's columns 0-6 at
 * counts + i * 7 * n_slots), n_samples >= 1.  Per slot, with t^i sample i's columns and depth^i = t^i[0] + ... +
 * t^i[5]:
 *   pooled mode (ref == NULL), only at positions (0 <= p < L): P = sum over the samples of t^i[0..5] in 64-bit,
 *     top = the first maximum of P; bit k (k = 0..5, k != top) is set when some sample has t^i[k] > abs_floor and
 *     (double)t^i[k] / (double)depth^i > rel_threshold (0 at depth 0).
 *   reference mode (ref as for K6r): bits 0-3 are K6r's SNV test of each sample against g, bit 6 K6r's
 *     insertion-candidate test with each sample's own DPa (depth^i(s - 1) for p >= 1, depth^i(s) for p = 0); each
 *     ORed over the samples, at K6r's positions.
 * At n_samples = 1 the bits are K6's (pooled) and K6r's (reference).  abs_floor / rel_threshold as for K6; counting,
 * scratch (kdl_variant_scratch_words) and the site total as for kdl_variant_count.  kdl_variant_multi_scatter writes,
 * in ascending slot order, site_slot[i] and site_mask[i] (the OR); the samples' rows are not written: the caller
 * gathers them from counts at the sites.  All pointers are device pointers. */
int kdl_variant_multi_count(const int32_t* counts, int32_t n_samples, int64_t n_slots, const int64_t* contig_slot,
                            const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                            double rel_threshold, uint32_t* block_sums, void* stream);
int kdl_variant_multi_scatter(const int32_t* counts, int32_t n_samples, int64_t n_slots, const int64_t* contig_slot,
                              const int32_t* contig_len, int32_t n_contigs, const uint8_t* ref, int64_t abs_floor,
                              double rel_threshold, const uint32_t* block_sums, int64_t n_sites, int64_t* site_slot,
                              uint8_t* site_mask, void* stream);

/* K7 -- the deletion events of a batch (extension, for `variants --vcf --reference`).  Every read's CIGAR is walked
 * with the reference's cursor (kindel.py:40-81: M/=/X and D advance; an S that is op #0 does not; any later S advances
 * while the cursor is below the contig length L; I, N, H, P do not); simple reads have no D op.  A D of length n >= 1
 * at cursor r is an event when 0 <= r and r + n <= L: (contig_slot + r, n).  kdl_deletion_count runs the per-CTA
 * counts and their scan; the number of events is then block_sums[words - 1], with block_sums device scratch of
 * words = kdl_deletion_scratch_words(n_reads) uint32.  kdl_deletion_scatter, on the same stream after it with
 * n_events = that number, writes ev_slot[i] and ev_len[i] in read order, then op order.  Device pointers. */
int64_t kdl_deletion_scratch_words(int64_t n_reads);
int kdl_deletion_count(const kdl_batch* batch, uint32_t* block_sums, void* stream);
int kdl_deletion_scatter(const kdl_batch* batch, const uint32_t* block_sums, int64_t n_events, int64_t* ev_slot,
                         int32_t* ev_len, void* stream);

/* K15d / K15i -- indel events left-aligned against the reference (extension: `variants --vcf --reference
 * --left-align`).  ref[n_slots]: K6r's codes (0-3 = A, C, G, T, 4 = anything else and every slot that is not a
 * position); s0 = contig_slot of the event's contig (the last contig with contig_slot <= the event's slot).
 * kdl_left_align_deletions: keys[i] = r << 28 | n, a K7 event (slot r, length n) or a group of them; while r > s0,
 * ref[r-1] < 4 and ref[r-1] == ref[r+n-1], r -= 1; keys_out[i] = the moved key (keys_out may be keys).  The caller
 * groups the moved keys again (equal keys: one group, the counts summed).
 * kdl_left_align_insertions: ins_events[n_events][4] = kdl_pileup's rows (slot p, read, q_off, len) of `batch`, 16-byte
 * aligned; t = the read's bases q_off .. min(q_off + len, SEQ) - 1 in seq4, m of them.  With k = 0: while m > 0,
 * p > s0, ref[p-1] < 4 and the base t[(m-1-k) mod m] is that code (A, C, G, T; any other nibble matches nothing),
 * p -= 1 and k += 1.  norm_slot[i] = p, rot[i] = k mod m (0 at m = 0): the normalised string is t rotated right by
 * rot[i]; hist[p] += 1 (atomics: hist is int32[n_slots], zeroed by the caller).  A row with dead[i] != 0 (dead may be
 * NULL) gets norm_slot -1, rot 0 and counts in no slot.  One thread per key / row.  Device pointers. */
int kdl_left_align_deletions(const int64_t* keys, int64_t n_keys, const int64_t* contig_slot, int32_t n_contigs,
                             const uint8_t* ref, int64_t* keys_out, void* stream);
int kdl_left_align_insertions(const kdl_batch* batch, const int32_t* ins_events, int64_t n_events, const uint8_t* dead,
                              const uint8_t* ref, int64_t* norm_slot, int32_t* rot, int32_t* hist, void* stream);

/* K8 (extension: `variants --vcf --strand`): the sub-batch of the reads with keep[r] != 0, built on the device.  The
 * result equals what the host's bamio.select_reads gives for np.flatnonzero(keep), field for field: the kept reads in
 * their order; seq_off dense; l_seq the parent's word (classification is per read); seq4 each kept read's bases and, for
 * a complex read, its [n_ops][evt_off][ops] trailer with evt_off the exclusive prefix of the kept reads' I-op counts;
 * contig_read_off, complex_idx and hard_idx remapped; reads_sorted recomputed over the kept reads; max_simple_len,
 * reach_right and reach_left the maxima over the kept reads (simple: the op length; tile-eligible: r_span + 1 and
 * lead + 1 of the CIGAR walk); the mask list with read_idx remapped, off rebuilt and the qpos runs copied.
 * contig_len / contig_slot / n_contigs are the parent's (the result may share them).
 *   kdl_select_count    per-CTA counts and maxima, then one CTA combines them.  scratch: device uint32
 *                       [kdl_select_scratch_words(n_reads)]; its last 16 words are the totals record, read back once:
 *                       [0] reads, [1] seq4 words, [2] complex reads, [3] hard reads, [4] insertion events, [5] reads
 *                       with masked bases, [6] masked bases, [7] reads_sorted, [8] max_simple_len, [9] reach_right,
 *                       [10] reach_left.
 *   kdl_select_scatter  on the same stream after it: writes the sub-batch into `out`, whose scalars the caller set
 *                       from the totals and whose arrays it sized by them (complex_idx / hard_idx may be NULL when
 *                       their count is 0; contig_read_off [n_contigs + 1]); out_mask (NULL when totals[5] == 0)
 *                       receives the mask list.
 * qmask may be NULL or empty.  One thread per read counts; the scatter copies each CTA's kept words as one coalesced
 * range. */
int64_t kdl_select_scratch_words(int64_t n_reads);
int kdl_select_count(const kdl_batch* batch, const kdl_qmask* qmask, const uint8_t* keep, uint32_t* scratch,
                     void* stream);
int kdl_select_scatter(const kdl_batch* batch, const kdl_qmask* qmask, const uint8_t* keep, const uint32_t* scratch,
                       const kdl_batch* out, const kdl_qmask* out_mask, void* stream);

/* K9 (extension: `--primers scheme.bed`): masks the bases of every read that copy an amplicon primer, as
 * min_base_quality masks a low-quality base (N in seq4, listed in the mask list for kdl_unmask), before the pileup.
 * Per read on contig c with at least one M/=/X base: s and e are the walk cursors (the reference's r_pos, before the
 * Python index wrap) of its first and its last M/=/X base.  Left: if a primer [a, b) of c has a <= s < b, B = the
 * largest such b, and every M/=/X base with cursor in [s, B) is masked.  Right: if a primer has a <= e < b, A = the
 * smallest such a, and every M/=/X base with cursor in [A, e] is masked.  Nothing else is masked (inserted and clipped
 * bases, deletions, clip events are untouched), and only bases inside the read's SEQ.  The primers of contig c, two
 * sorted views of the same intervals [contig_off[c], contig_off[c + 1]) (device pointers, int32 coordinates):
 *   start_sorted / end_max   starts ascending, end_max[i] = the largest end of the intervals up to i in that order
 *   end_sorted / start_min   ends ascending, start_min[i] = the smallest start of the intervals from i on in that order
 * (end_max and start_min restart at every contig).  n_contigs must be the batch's.
 *   kdl_primers_count  per-CTA counts and their scans.  scratch: device uint32[kdl_primers_scratch_words(n_reads)]; its
 *                      last 8 words are the totals record, read back once: [0] reads in the new mask list, [1] bases in
 *                      it, [2] reads with primer bases, [3] primer bases.
 *   kdl_primers_apply  on the same stream after it: writes the new mask list into out_mask (arrays sized by the
 *                      totals; NULL when totals[0] == 0) -- per read the sorted union of its entries in qmask (may be
 *                      NULL or empty) and its primer bases, each base once -- and sets the primer bases' nibbles to N
 *                      (15) in `seq4`: the batch's own seq4 (in place) or a copy of it.
 * One thread per 4 consecutive reads; a read owns whole words of seq4, so no atomics. */
typedef struct kdl_primers {
    int32_t n_contigs;
    int32_t reserved;
    int64_t n_intervals;
    const int64_t* contig_off; /* [n_contigs + 1] */
    const int32_t* start_sorted;
    const int32_t* end_max;
    const int32_t* end_sorted;
    const int32_t* start_min;
} kdl_primers;

int64_t kdl_primers_scratch_words(int64_t n_reads);
int kdl_primers_count(const kdl_batch* batch, const kdl_qmask* qmask, const kdl_primers* primers, uint32_t* scratch,
                      void* stream);
int kdl_primers_apply(const kdl_batch* batch, const kdl_qmask* qmask, const kdl_primers* primers,
                      const uint32_t* scratch, uint32_t* seq4, const kdl_qmask* out_mask, void* stream);

/* K10 (extension: `--mask-overlaps`): each read pair counted once where its mates overlap.  The decode gives every
 * kept read name_hash (64-bit FNV-1a of QNAME, NUL excluded), mate_start (PNEXT - 1, in ref_start's coordinates) and
 * pair_role: 1 for a first mate, 2 for a last mate, and 0 unless FLAG has 0x1, none of 0x8 / 0x100 / 0x800, exactly
 * one of 0x40 / 0x80, and RNEXT is the read's own contig (kdl_bam_fill_mates).
 *   Pair: two reads with roles 1 and 2 that are the only reads of the batch with pair_role != 0 and that name hash,
 *   on one contig, each one's ref_start the other's mate_start, neither KDL_HARD.  R1 is the role-1 read, R2 the
 *   role-2 read.  Anything else (singletons, groups of three or more, inconsistent coordinates) is left alone.
 *   Covers: R1 covers cursor x (the walk of K7) when it has there an M/=/X base inside SEQ whose nibble is not N --
 *   after the quality and primer masks, so a masked R1 base covers nothing -- or a D op.
 *   Masking R2: every M/=/X base of R2 at a covered cursor is masked as min_base_quality masks a base (N in seq4,
 *   listed in the mask list, its column-4 count taken back by kdl_unmask); a D op at [r, r + n) is dropped when R1
 *   covers r (its n column-5 counts are taken back, and it is no K7 event); an I op at slot p is dropped when R1
 *   covers p - 1 and p (its column-6 count is taken back, and its event row reaches no insertion string).  Clips
 *   and clip columns 7-18 are untouched.  So at a position R1 covers a pair adds at most one count to columns 0-3
 *   and 5, R1's, and where R1 covers nothing only R2 counts.  Exceptions where R1's information starts or stops: a
 *   real N in R1 is counted in column 4 and hides nothing; a kept R2 deletion (R1 does not cover its first position)
 *   also counts where R1 covers later positions of it; an R2 insertion next to an R1 end, N or masked base is kept
 *   beside an R1 insertion at the same slot.
 *   Order: decode, upload, K9, kdl_mates_pair, kdl_overlap_count / _apply, the pileup, kdl_unmask, kdl_overlap_untake.
 *   kdl_mates_pair     K10p.  order[n_order]: the indices of the reads with pair_role != 0, sorted by name_hash
 *                      (any order among equal hashes).  Writes mate[n_reads]: the R1 of every paired R2, -1 elsewhere.
 *                      The device sees only the hash: two names that hash alike are one group.
 *   kdl_overlap_count  K10's count.  scratch: device uint32[kdl_overlap_scratch_words(n_reads)]; its last 8 words are
 *                      the totals record, read back once: [0] reads in the merged mask list, [1] bases in it, [2] drop
 *                      rows, [3] pairs, [4] overlap bases, [5] dropped deletions, [6] dropped insertions.
 *   kdl_overlap_apply  on the same stream after it: writes the merged mask list into out_mask (sized by the totals;
 *                      NULL when totals[0] == 0) -- per read the sorted union of its entries in qmask (may be NULL)
 *                      and its overlap bases --, sets R2's overlap nibbles to N in `seq4` (the batch's own, in place,
 *                      or a copy), and writes drops[n_drops][4] int32 = (slot, len, read, evt) for every dropped op
 *                      in read, then op order: evt = the I op's row in ins_events, -1 for a D.
 *   kdl_overlap_untake K10u, after kdl_unmask on the same stream: subtracts each drop row's counts from column 5
 *                      (slots [slot, slot + len)) or column 6 (slot) of the table.
 * One thread per read (K10p: per sorted entry, K10u: per drop row); R1 is only read, so no atomics but K10u's. */
int kdl_mates_pair(const kdl_batch* batch, const uint64_t* name_hash, const int32_t* mate_start,
                   const uint8_t* pair_role, const int32_t* order, int64_t n_order, int32_t* mate, void* stream);
int64_t kdl_overlap_scratch_words(int64_t n_reads);
int kdl_overlap_count(const kdl_batch* batch, const kdl_qmask* qmask, const int32_t* mate, uint32_t* scratch,
                      void* stream);
int kdl_overlap_apply(const kdl_batch* batch, const kdl_qmask* qmask, const int32_t* mate, const uint32_t* scratch,
                      uint32_t* seq4, const kdl_qmask* out_mask, int32_t* drops, int64_t n_drops, void* stream);
int kdl_overlap_untake(const int32_t* drops, int64_t n_drops, int32_t* counts, int64_t n_slots, void* stream);

/* K11 (extension: `variants --vcf --qual`): the base qualities of the counted bases, summed per slot.  The counted
 * bases are exactly those the pileup counts in columns 0-3: M/=/X bases whose nibble in seq4 is A, C, G or T (so a base
 * masked by quality, primer or mate overlap -- an N nibble -- counts nowhere; clipped and inserted bases, N and
 * deletions add nothing), along K1g's walk for KDL_HARD reads (Python index wrap included).
 *   qual8[8 * seq4_words]  uint8, 8-byte aligned: the Phred quality of base k of read r at byte 8 * seq_off[r] + k
 *                          (kdl_bam_fill_qual); a tile's qualities are the bytes [8 * wa, 8 * wend) of its words
 *   qsum[4][n_slots]       uint32, 16-byte aligned: the summed Phred of the counted A / C / G / T bases of each slot
 *   emass[n_slots]         uint64, 16-byte aligned: the summed EPS[min(q, 93)] of each slot's counted bases, EPS[q] the
 *                          integer nearest to 2^32 * 10^(-q / 10)
 * Both tables are written whole (no zeroing needed); the sums are integers, so the result is independent of order.
 * With constant qualities q, qsum[k][s] == q * counts[k][s].  A coordinate-sorted batch with tile_index takes K0 (into
 * tile_index, so no ordering dependency on kdl_pileup) + K11 (one CTA per tile, plain stores) + K11g (KDL_HARD reads,
 * global atomics); any other batch a zeroing pass + K11g over every read.  Reads the batch's seq4 as it is: after K9 /
 * K10 when they run.  n_slots % 4 == 0.  Device pointers. */
int kdl_quality_pileup(const kdl_batch* batch, const uint8_t* qual8, uint32_t* qsum, uint64_t* emass, int64_t n_slots,
                       void* stream);

/* K11w (extension: `consensus --quality-vote`): the counted bases of kdl_quality_pileup, each weighted by its quality.
 *   wsum[4][n_slots]  uint64, 16-byte aligned: for k = A, C, G, T the summed W[min(q, 93)] of the slot's counted bases
 *                     of allele k, W[q] the integer nearest to 2^16 * 10 log10(3 (1 - e_q) / e_q) with
 *                     e_q = min(10^(-q / 10), 3/4): the log-likelihood ratio, in 1/65536 Phred, of "the true base is the
 *                     one read" against "it is one particular other base" (W[0] = W[1] = 0, W[20] = 1620546,
 *                     W[93] = 6407534; kindel_b200/quality.py holds the table)
 * The same branches as kdl_quality_pileup (K0 + K11w + K11g-w, or a zeroing pass + K11g-w); the table is written whole
 * and, as integer sums, does not depend on order.  With constant qualities q, wsum[k][s] == W[q] * counts[k][s].
 * n_slots % 4 == 0.  Device pointers. */
int kdl_quality_weights(const kdl_batch* batch, const uint8_t* qual8, uint64_t* wsum, int64_t n_slots, void* stream);

/* K2w (extension: `consensus --quality-vote`): the vote of kdl_vote with the base chosen by base-quality weights.  The
 * D, N and I decisions, their order and so the change bits of every call byte are kdl_vote's; where a base is emitted it
 * is b* = the base with the largest wsum[b][s] (kdl_quality_weights), and N (code 4) when that sum is 0 or two bases
 * share it.  The N column does not vote.  Bit 7 is never set.  qual (may be NULL): qual[s] = min(60, (wsum[b*][s] -
 * max over b != b* of wsum[b][s]) >> 16), and 0 for every call that emits N or nothing.  n_slots % 4 == 0. */
int kdl_vote_quality(const int32_t* counts, const uint64_t* wsum, int64_t n_slots, int64_t min_depth_ceil,
                     uint8_t* calls, uint8_t* qual, void* stream);

/* K12 / K12d (extension: `kindel amplicons --primers scheme.bed`): each read's amplicon, and the depth of each
 * amplicon's insert.  The amplicons are the scheme's on the batch's contigs, numbered 0 .. n_amplicons - 1; per contig c
 * and side (LEFT / RIGHT primers) the host gives the sorted breakpoints of that side's primer intervals,
 * [left_off[c], left_off[c + 1]) of left_at, and per breakpoint k the label of the segment [at[k], at[k + 1]): the
 * amplicon whose primers (alternates included) alone cover it, -3 where primers of several amplicons cover it, -1 where
 * none does (the last breakpoint of a contig is -1).  Device pointers, int32 coordinates.
 *   kdl_amplicons_assign  K12.  label[n_reads] int32: with s and e the walk cursors of the read's first and last M/=/X
 *                         base as K9 takes them (before the Python index wrap), l = the label of s among its contig's
 *                         LEFT segments and r = that of e among its RIGHT segments (-1 for a cursor outside [0, L) and
 *                         for both when the read has no M/=/X base): -1 (unprimed) when both are -1; -3 (ambiguous)
 *                         when either is -3; -2 (mispaired) when they are two different amplicons; else the amplicon
 *                         one or both name.  One thread per read.
 *   kdl_amplicons_depth   K12d.  With D(p) = A + C + G + T of `counts` (columns 0-3) at slot contig_slot[amp_contig[j]]
 *                         + p: stats[3 j] = the sum of D over amplicon j's insert [insert_start[j], insert_end[j]),
 *                         stats[3 j + 1] = its minimum and stats[3 j + 2] = the number of its positions with
 *                         D >= min_depth; all three 0 for an insert that does not lie in 0 <= start < end <= L.  One
 *                         warp per amplicon. */
typedef struct kdl_amplicons {
    int32_t n_contigs;
    int32_t n_amplicons;
    const int64_t* left_off;   /* [n_contigs + 1] */
    const int32_t* left_at;
    const int32_t* left_label;
    const int64_t* right_off;  /* [n_contigs + 1] */
    const int32_t* right_at;
    const int32_t* right_label;
    const int32_t* amp_contig;   /* [n_amplicons] */
    const int32_t* insert_start; /* [n_amplicons] */
    const int32_t* insert_end;   /* [n_amplicons] */
} kdl_amplicons;

int kdl_amplicons_assign(const kdl_batch* batch, const kdl_amplicons* amplicons, int32_t* label, void* stream);
int kdl_amplicons_depth(const int32_t* counts, int64_t n_slots, const int64_t* contig_slot, const int32_t* contig_len,
                        int32_t n_contigs, const kdl_amplicons* amplicons, int64_t min_depth, int64_t* stats,
                        void* stream);

/* K13 (extension: `--normalise N` with a named `--primers` scheme): the reads of each (amplicon, strand) group that
 * the cap keeps, in batch order.  Per read r: key = 2 label[r] + (reverse[r] != 0) when 0 <= label[r] < n_amplicons
 * (label: K12's), else none.  rank(r) = the reads before r in the batch with r's key.  keep[r] = 1 when r has no key
 * or rank(r) < cap, else 0; total[key] = the reads of each key (K = 2 n_amplicons entries); *dropped = the sum over
 * the keys of max(total - cap, 0) (int64).  cap >= 1.  Device pointers; `scratch` is int32 [scratch_words] with
 * scratch_words >= kdl_normalise_scratch_words(n_reads, n_amplicons) on the same device.
 *   K13c  G CTAs, CTA j over a contiguous run of the batch: its keys counted into row j of H[G][K] (scratch).
 *   K13s  one thread per key: H[.][key] replaced by its exclusive prefix over j, the total and the dropped reads.
 *   K13m  CTA j again, tile by tile in batch order: rank = H[j][key] + earlier warps' reads of the key in the tile +
 *         the read's rank among its warp's peers; keep.
 * G = min(2 SMs, tiles of 256 reads, KDL_NORMALISE_MAX_WORDS / K), at least 1: H takes at most
 * KDL_NORMALISE_MAX_WORDS int32 (64 MB) unless K alone exceeds it.  The result does not depend on G. */
#define KDL_NORMALISE_MAX_WORDS (1ll << 24)

int64_t kdl_normalise_scratch_words(int64_t n_reads, int32_t n_amplicons);
int kdl_normalise(const int32_t* label, const uint8_t* reverse, int64_t n_reads, int32_t n_amplicons, int64_t cap,
                  int32_t* scratch, int64_t scratch_words, uint8_t* keep, int32_t* total, int64_t* dropped,
                  void* stream);

/* K14 (extension: `--dedup`): duplicate reads and read pairs removed before the pileup, as samtools markdup -r and
 * Picard MarkDuplicates remove them.  Over the batch's reads (after min_mapq / exclude_flags; a 0x400 in the file is
 * ignored):
 *   Left alone: dup_score[r] < 0 (the decode gives -1 where FLAG & 0x900), or no M/D/N/=/X op.  Never removed, never
 *   anyone's duplicate.
 *   End: (contig, u, strand), strand = reverse[r] (FLAG & 0x10), u the unclipped 5' position in SAM arithmetic:
 *   forward u = POS0 - the S and H ops before the first M/D/N/=/X op; reverse u = POS0 + the M/D/N/=/X lengths - 1 +
 *   the S and H ops after the last one.  Encoded e = 2 u + strand (int64), so (u, strand) order is e order.
 *   Score: dup_score[r], the sum of the read's Phred qualities >= 15 over all of SEQ (0 without qualities).
 *   Pair: an R2 (mate[r] >= 0, K10p's) and its R1, neither left alone.  Single: any other read not left alone (a
 *   pair's mate whose partner is left alone included).
 *   Pairs: key (contig, E1, E2), E1 <= E2 the mates' ends; of each key the pair with the largest score R1 + R2 (int64)
 *   stays, ties to the smallest min(R1, R2); the others are removed, both mates.
 *   Singles: removed when a pair (kept or removed) has a mate end equal to theirs; otherwise of each end the single
 *   with the largest score stays, ties to the smallest index.
 * keep[r] = 0 for a removed read, else 1.
 *   kdl_dedup_entries  K14k (three launches, one thread per read): keep = 1, end[], paired[], then the two entry
 *                      lists, compacted in any order.  Pair list: pair_contig / pair_e1 (E1) / pair_e2 (E2) /
 *                      pair_rank / pair_r1 / pair_r2, capacity n_reads / 2.  Single list: single_contig, single_key =
 *                      2 e + 0 for a pair mate's end (two markers per pair) or 2 e + 1 for a single's, single_rank,
 *                      single_read (-1 for a marker), capacity n_reads.  rank = (0xffffffff - score) << 32 | index
 *                      (pair: the summed score, the smaller mate index): the best entry has the smallest rank.  end
 *                      int64 [n_reads] and paired uint8 [n_reads] are scratch.  mate may be NULL (no pairs).  Zeroes
 *                      the totals record (KDL_DEDUP_TOTALS int64) and writes [0] pair entries, [1] single-list
 *                      entries: one read-back sizes the sort.
 *   kdl_dedup_select   K14s (four launches per list, one thread per sorted entry, no thread walking a run): over the
 *                      lists sorted by key -- pair_order[n_pairs] by (contig, E1, E2), single_order[n_singles] by
 *                      (contig, single_key), the entry indices in key order -- each run's best candidate stays and
 *                      the others get keep 0.  Adds [2] pairs removed, [3] singles removed, [4] of those singles the
 *                      ones a pair end shadowed.  scratch: int32 [kdl_dedup_scratch_words(max(n_pairs, n_singles))],
 *                      8-byte aligned.  On the stream after kdl_dedup_entries.
 * Device pointers. */
#define KDL_DEDUP_TOTALS 8
#define KDL_DEDUP_ALONE ((int64_t)(-0x7fffffffffffffffll - 1))  /* end[r] of a read left alone */

typedef struct kdl_dedup_lists {
    int32_t* pair_contig;
    int64_t* pair_e1;
    int64_t* pair_e2;
    uint64_t* pair_rank;
    int32_t* pair_r1;
    int32_t* pair_r2;
    int32_t* single_contig;
    int64_t* single_key;
    uint64_t* single_rank;
    int32_t* single_read;
    int64_t* end;     /* [n_reads] scratch */
    uint8_t* paired;  /* [n_reads] scratch */
} kdl_dedup_lists;

int kdl_dedup_entries(const kdl_batch* batch, const uint8_t* reverse, const int32_t* dup_score, const int32_t* mate,
                      const kdl_dedup_lists* lists, uint8_t* keep, int64_t* totals, void* stream);
int64_t kdl_dedup_scratch_words(int64_t n_entries);
int kdl_dedup_select(const kdl_dedup_lists* lists, const int64_t* pair_order, int64_t n_pairs,
                     const int64_t* single_order, int64_t n_singles, int32_t* scratch, int64_t scratch_words,
                     uint8_t* keep, int64_t* totals, void* stream);

/* Fused cross-GPU count reduction + vote (SURVEY.md 8e): sums the 7 vote columns of `n_peers`
 * tables that live on this and on peer GPUs (peer pointers mapped with CUDA IPC / P2P), votes on
 * slots [slot_lo, slot_hi) and writes calls for that range; optionally stores the reduced
 * columns into reduced[7][n_slots] (may be NULL). */
int kdl_vote_peers(const int32_t* const* peer_counts, int32_t n_peers, int64_t n_slots,
                   int64_t slot_lo, int64_t slot_hi, int64_t min_depth_ceil, uint8_t* calls,
                   int32_t* reduced, void* stream);
/* Same, with each table's footprint: peer p only holds non-zero counts in slots
 * [foot_lo[p], foot_hi[p]) (host int64 arrays, multiples of 4), so a read-sharded, coordinate-sorted
 * job pulls only the halo of its neighbours over NVLink instead of every table. */
int kdl_vote_peers_sparse(const int32_t* const* peer_counts, const int64_t* foot_lo, const int64_t* foot_hi,
                          int32_t n_peers, int64_t n_slots, int64_t slot_lo, int64_t slot_hi,
                          int64_t min_depth_ceil, uint8_t* calls, int32_t* reduced, void* stream);

/* ---- fully fused exchange (no NCCL on the data path) ------------------------------------------
 * Every rank owns one IPC block: [count table 19 x n_slots int32][calls n_slots bytes][flags].
 * Per step (epoch e = 1, 2, ...), on every rank, in stream order:
 *   kdl_pileup(...)                       its shard into its own table
 *   kdl_exchange_signal(x, e)             optional early "my table is complete" -> ready[p][rank] = e in
 *                                         every peer p (kdl_exchange_vote publishes it too, first thing)
 *   kdl_exchange_vote(x, ..., e)          K2x: waits for ready[rank][*] >= e, sums the 7 vote columns
 *                                         of its slot slice [slice_lo[rank], slice_hi[rank]) over the
 *                                         (footprint-clipped) peer tables through NVLink, votes,
 *                                         stores the call bytes of the slice locally; the last CTA
 *                                         out publishes done[p][rank] = e to every peer p
 *   kdl_exchange_wait(x, e)               K2g: per peer p, waits for done[rank][p] >= e and pulls p's
 *                                         call slice over NVLink into the local call buffer; when it
 *                                         ends every slice is here and nobody still reads this
 *                                         rank's table
 * All pointers of rank p (tables[p], calls[p], ready[p], done[p]) are this process's mappings of
 * rank p's block (own block: the local pointer). */
typedef struct kdl_exchange {
    int32_t n_ranks, rank;
    const int32_t* tables[16];
    uint8_t* calls[16];
    int32_t* ready[16]; /* int32[16] per rank */
    int32_t* done[16];  /* int32[16] per rank */
    int64_t foot_lo[16], foot_hi[16];   /* table p is zero outside [foot_lo[p], foot_hi[p]) */
    int64_t slice_lo[16], slice_hi[16]; /* slots rank p votes on (multiples of 4, a partition) */
    int32_t* counter;   /* local device int32, zero-initialised */
} kdl_exchange;

int kdl_exchange_signal(const kdl_exchange* x, int32_t epoch, void* stream);
int kdl_exchange_vote(const kdl_exchange* x, int64_t n_slots, int64_t min_depth_ceil, int32_t epoch,
                      void* stream);
/* K2x with the IUPAC vote of kdl_vote_iupac (same threshold rule, same call bytes as one table). */
int kdl_exchange_vote_iupac(const kdl_exchange* x, int64_t n_slots, int64_t min_depth_ceil, double threshold,
                            int32_t epoch, void* stream);
int kdl_exchange_wait(const kdl_exchange* x, int32_t epoch, void* stream);

/* Count tables that peer GPUs (other processes of the same node) can map: plain cudaMalloc
 * memory exported / opened with CUDA IPC.  kdl_table_alloc zero-fills. */
int kdl_table_alloc(int64_t bytes, void** dev_ptr);
int kdl_table_free(void* dev_ptr);
int kdl_ipc_export(void* dev_ptr, uint8_t handle[64]);
int kdl_ipc_open(const uint8_t handle[64], void** dev_ptr);
int kdl_ipc_close(void* dev_ptr);

/* ---- host-buffer path (what a cgo/JNI/ctypes caller without its own CUDA runtime uses) ---- */
typedef struct kdl_ctx kdl_ctx;

int kdl_ctx_create(int device, kdl_ctx** out);
void kdl_ctx_destroy(kdl_ctx* ctx);

/* batch holds HOST pointers.  batch->seq_off may be NULL: the packed bases are then taken to be DENSE (read i
 * starts at the sum of ceil(l_seq[j] / 8) words over j < i, as every flattener here lays them out) and the
 * offsets are computed on the device instead of being copied (4 bytes per read less over PCIe).
 * Outputs (host, caller-allocated, any may be NULL to skip):
 *   calls_out[n_slots] uint8, counts_out[KDL_NCOL][n_slots] int32,
 *   ins_events_out[n_events][4] int32.  diag_out is always filled.
 * Returns KDL_OK, or KDL_ERR_INDEX / KDL_ERR_KEY with diag_out describing the first offender. */
int kdl_ctx_consensus(kdl_ctx* ctx, const kdl_batch* batch, int64_t n_slots, int64_t n_events,
                      int64_t min_depth_ceil, uint8_t* calls_out, int32_t* counts_out,
                      int32_t* ins_events_out, kdl_diag* diag_out);

/* kdl_ctx_consensus of a batch with masked bases: the same contract, plus the batch's mask list (HOST pointers),
 * uploaded with the rest; K1q runs between the pileup and the vote. */
int kdl_ctx_consensus_masked(kdl_ctx* ctx, const kdl_batch* batch, const kdl_qmask* qmask, int64_t n_slots,
                             int64_t n_events, int64_t min_depth_ceil, uint8_t* calls_out, int32_t* counts_out,
                             int32_t* ins_events_out, kdl_diag* diag_out);

/* device time (ms) of the last kdl_ctx_consensus call, H2D / kernels / D2H, from CUDA events */
int kdl_ctx_last_timing(kdl_ctx* ctx, float* h2d_ms, float* kernel_ms, float* d2h_ms);

/* ---- host-side BAM decode (no GPU involved; kindel_b200/csrc/bam_host.cpp) ----
 * Replaces the simplesam -> `samtools view` text round trip of kindel/kindel.py:136-145 for .bam input: BGZF blocks
 * inflated by zlib in C++ threads, records filtered (kindel.py:43-46), classified and written straight into the
 * layout above -- into caller-owned buffers, which may be pinned memory.
 *   kdl_bam_open     read + inflate + parse the header (text, reference dictionary).  Takes BGZF / gzip / plain BAM
 *                    and SAM text (plain or gzip): text lines are turned into BAM records in threads by a strict
 *                    parser that gives up (error) on anything unusual -- the caller then uses its own text reader
 *   kdl_bam_prepare  ref_len[n_ref] = contig lengths to classify against (the @SQ LN values the reference uses;
 *                    NULL = the binary dictionary's).  info[16] out: 0 records, 1 kept reads, 2 contigs seen,
 *                    3 CIGAR ops of kept reads, 4 words of seq4, 5 complex reads, 6 hard reads, 7 aligned bases,
 *                    9 reach_right, 10 reach_left, 11 longest simple read
 *   kdl_bam_contigs  order[n_seen] = reference ids in first-seen order (kindel.py:143-151), read_off[n_seen + 1]
 *   kdl_bam_fill     ref_start / seq_off / l_seq / seq_len [kept], cig_off [kept + 1], cigar [ops] (may be NULL),
 *                    seq4 [words], complex_idx [complex], hard_idx [hard] (may be NULL); contig_slot[n_seen] = the slot
 *                    layout; fills info[8] = insertion events, info[12] = reads_sorted
 * Extension, all off by default:
 *   kdl_bam_set_filter  before prepare: a record with MAPQ < min_mapq or FLAG & exclude_flags is treated as unmapped;
 *                    a base with Phred quality < min_base_quality (record with qualities only) is masked -- N in seq4,
 *                    before classification.  Refused (KDL_ERR_INVALID_ARG) for SAM text whose MAPQ / QUAL fields the
 *                    text parser could not carry when the filter would read them.  prepare's info[13] = masked bases,
 *                    info[14] = reads with masked bases
 *   kdl_bam_fill_mask   after fill: the kdl_qmask arrays, read_idx [info[14]], off [info[14] + 1], qpos [info[13]]
 *   kdl_bam_fill_strand after fill (extension): reverse [n_kept], 1 where the kept read's FLAG has 0x10, in read order
 *   kdl_bam_fill_mates  after fill (extension): name_hash / mate_start / pair_role [n_kept] of K10, in read order
 *   kdl_bam_fill_qual   after fill (extension): qual8 [8 * words of seq4], the Phred quality of base k of read r at byte
 *                    8 * seq_off[r] + k, 0xff for a complex read's trailer words and the padding.  prepare's info[15] =
 *                    kept reads without qualities (BAM 0xff, SAM `*`): their bytes are 0xff too
 *   kdl_bam_fill_dup    after fill (extension, K14): dup_score [n_kept] int32 in read order, -1 where FLAG & 0x900, else
 *                    the sum of the read's Phred qualities >= 15 over all of SEQ (0 without qualities), saturating at
 *                    2^31 - 1 */
typedef struct kdl_bam kdl_bam;
int kdl_bam_open(const char* path, int threads, kdl_bam** out);
void kdl_bam_close(kdl_bam* h);
const char* kdl_bam_header_text(const kdl_bam* h, int64_t* len);
int32_t kdl_bam_n_ref(const kdl_bam* h);
const char* kdl_bam_ref_name(const kdl_bam* h, int32_t ref_id);
int32_t kdl_bam_ref_len(const kdl_bam* h, int32_t ref_id);
int kdl_bam_prepare(kdl_bam* h, const int32_t* ref_len, int threads, int64_t* info);
int kdl_bam_contigs(const kdl_bam* h, int32_t* order, int64_t* read_off);
int kdl_bam_fill(kdl_bam* h, int threads, const int64_t* contig_slot, int32_t* ref_start, uint32_t* seq_off,
                 int32_t* l_seq, int32_t* seq_len, uint32_t* cig_off, uint32_t* cigar, uint32_t* seq4,
                 uint32_t* complex_idx, uint32_t* hard_idx, int64_t* info);
int kdl_bam_set_filter(kdl_bam* h, int32_t min_mapq, int32_t exclude_flags, int32_t min_base_quality);
int kdl_bam_fill_mask(kdl_bam* h, int threads, uint32_t* read_idx, uint32_t* off, uint32_t* qpos);
int kdl_bam_fill_strand(kdl_bam* h, int threads, uint8_t* reverse);
int kdl_bam_fill_mates(kdl_bam* h, int threads, uint64_t* name_hash, int32_t* mate_start, uint8_t* pair_role);
int kdl_bam_fill_qual(kdl_bam* h, int threads, uint8_t* qual8);
int kdl_bam_fill_dup(kdl_bam* h, int threads, int32_t* dup_score);

#ifdef __cplusplus
}
#endif
#endif /* KINDEL_B200_H */
