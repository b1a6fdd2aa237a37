"""Host-side decode of BAM / SAM into the engine's flattened read layout (stays on the host).

Replaces the record materialisation of the reference's `parse_bam`
(reference kindel/kindel.py:131-153: `simplesam.Reader` -> `samtools view` text -> one Python
object per record) with:

  .bam : BGZF blocks inflated with zlib in a thread pool, then one C++ pass over the byte stream
         (`kdl_bam_count` / `kdl_bam_fill`, kindel_b200/csrc/bam_host.cpp) that copies each kept
         record's CIGAR words and packed bases straight into the device layout.
  .sam : text parse in Python (SAM input is small in practice; the reference's test-suite uses it
         for three ONT fixtures).

Semantics kept from the reference:
  * records are bucketed by RNAME in first-seen order over ALL records (kindel.py:143-145), `*`
    is dropped (kindel.py:147-148); a contig whose records are all filtered still appears, with
    empty tables;
  * a record contributes only if `mapped and len(seq) > 1` (kindel.py:43-46): FLAG & 0x4 clear and
    SEQ longer than one base (SEQ `*` has length 1).  Secondary / supplementary / duplicate
    records count (SURVEY.md A-11);
  * contig lengths come from the @SQ header lines (kindel.py:138-141).

Extension (the reference has no such options), all off by default: `min_mapq`, `exclude_flags` and
`min_base_quality`.  A record with MAPQ < min_mapq or FLAG & exclude_flags is treated exactly like an unmapped one
(it still counts for the first-seen order of contigs).  A base with Phred quality < min_base_quality is MASKED: its
nibble becomes N (15) in `seq4` before the reads are classified, and its query offset goes into the batch's mask list
(`mask_read` / `mask_off` / `mask_qpos`), from which K1q (csrc/pileup_mask.cu) takes back the count the N added to a
base column.  A record without qualities (SAM `*`, BAM 0xff) is never masked; with min_base_quality == 0 QUAL is not
read at all.
With `strand=True` the batch also keeps each kept read's strand (`reverse`, FLAG & 0x10), which `variants --vcf
--strand` splits the pileup by; it costs nothing when off.  With `mates=True` it keeps what `--mask-overlaps` pairs the
reads by (`name_hash`, `mate_start`, `pair_role`: include/kindel_b200.h K10 has the rule); nothing is decoded when off.
With `qual=True` it keeps every base's quality beside its bases (`qual8`, which K11 sums for `variants --vcf --qual`);
a kept read without qualities is then a ValueError naming the file: nothing is guessed.

The result is a `ReadBatch` (numpy arrays in host memory) described in include/kindel_b200.h.
"""
from __future__ import annotations

import gzip
import os
import struct
import zlib
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np

from . import _ffi

CIGAR_OPS = "MIDNSHP=X"
NIBBLES = "=ACMGRSVTWYHKDBN"
SLOT_ALIGN = _ffi.KDL_TILE  # table slots are padded to whole tiles of the owner-computes pileup

_OP_CODE = {c: i for i, c in enumerate(CIGAR_OPS)}
_ENC = np.full(256, 255, dtype=np.uint8)
for _i, _c in enumerate(NIBBLES):
    _ENC[ord(_c)] = _i
    _ENC[ord(_c.lower())] = _i


@dataclass
class ReadBatch:
    """Flattened reads of one alignment file (host memory).  Field meanings: include/kindel_b200.h.
    Host-only companions of the device layout: `seq_len` (plain SEQ lengths), `cig_off` / `cigar` (the CIGARs of
    ALL reads: what the CPU checker, the sharder and the insertion-string builder read) and `complex_idx`."""

    contig_names: list
    contig_len: np.ndarray        # int32 [nc]
    contig_read_off: np.ndarray   # int64 [nc+1]
    contig_slot: np.ndarray       # int64 [nc]
    n_slots: int
    ref_start: np.ndarray         # int32 [n]
    seq_off: np.ndarray           # uint32 [n]  (4-byte words) start of the read's block in seq4
    l_seq: np.ndarray             # int32 [n]   device word: length | op-count field | KDL_COMPLEX | KDL_HARD
    seq_len: np.ndarray           # int32 [n]   plain SEQ length (host only)
    cig_off: np.ndarray           # uint32 [n+1]  (host only)
    cigar: np.ndarray             # uint32 [n_ops] (host only)
    seq4: np.ndarray              # uint32 [words]: per read its bases, complex reads followed by [n_ops][evt_off][ops]
    hard_idx: np.ndarray = field(default=None)      # uint32 [n_hard]: KDL_HARD reads (K1g walks them)
    complex_idx: np.ndarray = field(default=None)   # uint32 [n_complex]: all complex reads (K1e walks the tile-eligible ones)
    n_events: int = 0
    reads_sorted: bool = False
    aligned_bases: int = 0        # sum of M/=/X lengths = sum of the weights table (the metric's unit)
    n_records: int = 0            # records in the file, before filtering
    max_simple_len: int = 0       # longest simple read
    reach_right: int = 0          # see include/kindel_b200.h
    reach_left: int = 0
    # masked bases (min_base_quality; include/kindel_b200.h kdl_qmask).  None = no masked base.
    mask_read: np.ndarray = field(default=None)     # uint32 [m]: ascending indices of the reads with masked bases
    mask_off: np.ndarray = field(default=None)      # uint32 [m+1]: their entries in mask_qpos
    mask_qpos: np.ndarray = field(default=None)     # uint32 [n_masked]: query offsets, ascending per read
    # strand (extension; `strand=True` at decode): 1 where the read's FLAG has 0x10.  None = not asked for.
    reverse: np.ndarray = field(default=None)       # uint8 [n]
    # mates (extension; `mates=True` at decode, K10): FNV-1a of QNAME, PNEXT - 1, 1 / 2 = first / last mate of a pair
    # on one contig (0 otherwise).  None = not asked for.
    name_hash: np.ndarray = field(default=None)     # uint64 [n]
    mate_start: np.ndarray = field(default=None)    # int32 [n]
    pair_role: np.ndarray = field(default=None)     # uint8 [n]
    # base qualities (extension; `qual=True` at decode, K11): base k of read r at byte 8 * seq_off[r] + k, 0xff for the
    # padding and a complex read's trailer words.  None = not asked for; select_reads and the shards leave it behind.
    qual8: np.ndarray = field(default=None)         # uint8 [8 * words of seq4]

    @property
    def mates(self):
        """(name_hash, mate_start, pair_role), or None when the batch was decoded without them."""
        return None if self.pair_role is None else (self.name_hash, self.mate_start, self.pair_role)

    @property
    def n_reads(self) -> int:
        return int(self.ref_start.shape[0])

    @property
    def n_contigs(self) -> int:
        return len(self.contig_names)

    @property
    def n_complex(self) -> int:
        return int(self.complex_idx.shape[0])

    @property
    def n_hard(self) -> int:
        return int(self.hard_idx.shape[0])

    @property
    def n_masked(self) -> int:
        return 0 if self.mask_qpos is None else int(self.mask_qpos.shape[0])

    @property
    def n_mask_reads(self) -> int:
        return 0 if self.mask_read is None else int(self.mask_read.shape[0])

    def mask_counts(self) -> np.ndarray:
        """Masked bases per read (int64 [n_reads])."""
        out = np.zeros(self.n_reads, dtype=np.int64)
        if self.n_mask_reads:
            out[self.mask_read.astype(np.int64)] = np.diff(self.mask_off.astype(np.int64))
        return out

    def mask_bytes(self) -> int:
        """Bytes of the mask list (what K1q reads on top of the batch)."""
        arrs = (self.mask_read, self.mask_off, self.mask_qpos)
        return int(sum(a.nbytes for a in arrs if a is not None)) if self.n_masked else 0

    def input_bytes(self) -> int:
        """Bytes of read data the device consumes (what the e2e path copies host->device)."""
        arrs = (self.ref_start, self.seq_off, self.l_seq, self.seq4, self.complex_idx, self.hard_idx, self.contig_len,
                self.contig_read_off, self.contig_slot)
        return int(sum(a.nbytes for a in arrs if a is not None)) + self.mask_bytes()


def seq_lengths(l_seq: np.ndarray) -> np.ndarray:
    """SEQ length (int64) of every read from the device word l_seq (include/kindel_b200.h)."""
    w = np.asarray(l_seq).astype(np.int64) & 0xFFFFFFFF
    cx = (w & _ffi.KDL_COMPLEX) != 0
    hard = (w & _ffi.KDL_HARD) != 0
    return np.where(cx, np.where(hard, w & 0x3FFFFFFF, w & _ffi.KDL_LEN_MASK), w)


def _reads_with_exotic_bases(seq4: np.ndarray, seq_off: np.ndarray, lseq: np.ndarray) -> np.ndarray:
    """True for reads holding a base outside A,C,G,T,N (nibbles 1,2,4,8,15) inside their SEQ.
    Such reads take the general kernel, which reproduces the reference's KeyError semantics; the
    fast kernel relies on simple reads being clean (include/kindel_b200.h).  Vectorised: per word,
    nibbles with popcount 2 or 3 are exotic; zero nibbles ('=') are exotic unless they are the
    padding behind the last base of a read."""
    n = seq_off.shape[0]
    out = np.zeros(n, dtype=bool)
    if n == 0 or seq4.size == 0:
        return out
    w = seq4.astype(np.uint32)
    h = w | (w >> 1)
    pair = w & (w >> 1)
    two_plus = (pair | (pair >> 2) | (h & (h >> 2))) & 0x11111111
    all4 = pair & (pair >> 2) & 0x11111111
    zero = ~(h | (h >> 2)) & 0x11111111
    starts = seq_off.astype(np.int64)
    lens = np.maximum(lseq.astype(np.int64), 0)
    has = lens > 0
    last = starts + (lens + 7) // 8 - 1
    pad_nibbles = ((lens + 7) // 8) * 8 - lens                       # 0..7 zero nibbles behind the last base
    pad_mask = ((np.uint64(1) << (4 * pad_nibbles).astype(np.uint64)) - np.uint64(1)).astype(np.uint32)
    zero_ok = np.zeros_like(zero)
    zero_ok[last[has]] = pad_mask[has]
    flagged = np.flatnonzero(((two_plus & ~all4) | (zero & ~zero_ok)) != 0)
    if flagged.size:
        owner = np.searchsorted(starts, flagged, side="right") - 1
        ok = (owner >= 0) & (flagged <= last[np.maximum(owner, 0)])   # ignore words that belong to no read
        out[np.unique(owner[ok])] = True
    return out


def layout_slots(contig_len: np.ndarray):
    """Every contig owns ref_len + 1 consecutive slots (kindel.py:36-39 sizes); total padded."""
    lens = np.asarray(contig_len, dtype=np.int64) + 1
    slot = np.zeros(len(lens), dtype=np.int64)
    if len(lens) > 1:
        slot[1:] = np.cumsum(lens[:-1])
    total = int(lens.sum()) if len(lens) else 0
    n_slots = max(SLOT_ALIGN, (total + SLOT_ALIGN - 1) // SLOT_ALIGN * SLOT_ALIGN)
    return slot, n_slots


def _per_read_sum(values: np.ndarray, cig_off: np.ndarray) -> np.ndarray:
    """Sum of `values` (one per CIGAR op) over each read's ops."""
    c = np.concatenate(([0], np.cumsum(values, dtype=np.int64)))
    return c[cig_off[1:]] - c[cig_off[:-1]]


def check_filters(min_mapq=0, exclude_flags=0, min_base_quality=0):
    """The three read / base filters as ints, validated (ValueError)."""
    vals = (int(min_mapq), int(exclude_flags), int(min_base_quality))
    if not 0 <= vals[0] <= 255:
        raise ValueError("min_mapq must lie in 0..255, got %r" % (min_mapq,))
    if not 0 <= vals[1] <= 0xFFFF:
        raise ValueError("exclude_flags must lie in 0..0xffff, got %r" % (exclude_flags,))
    if not 0 <= vals[2] <= 255:
        raise ValueError("min_base_quality must lie in 0..255, got %r" % (min_base_quality,))
    return vals


def low_quality_mask(qual: np.ndarray, lseq: np.ndarray, min_base_quality: int):
    """(masked bases per read int64 [n], their query offsets uint32 ascending per read) from the concatenated
    Phred qualities of all reads (exactly SEQ-length bytes per read; 0xff for a read without qualities)."""
    lseq = np.asarray(lseq, dtype=np.int64)
    qual = np.asarray(qual, dtype=np.uint8)
    if qual.shape[0] != int(lseq.sum()):
        raise ValueError("qualities must hold exactly one byte per base")
    pos = np.flatnonzero(qual < min_base_quality)
    starts = np.concatenate(([0], np.cumsum(lseq)))
    owner = np.searchsorted(starts, pos, side="right") - 1
    counts = np.bincount(owner, minlength=lseq.shape[0]).astype(np.int64)
    return counts, (pos - starts[owner]).astype(np.uint32)


def mask_bases(seq4: np.ndarray, seq_off: np.ndarray, counts: np.ndarray, qpos: np.ndarray) -> np.ndarray:
    """Copy of `seq4` with the listed bases (counts per read, query offsets) set to N (nibble 15)."""
    out = np.array(seq4, dtype=np.uint32, copy=True)
    if qpos.shape[0]:
        owner = np.repeat(np.arange(counts.shape[0], dtype=np.int64), counts)
        q = qpos.astype(np.int64)
        word = np.asarray(seq_off, dtype=np.int64)[owner] + (q >> 3)
        bits = (np.uint32(0xF) << (28 - 4 * (q & 7)).astype(np.uint32)).astype(np.uint32)
        np.bitwise_or.at(out, word, bits)
    return out


def finalize(contig_names, contig_len, contig_read_off, ref_start, seq_off, l_seq, cig_off, cigar, seq4,
             n_records=0, exotic=None, qual=None, min_base_quality=0, mask=None, reverse=None, mates=None) -> ReadBatch:
    """Classify reads (simple / tile-eligible complex / hard), lay the complex reads' CIGARs behind their bases,
    detect coordinate order.  All vectorised numpy; shared by the BAM, SAM and synthetic paths.

    In: per read its start, SEQ length, CIGAR (cig_off / cigar over ALL reads) and the offset of its packed
    bases in `seq4` (any layout: gaps and extra words between reads are allowed and dropped).
    qual + min_base_quality > 0: concatenated Phred qualities (one byte per base, 0xff = none); the bases below the
    threshold are masked (N in seq4, listed in the mask) BEFORE classification.  mask = (per-read counts, query
    offsets): a mask already applied to `seq4` (re-finalizing a masked batch), carried into the result.
    reverse: the reads' strand bytes (1 = FLAG & 0x10), carried into the result.  mates: (name_hash, mate_start,
    pair_role) of the reads, carried into the result."""
    contig_len = np.ascontiguousarray(contig_len, dtype=np.int32)
    contig_read_off = np.ascontiguousarray(contig_read_off, dtype=np.int64)
    ref_start = np.ascontiguousarray(ref_start, dtype=np.int32)
    seq_off_in = np.ascontiguousarray(seq_off).astype(np.int64)
    lseq = np.ascontiguousarray(l_seq).astype(np.int64)
    cig_off = np.ascontiguousarray(cig_off, dtype=np.uint32)
    cigar = np.ascontiguousarray(cigar, dtype=np.uint32)
    seq4 = np.ascontiguousarray(seq4, dtype=np.uint32)
    n = ref_start.shape[0]
    if lseq.size and (lseq.min() < 0 or lseq.max() >= (1 << 30)):
        raise ValueError("finalize() takes plain SEQ lengths below 2^30 (use ReadBatch.seq_len, not the device word l_seq)")
    if qual is not None and min_base_quality > 0:
        mask = low_quality_mask(qual, lseq, min_base_quality)
        if mask[1].shape[0]:
            seq4 = mask_bases(seq4, seq_off_in, *mask)
            exotic = None  # masked bases are N now
    slot, n_slots = layout_slots(contig_len)
    per_contig = np.diff(contig_read_off)
    read_L = np.repeat(contig_len.astype(np.int64), per_contig)
    co = cig_off.astype(np.int64)

    n_cig = np.diff(co)
    first = np.zeros(n, dtype=np.uint32)
    has = n_cig > 0
    first[has] = cigar[co[:-1][has]]
    op = first & 15
    oplen = (first >> 4).astype(np.int64)
    is_m = (op == 0) | (op == 7) | (op == 8)
    start = ref_start.astype(np.int64)
    simple = (n_cig == 1) & is_m & (oplen == lseq) & (start >= 0) & (start + oplen <= read_L)
    simple &= oplen <= _ffi.KDL_FAST_MAXLEN
    # reads with a base outside A,C,G,T,N (flagged by the C++ gather for BAM input, else found here)
    exo = (np.asarray(exotic, dtype=bool) if exotic is not None
           else _reads_with_exotic_bases(seq4, seq_off_in.astype(np.uint32), lseq))
    simple &= ~exo

    # ---- complex reads: which of them the tile kernel may walk (include/kindel_b200.h: "tile-eligible")
    ops_all = (cigar & 15).astype(np.int64)
    len_all = (cigar >> 4).astype(np.int64)
    is_match = (ops_all == 0) | (ops_all == 7) | (ops_all == 8)
    is_first = np.zeros(cigar.shape[0], dtype=bool)
    is_first[co[:-1][has]] = True
    later_clip = (ops_all == 4) & ~is_first
    q_span = _per_read_sum(len_all * (is_match | (ops_all == 1) | (ops_all == 4)), co)
    r_span = _per_read_sum(len_all * (is_match | (ops_all == 2) | later_clip), co)  # a non-first S advances r_pos too
    n_match = _per_read_sum(is_match.astype(np.int64), co)
    ins_per_read = _per_read_sum((ops_all == 1).astype(np.int64), co)
    lead = np.where(has & (op == 4), oplen, 0)
    tile_ok = (~simple & ~exo & (n_cig <= _ffi.KDL_TILE_MAXOPS) & (lseq <= _ffi.KDL_FAST_MAXLEN) & (q_span <= lseq)
               & (start - lead - 1 >= 0) & (start + r_span <= read_L - 1)
               & (r_span + 1 <= _ffi.KDL_TILE_MAXREACH) & (lead + 1 <= _ffi.KDL_TILE_MAXREACH))
    hard = ~simple & ~tile_ok
    l_out = np.where(simple, oplen,
                     np.where(tile_ok, lseq | (n_match << _ffi.KDL_NM_SHIFT) | _ffi.KDL_COMPLEX,
                              lseq | _ffi.KDL_COMPLEX | _ffi.KDL_HARD)).astype(np.uint32).view(np.int32)
    complex_idx = np.flatnonzero(~simple).astype(np.uint32)
    hard_idx = np.flatnonzero(hard).astype(np.uint32)
    evt = np.concatenate(([0], np.cumsum(ins_per_read)))  # row of each read's first insertion event
    n_events = int(evt[-1])
    aligned = int((len_all * is_match).sum())
    reach_right = int(max(oplen[simple].max() if simple.any() else 0, (r_span[tile_ok] + 1).max() if tile_ok.any() else 0))
    reach_left = int((lead[tile_ok] + 1).max()) if tile_ok.any() else 0

    # ---- the read stream: bases of every read in read order, complex reads followed by [n_ops][evt_off][ops...]
    words = (lseq + 7) // 8
    extra = np.where(simple, 0, 2 + n_cig)
    new_off = np.concatenate(([0], np.cumsum(words + extra)))
    dense_in = bool(n == 0 or (seq_off_in[0] == 0 and np.array_equal(seq_off_in[1:], np.cumsum(words[:-1]))
                               and int(words.sum()) == seq4.shape[0]))
    if dense_in and not extra.any():
        stream = seq4  # already the device layout: no copy
    else:
        if new_off[-1] >= (1 << 32):
            raise ValueError("alignment too large for 32-bit word offsets; split it by contig")
        stream = np.zeros(int(new_off[-1]), dtype=np.uint32)
        total = int(words.sum())
        ramp = np.arange(total, dtype=np.int64) - np.repeat(np.cumsum(words) - words, words)
        stream[np.repeat(new_off[:-1], words) + ramp] = seq4[np.repeat(seq_off_in, words) + ramp]
        cx = np.flatnonzero(~simple)
        if cx.size:
            hdr = new_off[:-1][cx] + words[cx]
            stream[hdr] = n_cig[cx]
            stream[hdr + 1] = evt[:-1][cx]
            nc = n_cig[cx]
            tot = int(nc.sum())
            ramp2 = np.arange(tot, dtype=np.int64) - np.repeat(np.cumsum(nc) - nc, nc)
            stream[np.repeat(hdr + 2, nc) + ramp2] = cigar[np.repeat(co[:-1][cx], nc) + ramp2]
    seq_off_out = new_off[:-1].astype(np.uint32)

    # coordinate order: the global start slot (contig_slot + ref_start) must be non-decreasing over
    # ALL reads (the blocks of seq4 are in read order by construction: the tile-owner kernel stages
    # the reads of a tile as one contiguous index range and one contiguous byte range)
    sorted_ok = True
    if n > 1:
        gstart = np.repeat(slot, per_contig) + start
        sorted_ok = bool((np.diff(gstart) >= 0).all())

    mask_read = mask_off = mask_qpos = None
    if mask is not None and np.asarray(mask[1]).shape[0]:
        mcount = np.asarray(mask[0], dtype=np.int64)
        mask_read = np.flatnonzero(mcount).astype(np.uint32)
        mask_off = np.concatenate(([0], np.cumsum(mcount[mask_read]))).astype(np.uint32)
        mask_qpos = np.ascontiguousarray(mask[1], dtype=np.uint32)

    return ReadBatch(
        contig_names=list(contig_names), contig_len=contig_len, contig_read_off=contig_read_off,
        contig_slot=slot, n_slots=n_slots, ref_start=ref_start, seq_off=seq_off_out, l_seq=l_out,
        seq_len=lseq.astype(np.int32), cig_off=cig_off, cigar=cigar, seq4=stream, hard_idx=hard_idx,
        complex_idx=complex_idx, n_events=n_events, reads_sorted=sorted_ok, aligned_bases=aligned,
        n_records=int(n_records), max_simple_len=int(oplen[simple].max()) if simple.any() else 0,
        reach_right=reach_right, reach_left=reach_left, mask_read=mask_read, mask_off=mask_off, mask_qpos=mask_qpos,
        reverse=None if reverse is None else np.ascontiguousarray(reverse, dtype=np.uint8),
        **_mate_fields(mates),
    )


def _mate_fields(mates) -> dict:
    if mates is None:
        return {}
    h, m, r = mates
    return dict(name_hash=np.ascontiguousarray(h, dtype=np.uint64), mate_start=np.ascontiguousarray(m, dtype=np.int32),
                pair_role=np.ascontiguousarray(r, dtype=np.uint8))


def _mates_at(batch: ReadBatch, idx):
    return None if batch.mates is None else tuple(a[idx] for a in batch.mates)


_FNV_OFFSET, _FNV_PRIME = 0xCBF29CE484222325, 0x100000001B3


def name_hash(qname) -> int:
    """64-bit FNV-1a of a QNAME's bytes (str or bytes), the hash K10 pairs mates by."""
    h = _FNV_OFFSET
    for c in qname.encode() if isinstance(qname, str) else bytes(qname):
        h = ((h ^ c) * _FNV_PRIME) & 0xFFFFFFFFFFFFFFFF
    return h


def pair_role(flag: int, same_contig: bool) -> int:
    """1 / 2 for the first / last mate of a pair whose mates sit on one contig, else 0 (include/kindel_b200.h K10)."""
    if not flag & 0x1 or flag & (0x8 | 0x100 | 0x800) or bool(flag & 0x40) == bool(flag & 0x80) or not same_contig:
        return 0
    return 1 if flag & 0x40 else 2


def _mask_of(batch: ReadBatch, idx: np.ndarray):
    """(per-read counts, query offsets) of the reads `idx` of `batch`, in that order; None when nothing is masked."""
    if not batch.n_masked:
        return None
    counts = batch.mask_counts()
    start = np.zeros(batch.n_reads, dtype=np.int64)
    start[batch.mask_read.astype(np.int64)] = batch.mask_off[:-1].astype(np.int64)
    return counts[idx], _ragged_gather(batch.mask_qpos, start[idx], counts[idx])


def with_mask(batch: ReadBatch, counts: np.ndarray, qpos: np.ndarray) -> ReadBatch:
    """`batch` with the listed bases (masked bases per read, their query offsets ascending per read) masked, as if
    they had been below min_base_quality at decode (re-classified: a read whose only exotic bases are masked may
    become simple)."""
    counts = np.asarray(counts, dtype=np.int64)
    qpos = np.asarray(qpos, dtype=np.uint32)
    seq4 = mask_bases(batch.seq4, batch.seq_off, counts, qpos)
    return finalize(batch.contig_names, batch.contig_len, batch.contig_read_off, batch.ref_start, batch.seq_off,
                    batch.seq_len, batch.cig_off, batch.cigar, seq4, n_records=batch.n_records, mask=(counts, qpos),
                    reverse=batch.reverse, mates=batch.mates)


def select_reads(batch: ReadBatch, idx) -> ReadBatch:
    """The sub-batch made of reads `idx` (any order; kept grouped by contig, the given order inside a contig),
    over the same contigs and slot layout."""
    idx = np.asarray(idx, dtype=np.int64)
    contig_of = np.searchsorted(batch.contig_read_off, idx, side="right") - 1
    order = np.argsort(contig_of, kind="stable")
    idx, contig_of = idx[order], contig_of[order]
    read_off = np.concatenate(([0], np.cumsum(np.bincount(contig_of, minlength=batch.n_contigs))))
    n = idx.shape[0]
    lseq = batch.seq_len[idx].astype(np.int64)
    co = batch.cig_off.astype(np.int64)
    n_cig = np.diff(co)[idx]
    # gather the ragged CIGAR and base ranges of the kept reads
    cig_off = np.concatenate(([0], np.cumsum(n_cig)))
    cig_src = np.repeat(co[:-1][idx], n_cig) + (np.arange(int(cig_off[-1])) - np.repeat(cig_off[:-1], n_cig))
    words = (lseq + 7) // 8
    seq_off = np.concatenate(([0], np.cumsum(words)))
    seq_src = np.repeat(batch.seq_off.astype(np.int64)[idx], words) + (
        np.arange(int(seq_off[-1])) - np.repeat(seq_off[:-1], words))
    return finalize(batch.contig_names, batch.contig_len, read_off, batch.ref_start[idx], seq_off[:-1], lseq,
                          cig_off, batch.cigar[cig_src], batch.seq4[seq_src], n_records=n, mask=_mask_of(batch, idx),
                          reverse=None if batch.reverse is None else batch.reverse[idx], mates=_mates_at(batch, idx))



def _ragged_gather(src: np.ndarray, starts: np.ndarray, lens: np.ndarray) -> np.ndarray:
    """Concatenation of src[starts[i] : starts[i] + lens[i]] over i."""
    lens = lens.astype(np.int64)
    total = int(lens.sum())
    ramp = np.arange(total, dtype=np.int64) - np.repeat(np.cumsum(lens) - lens, lens)
    return src[np.repeat(starts.astype(np.int64), lens) + ramp]


def merge_batches(batches) -> ReadBatch:
    """All reads of several batches over the SAME contigs as one batch, coordinate-sorted inside every contig
    (stable: ties keep batch order).  Used to mix synthetic read populations; not a hot path.  The strand bytes and the
    mates are carried when every batch has them."""
    first = batches[0]
    for b in batches[1:]:
        if list(b.contig_names) != list(first.contig_names) or not np.array_equal(b.contig_len, first.contig_len):
            raise ValueError("merge_batches needs batches over the same contigs")
    nc = first.n_contigs
    contig_of = np.concatenate([np.repeat(np.arange(nc), np.diff(b.contig_read_off)) for b in batches])
    ref_start = np.concatenate([b.ref_start for b in batches]).astype(np.int64)
    lseq = np.concatenate([b.seq_len for b in batches]).astype(np.int64)
    n_cig = np.concatenate([np.diff(b.cig_off.astype(np.int64)) for b in batches])
    cigar = np.concatenate([b.cigar for b in batches])
    cig_base = np.concatenate(([0], np.cumsum([b.cigar.shape[0] for b in batches])))
    cig_at = np.concatenate([b.cig_off[:-1].astype(np.int64) + cig_base[k] for k, b in enumerate(batches)])
    words = (lseq + 7) // 8
    bases = np.concatenate([_ragged_gather(b.seq4, b.seq_off, (b.seq_len.astype(np.int64) + 7) // 8) for b in batches])
    base_at = np.cumsum(words) - words
    order = np.lexsort((ref_start, contig_of))  # stable
    read_off = np.concatenate(([0], np.cumsum(np.bincount(contig_of, minlength=nc))))
    nco = n_cig[order]
    cig_off = np.concatenate(([0], np.cumsum(nco)))
    mask = None
    if any(b.n_masked for b in batches):
        mcount = np.concatenate([b.mask_counts() for b in batches])
        mq = np.concatenate([b.mask_qpos if b.n_masked else np.zeros(0, dtype=np.uint32) for b in batches])
        mask = (mcount[order], _ragged_gather(mq, (np.cumsum(mcount) - mcount)[order], mcount[order]))
    reverse = None
    if all(b.reverse is not None for b in batches):
        reverse = np.concatenate([b.reverse for b in batches])[order]
    mates = None
    if all(b.mates is not None for b in batches):
        mates = tuple(np.concatenate([b.mates[k] for b in batches])[order] for k in range(3))
    return finalize(first.contig_names, first.contig_len, read_off, ref_start[order], base_at[order], lseq[order],
                    cig_off, _ragged_gather(cigar, cig_at[order], nco), bases, n_records=int(order.shape[0]), mask=mask,
                    reverse=reverse, mates=mates)


_SAVE_FIELDS = ("contig_len", "contig_read_off", "contig_slot", "ref_start", "seq_off", "l_seq", "seq_len", "cig_off",
                "cigar", "seq4", "hard_idx", "complex_idx")
_SAVE_SCALARS = ("n_slots", "n_events", "reads_sorted", "aligned_bases", "n_records", "max_simple_len", "reach_right",
                 "reach_left")
_MASK_FIELDS = ("mask_read", "mask_off", "mask_qpos")  # saved only when the batch has masked bases
_STRAND_FIELDS = ("reverse",)  # saved only when the batch has its strands
_MATE_FIELDS = ("name_hash", "mate_start", "pair_role")  # saved only when the batch has its mates


def save_batch(directory: str, batch: ReadBatch) -> None:
    """One .npy per array (so that several processes can map them) + a small json."""
    import json

    os.makedirs(directory, exist_ok=True)
    for f in _MASK_FIELDS + _STRAND_FIELDS + _MATE_FIELDS:
        if os.path.exists(os.path.join(directory, f + ".npy")):
            os.remove(os.path.join(directory, f + ".npy"))
    for f in (_SAVE_FIELDS + (_MASK_FIELDS if batch.n_masked else ())
              + (_STRAND_FIELDS if batch.reverse is not None else ()) + (_MATE_FIELDS if batch.mates is not None else ())):
        np.save(os.path.join(directory, f + ".npy"), np.ascontiguousarray(getattr(batch, f)))
    meta = {k: (bool(getattr(batch, k)) if k == "reads_sorted" else int(getattr(batch, k))) for k in _SAVE_SCALARS}
    meta["contig_names"] = list(batch.contig_names)
    with open(os.path.join(directory, "batch.json"), "w") as fh:
        json.dump(meta, fh)


def load_batch(directory: str, mmap: bool = True) -> ReadBatch:
    import json

    with open(os.path.join(directory, "batch.json")) as fh:
        meta = json.load(fh)
    arrays = {f: np.load(os.path.join(directory, f + ".npy"), mmap_mode="r" if mmap else None) for f in _SAVE_FIELDS}
    for f in _MASK_FIELDS + _STRAND_FIELDS + _MATE_FIELDS:
        if os.path.exists(os.path.join(directory, f + ".npy")):
            arrays[f] = np.load(os.path.join(directory, f + ".npy"), mmap_mode="r" if mmap else None)
    return ReadBatch(contig_names=meta.pop("contig_names"), **arrays, **meta)


# --------------------------------------------------------------------------------------- BGZF
def _bgzf_blocks(data: bytes):
    """Yield (payload_start, payload_end, isize) for each BGZF block; None if not BGZF."""
    out = []
    off, n = 0, len(data)
    while off < n:
        if n - off < 18 or data[off:off + 4] != b"\x1f\x8b\x08\x04":
            return None
        xlen = struct.unpack_from("<H", data, off + 10)[0]
        p, end_x, bsize = off + 12, off + 12 + xlen, None
        while p + 4 <= end_x:
            si1, si2, slen = data[p], data[p + 1], struct.unpack_from("<H", data, p + 2)[0]
            if si1 == 66 and si2 == 67 and slen == 2:
                bsize = struct.unpack_from("<H", data, p + 4)[0]
            p += 4 + slen
        if bsize is None:
            return None
        blk_end = off + bsize + 1
        isize = struct.unpack_from("<I", data, blk_end - 4)[0]
        out.append((end_x, blk_end - 8, isize))
        off = blk_end
    return out


def inflate_bam(path) -> np.ndarray:
    """Whole-file inflate of a BAM (BGZF, plain gzip or uncompressed) -> uint8 array."""
    with open(path, "rb") as fh:
        data = fh.read()
    if data[:4] == b"BAM\x01":
        return np.frombuffer(data, dtype=np.uint8)
    blocks = _bgzf_blocks(data)
    if blocks is None:
        return np.frombuffer(gzip.decompress(data), dtype=np.uint8)
    sizes = np.fromiter((b[2] for b in blocks), dtype=np.int64, count=len(blocks))
    offs = np.concatenate(([0], np.cumsum(sizes)))
    out = np.empty(int(offs[-1]), dtype=np.uint8)
    mv = memoryview(data)

    def work(k):
        s, e, isz = blocks[k]
        if isz:
            out[offs[k]:offs[k + 1]] = np.frombuffer(zlib.decompress(mv[s:e], -15), dtype=np.uint8)

    if len(blocks) > 8:
        with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as pool:
            list(pool.map(work, range(len(blocks)), chunksize=16))
    else:
        for k in range(len(blocks)):
            work(k)
    return out


def _sq_from_text(text: str):
    """@SQ lines -> (names, lengths) in header order (the dict the reference builds, kindel.py:138-141)."""
    names, lens = [], []
    for line in text.splitlines():
        if line.startswith("@SQ"):
            sn = ln = None
            for f in line.split("\t")[1:]:
                if f.startswith("SN:"):
                    sn = f[3:]
                elif f.startswith("LN:"):
                    ln = int(f[3:])
            if sn is not None and ln is not None:
                names.append(sn)
                lens.append(ln)
    return names, lens


def decode_threads() -> int:
    """Threads of the C++ BAM decoder: $KINDEL_DECODE_THREADS, else the cores this process may use (at most 64)."""
    ev = os.environ.get("KINDEL_DECODE_THREADS")
    if ev:
        return max(1, int(ev))
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    return max(1, min(64, n))


def read_bam(path, threads: int = None, pinned: bool = False, min_mapq: int = 0, exclude_flags: int = 0,
             min_base_quality: int = 0, strand: bool = False, mates: bool = False, qual: bool = False) -> ReadBatch:
    """.bam -> ReadBatch through the C++ decoder (bam_host.cpp): BGZF inflate, filter, classification and the
    device layout (inline CIGAR blocks included) in threads, no Python per-record or per-array work.
    pinned=True puts the arrays the device consumes into page-locked memory (needs torch + CUDA).
    min_mapq / exclude_flags / min_base_quality: the filters of this module's docstring (extension).  strand=True
    (extension): also the kept reads' strands, `reverse` (kdl_bam_fill_strand).  mates=True (extension): also
    `name_hash`, `mate_start` and `pair_role` (kdl_bam_fill_mates).  qual=True (extension): also `qual8`, the
    qualities beside the bases (kdl_bam_fill_qual); a kept read without qualities is a ValueError."""
    import ctypes as C

    filters = check_filters(min_mapq, exclude_flags, min_base_quality)
    lib = _ffi.load()
    threads = threads or decode_threads()
    h = C.c_void_p()
    rc = lib.kdl_bam_open(os.fspath(path).encode(), threads, C.byref(h))
    if rc != 0:
        raise ValueError("not a (readable) BAM file: %s" % path)
    try:
        if any(filters):
            # refused for SAM text whose MAPQ / QUAL fields the strict parser could not carry: the text reader's case
            if lib.kdl_bam_set_filter(h, *filters) != 0:
                raise ValueError("%s: MAPQ / QUAL fields the C++ text parser does not take" % path)
        n_ref = lib.kdl_bam_n_ref(h)
        tl = C.c_int64()
        tp = lib.kdl_bam_header_text(h, C.byref(tl))
        text = C.string_at(tp, tl.value).decode("utf-8", "replace") if tp and tl.value else ""
        bin_names = [lib.kdl_bam_ref_name(h, k).decode() for k in range(n_ref)]
        bin_lens = [lib.kdl_bam_ref_len(h, k) for k in range(n_ref)]
        text_names, text_lens = _sq_from_text(text)
        text_len = dict(zip(text_names, text_lens))
        ref_len = np.array([text_len.get(nm, ln) for nm, ln in zip(bin_names, bin_lens)], dtype=np.int32)
        info = np.zeros(16, dtype=np.int64)
        rc = lib.kdl_bam_prepare(h, ref_len.ctypes.data if n_ref else None, threads, info.ctypes.data)
        if rc != 0:
            raise ValueError("malformed BAM record stream in %s (or too large for 32-bit offsets)" % path)
        n_rec, n, n_seen, n_ops, n_words, n_cx, n_hard = (int(x) for x in info[:7])
        order = np.zeros(max(n_seen, 1), dtype=np.int32)[:n_seen]
        read_off = np.zeros(n_seen + 1, dtype=np.int64)
        _ffi.check(lib.kdl_bam_contigs(h, order.ctypes.data if n_seen else None, read_off.ctypes.data)
                   if n_seen else 0, "kdl_bam_contigs")
        contig_len = ref_len[order].astype(np.int32)
        slot, n_slots = layout_slots(contig_len)

        def buf(count, dtype):
            if pinned:
                import torch

                tdt = {np.int32: torch.int32, np.uint32: torch.int32}[dtype]
                return torch.empty(max(count, 1), dtype=tdt).pin_memory().numpy().view(dtype)[:count]
            return np.empty(max(count, 1), dtype=dtype)[:count]

        ref_start, seq_off, l_seq = buf(n, np.int32), buf(n, np.uint32), buf(n, np.int32)
        seq_len = np.empty(max(n, 1), dtype=np.int32)[:n]
        cig_off = np.empty(n + 1, dtype=np.uint32)
        cigar = np.empty(max(n_ops, 1), dtype=np.uint32)[:n_ops]
        stream = buf(n_words, np.uint32)
        cx_idx, hard_idx = buf(n_cx, np.uint32), buf(n_hard, np.uint32)
        rc = lib.kdl_bam_fill(h, threads, slot.ctypes.data if n_seen else None, ref_start.ctypes.data, seq_off.ctypes.data,
                              l_seq.ctypes.data, seq_len.ctypes.data, cig_off.ctypes.data, cigar.ctypes.data,
                              stream.ctypes.data, cx_idx.ctypes.data, hard_idx.ctypes.data, info.ctypes.data)
        if rc != 0:
            raise ValueError("malformed BAM record stream in %s" % path)
        mask = {}
        n_masked, n_mreads = int(info[13]), int(info[14])
        if n_masked:
            mask = dict(mask_read=buf(n_mreads, np.uint32), mask_off=buf(n_mreads + 1, np.uint32),
                        mask_qpos=buf(n_masked, np.uint32))
            _ffi.check(lib.kdl_bam_fill_mask(h, threads, mask["mask_read"].ctypes.data, mask["mask_off"].ctypes.data,
                                             mask["mask_qpos"].ctypes.data), "kdl_bam_fill_mask")
        if strand:
            mask["reverse"] = np.zeros(n, dtype=np.uint8)
            _ffi.check(lib.kdl_bam_fill_strand(h, threads, mask["reverse"].ctypes.data if n else None),
                       "kdl_bam_fill_strand")
        if mates:
            mask.update(name_hash=np.zeros(n, dtype=np.uint64), mate_start=np.zeros(n, dtype=np.int32),
                        pair_role=np.zeros(n, dtype=np.uint8))
            ptrs = [mask[f].ctypes.data if n else None for f in _MATE_FIELDS]
            _ffi.check(lib.kdl_bam_fill_mates(h, threads, *ptrs), "kdl_bam_fill_mates")
        if qual:
            if int(info[15]):
                raise ValueError(missing_qualities(path, int(info[15])))
            mask["qual8"] = np.empty(8 * n_words, dtype=np.uint8)
            _ffi.check(lib.kdl_bam_fill_qual(h, threads, mask["qual8"].ctypes.data if n else None), "kdl_bam_fill_qual")
    finally:
        lib.kdl_bam_close(h)
    return ReadBatch(
        contig_names=[bin_names[i] for i in order], contig_len=contig_len, contig_read_off=read_off, contig_slot=slot,
        n_slots=n_slots, ref_start=ref_start, seq_off=seq_off, l_seq=l_seq, seq_len=seq_len, cig_off=cig_off,
        cigar=cigar, seq4=stream, hard_idx=hard_idx, complex_idx=cx_idx, n_events=int(info[8]),
        reads_sorted=bool(info[12]) or n < 2, aligned_bases=int(info[7]), n_records=n_rec,
        max_simple_len=int(info[11]), reach_right=int(info[9]), reach_left=int(info[10]), **mask)


def missing_qualities(path, n: int) -> str:
    return "%s: %d kept read(s) without base qualities (QUAL `*` or 0xff); --qual and --quality-vote need them" % (
        os.fspath(path), n)


def qual_layout(batch: ReadBatch, qual: np.ndarray) -> np.ndarray:
    """The qual8 of a batch from its reads' qualities concatenated in read order (seq_len bytes per read): base k of
    read r at byte 8 * seq_off[r] + k, 0xff elsewhere (include/kindel_b200.h kdl_quality_pileup)."""
    qual = np.asarray(qual, dtype=np.uint8)
    lens = np.asarray(batch.seq_len, dtype=np.int64)
    if qual.shape[0] != int(lens.sum()):
        raise ValueError("qualities must hold exactly one byte per base")
    out = np.full(8 * int(batch.seq4.shape[0]), 0xFF, dtype=np.uint8)
    starts = 8 * np.asarray(batch.seq_off, dtype=np.int64)
    out[np.repeat(starts - (np.cumsum(lens) - lens), lens) + np.arange(qual.shape[0], dtype=np.int64)] = qual
    return out


# ---------------------------------------------------------------------------------------- SAM
def encode_seq(seq: str) -> np.ndarray:
    """Text bases -> uint32 words, 8 nibbles each, first base in the most significant nibble,
    zero-padded.  Case is folded (the reference upper-cases every base it touches:
    kindel.py:51,56,69,77)."""
    codes = _ENC[np.frombuffer(seq.encode("ascii"), dtype=np.uint8)]
    if codes.size and codes.max() == 255:
        bad = seq[int(np.argmax(codes == 255))]
        raise ValueError("base %r is outside the BAM alphabet %s and cannot be packed" % (bad, NIBBLES))
    n_words = (len(seq) + 7) // 8
    padded = np.zeros(n_words * 8, dtype=np.uint32)
    padded[: codes.size] = codes
    return pack_nibbles(padded.reshape(-1, 8)).reshape(-1)


_SHIFTS = np.arange(28, -4, -4, dtype=np.uint32)


def pack_nibbles(nib: np.ndarray) -> np.ndarray:
    """[..., 8k] nibble codes -> [..., k] uint32 words (first base in the top nibble)."""
    shape = nib.shape[:-1] + (nib.shape[-1] // 8, 8)
    return (nib.reshape(shape).astype(np.uint32) << _SHIFTS).sum(axis=-1, dtype=np.uint32)


def unpack_nibbles(words: np.ndarray) -> np.ndarray:
    """uint32 words [..., k] -> nibble codes [..., 8k] uint8."""
    w = np.asarray(words, dtype=np.uint32)
    return ((w[..., None] >> _SHIFTS) & 0xF).astype(np.uint8).reshape(w.shape[:-1] + (w.shape[-1] * 8,))


def words_to_bam_bytes(words: np.ndarray, l_seq: int) -> bytes:
    """The BAM on-disk packing of a read (two bases per byte, first in the high nibble)."""
    return np.asarray(words, dtype=">u4").tobytes()[: (l_seq + 1) // 2]


def parse_cigar_text(text: str):
    if text == "*":
        return []
    out, num = [], 0
    for ch in text:
        if ch.isdigit():
            num = num * 10 + ord(ch) - 48
        else:
            out.append((num << 4) | _OP_CODE.get(ch, 15))  # unknown op letters are no-ops
            num = 0
    return out


def _sam_qual(text: str, seq: str) -> bytes:
    """Phred qualities of a SAM QUAL field (b"\\xff" * len(seq) for `*`); ValueError for a malformed one."""
    if text == "*":
        return b"\xff" * len(seq)
    raw = text.encode("ascii", "replace")
    if len(raw) != len(seq) or any(c < 33 or c > 126 for c in raw):
        raise ValueError("QUAL %r does not match SEQ of length %d" % (text[:40], len(seq)))
    return bytes(c - 33 for c in raw)


def read_sam(path, min_mapq: int = 0, exclude_flags: int = 0, min_base_quality: int = 0,
             strand: bool = False, mates: bool = False, qual: bool = False) -> ReadBatch:
    min_mapq, exclude_flags, min_base_quality = check_filters(min_mapq, exclude_flags, min_base_quality)
    header = []
    groups = {}  # rname -> list of (pos0, cigar words, seq, qualities, reverse, (name hash, PNEXT - 1, role))
    n_records = n_noqual = 0
    with open(path, "rt") as fh:
        for line in fh:
            if line.startswith("@"):
                header.append(line.rstrip("\n"))
                continue
            f = line.rstrip("\n").split("\t")
            if len(f) < 11:
                continue
            n_records += 1
            rname = f[2]
            g = groups.get(rname)
            if g is None:
                g = groups[rname] = []
            flag, seq = int(f[1]), f[9]
            if (flag & 0x4) or len(seq) <= 1:  # kindel.py:43-46
                continue
            if flag & exclude_flags:  # excluded == unmapped (extension)
                continue
            if min_mapq:
                mapq = int(f[4])
                if not 0 <= mapq <= 255:
                    raise ValueError("MAPQ %d out of range" % mapq)
                if mapq < min_mapq:
                    continue
            qv = _sam_qual(f[10], seq) if (min_base_quality or qual) else None
            if qual and f[10] == "*":
                n_noqual += 1
            mate = None
            if mates:
                try:
                    pnext = int(f[7])
                except ValueError:
                    pnext = -1
                mate = (name_hash(f[0]), pnext - 1 if 0 <= pnext < (1 << 31) else -1,
                        pair_role(flag, f[6] == "=" or f[6] == rname))
            g.append((int(f[3]) - 1, parse_cigar_text(f[5]), seq, qv, 1 if flag & 0x10 else 0, mate))
    groups.pop("*", None)  # kindel.py:147-148
    names, lens = _sq_from_text("\n".join(header))
    sq = dict(zip(names, lens))
    contig_names = list(groups)
    for nm in contig_names:
        if nm not in sq:
            raise KeyError(nm)  # refs_lens[ref_id], kindel.py:151
    ref_start, l_seq, cig_off, cigar, seq_off, seq_parts, quals, rev, mate_rows = [], [], [0], [], [], [], [], [], []
    read_off = [0]
    words = 0
    for nm in contig_names:
        for pos0, cig, seq, qual, is_rev, mate in groups[nm]:
            ref_start.append(pos0)
            l_seq.append(len(seq))
            cigar.extend(cig)
            cig_off.append(len(cigar))
            enc = encode_seq(seq)
            seq_off.append(words)
            words += enc.size
            seq_parts.append(enc)
            quals.append(qual)
            rev.append(is_rev)
            mate_rows.append(mate)
        read_off.append(len(ref_start))
    seq4 = np.concatenate(seq_parts) if seq_parts else np.zeros(0, dtype=np.uint32)
    if n_noqual:
        raise ValueError(missing_qualities(path, n_noqual))
    quals = np.frombuffer(b"".join(quals), dtype=np.uint8) if (min_base_quality or qual) else None
    batch = finalize(contig_names, np.array([sq[nm] for nm in contig_names], dtype=np.int64),
                    np.array(read_off, dtype=np.int64), np.array(ref_start, dtype=np.int64),
                    np.array(seq_off, dtype=np.int64), np.array(l_seq, dtype=np.int64),
                    np.array(cig_off, dtype=np.int64), np.array(cigar, dtype=np.int64), seq4,
                     n_records=n_records, qual=quals, min_base_quality=min_base_quality,
                     reverse=np.array(rev, dtype=np.uint8) if strand else None,
                     mates=tuple(np.array([m[k] for m in mate_rows], dtype=dt) for k, dt in
                                 enumerate((np.uint64, np.int64, np.uint8))) if mates else None)
    if qual:
        batch.qual8 = qual_layout(batch, quals)
    return batch


def read_alignment(path, min_mapq: int = 0, exclude_flags: int = 0, min_base_quality: int = 0,
                   strand: bool = False, mates: bool = False, qual: bool = False) -> ReadBatch:
    """.bam or .sam (by content, not by suffix) -> ReadBatch.  The filters, strand, mates and qualities (extensions):
    see the module docstring."""
    path = os.fspath(path)
    filters = dict(zip(("min_mapq", "exclude_flags", "min_base_quality"),
                       check_filters(min_mapq, exclude_flags, min_base_quality)), strand=bool(strand))
    if mates:  # (the keyword only when asked: a reader without it stays as it was)
        filters["mates"] = True
    if qual:
        filters["qual"] = True
    with open(path, "rb") as fh:
        magic = fh.read(4)
    if magic[:2] == b"\x1f\x8b" or magic == b"BAM\x01":
        return read_bam(path, **filters)
    # SAM text: the C++ decoder turns the lines into BAM records in threads and shares everything downstream.  Its
    # parser is strict; whatever it refuses (an RNAME without @SQ line, a base that cannot be packed, odd integers ...)
    # goes through the Python text reader below, which raises what the reference's path would
    try:
        return read_bam(path, **filters)
    except ValueError:
        return read_sam(path, **filters)


# ------------------------------------------------------------------------------ BAM writing
def write_bam(path, contigs, records, header_text=None, level=6):
    """Minimal BAM writer (used for synthetic inputs and test fixtures).

    contigs: list of (name, length).  records: iterable of tuples
    (ref_id, pos0, flag, cigar_words, seq_text[, qname[, mapq[, qual[, next_ref_id, next_pos0]]]]): mapq defaults to
    60, qual (Phred values, bytes or a sequence of ints, one per base; None = none, stored as 0xff) to none, RNEXT /
    PNEXT (the mate's reference id and 0-based position) to -1.  One BGZF block per ~60 KB + EOF
    block.
    """
    if header_text is None:
        header_text = "@HD\tVN:1.6\tSO:unknown\n" + "".join(
            "@SQ\tSN:%s\tLN:%d\n" % (n, l) for n, l in contigs)
    ht = header_text.encode()
    body = bytearray()
    body += b"BAM\x01" + struct.pack("<i", len(ht)) + ht + struct.pack("<i", len(contigs))
    for name, length in contigs:
        nb = name.encode() + b"\x00"
        body += struct.pack("<i", len(nb)) + nb + struct.pack("<i", length)
    for k, rec in enumerate(records):
        ref_id, pos0, flag, cig, seq = rec[:5]
        qname = (rec[5] if len(rec) > 5 and rec[5] is not None else "r%d" % k).encode() + b"\x00"
        mapq = int(rec[6]) if len(rec) > 6 and rec[6] is not None else 60
        if seq == "*":
            l_seq, packed = 0, b""
        else:
            l_seq = len(seq)
            packed = words_to_bam_bytes(encode_seq(seq), l_seq)
        qual = bytes(rec[7]) if len(rec) > 7 and rec[7] is not None else b"\xff" * l_seq
        if len(qual) != l_seq:
            raise ValueError("record %d: %d qualities for %d bases" % (k, len(qual), l_seq))
        next_ref = int(rec[8]) if len(rec) > 8 and rec[8] is not None else -1
        next_pos = int(rec[9]) if len(rec) > 9 and rec[9] is not None else -1
        core = struct.pack("<iiBBHHHiiii", ref_id, pos0, len(qname), mapq, 4680, len(cig), flag, l_seq, next_ref, next_pos,
                           0)
        data = core + qname + struct.pack("<%dI" % len(cig), *cig) + packed + qual
        body += struct.pack("<i", len(data)) + data
    with open(path, "wb") as fh:
        for s in range(0, len(body), 60000):
            fh.write(_bgzf_block(bytes(body[s:s + 60000]), level))
        fh.write(_bgzf_block(b"", level))


def _bgzf_block(chunk: bytes, level: int) -> bytes:
    comp = zlib.compressobj(level, zlib.DEFLATED, -15)
    payload = comp.compress(chunk) + comp.flush()
    bsize = len(payload) + 25
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", bsize) + payload
            + struct.pack("<II", zlib.crc32(chunk) & 0xFFFFFFFF, len(chunk)))
