"""TEST INFRASTRUCTURE ONLY -- an independent restatement of amplicon primer masking (`--primers`, an extension: the
reference has no such option), as a per-record loop over plain Python ints and lists.

Records are objects with .pos (1-based), .mapped, .seq and .cigars ((length, op letter) pairs), as oracle/samdecode.py
gives them; primers are plain (chrom, start, end) rows.  Per record, on a contig of length L:

  walk    the reference's loop (kindel.py:40-81) for the cursors alone: M/=/X give each base the cursor r_pos and
          advance r_pos and q_pos; I advances q_pos; D advances r_pos; an S that is op #0 advances q_pos; any later S
          advances both while r_pos < L; N, H, P nothing
  ends    s, e = the cursors of the first and the last M/=/X base (a record without one is left alone)
  left    the primers [a, b) with a <= s < b: every M/=/X base with s <= cursor < max(b)
  right   the primers with a <= e < b: every M/=/X base with min(a) <= cursor <= e
  only bases inside SEQ (q < len(seq)) are masked.

The masked bases become a quality vector (0 where masked, the given quality or 0xff elsewhere) for
oracle.qoracle.pileup, whose C walk reads a base below the threshold as N and does not count it.  With
min_base_quality as well, a base is masked when either rule masks it.  masked_qpos checks every interval against both
ends, with no sorting and no search (masked_arrays, its form for batches of millions of reads, walks the intervals
instead); the engine's arrays and mask list are never read.  Nothing here imports kindel_b200."""
from __future__ import annotations

import numpy as np

from . import qoracle, samdecode


def masked_qpos(rec, L, intervals):
    """Sorted query offsets of the record's primer bases; intervals = [(start, end)] of its contig."""
    r_pos, q_pos = rec.pos - 1, 0
    bases = []  # (query offset, cursor) of every M/=/X base
    for i, (length, op) in enumerate(rec.cigars):
        if op in ("M", "=", "X"):
            for _ in range(length):
                bases.append((q_pos, r_pos))
                r_pos += 1
                q_pos += 1
        elif op == "I":
            q_pos += length
        elif op == "D":
            r_pos += length
        elif op == "S":
            if i == 0:
                q_pos += length
            else:
                for _ in range(length):
                    if r_pos < L:
                        r_pos += 1
                        q_pos += 1
    if not bases:
        return []
    s, e = bases[0][1], bases[-1][1]
    left = [b for a, b in intervals if a <= s < b]
    right = [a for a, b in intervals if a <= e < b]
    B = max(left) if left else s
    A = min(right) if right else e + 1
    return [q for q, c in bases if (s <= c < B or A <= c <= e) and q < len(rec.seq)]


def contig_intervals(rows, name):
    return [(int(a), int(b)) for c, a, b in rows if c == name]


def read_bed_rows(path):
    """[(chrom, start, end)] of a plain-text BED, read the simplest way (tests write plain files)."""
    rows = []
    with open(path) as fh:
        for line in fh:
            line = line.rstrip("\r\n")
            if not line.strip() or line.startswith(("#", "track", "browser")):
                continue
            f = line.split()
            rows.append((f[0], int(f[1]), int(f[2])))
    return rows


def kept_records(path, contig_names):
    """({name: L}, the records the engine keeps without filters, in its read order: by contig in `contig_names`
    order, file order inside a contig)."""
    header, records = samdecode.read_alignment_file(path)
    lengths = {}
    for sn, fields in header["@SQ"].items():
        ln = next(f for f in fields if f.startswith("LN:"))
        lengths[sn[3:]] = int(ln[3:])
    groups = {}
    for r in records:
        groups.setdefault(r.rname, []).append(r)
    out = [(nm, r) for nm in contig_names for r in groups.get(nm, []) if r.mapped and len(r.seq) > 1]
    return lengths, out


def masked_by_read(path, contig_names, rows):
    """Per kept record (engine read order): its sorted primer query offsets."""
    lengths, recs = kept_records(path, contig_names)
    return [masked_qpos(r, lengths[nm], contig_intervals(rows, nm)) for nm, r in recs]


class _Rec:
    __slots__ = ("pos", "seq", "cigars")

    def __init__(self, pos, seq, cigars):
        self.pos, self.seq, self.cigars = pos, seq, cigars


def masked_arrays(batch, rows):
    """The primer bases of a large batch (any object with the flattened-batch attributes) as (per-read counts int64,
    query offsets int64, ascending per read): every read with a CIGAR other than one M op of its SEQ length goes
    through masked_qpos; for the one-M-op reads the same rule is applied interval by interval, each interval to the
    reads whose first or last base it holds (found in the reads' ends, sorted)."""
    n = int(batch.ref_start.shape[0])
    cig_off = np.asarray(batch.cig_off, dtype=np.int64)
    cigar = np.asarray(batch.cigar, dtype=np.int64)
    lseq = np.asarray(batch.seq_len, dtype=np.int64)
    start = np.asarray(batch.ref_start, dtype=np.int64)
    n_ops = np.diff(cig_off)
    first = np.where(n_ops > 0, cigar[np.minimum(cig_off[:-1], max(cigar.shape[0] - 1, 0))], 0) if n else np.zeros(0)
    one_m = (n_ops == 1) & np.isin(first & 15, (0, 7, 8)) & ((first >> 4) == lseq) & (lseq > 0)
    left = np.zeros(n, dtype=np.int64)        # one-M-op reads: q in [0, left) and [right, lseq) are masked
    right = lseq.copy()
    other = {}
    for c, name in enumerate(batch.contig_names):
        lo, hi = int(batch.contig_read_off[c]), int(batch.contig_read_off[c + 1])
        iv = contig_intervals(rows, name)
        idx = np.arange(lo, hi)[one_m[lo:hi]]
        s, e = start[idx], start[idx] + lseq[idx] - 1
        B, A = s.copy(), e + 1
        s_ord, e_ord = np.argsort(s, kind="stable"), np.argsort(e, kind="stable")
        s_srt, e_srt = s[s_ord], e[e_ord]
        for a, b in iv:  # the reads whose first / last base lies in [a, b)
            hit = s_ord[np.searchsorted(s_srt, a):np.searchsorted(s_srt, b)]
            B[hit] = np.maximum(B[hit], b)
            hit = e_ord[np.searchsorted(e_srt, a):np.searchsorted(e_srt, b)]
            A[hit] = np.minimum(A[hit], a)
        left[idx] = np.minimum(B - s, lseq[idx])
        right[idx] = np.minimum(np.maximum(A - s, left[idx]), lseq[idx])
        for r in np.flatnonzero(~one_m[lo:hi]) + lo:
            ops = [(int(w >> 4), "MIDNSHP=X"[w & 15] if (w & 15) < 9 else None)
                   for w in cigar[cig_off[r]:cig_off[r + 1]].tolist()]
            rec = _Rec(int(start[r]) + 1, "N" * int(lseq[r]), ops)
            other[int(r)] = np.array(masked_qpos(rec, int(batch.contig_len[c]), iv), dtype=np.int64)
    counts = np.where(one_m, left + (lseq - right), 0)
    for r, q in other.items():
        counts[r] = q.shape[0]
    # per read: its left run, then its right run (or its walked list)
    total = int(counts.sum())
    ramp = np.arange(total, dtype=np.int64) - np.repeat(np.cumsum(counts) - counts, counts)
    rr = np.repeat(np.arange(n), counts)
    flat = np.where(ramp < left[rr], ramp, ramp - left[rr] + right[rr])
    at = np.cumsum(counts) - counts
    for r, q in other.items():
        flat[at[r]:at[r] + q.shape[0]] = q
    return counts, flat


def masked_by_batch(batch, rows):
    """masked_arrays as per-read arrays (the shape masked_by_read gives)."""
    counts, flat = masked_arrays(batch, rows)
    return np.split(flat, np.cumsum(counts)[:-1]) if counts.shape[0] else []


def quality_vector(batch, masked, qual=None):
    """Qualities of the reads concatenated (batch.seq_len bytes each): `qual` (or 0xff = none) with every primer base 0.
    masked: per-read lists, or masked_arrays' (counts, offsets)."""
    lseq = np.asarray(batch.seq_len, dtype=np.int64)
    out = np.full(int(lseq.sum()), 0xFF, dtype=np.uint8) if qual is None else np.array(qual, dtype=np.uint8)
    starts = np.cumsum(lseq) - lseq
    if isinstance(masked, tuple):  # masked_arrays' (counts, offsets)
        lens, flat = masked
    else:
        lens = np.array([len(x) for x in masked], dtype=np.int64)
        flat = np.concatenate([np.asarray(x, dtype=np.int64) for x in masked]) if lens.sum() else np.zeros(0, np.int64)
    if lens.sum():
        out[np.repeat(starts, lens) + flat] = 0
    return out


def pileup(batch, masked, qual=None, min_base_quality=0):
    """(counts, events) of the unmasked `batch` with the primer bases `masked` (masked_by_read) -- and, given
    `qual`, the bases below min_base_quality -- read as N and not counted (oracle.qoracle)."""
    return qoracle.pileup(batch, quality_vector(batch, masked, qual), max(int(min_base_quality), 1))


def merged_mask(masked, qual, lseq, min_base_quality):
    """Per read, the sorted union of its primer bases and its bases below min_base_quality (qual: concatenated,
    0xff = none): the mask list K9 must write."""
    out = []
    at = 0
    for r, qs in enumerate(masked):
        n = int(lseq[r])
        low = [q for q in range(n) if qual is not None and qual[at + q] < min_base_quality] if min_base_quality else []
        out.append(sorted(set(qs) | set(low)))
        at += n
    return out
