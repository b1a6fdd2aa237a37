"""Amplicon primer schemes for `--primers scheme.bed` (extension): the BED loader and the per-contig arrays K9 searches.

    load_primers(path) -> PrimerSet(name, chrom, start, end, line)
    primer_arrays(primer_set, contig_names, contig_len) -> PrimerArrays (the kdl_primers arrays, host numpy)

The file is BED text, plain or gzip, told apart by its magic bytes.  Columns 1-3 are read: chrom, 0-based start,
exclusive end; further columns (an ARTIC `*.primer.bed`'s name, pool and strand) are ignored.  Blank lines and lines
starting with `#`, `track` or `browser` are skipped, and CR is dropped.  A row with fewer than 3 fields or with
coordinates that are not integers raises ValueError naming its line, and so does, once the alignment's contigs are
known, a row with start < 0, start >= end or end > the @SQ LN of its contig.  Rows of contigs the alignment does not
have are ignored.  Overlapping and duplicate intervals are allowed.

What K9 does with them (kindel_b200/csrc/primers.cu): a read whose first M/=/X base lies in a primer has its bases up
to the end of the longest such primer masked, and a read whose last M/=/X base lies in one has its bases from the
start of the earliest such primer masked.  To find both with one binary search each, every contig's intervals are
kept twice: sorted by start with the running maximum of the end, and sorted by end with the suffix minimum of the
start.
"""
from __future__ import annotations

import gzip
import os
from dataclasses import dataclass

import numpy as np


@dataclass(frozen=True)
class PrimerSet:
    name: str           # the BED's file name, without directories (REPORT and VCF header)
    chrom: tuple        # per row
    start: np.ndarray   # int64 per row, 0-based
    end: np.ndarray     # int64 per row, exclusive
    line: np.ndarray    # int64 per row: its 1-based line number in the file

    @property
    def n_rows(self) -> int:
        return len(self.chrom)


@dataclass(frozen=True)
class PrimerArrays:
    """The kdl_primers arrays of one alignment's contigs (include/kindel_b200.h, K9)."""

    contig_off: np.ndarray    # int64 [n_contigs + 1]
    start_sorted: np.ndarray  # int32 [n]
    end_max: np.ndarray       # int32 [n]
    end_sorted: np.ndarray    # int32 [n]
    start_min: np.ndarray     # int32 [n]

    @property
    def n_contigs(self) -> int:
        return int(self.contig_off.shape[0]) - 1

    @property
    def n_intervals(self) -> int:
        return int(self.start_sorted.shape[0])


_SKIP = (b"#", b"track", b"browser")


def read_bed(data: bytes, name: str = "<bed>") -> PrimerSet:
    """The rows of BED text (bytes, already inflated)."""
    chrom, start, end, line = [], [], [], []
    for k, raw in enumerate(data.split(b"\n"), start=1):
        text = raw.replace(b"\r", b"")
        if not text.strip() or text.startswith(_SKIP):
            continue
        fields = text.split(b"\t") if b"\t" in text else text.split()
        if len(fields) < 3:
            raise ValueError("%s line %d: a BED row needs chrom, start and end, got %d field(s)" % (name, k, len(fields)))
        try:
            a, b = int(fields[1]), int(fields[2])
        except ValueError:
            raise ValueError("%s line %d: start and end must be integers, got %r and %r"
                             % (name, k, fields[1].decode("utf-8", "replace"), fields[2].decode("utf-8", "replace")))
        chrom.append(fields[0].decode("utf-8", "replace"))
        start.append(a)
        end.append(b)
        line.append(k)
    return PrimerSet(name, tuple(chrom), np.array(start, dtype=np.int64), np.array(end, dtype=np.int64),
                     np.array(line, dtype=np.int64))


def load_primers(path) -> PrimerSet:
    """The rows of the BED file at `path` (plain or gzip)."""
    with open(path, "rb") as fh:
        data = fh.read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)  # every member of a (b)gzip file
    name = os.path.basename(os.fspath(path))
    return read_bed(data, name)


def as_primer_set(primers):
    """None, a PrimerSet, or a path to load."""
    if primers is None or isinstance(primers, PrimerSet):
        return primers
    return load_primers(primers)


def primer_arrays(primer_set: PrimerSet, contig_names, contig_len) -> PrimerArrays:
    """The per-contig arrays of the rows on the given contigs (in their order); the other rows are ignored.  A row
    with start < 0, start >= end or end > its contig's length raises ValueError naming its line."""
    index = {nm: c for c, nm in enumerate(contig_names)}
    contig_len = np.asarray(contig_len, dtype=np.int64)
    c_of = np.array([index.get(nm, -1) for nm in primer_set.chrom], dtype=np.int64)
    on = c_of >= 0
    a, b, c, ln = primer_set.start[on], primer_set.end[on], c_of[on], primer_set.line[on]
    bad = (a < 0) | (a >= b) | (b > contig_len[c])
    if bad.any():
        k = int(np.flatnonzero(bad)[0])
        raise ValueError("%s line %d: interval [%d, %d) of %r does not lie in 0 <= start < end <= %d (its @SQ LN)"
                         % (primer_set.name, int(ln[k]), int(a[k]), int(b[k]), contig_names[int(c[k])],
                            int(contig_len[c[k]])))
    n_contigs = len(contig_names)
    off = np.zeros(n_contigs + 1, dtype=np.int64)
    off[1:] = np.cumsum(np.bincount(c, minlength=n_contigs))
    by_start = np.lexsort((b, a, c))
    by_end = np.lexsort((a, b, c))
    start_sorted, end_sorted = a[by_start], b[by_end]
    end_max = b[by_start].copy()
    start_min = a[by_end].copy()
    for k in range(n_contigs):  # running max / suffix min, restarted per contig
        lo, hi = int(off[k]), int(off[k + 1])
        if hi > lo:
            end_max[lo:hi] = np.maximum.accumulate(end_max[lo:hi])
            start_min[lo:hi] = np.minimum.accumulate(start_min[lo:hi][::-1])[::-1]
    i32 = lambda x: np.ascontiguousarray(x, dtype=np.int32)  # noqa: E731  (coordinates <= @SQ LN < 2^31)
    return PrimerArrays(off, i32(start_sorted), i32(end_max), i32(end_sorted), i32(start_min))


def window(arrays: PrimerArrays, c: int, s: int, e: int):
    """(B, A) of a read on contig c whose first / last M/=/X base is at cursor s / e, from the arrays as K9 searches
    them: bases with cursor in [s, B) and [A, e] are masked (B = s, A = e + 1 where no primer holds that end)."""
    lo, hi = int(arrays.contig_off[c]), int(arrays.contig_off[c + 1])
    B, A = s, e + 1
    kl = lo + int(np.searchsorted(arrays.start_sorted[lo:hi], s, side="right"))
    if kl > lo and int(arrays.end_max[kl - 1]) > s:
        B = int(arrays.end_max[kl - 1])
    kr = lo + int(np.searchsorted(arrays.end_sorted[lo:hi], e, side="right"))
    if kr < hi and int(arrays.start_min[kr]) <= e:
        A = int(arrays.start_min[kr])
    return B, A


def save_arrays(path: str, arrays: PrimerArrays) -> None:
    np.savez(path, **{f: getattr(arrays, f) for f in _ARRAY_FIELDS})


def load_arrays(path: str) -> PrimerArrays:
    with np.load(path) as z:
        return PrimerArrays(**{f: z[f] for f in _ARRAY_FIELDS})


_ARRAY_FIELDS = ("contig_off", "start_sorted", "end_max", "end_sorted", "start_min")
