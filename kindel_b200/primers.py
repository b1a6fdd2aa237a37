"""Amplicon primer schemes for `--primers scheme.bed` (extension): the BED loader and the per-contig arrays K9 searches.

    load_primers(path) -> PrimerSet(name, chrom, start, end, line)
    primer_arrays(primer_set, contig_names, contig_len) -> PrimerArrays (the kdl_primers arrays, host numpy)
    load_scheme(path) -> AmpliconScheme (`kindel amplicons`: the amplicons the name column defines, below)
    amplicon_arrays(scheme, contig_names, contig_len) -> AmpliconArrays (the kdl_amplicons arrays K12 searches)

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


def _bed_rows(data: bytes, name: str):
    """(line number, fields, start, end) of every row of BED text: skipped lines left out, CR dropped, columns 2-3
    parsed (ValueError naming the line)."""
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
        yield k, fields, a, b


def read_bed(data: bytes, name: str = "<bed>") -> PrimerSet:
    """The rows of BED text (bytes, already inflated)."""
    chrom, start, end, line = [], [], [], []
    for k, fields, a, b in _bed_rows(data, name):
        chrom.append(fields[0].decode("utf-8", "replace"))
        start.append(a)
        end.append(b)
        line.append(k)
    return PrimerSet(name, tuple(chrom), np.array(start, dtype=np.int64), np.array(end, dtype=np.int64),
                     np.array(line, dtype=np.int64))


def _read_file(path):
    """(bytes inflated, file name without directories) of a plain or gzip file."""
    with open(path, "rb") as fh:
        data = fh.read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)  # every member of a (b)gzip file
    return data, os.path.basename(os.fspath(path))


def load_primers(path) -> PrimerSet:
    """The rows of the BED file at `path` (plain or gzip)."""
    data, name = _read_file(path)
    return read_bed(data, name)


def as_primer_set(primers):
    """None, a PrimerSet, or a path to load."""
    if primers is None or isinstance(primers, PrimerSet):
        return primers
    return load_primers(primers)


def _rows_on(primer_set: PrimerSet, contig_names, contig_len):
    """(bool per row: on one of the contigs, int64 per row: its contig index or -1); a row on them with start < 0,
    start >= end or end > its contig's length raises ValueError naming its line."""
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
    return on, c_of


def primer_arrays(primer_set: PrimerSet, contig_names, contig_len) -> PrimerArrays:
    """The per-contig arrays of the rows on the given contigs (in their order); the other rows are ignored.  A row
    with start < 0, start >= end or end > its contig's length raises ValueError naming its line."""
    on, c_of = _rows_on(primer_set, contig_names, contig_len)
    a, b, c = primer_set.start[on], primer_set.end[on], c_of[on]
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


# ------------------------------------------------------------------------------------- amplicon schemes
# `kindel amplicons --primers scheme.bed`: the amplicons the BED's name column defines, and the per-contig segment
# arrays K12 (csrc/amplicons.cu) searches to give each read its amplicon.

@dataclass(frozen=True)
class AmpliconScheme:
    """The amplicons of a named primer BED (load_scheme), in file order of their first row, and its rows."""

    primers: PrimerSet       # every row, as load_primers reads it (the masking of the pileup)
    row_amplicon: np.ndarray  # int64 per row: its amplicon
    row_left: np.ndarray      # bool per row: a left primer (else a right one)
    names: tuple             # per amplicon: the primer names' text before `_LEFT` / `_RIGHT`
    chrom: tuple
    pool: tuple              # column 5's text, `.` when absent
    start: np.ndarray        # int64: the smallest left-primer start
    end: np.ndarray          # int64: the largest right-primer end
    insert_start: np.ndarray  # int64: the largest left-primer end
    insert_end: np.ndarray    # int64: the smallest right-primer start

    @property
    def name(self) -> str:
        return self.primers.name

    @property
    def n_amplicons(self) -> int:
        return len(self.names)


@dataclass(frozen=True)
class AmpliconArrays:
    """The kdl_amplicons arrays of one alignment's contigs (include/kindel_b200.h, K12): the scheme's amplicons on those
    contigs in contig order, then start, then name -- a read's label is an index into this order -- and per contig and
    side the breakpoints of its primers' intervals, each with the label of the segment from it to the next breakpoint:
    the one amplicon whose primers cover it, -3 where primers of several amplicons do, -1 where none does (so the last
    breakpoint of a contig is always -1)."""

    amplicon: np.ndarray      # int64 [n]: index into the scheme
    contig: np.ndarray        # int32 [n]
    insert_start: np.ndarray  # int32 [n]
    insert_end: np.ndarray    # int32 [n]
    left_off: np.ndarray      # int64 [n_contigs + 1]
    left_at: np.ndarray       # int32: breakpoints, ascending per contig
    left_label: np.ndarray    # int32
    right_off: np.ndarray
    right_at: np.ndarray
    right_label: np.ndarray

    @property
    def n_contigs(self) -> int:
        return int(self.left_off.shape[0]) - 1

    @property
    def n_amplicons(self) -> int:
        return int(self.amplicon.shape[0])


UNPRIMED, MISPAIRED, AMBIGUOUS = -1, -2, -3  # K12's labels of a read that no one amplicon takes


def read_scheme(data: bytes, name: str = "<bed>") -> AmpliconScheme:
    """The amplicons of BED text (bytes, already inflated) whose column 4 names each primer `<amplicon>_LEFT...` or
    `<amplicon>_RIGHT...` (ARTIC / primalscheme style); column 5, when present, is the pool."""
    chrom, start, end, line, amp, left = [], [], [], [], [], []
    index, names, achrom, pools, pool_line = {}, [], [], [], []
    for k, fields, a, b in _bed_rows(data, name):
        if len(fields) < 4:
            raise ValueError("%s line %d: an amplicon scheme row needs a primer name in column 4" % (name, k))
        if a < 0 or a >= b:
            raise ValueError("%s line %d: interval [%d, %d) does not lie in 0 <= start < end" % (name, k, a, b))
        pname = fields[3].decode("utf-8", "replace")
        at = {tok: pname.find(tok) for tok in ("_LEFT", "_RIGHT") if tok in pname}
        if not at:
            raise ValueError("%s line %d: primer name %r has neither _LEFT nor _RIGHT" % (name, k, pname))
        tok = min(at, key=at.get)  # the first token in the name decides
        c = fields[0].decode("utf-8", "replace")
        key = (c, pname[:at[tok]])
        pool = fields[4].decode("utf-8", "replace") if len(fields) > 4 else "."
        j = index.get(key)
        if j is None:
            j = index[key] = len(names)
            names.append(key[1])
            achrom.append(c)
            pools.append(pool)
            pool_line.append(k)
        elif pools[j] != pool:
            raise ValueError("%s line %d: amplicon %r is in pool %r here and in pool %r on line %d"
                             % (name, k, key[1], pool, pools[j], pool_line[j]))
        chrom.append(c)
        start.append(a)
        end.append(b)
        line.append(k)
        amp.append(j)
        left.append(tok == "_LEFT")
    primers = PrimerSet(name, tuple(chrom), np.array(start, dtype=np.int64), np.array(end, dtype=np.int64),
                        np.array(line, dtype=np.int64))
    amp, left = np.array(amp, dtype=np.int64), np.array(left, dtype=bool)
    n = len(names)
    big = np.iinfo(np.int64).max
    lo, hi = np.full(n, big), np.full(n, -1, dtype=np.int64)           # start, end
    ins_lo, ins_hi = np.full(n, -1, dtype=np.int64), np.full(n, big)   # insert_start, insert_end
    np.minimum.at(lo, amp[left], primers.start[left])
    np.maximum.at(ins_lo, amp[left], primers.end[left])
    np.maximum.at(hi, amp[~left], primers.end[~left])
    np.minimum.at(ins_hi, amp[~left], primers.start[~left])
    for j in range(n):
        if hi[j] < 0 or lo[j] == big:
            raise ValueError("%s: amplicon %r on %r has no %s primer"
                             % (name, names[j], achrom[j], "left" if lo[j] == big else "right"))
        if ins_lo[j] >= ins_hi[j]:
            raise ValueError("%s: amplicon %r on %r leaves no insert between its primers (%d >= %d)"
                             % (name, names[j], achrom[j], ins_lo[j], ins_hi[j]))
    return AmpliconScheme(primers, amp, left, tuple(names), tuple(achrom), tuple(pools), lo, hi, ins_lo, ins_hi)


def load_scheme(path) -> AmpliconScheme:
    """The amplicons of the named primer BED at `path` (plain or gzip); see read_scheme."""
    data, name = _read_file(path)
    return read_scheme(data, name)


def as_scheme(scheme) -> AmpliconScheme:
    """An AmpliconScheme, or a path to load."""
    return scheme if isinstance(scheme, AmpliconScheme) else load_scheme(scheme)


def _segments(n_contigs, c, a, b, amp):
    """(offsets, breakpoints, labels) of the intervals [a, b) of amplicon amp on contig c (one side's primers)."""
    off = np.zeros(n_contigs + 1, dtype=np.int64)
    at, lab = [], []
    for k in range(n_contigs):
        on = c == k
        bp = np.unique(np.concatenate([a[on], b[on]]))
        owner = np.full(bp.shape[0], UNPRIMED, dtype=np.int64)
        for x, y, j in zip(np.searchsorted(bp, a[on]).tolist(), np.searchsorted(bp, b[on]).tolist(), amp[on].tolist()):
            seg = owner[x:y]
            owner[x:y] = np.where((seg == UNPRIMED) | (seg == j), j, AMBIGUOUS)
        at.append(bp)
        lab.append(owner)
        off[k + 1] = off[k] + bp.shape[0]
    i32 = lambda parts: np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0), dtype=np.int32)  # noqa: E731
    return off, i32(at), i32(lab)


def amplicon_arrays(scheme: AmpliconScheme, contig_names, contig_len) -> AmpliconArrays:
    """The K12 arrays of the scheme's amplicons on the given contigs (in their order); amplicons of other contigs are
    left out.  A row on them with start < 0, start >= end or end > its contig's length raises ValueError naming its
    line."""
    ps = scheme.primers
    on, c_of = _rows_on(ps, contig_names, contig_len)
    index = {nm: c for c, nm in enumerate(contig_names)}
    amp_c = np.array([index.get(nm, -1) for nm in scheme.chrom], dtype=np.int64)
    keep = np.flatnonzero(amp_c >= 0)
    order = keep[sorted(range(keep.shape[0]),
                        key=lambda i: (amp_c[keep[i]], scheme.start[keep[i]], scheme.names[keep[i]]))]
    label = np.full(scheme.n_amplicons, -1, dtype=np.int64)
    label[order] = np.arange(order.shape[0])
    n_contigs = len(contig_names)
    sides = []
    for side in (scheme.row_left, ~scheme.row_left):
        r = on & side
        sides.append(_segments(n_contigs, c_of[r], ps.start[r], ps.end[r], label[scheme.row_amplicon[r]]))
    i32 = lambda x: np.ascontiguousarray(x, dtype=np.int32)  # noqa: E731
    return AmpliconArrays(order.astype(np.int64), i32(amp_c[order]), i32(scheme.insert_start[order]),
                          i32(scheme.insert_end[order]), *sides[0], *sides[1])


def segment_label(off, at, label, c: int, x: int) -> int:
    """The label of cursor x on contig c in one side's segment arrays, as K12 searches them."""
    lo, hi = int(off[c]), int(off[c + 1])
    k = lo + int(np.searchsorted(at[lo:hi], x, side="right")) - 1
    return int(label[k]) if k >= lo else UNPRIMED
