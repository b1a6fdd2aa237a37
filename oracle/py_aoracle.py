"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `kindel amplicons` (an extension: the reference has no such
command): which amplicon of a named primer scheme each read comes from, and the depth of each amplicon's insert, as
plain loops over Python ints and lists.

Scheme rows are (chrom, start, end, amplicon, side) with side "L" or "R": the amplicon is a primer name's text before
its first `_LEFT` or `_RIGHT`, which also gives the side (read_scheme_rows).  Per amplicon, start / end are the
smallest left-primer start and the largest right-primer end, insert_start / insert_end the largest left-primer end and
the smallest right-primer start.

Per record (oracle/samdecode.py), on a contig of length L:
  walk    the reference's loop (kindel.py:40-81) for the cursors alone -- M/=/X and D advance r_pos, an S that is op #0
          does not, any later S advances it while r_pos < L; I, N, H, P do not
  ends    s, e = the cursors of the first and the last M/=/X base; a record without one is unprimed
  sides   left = the amplicons with a left primer [a, b) with a <= s < b, right = those with a right primer holding e
          (every interval of the contig is tested; a cursor outside [0, L) is in no primer)
  label   -1 when both are empty, -3 when either names two or more amplicons, -2 when they name two different ones,
          else the one amplicon named, as its index in amplicon_table's order (contig order, then start, then name)

The insert statistics sum columns 0-3 of a count table (the oracle's or the product's) position by position.  Nothing
here imports kindel_b200."""
from __future__ import annotations

import numpy as np

from . import samdecode

UNPRIMED, MISPAIRED, AMBIGUOUS = -1, -2, -3


def split_name(name):
    """(amplicon, side) of a primer name, or None when it has neither token."""
    hits = [(name.find(tok), tok) for tok in ("_LEFT", "_RIGHT") if tok in name]
    if not hits:
        return None
    at, tok = min(hits)
    return name[:at], "L" if tok == "_LEFT" else "R"


def read_scheme_rows(path):
    """[(chrom, start, end, amplicon, side)] of a plain-text named BED, read the simplest way."""
    rows = []
    with open(path) as fh:
        for line in fh:
            line = line.rstrip("\r\n")
            if not line.strip() or line.startswith(("#", "track", "browser")):
                continue
            f = line.split("\t") if "\t" in line else line.split()
            amp, side = split_name(f[3])
            rows.append((f[0], int(f[1]), int(f[2]), amp, side))
    return rows


def amplicon_table(rows, contig_names):
    """[(contig, amplicon, start, end, insert_start, insert_end)] of the amplicons on contig_names, in contig order,
    then start, then name."""
    groups = {}
    for ch, a, b, amp, sd in rows:
        if ch in contig_names:
            groups.setdefault((ch, amp), []).append((a, b, sd))
    out = []
    for (c, nm), prs in groups.items():
        left = [(a, b) for a, b, sd in prs if sd == "L"]
        right = [(a, b) for a, b, sd in prs if sd == "R"]
        out.append((c, nm, min(a for a, _ in left), max(b for _, b in right), max(b for _, b in left),
                    min(a for a, _ in right)))
    out.sort(key=lambda t: (contig_names.index(t[0]), t[2], t[1]))
    return out


def ends(rec, L):
    """(s, e) of the record's first and last M/=/X base, or None."""
    r_pos = rec.pos - 1
    s = e = None
    for i, (length, op) in enumerate(rec.cigars):
        if op in ("M", "=", "X"):
            if length > 0:
                if s is None:
                    s = r_pos
                e = r_pos + length - 1
            r_pos += length
        elif op == "D":
            r_pos += length
        elif op == "S" and i != 0:
            for _ in range(length):
                if r_pos < L:
                    r_pos += 1
    return None if s is None else (s, e)


def label(se, L, rows_c, index):
    """The label of a read with ends se (or None) on a contig of length L; rows_c: that contig's scheme rows, index:
    {amplicon name: its index}."""
    if se is None:
        return UNPRIMED
    s, e = se
    left = {amp for _, a, b, amp, sd in rows_c if sd == "L" and a <= s < b and 0 <= s < L}
    right = {amp for _, a, b, amp, sd in rows_c if sd == "R" and a <= e < b and 0 <= e < L}
    if not left and not right:
        return UNPRIMED
    if len(left) > 1 or len(right) > 1:
        return AMBIGUOUS
    if left and right and left != right:
        return MISPAIRED
    return index[next(iter(left or right))]


def kept_records(path, contig_names, min_mapq=0, exclude_flags=0):
    """({name: L}, [(contig name, record)]) of the records the engine keeps under the read filters, in its read order:
    by contig in `contig_names` order, file order inside a contig."""
    header, records = samdecode.read_alignment_file(path)
    lengths = {}
    for sn, fields in header["@SQ"].items():
        ln = next(f for f in fields if f.startswith("LN:"))
        lengths[sn[3:]] = int(ln[3:])
    groups = {}
    for r in records:
        groups.setdefault(r.rname, []).append(r)
    keep = lambda r: (r.mapped and len(r.seq) > 1 and r.mapq >= min_mapq  # noqa: E731
                      and not (r.flag & exclude_flags))
    return lengths, [(nm, r) for nm in contig_names for r in groups.get(nm, []) if keep(r)]


def labels_by_read(path, contig_names, rows, min_mapq=0, exclude_flags=0):
    """int64 labels of the kept records in the engine's read order."""
    lengths, recs = kept_records(path, contig_names, min_mapq, exclude_flags)
    table = amplicon_table(rows, contig_names)
    index = {(t[0], t[1]): k for k, t in enumerate(table)}
    out = []
    for nm, r in recs:
        rows_c = [x for x in rows if x[0] == nm]
        idx = {amp: k for (c, amp), k in index.items() if c == nm}
        out.append(label(ends(r, lengths[nm]), lengths[nm], rows_c, idx))
    return np.array(out, dtype=np.int64)


def labels_of_batch(batch, rows):
    """The labels of a large flattened batch (any object with its attributes: contig_names, contig_len,
    contig_read_off, ref_start, seq_len, cig_off, cigar): each contig's primers are painted position by position,
    interval by interval (a position one amplicon's primers cover gets its index, one that several cover -3), and a
    read's ends are looked up there; a read with a CIGAR other than one M op of its SEQ length goes through ends()."""
    names = list(batch.contig_names)
    table = amplicon_table(rows, names)
    index = {(t[0], t[1]): k for k, t in enumerate(table)}
    n = int(np.asarray(batch.ref_start).shape[0])
    cig_off = np.asarray(batch.cig_off, dtype=np.int64)
    cigar = np.asarray(batch.cigar, dtype=np.int64)
    lseq = np.asarray(batch.seq_len, dtype=np.int64)
    start = np.asarray(batch.ref_start, dtype=np.int64)
    n_ops = np.diff(cig_off)
    first = cigar[np.minimum(cig_off[:-1], max(cigar.shape[0] - 1, 0))] if n and cigar.shape[0] else np.zeros(n, np.int64)
    one_m = (n_ops == 1) & np.isin(first & 15, (0, 7, 8)) & ((first >> 4) == lseq) & (lseq > 0)
    out = np.full(n, UNPRIMED, dtype=np.int64)
    rows_by_contig = {}
    for r in rows:
        rows_by_contig.setdefault(r[0], []).append(r)
    for c, nm in enumerate(names):
        L = int(batch.contig_len[c])
        paint = {}
        for side in ("L", "R"):
            own = np.full(L + 1, UNPRIMED, dtype=np.int64)  # (L: a cursor past the contig, in no primer)
            for ch, a, b, amp, sd in rows_by_contig.get(nm, []):
                if sd == side:
                    k = index[(nm, amp)]
                    seg = own[a:b]
                    own[a:b] = np.where((seg == UNPRIMED) | (seg == k), k, AMBIGUOUS)
            paint[side] = own
        lo, hi = int(batch.contig_read_off[c]), int(batch.contig_read_off[c + 1])
        s, e = start[lo:hi].copy(), start[lo:hi] + lseq[lo:hi] - 1
        has = one_m[lo:hi].copy()
        for r in (np.flatnonzero(~one_m[lo:hi]) + lo).tolist():
            ops = cigar[cig_off[r]:cig_off[r + 1]].tolist()
            rec = samdecode.Record("", 0, nm, int(start[r]) + 1, "N" * int(lseq[r]),
                                   [(w >> 4, "MIDNSHP=X"[w & 15] if (w & 15) < 9 else None) for w in ops])
            se = ends(rec, L)
            if se is not None:
                s[r - lo], e[r - lo], has[r - lo] = se[0], se[1], True
        inside = lambda x: (x >= 0) & (x < L)  # noqa: E731
        left = np.where(has & inside(s), paint["L"][np.clip(s, 0, L)], UNPRIMED)
        right = np.where(has & inside(e), paint["R"][np.clip(e, 0, L)], UNPRIMED)
        lab = np.where(left >= 0, left, right)
        lab = np.where((left >= 0) & (right >= 0) & (left != right), MISPAIRED, lab)
        lab = np.where((left == AMBIGUOUS) | (right == AMBIGUOUS), AMBIGUOUS, lab)
        out[lo:hi] = lab
    return out


def insert_stats(counts, contig_slot, contig_names, table, min_depth):
    """[(sum, lowest, covered)] of A+C+G+T (columns 0-3 of `counts`) over each amplicon's insert."""
    out = []
    for c, _, _, _, i0, i1 in table:
        base = int(contig_slot[contig_names.index(c)])
        d = np.asarray(counts[0:4, base + i0:base + i1], dtype=np.int64).sum(axis=0)
        out.append((int(d.sum()), int(d.min()), int((d >= min_depth).sum())))
    return out
