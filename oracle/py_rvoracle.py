"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `variants --vcf --reference` (an extension: the reference
has no variant caller), as per-record and per-position loops over plain Python ints, floats, strings and dicts.

Records are objects with .pos (1-based), .mapped, .seq and .cigars ((length, op letter) pairs): oracle/samdecode.py's,
or py_oracle.Rec.  The pileup of a contig is py_oracle.pileup (the reference's own loop, Python index wrap included);
this file adds what the count table does not keep and the VCF rules:

  deletion events   each D op of length n >= 1 at cursor r with 0 <= r and r + n <= L, the cursor moved as in the
                    reference's loop (M/=/X and D advance; an S that is op #0 does not; any later S advances while
                    r < L; I, N, H, P do not)
  SNV               at position p < L with six counts t (A, C, G, T, N, deletions), depth = their sum and reference
                    base g: every base k of A, C, G, T other than g with t[k] > abs and t[k] / depth > rel (0 at depth 0)
  insertion         string s (not empty) of insertions[p], 0 <= p <= L, count c: c > abs and c / DPa > rel, DPa =
                    depth(p - 1) for p >= 1 and depth(0) for p = 0; depth(L) counts only the deletions at slot L
  deletion          event (r, n) with count c: c > abs and c / depth(r) > rel

and writes the lines as kindel_b200/vcf.py's docstring of records states them.  Reference letters are
A, C, G, T or N (anything else reads as N).  Nothing here imports kindel_b200."""
from __future__ import annotations

import numpy as np

from .py_oracle import pileup

_NUC = "ACGT"


def deletion_events(ref_len, records):
    """[(r, n)] of every deletion event, in record order and then op order."""
    out = []
    for rec in records:
        if not rec.mapped or len(rec.seq) <= 1:
            continue
        r = rec.pos - 1
        for i, (n, op) in enumerate(rec.cigars):
            if op in ("M", "=", "X"):
                r += n
            elif op == "D":
                if n >= 1 and r >= 0 and r + n <= ref_len:
                    out.append((r, n))
                r += n
            elif op == "S" and i != 0:
                for _ in range(n):
                    if r < ref_len:
                        r += 1
    return out


def ref_letters(seq):
    return "".join(ch if ch in _NUC else "N" for ch in seq.upper())


def _share(c, d):
    return c / d if d > 0 else 0.0


def _af(c, d):
    return repr(float(np.round(np.float64(_share(c, d)), 4)))


def contig_records(name, ref, records, abs_threshold, rel_threshold):
    """[(POS, kind, deletion length, insertion slot, rank, line)] of one contig; ref: its reference text (length L)."""
    L = len(ref)
    ref = ref_letters(ref)
    p = pileup(L, records)

    def counts(pos):
        if pos < L:
            w = p.weights[pos]
            return [w["A"], w["C"], w["G"], w["T"], w["N"], p.deletions[pos]]
        return [0, 0, 0, 0, 0, p.deletions[pos]]

    def depth(pos):
        return sum(counts(pos))

    out = []
    for pos in range(L):
        t = counts(pos)
        d = sum(t)
        g = _NUC.find(ref[pos])
        alts = [k for k in range(4) if k != g and t[k] > abs_threshold and _share(t[k], d) > rel_threshold]
        if alts:
            ad = [t[g] if g >= 0 else 0] + [t[k] for k in alts]
            out.append((pos + 1, 0, 0, 0, 0, "%s\t%d\t.\t%s\t%s\t.\tPASS\tDP=%d;AD=%s;AF=%s" % (
                name, pos + 1, ref[pos], ",".join(_NUC[k] for k in alts), d, ",".join(map(str, ad)),
                ",".join(_af(t[k], d) for k in alts))))
    if L > 0:
        for pos in range(L + 1):
            dpa = depth(pos - 1) if pos >= 1 else depth(0)
            for rank, (s, c) in enumerate(p.insertions[pos].items()):
                if not s or not (c > abs_threshold and _share(c, dpa) > rel_threshold):
                    continue
                s = "".join(ch if ch in _NUC + "N" else "N" for ch in s)
                if pos >= 1:
                    rec = (pos, ref[pos - 1], ref[pos - 1] + s)
                else:
                    rec = (1, ref[0], s + ref[0])
                out.append((rec[0], 2, 0, pos, rank, "%s\t%d\t.\t%s\t%s\t.\tPASS\tINDEL;DP=%d;AO=%d;AF=%s" % (
                    name, rec[0], rec[1], rec[2], dpa, c, _af(c, dpa))))
    groups = {}
    for ev in deletion_events(L, records):
        groups[ev] = groups.get(ev, 0) + 1
    for (r, n), c in groups.items():
        d = depth(r)
        if not (c > abs_threshold and _share(c, d) > rel_threshold):
            continue
        if r >= 1:
            rec = (r, ref[r - 1:r + n], ref[r - 1])
        elif n < L:
            rec = (1, ref[0:n + 1], ref[n])
        else:
            continue
        out.append((rec[0], 1, n, 0, 0, "%s\t%d\t.\t%s\t%s\t.\tPASS\tINDEL;DP=%d;AO=%d;AF=%s" % (
            name, rec[0], rec[1], rec[2], d, c, _af(c, d))))
    out.sort(key=lambda x: x[:5])
    return out


def vcf_lines(contigs, abs_threshold, rel_threshold):
    """The data lines of the VCF: contigs = [(name, reference text, records)] in the file's contig order."""
    lines = []
    for name, ref, records in contigs:
        lines += [x[5] for x in contig_records(name, ref, records, abs_threshold, rel_threshold)]
    return lines


def sites(table, contig_slot, contig_len, ref_codes, abs_threshold, rel_threshold):
    """K6r restated over a count table [>= 7, n_slots] and reference codes (0-3 = A, C, G, T, 4 = other): (slot
    int64[n], counts int32[7, n], dpa int64[n], mask uint8[n]) in ascending slot order -- bits 0-3 the SNV bases,
    bit 6 the insertion candidate (t6 > abs and t6 / DPa > rel at 0 <= p <= L)."""
    cols = [np.asarray(table[k]).tolist() for k in range(7)]
    codes = np.asarray(ref_codes).tolist()
    out = []

    def depth(s):
        return cols[0][s] + cols[1][s] + cols[2][s] + cols[3][s] + cols[4][s] + cols[5][s]

    for s0, L in zip(np.asarray(contig_slot).tolist(), np.asarray(contig_len).tolist()):
        for s in range(s0, s0 + L + 1):
            p = s - s0
            t = [cols[k][s] for k in range(7)]
            d = depth(s)
            mask = 0
            if p < L:
                for k in range(4):
                    if k != codes[s] and t[k] > abs_threshold and _share(t[k], d) > rel_threshold:
                        mask |= 1 << k
            dpa = depth(s - 1) if p >= 1 else d
            if t[6] > abs_threshold and _share(t[6], dpa) > rel_threshold:
                mask |= 1 << 6
            if mask:
                out.append((s, t, dpa, mask))
    counts = np.array([x[1] for x in out], dtype=np.int32).reshape(-1, 7).T.copy()
    return (np.array([x[0] for x in out], dtype=np.int64), counts, np.array([x[2] for x in out], dtype=np.int64),
            np.array([x[3] for x in out], dtype=np.uint8))
