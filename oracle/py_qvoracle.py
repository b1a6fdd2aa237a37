"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `variants --vcf --qual` (DESIGN.md section 1, twelfth
extension) as per-record loops over plain Python ints.

  EPS       EPS[q] = the integer nearest to 2^32 * 10^(-q / 10), q = 0..93, computed with `decimal`
  sums      per contig, qsum[k][p] (k = A, C, G, T) and emass[p]: every M/=/X base of a piled record whose query offset
            is not masked and whose letter is A, C, G or T adds its Phred q to qsum and EPS[min(q, 93)] to emass, at
            the reference's cursor (kindel.py:40-81, Python's negative index wrap included); clips, insertions, N and
            deletions add nothing
  masks     the records and masks of oracle/py_cvoracle.py (quality and primer masks) or, with mates, of
            oracle/py_moracle.py's ComposedMates (each R2's overlap bases added to its mask)
  records   the text of py_cvoracle / py_moracle with, on every record with a base ALT: QUAL = the largest AQ of the
            base ALTs, FILTER `lowqual` after `sor` when QUAL < min_qual, INFO ;BQ= (REF then ALTs, the mean Phred
            "%.1f", `.` without counted bases or for a non-base allele) and ;AQ= (per ALT, `.` for `*`); AQ from
            p = scipy.special.gammainc(k, emass / (3 * 2^32)), -10 log10(p) rounded half up, clamped to [0, 3000]
            (3000 when p == 0), 0 for k = 0

Nothing here imports kindel_b200."""
from __future__ import annotations

import math
from decimal import ROUND_HALF_EVEN, Decimal, getcontext

from . import py_cvoracle, py_moracle, py_poracle, samdecode


def eps_table():
    getcontext().prec = 60
    out = []
    for q in range(94):
        x = Decimal(2) ** 32 * Decimal(10) ** (Decimal(-q) / Decimal(10))
        out.append(int(x.to_integral_value(rounding=ROUND_HALF_EVEN)))
    return out


EPS = eps_table()


def walk(L, rec, qual, masked, qsum, emass):
    """Add one record's counted bases to qsum [4][L] and emass [L] (lists of ints)."""
    r, q = rec.pos - 1, 0
    for i, (n, op) in enumerate(rec.cigars):
        if op in ("M", "=", "X"):
            for _ in range(n):
                b = rec.seq[q].upper()
                if q not in masked and b in "ACGT":
                    s = r + L if r < 0 else r
                    qsum["ACGT".index(b)][s] += qual[q]
                    emass[s] += EPS[min(qual[q], 93)]
                r += 1
                q += 1
        elif op == "I":
            q += n
        elif op == "D":
            r += n
        elif op == "S":
            if i == 0:
                q += n
            else:
                for _ in range(n):
                    if r < L:
                        r += 1
                        q += 1


def quality_sums(path, min_base_quality=0, min_mapq=0, exclude_flags=0, primer_rows=None, mates=False):
    """{contig: (qsum [4][L], emass [L])} of one alignment file, with the masks of py_cvoracle / py_moracle."""
    header, records = samdecode.read_alignment_file(path)
    lengths = {sn[3:]: int(next(f for f in fl if f.startswith("LN:"))[3:]) for sn, fl in header["@SQ"].items()}
    mf = py_moracle.mate_fields(path) if mates else [None] * len(records)
    groups = {}
    for rec, m in zip(records, mf):
        groups.setdefault(rec.rname, []).append((rec, m))
    groups.pop("*", None)
    kept = []  # (contig, record, QNAME, role, PNEXT - 1, mask)
    for nm, items in groups.items():
        L = lengths[nm]
        iv = py_poracle.contig_intervals(primer_rows, nm) if primer_rows is not None else None
        for rec, m in items:
            if rec.flag & 0x4 or rec.mapq < min_mapq or rec.flag & exclude_flags or len(rec.seq) <= 1:
                continue
            mask = py_cvoracle.record_mask(rec, L, iv, min_base_quality)
            if mates:
                qn, same, pn = m
                kept.append((nm, rec, qn, py_moracle.role(rec.flag, same), pn, mask))
            else:
                kept.append((nm, rec, None, 0, -1, mask))
    if mates:
        for r2, r1 in py_moracle.pairs(lengths, [x[:5] for x in kept]).items():
            b, _, _ = py_moracle.overlap(kept[r2][1], py_moracle.covered(kept[r1][1], kept[r1][5]))
            kept[r2][5].update(b)
    out = {nm: ([[0] * lengths[nm] for _ in range(4)], [0] * lengths[nm]) for nm in groups}
    for nm, rec, _, _, _, mask in kept:
        if rec.qual is None:
            raise ValueError("a kept record without qualities")
        walk(lengths[nm], rec, rec.qual, mask, *out[nm])
    return out


def allele_quality(k, emass):
    from scipy.special import gammainc

    if k <= 0:
        return 0
    p = float(gammainc(float(k), float(emass) / (3.0 * 2.0 ** 32)))
    if p <= 0.0:
        return 3000
    return min(max(int(math.floor(-10.0 * math.log10(p) + 0.5)), 0), 3000)


_COL = {"A": 0, "C": 1, "G": 2, "T": 3, "*": 5}


def with_quality(text, sums, min_qual=None):
    """The VCF text of py_cvoracle / py_moracle (`text`) with the quality header lines and fields added."""
    lines = text.rstrip("\n").split("\n")
    head = [x for x in lines if x.startswith("#")]
    at = next(k for k, x in enumerate(head) if x.startswith(("##reference=", "##contig=", "##INFO=")))
    head.insert(at, "##kindelQual=model=poisson;min_qual=%s" % ("." if min_qual is None else min_qual))
    extra = ['##INFO=<ID=BQ,Number=R,Type=Float,Description="Mean base quality of the counted bases of REF and of '
             'each ALT allele">',
             '##INFO=<ID=AQ,Number=A,Type=Integer,Description="Phred-scaled probability that sequencing errors alone '
             'give the ALT base its count (Poisson model)">']
    if min_qual is not None:
        extra.append('##FILTER=<ID=lowqual,Description="QUAL is below %s">' % min_qual)
    head[-1:-1] = extra
    out = head
    for x in lines:
        if x.startswith("#"):
            continue
        f = x.split("\t")
        if f[7].startswith("INDEL"):
            out.append(x)
            continue
        alts = [_COL[a] for a in f[4].split(",")]
        if not any(k < 4 for k in alts):
            out.append(x)
            continue
        info = dict(kv.split("=", 1) for kv in f[7].split(";"))
        ad = [int(v) for v in info["AD"].split(",")]
        qsum, emass = sums[f[0]]
        p = int(f[1]) - 1
        ref = "ACGT".find(f[3])
        cols = [ref if ref >= 0 else None] + alts
        bq = ["." if k is None or k > 3 or c == 0 else "%.1f" % (qsum[k][p] / c) for k, c in zip(cols, ad)]
        aq = [allele_quality(c, emass[p]) if k < 4 else None for k, c in zip(alts, ad[1:])]
        qual = max(a for a in aq if a is not None)
        failed = [x for x in f[6].split(";") if x != "PASS"]
        if min_qual is not None and qual < min_qual:
            failed.append("lowqual")
        f[5] = str(qual)
        f[6] = ";".join(failed) if failed else "PASS"
        f[7] += ";BQ=%s;AQ=%s" % (",".join(bq), ",".join("." if a is None else str(a) for a in aq))
        out.append("\t".join(f))
    return "\n".join(out) + "\n"
