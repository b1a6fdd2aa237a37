"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `variants --vcf --strand` (an extension: the reference has
no variant caller), as per-record and per-position loops over plain Python ints, floats, strings and dicts.

Records are objects with .pos (1-based), .mapped, .seq, .cigars ((length, op letter) pairs) and the strand: .flag
(oracle/samdecode.py's records; 0x10 = reverse) or .reverse (`Rec` below).  The forward-strand records and the
reverse-strand records are piled SEPARATELY with py_oracle.pileup (the reference's own loop), and so are their
deletion events (py_rvoracle.deletion_events): nothing is derived by subtraction.  The records of both strands
together give the sites and the totals, by the rules of py_rvoracle (against a reference) or of the sites-only VCF
(without one: REF = the most frequent of A, C, G, T, N, deletion; ALT the other alleles among A, C, G, T, deletion
that pass both thresholds).  Then per record:

  ADF / ADR   forward / reverse count of REF and of each ALT.  Without a reference: the strand pileups' counts of the
              AD columns.  Against a reference, SNV: the same, REF 0 where the reference base is not A, C, G or T;
              indel: the ALT's carriers on that strand, REF max(DP_s - AO_s, 0) with DP_s the record's DP (depth(r)
              or DPa) in strand s's pileup
  SOR         per ALT k: t00 = ADF[0] + 1, t01 = ADR[0] + 1, t10 = ADF[k] + 1, t11 = ADR[k] + 1,
              log((t00/t01)(t11/t10) + (t01/t00)(t10/t11)) + log(min(t00,t01)/max(t00,t01))
              - log(min(t10,t11)/max(t10,t11)), written "%.3f"
  FILTER      `sor` when max_sor is set and some ALT's SOR, as written, is above it; else PASS

Nothing here imports kindel_b200."""
from __future__ import annotations

import math

from .py_oracle import pileup
from .py_rvoracle import _af, _share, deletion_events, ref_letters

_NUC = "ACGT"


class Rec:
    __slots__ = ("pos", "mapped", "seq", "cigars", "reverse")

    def __init__(self, pos, seq, cigars, reverse, mapped=True):
        self.pos, self.seq, self.cigars, self.reverse, self.mapped = pos, seq, cigars, bool(reverse), mapped


def is_reverse(rec) -> bool:
    return bool(rec.reverse) if hasattr(rec, "reverse") else bool(rec.flag & 0x10)


def sor(adf, adr, k):
    t00, t01, t10, t11 = adf[0] + 1.0, adr[0] + 1.0, adf[k] + 1.0, adr[k] + 1.0
    ratio = (t00 / t01) * (t11 / t10) + (t01 / t00) * (t10 / t11)
    return math.log(ratio) + math.log(min(t00, t01) / max(t00, t01)) - math.log(min(t10, t11) / max(t10, t11))


def strand_tail(adf, adr, max_sor):
    """(FILTER, ";ADF=..;ADR=..;SOR=..")."""
    sors = ["%.3f" % sor(adf, adr, k) for k in range(1, len(adf))]
    filt = "PASS"
    if max_sor is not None and any(float(x) > max_sor for x in sors):
        filt = "sor"
    return filt, ";ADF=%s;ADR=%s;SOR=%s" % (",".join(map(str, adf)), ",".join(map(str, adr)), ",".join(sors))


class _Piles:
    """The pileups of one contig: all records, the forward ones, the reverse ones."""

    def __init__(self, L, records):
        self.L = L
        self.recs = [r for r in records if r.mapped and len(r.seq) > 1]
        self.fwd = [r for r in self.recs if not is_reverse(r)]
        self.rev = [r for r in self.recs if is_reverse(r)]
        self.all, self.f, self.r = pileup(L, self.recs), pileup(L, self.fwd), pileup(L, self.rev)

    def counts(self, p, pos):
        if pos < self.L:
            w = p.weights[pos]
            return [w["A"], w["C"], w["G"], w["T"], w["N"], p.deletions[pos]]
        return [0, 0, 0, 0, 0, p.deletions[pos]]

    def depth(self, p, pos):
        return sum(self.counts(p, pos))


def sites_lines(name, L, records, abs_threshold, rel_threshold, max_sor=None):
    """The data lines of `variants --vcf --strand` (no reference) of one contig of length L."""
    P = _Piles(L, records)
    out = []
    for pos in range(L):
        t = P.counts(P.all, pos)
        d = sum(t)
        top = max(range(6), key=lambda k: (t[k], -k))  # the first maximum
        alts = [k for k in (0, 1, 2, 3, 5) if k != top and t[k] > abs_threshold and _share(t[k], d) > rel_threshold]
        if not alts:
            continue
        ks = [top] + alts
        tf, tr = P.counts(P.f, pos), P.counts(P.r, pos)
        filt, tail = strand_tail([tf[k] for k in ks], [tr[k] for k in ks], max_sor)
        out.append("%s\t%d\t.\t%s\t%s\t.\t%s\tDP=%d;AD=%s;AF=%s%s" % (
            name, pos + 1, _NUC[top] if top < 4 and d > 0 else "N", ",".join("ACGT*"[min(k, 4)] for k in alts), filt,
            d, ",".join(str(t[k]) for k in ks), ",".join(_af(t[k], d) for k in alts), tail))
    return out


def reference_records(name, ref, records, abs_threshold, rel_threshold, max_sor=None):
    """[(POS, kind, deletion length, insertion slot, rank, line)] of `variants --vcf --reference --strand` of one
    contig; ref: its reference text (length L)."""
    L = len(ref)
    ref = ref_letters(ref)
    P = _Piles(L, records)
    out = []

    def indel_tail(dp_f, dp_r, ao_f, ao_r):
        return strand_tail([max(dp_f - ao_f, 0), ao_f], [max(dp_r - ao_r, 0), ao_r], max_sor)

    for pos in range(L):
        t = P.counts(P.all, pos)
        d = sum(t)
        g = _NUC.find(ref[pos])
        alts = [k for k in range(4) if k != g and t[k] > abs_threshold and _share(t[k], d) > rel_threshold]
        if alts:
            tf, tr = P.counts(P.f, pos), P.counts(P.r, pos)
            ad = [t[g] if g >= 0 else 0] + [t[k] for k in alts]
            filt, tail = strand_tail([tf[g] if g >= 0 else 0] + [tf[k] for k in alts],
                                     [tr[g] if g >= 0 else 0] + [tr[k] for k in alts], max_sor)
            out.append((pos + 1, 0, 0, 0, 0, "%s\t%d\t.\t%s\t%s\t.\t%s\tDP=%d;AD=%s;AF=%s%s" % (
                name, pos + 1, ref[pos], ",".join(_NUC[k] for k in alts), filt, d, ",".join(map(str, ad)),
                ",".join(_af(t[k], d) for k in alts), tail)))
    if L > 0:
        for pos in range(L + 1):
            at = pos - 1 if pos >= 1 else 0
            dpa = P.depth(P.all, at)
            for rank, (s, c) in enumerate(P.all.insertions[pos].items()):
                if not s or not (c > abs_threshold and _share(c, dpa) > rel_threshold):
                    continue
                filt, tail = indel_tail(P.depth(P.f, at), P.depth(P.r, at), P.f.insertions[pos].get(s, 0),
                                        P.r.insertions[pos].get(s, 0))
                s = "".join(ch if ch in _NUC + "N" else "N" for ch in s)
                rec = (pos, ref[pos - 1], ref[pos - 1] + s) if pos >= 1 else (1, ref[0], s + ref[0])
                out.append((rec[0], 2, 0, pos, rank, "%s\t%d\t.\t%s\t%s\t.\t%s\tINDEL;DP=%d;AO=%d;AF=%s%s" % (
                    name, rec[0], rec[1], rec[2], filt, dpa, c, _af(c, dpa), tail)))

    def groups(recs):
        out = {}
        for ev in deletion_events(L, recs):
            out[ev] = out.get(ev, 0) + 1
        return out

    g_all, g_f, g_r = groups(P.recs), groups(P.fwd), groups(P.rev)
    for (r, n), c in g_all.items():
        d = P.depth(P.all, r)
        if not (c > abs_threshold and _share(c, d) > rel_threshold):
            continue
        if r >= 1:
            rec = (r, ref[r - 1:r + n], ref[r - 1])
        elif n < L:
            rec = (1, ref[0:n + 1], ref[n])
        else:
            continue
        filt, tail = indel_tail(P.depth(P.f, r), P.depth(P.r, r), g_f.get((r, n), 0), g_r.get((r, n), 0))
        out.append((rec[0], 1, n, 0, 0, "%s\t%d\t.\t%s\t%s\t.\t%s\tINDEL;DP=%d;AO=%d;AF=%s%s" % (
            name, rec[0], rec[1], rec[2], filt, d, c, _af(c, d), tail)))
    out.sort(key=lambda x: x[:5])
    return out


def vcf_lines(contigs, abs_threshold, rel_threshold, max_sor=None, reference=False):
    """The data lines: contigs = [(name, L, records)] without a reference, [(name, reference text, records)] with
    reference=True, in the file's contig order."""
    lines = []
    for name, L_or_ref, records in contigs:
        if reference:
            lines += [x[5] for x in reference_records(name, L_or_ref, records, abs_threshold, rel_threshold, max_sor)]
        else:
            lines += sites_lines(name, L_or_ref, records, abs_threshold, rel_threshold, max_sor)
    return lines


def header_lines(max_sor=None):
    """The lines variants_vcf adds to its header with strand on."""
    out = ["##kindelStrand=max_sor=%s" % ("." if max_sor is None else max_sor)]
    return out + (['##FILTER=<ID=sor,Description="The strand odds ratio of an ALT allele is above %s">' % max_sor]
                  if max_sor is not None else [])

