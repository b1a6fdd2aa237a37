"""TEST INFRASTRUCTURE ONLY -- an independent restatement of the multi-sample VCF (`kindel variants --vcf a.bam b.bam
...`, DESIGN.md section 1, eleventh extension) as per-position loops over plain Python ints, strings and dicts.

Each sample is piled on its own by the existing oracles (py_cvoracle.Composed, or py_moracle.ComposedMates with
`--mask-overlaps`), or given as a count table (from_table: the pooled mode needs nothing else).  Its tables are held by
contig NAME, never by slot: a contig a sample lacks has zero counts there.  The contigs are the union of the samples'
contigs: the first sample's order, then each contig a later sample shows first.  Per position:

  pooled      P = the samples' counts summed, top = the first maximum of P; allele k (A, C, G, T, deletion; k != top)
              is an ALT when some sample has count > a and count / depth > r; REF the top allele's letter (N for N, a
              deletion or depth 0); INFO DP, AD (REF, then the ALTs) and AF over P
  reference   SNV alleles k != the reference base that pass in some sample; insertion strings at p (0 <= p <= L) that
              pass in some sample against its own DPa, in the order: first sample that has the string, then its
              first-seen rank there; deletions (r, n) that pass in some sample against its depth at r
  FORMAT      DP:AD:AF per sample -- SNV / allele: the sample's depth, its counts of REF and the ALTs, the ALTs'
              shares; indel: DP the sample's depth at r (deletion) or DPa (insertion), AD max(DP - AO, 0),AO

Nothing here imports kindel_b200, and nothing is shared with kindel_b200/cohort.py."""
from __future__ import annotations

from .py_cvoracle import Composed
from .py_moracle import ComposedMates
from .py_rvoracle import _af, _share, ref_letters

_NUC = "ACGT"


class Sample:
    """One sample's tables by contig name: counts(name, pos) -> [A, C, G, T, N, deletions], insertions(name, pos) ->
    {string: count} in first-seen order, deletions(name) -> {(r, n): count}."""

    def __init__(self, contigs, counts, insertions=None, deletions=None):
        self.contigs = list(contigs)  # [(name, L)] in the sample's order
        self._counts, self._ins, self._del = counts, insertions or {}, deletions or {}

    @classmethod
    def from_path(cls, path, min_base_quality=0, min_mapq=0, exclude_flags=0, primer_rows=None, mates=False):
        comp = (ComposedMates if mates else Composed)(path, min_base_quality, min_mapq, exclude_flags, primer_rows)
        piles = {nm: comp.piles[nm][0] for nm, _ in comp.contigs}
        return cls(comp.contigs, {nm: p.counts for nm, p in piles.items()},
                   {nm: p.insertions for nm, p in piles.items()}, {nm: p.del_events for nm, p in piles.items()})

    @classmethod
    def from_table(cls, names, lengths, slots, table):
        """A count table [7][n_slots] laid out at `slots`: no insertion strings and no deletion events, so the records
        it gives are the pooled mode's; site_bits reads its column 6 (insertion ops)."""
        cols = {}
        for nm, L, s0 in zip(names, lengths, slots):
            cols[nm] = [[int(x) for x in table[k][int(s0):int(s0) + int(L) + 1]] for k in range(7)]
        smp = cls(list(zip(names, [int(x) for x in lengths])),
                  {nm: (lambda c: lambda pos: [col[pos] for col in c[:6]])(c) for nm, c in cols.items()})
        smp._ops = {nm: c[6] for nm, c in cols.items()}
        return smp

    def ins_ops(self, nm, pos):
        c = getattr(self, "_ops", {}).get(nm)
        return c[pos] if c is not None else 0

    def counts(self, nm, pos):
        f = self._counts.get(nm)
        return f(pos) if f is not None else [0] * 6

    def depth(self, nm, pos):
        return sum(self.counts(nm, pos))

    def insertions(self, nm, pos):
        d = self._ins.get(nm)
        return d[pos] if d is not None else {}

    def deletions(self, nm):
        return self._del.get(nm, {})


def contigs_of(samples):
    out, seen = [], set()
    for smp in samples:
        for nm, L in smp.contigs:
            if nm not in seen:
                seen.add(nm)
                out.append((nm, L))
    return out


def site_bits(samples, a, r, reference=None):
    """[(contig, p, bits)] of every slot with a bit set, contigs in union order, p ascending (p = L is the slot behind
    the contig): pooled, bit k (k = 0..5, N included) for an allele other than the pooled top that passes in some
    sample; with reference ({contig: text}), bits 0-3 SNV alleles other than the reference base and bit 6 when some
    sample's insertion ops pass against its DPa."""
    out = []
    for nm, L in contigs_of(samples):
        for pos in range(L + 1):
            bits = 0
            ts = [smp.counts(nm, pos) for smp in samples]
            if reference is None:
                if pos == L:
                    continue
                P = [sum(t[k] for t in ts) for k in range(6)]
                top = max(range(6), key=lambda k: (P[k], -k))
                for k in range(6):
                    if k != top and any(_passes(t[k], sum(t), a, r) for t in ts):
                        bits |= 1 << k
            else:
                g = _NUC.find(ref_letters(reference[nm][pos])) if pos < L else -1
                for k in range(4):
                    if pos < L and k != g and any(_passes(t[k], sum(t), a, r) for t in ts):
                        bits |= 1 << k
                at = pos - 1 if pos >= 1 else 0
                if any(_passes(smp.ins_ops(nm, pos), smp.depth(nm, at), a, r) for smp in samples):
                    bits |= 64
            if bits:
                out.append((nm, pos, bits))
    return out


def _fields(dp, ad):
    return "%d:%s:%s" % (dp, ",".join(str(x) for x in ad), ",".join(_af(x, dp) for x in ad[1:]))


def _passes(c, d, a, r):
    return c > a and _share(c, d) > r


def pooled_lines(samples, nm, L, a, r):
    out = []
    for pos in range(L):
        ts = [smp.counts(nm, pos) for smp in samples]
        P = [sum(t[k] for t in ts) for k in range(6)]
        d = sum(P)
        top = max(range(6), key=lambda k: (P[k], -k))
        alts = [k for k in (0, 1, 2, 3, 5) if k != top and any(_passes(t[k], sum(t), a, r) for t in ts)]
        if not alts:
            continue
        ks = [top] + alts
        cols = [_fields(sum(t), [t[k] for k in ks]) for t in ts]
        out.append("\t".join(["%s\t%d\t.\t%s\t%s\t.\tPASS\tDP=%d;AD=%s;AF=%s\tDP:AD:AF" % (
            nm, pos + 1, _NUC[top] if top < 4 and d > 0 else "N", ",".join("ACGT*"[min(k, 4)] for k in alts), d,
            ",".join(str(P[k]) for k in ks), ",".join(_af(P[k], d) for k in alts))] + cols))
    return out


def reference_lines(samples, nm, ref, a, r):
    L = len(ref)
    ref = ref_letters(ref)
    out = []
    for pos in range(L):
        ts = [smp.counts(nm, pos) for smp in samples]
        g = _NUC.find(ref[pos])
        alts = [k for k in range(4) if k != g and any(_passes(t[k], sum(t), a, r) for t in ts)]
        if not alts:
            continue
        ads = [[t[g] if g >= 0 else 0] + [t[k] for k in alts] for t in ts]
        tot = [sum(x[j] for x in ads) for j in range(len(alts) + 1)]
        d = sum(sum(t) for t in ts)
        out.append((pos + 1, 0, 0, 0, 0, "\t".join(["%s\t%d\t.\t%s\t%s\t.\tPASS\tDP=%d;AD=%s;AF=%s\tDP:AD:AF" % (
            nm, pos + 1, ref[pos], ",".join(_NUC[k] for k in alts), d, ",".join(map(str, tot)),
            ",".join(_af(x, d) for x in tot[1:]))] + [_fields(sum(t), x) for t, x in zip(ts, ads)])))
    if L > 0:
        for pos in range(L + 1):
            at = pos - 1 if pos >= 1 else 0
            dpa = [smp.depth(nm, at) for smp in samples]
            dicts = [smp.insertions(nm, pos) for smp in samples]
            order = []
            for dct in dicts:
                for s in dct:
                    if s not in order:
                        order.append(s)
            for rank, s in enumerate(order):
                ao = [dct.get(s, 0) for dct in dicts]
                if not s or not any(_passes(c, d, a, r) for c, d in zip(ao, dpa)):
                    continue
                alt = "".join(ch if ch in _NUC + "N" else "N" for ch in s)
                rec = (pos, ref[pos - 1], ref[pos - 1] + alt) if pos >= 1 else (1, ref[0], alt + ref[0])
                out.append((rec[0], 2, 0, pos, rank, "\t".join(
                    ["%s\t%d\t.\t%s\t%s\t.\tPASS\tINDEL;DP=%d;AO=%d;AF=%s\tDP:AD:AF" % (
                        nm, rec[0], rec[1], rec[2], sum(dpa), sum(ao), _af(sum(ao), sum(dpa)))]
                    + [_fields(d, [max(d - c, 0), c]) for c, d in zip(ao, dpa)])))
    keys = set()
    for smp in samples:
        for (rr, n), c in smp.deletions(nm).items():
            if _passes(c, smp.depth(nm, rr), a, r):
                keys.add((rr, n))
    for rr, n in keys:
        if rr >= 1:
            rec = (rr, ref[rr - 1:rr + n], ref[rr - 1])
        elif n < L:
            rec = (1, ref[0:n + 1], ref[n])
        else:
            continue
        ao = [smp.deletions(nm).get((rr, n), 0) for smp in samples]
        dp = [smp.depth(nm, rr) for smp in samples]
        out.append((rec[0], 1, n, 0, 0, "\t".join(["%s\t%d\t.\t%s\t%s\t.\tPASS\tINDEL;DP=%d;AO=%d;AF=%s\tDP:AD:AF" % (
            nm, rec[0], rec[1], rec[2], sum(dp), sum(ao), _af(sum(ao), sum(dp)))]
            + [_fields(d, [max(d - c, 0), c]) for c, d in zip(ao, dp)])))
    out.sort(key=lambda x: x[:5])
    return [x[5] for x in out]


def vcf(samples, names, source, abs_threshold, rel_threshold, filters=(0, 0, 0), primers_name=None, reference=None,
        mates=False):
    """The whole text.  samples: [Sample]; names: the column names; reference: None or (file name, {contig: text})."""
    mbq, mapq, flags = filters
    contigs = contigs_of(samples)
    lines = ["##fileformat=VCFv4.2", "##source=%s" % source,
             "##kindelVariants=abs_threshold=%s;rel_threshold=%s;min_base_quality=%d;min_mapq=%d;exclude_flags=%s"
             % (abs_threshold, rel_threshold, mbq, mapq, hex(flags))]
    if primers_name is not None:
        lines.append("##kindelPrimers=%s" % primers_name)
    if mates:
        lines.append("##kindelMateOverlaps=R2 masked where R1 covers")
    if reference is not None:
        lines.append("##reference=%s" % reference[0])
    lines += ["##contig=<ID=%s,length=%d>" % c for c in contigs]
    lines.append('##INFO=<ID=DP,Number=1,Type=Integer,Description="Depth: A + C + G + T + N + deletions">')
    if reference is None:
        lines.append('##INFO=<ID=AD,Number=R,Type=Integer,Description="Count of REF (the most frequent allele) and of '
                     'each ALT allele">')
    else:
        lines.append('##INFO=<ID=AD,Number=R,Type=Integer,Description="Count of the REF base and of each ALT base '
                     '(SNVs)">')
    lines.append('##INFO=<ID=AF,Number=A,Type=Float,Description="Share of the depth of each ALT allele, rounded to 4 '
                 'decimals">')
    if reference is not None:
        lines += ['##INFO=<ID=INDEL,Number=0,Type=Flag,Description="The record is an insertion or a deletion">',
                  '##INFO=<ID=AO,Number=A,Type=Integer,Description="Count of the reads carrying the ALT allele">']
    lines += ['##FORMAT=<ID=DP,Number=1,Type=Integer,Description="The sample\'s depth: A + C + G + T + N + deletions '
              '(indels: the depth the allele is measured against)">',
              '##FORMAT=<ID=AD,Number=R,Type=Integer,Description="The sample\'s count of REF and of each ALT allele">',
              '##FORMAT=<ID=AF,Number=A,Type=Float,Description="The sample\'s share of DP of each ALT allele, rounded '
              'to 4 decimals">',
              "##kindelSamples=%d" % len(samples),
              "\t".join(["#CHROM", "POS", "ID", "REF", "ALT", "QUAL", "FILTER", "INFO", "FORMAT"] + list(names))]
    for nm, L in contigs:
        if reference is None:
            lines += pooled_lines(samples, nm, L, abs_threshold, rel_threshold)
        else:
            lines += reference_lines(samples, nm, reference[1][nm], abs_threshold, rel_threshold)
    return "\n".join(lines) + "\n"
