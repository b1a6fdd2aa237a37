"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `variants --vcf` with every option at once (base and read
filters, primers, reference, strand), as per-record and per-position loops over plain Python ints, strings and dicts.

Records are oracle/samdecode.py's (.rname, .flag, .mapq, .pos 1-based, .seq, .cigars, .qual); primers are plain
(chrom, start, end) rows.  Per alignment file:

  contigs   first-seen order of the records' RNAME (`*` dropped), every record counting, filtered or not
  filters   a record with MAPQ < min_mapq or FLAG & exclude_flags is treated as unmapped (FLAG 0x4); a record is piled
            when mapped and len(SEQ) > 1 (kindel.py:43-46)
  mask      per record, the union of the query offsets whose QUAL is below min_base_quality (never for QUAL `*`) and
            its primer bases (py_poracle.masked_qpos)
  walk      the reference's loop (kindel.py:40-81, Python list indexing and its wrap included) with masked bases:
            a masked M/=/X base advances both cursors and adds nothing to the weights; a masked clipped base adds
            nothing to the clip weights (clip_starts / clip_ends count as before); a masked inserted base is `N` in the
            insertion string; deletions are unchanged; a masked base raises no KeyError, whatever its letter
  strand    the forward (FLAG & 0x10 clear) and the reverse records are piled separately, with their own deletion
            events (py_rvoracle.deletion_events' rule); nothing is derived by subtraction

The VCF text -- header and records -- follows DESIGN.md section 1 (sites-only VCF, seventh, eighth and ninth
extensions); the record rules are py_voracle's / py_rvoracle's, the strand fields py_soracle's.  `tables` gives the
walk's 19-column count table and insertion dicts, for pinning against oracle/kindel_qoracle.c.  Nothing here imports
kindel_b200."""
from __future__ import annotations

from . import samdecode
from .py_poracle import contig_intervals, masked_qpos
from .py_rvoracle import _af, _share, ref_letters
from .py_soracle import is_reverse, strand_tail

_NUC = "ACGT"
_KEYS = "ACGTN"


def _fresh(n):
    return [{"A": 0, "C": 0, "G": 0, "T": 0, "N": 0} for _ in range(n)]


class Pile:
    """The masked walk's tables of one contig of length L over some records."""

    def __init__(self, L):
        self.L = L
        self.weights, self.csw, self.cew = _fresh(L), _fresh(L), _fresh(L)
        self.deletions, self.clip_starts, self.clip_ends = [0] * (L + 1), [0] * (L + 1), [0] * (L + 1)
        self.ins_ops = [0] * (L + 1)              # every I op, empty strings included (column 6)
        self.insertions = [{} for _ in range(L + 1)]  # first-seen order
        self.del_events = {}                       # (r, n) -> count
        self.masked_n_inserts = 0                  # inserted strings holding a masked base

    def add(self, rec, masked):
        seq, L = rec.seq, self.L
        r, q = rec.pos - 1, 0
        for i, (n, op) in enumerate(rec.cigars):
            if op in ("M", "=", "X"):
                for _ in range(n):
                    w, b = self.weights[r], seq[q].upper()
                    if q not in masked:
                        w[b] += 1
                    r += 1
                    q += 1
            elif op == "I":
                s = "".join("N" if k in masked else seq[k].upper() for k in range(q, min(q + n, len(seq))))
                self.ins_ops[r] += 1
                d = self.insertions[r]
                d[s] = d.get(s, 0) + 1
                self.masked_n_inserts += any(k in masked for k in range(q, min(q + n, len(seq))))
                q += n
            elif op == "D":
                if n >= 1 and r >= 0 and r + n <= L:
                    self.del_events[(r, n)] = self.del_events.get((r, n), 0) + 1
                for k in range(n):
                    self.deletions[r + k] += 1
                r += n
            elif op == "S":
                if i == 0:
                    self.clip_ends[r] += 1
                    for g in range(n):
                        b = seq[g].upper()
                        rel = r - n + g
                        if rel >= 0:
                            w = self.cew[rel]
                            if g not in masked:
                                w[b] += 1
                    q += n
                else:
                    self.clip_starts[r - 1] += 1
                    for _ in range(n):
                        b = seq[q].upper()
                        if r < L:
                            w = self.csw[r]
                            if q not in masked:
                                w[b] += 1
                            r += 1
                            q += 1

    def counts(self, pos):
        """A, C, G, T, N, deletions at pos (0 <= pos <= L; slot L holds deletions only)."""
        if pos < self.L:
            w = self.weights[pos]
            return [w["A"], w["C"], w["G"], w["T"], w["N"], self.deletions[pos]]
        return [0, 0, 0, 0, 0, self.deletions[pos]]

    def depth(self, pos):
        return sum(self.counts(pos))


def record_mask(rec, L, intervals, min_base_quality):
    """The masked query offsets of one record: low-quality bases, and primer bases when intervals is not None."""
    out = set()
    if min_base_quality and rec.qual is not None:
        out = {q for q, v in enumerate(rec.qual) if v < min_base_quality}
    if intervals is not None:
        out |= set(masked_qpos(rec, L, intervals))
    return out


class Composed:
    """The masked piles of one alignment file at one (min_base_quality, min_mapq, exclude_flags, primer rows)."""

    def __init__(self, path, min_base_quality=0, min_mapq=0, exclude_flags=0, primer_rows=None):
        header, records = samdecode.read_alignment_file(path)
        lengths = {}
        for sn, fields in header["@SQ"].items():
            lengths[sn[3:]] = int(next(f for f in fields if f.startswith("LN:"))[3:])
        groups = {}
        for rec in records:
            groups.setdefault(rec.rname, []).append(rec)
        groups.pop("*", None)
        self.contigs = [(nm, lengths[nm]) for nm in groups]
        self.piles = {}  # name -> (all, forward, reverse)
        for nm, L in self.contigs:
            iv = contig_intervals(primer_rows, nm) if primer_rows is not None else None
            piles = (Pile(L), Pile(L), Pile(L))
            for rec in groups[nm]:
                if rec.flag & 0x4 or rec.mapq < min_mapq or rec.flag & exclude_flags or len(rec.seq) <= 1:
                    continue
                m = record_mask(rec, L, iv, min_base_quality)
                piles[0].add(rec, m)
                piles[2 if is_reverse(rec) else 1].add(rec, m)
            self.piles[nm] = piles

    # ---------------------------------------------------------------------------------------------- tables
    def tables(self, strand=0):
        """[(name, counts [19][L + 1] as lists, insertion dicts)] of the piles of strand 0 (all), 1 (fwd), 2 (rev),
        in the columns of oracle/kindel_qoracle.c."""
        out = []
        for nm, L in self.contigs:
            p = self.piles[nm][strand]
            cols = [[0] * (L + 1) for _ in range(19)]
            for pos in range(L):
                for k, b in enumerate(_KEYS):
                    cols[k][pos] = p.weights[pos][b]
                    cols[9 + k][pos] = p.csw[pos][b]
                    cols[14 + k][pos] = p.cew[pos][b]
            cols[5], cols[6], cols[7], cols[8] = list(p.deletions), list(p.ins_ops), list(p.clip_starts), \
                list(p.clip_ends)
            out.append((nm, cols, p.insertions))
        return out

    # ---------------------------------------------------------------------------------------------- records
    def _sites_lines(self, nm, L, a, r, strand, max_sor):
        P, F, R = self.piles[nm]
        out = []
        for pos in range(L):
            t = P.counts(pos)
            d = sum(t)
            top = max(range(6), key=lambda k: (t[k], -k))
            alts = [k for k in (0, 1, 2, 3, 5) if k != top and t[k] > a and _share(t[k], d) > r]
            if not alts:
                continue
            ks = [top] + alts
            filt, tail = "PASS", ""
            if strand:
                tf, tr = F.counts(pos), R.counts(pos)
                filt, tail = strand_tail([tf[k] for k in ks], [tr[k] for k in ks], max_sor)
            out.append("%s\t%d\t.\t%s\t%s\t.\t%s\tDP=%d;AD=%s;AF=%s%s" % (
                nm, pos + 1, _NUC[top] if top < 4 and d > 0 else "N", ",".join("ACGT*"[min(k, 4)] for k in alts),
                filt, d, ",".join(str(t[k]) for k in ks), ",".join(_af(t[k], d) for k in alts), tail))
        return out

    def _reference_lines(self, nm, ref, a, r, strand, max_sor, stats):
        L = len(ref)
        ref = ref_letters(ref)
        P, F, R = self.piles[nm]
        out = []

        def indel_tail(dp_f, dp_r, ao_f, ao_r):
            if stats is not None and (dp_f < ao_f or dp_r < ao_r):
                stats["clamp"] = stats.get("clamp", 0) + 1
            return strand_tail([max(dp_f - ao_f, 0), ao_f], [max(dp_r - ao_r, 0), ao_r], max_sor)

        for pos in range(L):
            t = P.counts(pos)
            d = sum(t)
            g = _NUC.find(ref[pos])
            alts = [k for k in range(4) if k != g and t[k] > a and _share(t[k], d) > r]
            if not alts:
                continue
            ad = [t[g] if g >= 0 else 0] + [t[k] for k in alts]
            filt, tail = "PASS", ""
            if strand:
                tf, tr = F.counts(pos), R.counts(pos)
                filt, tail = strand_tail([tf[g] if g >= 0 else 0] + [tf[k] for k in alts],
                                         [tr[g] if g >= 0 else 0] + [tr[k] for k in alts], max_sor)
            out.append((pos + 1, 0, 0, 0, 0, "%s\t%d\t.\t%s\t%s\t.\t%s\tDP=%d;AD=%s;AF=%s%s" % (
                nm, pos + 1, ref[pos], ",".join(_NUC[k] for k in alts), filt, d, ",".join(map(str, ad)),
                ",".join(_af(t[k], d) for k in alts), tail)))
        if L > 0:
            for pos in range(L + 1):
                at = pos - 1 if pos >= 1 else 0
                dpa = P.depth(at)
                for rank, (s, c) in enumerate(P.insertions[pos].items()):
                    if not s or not (c > a and _share(c, dpa) > r):
                        continue
                    filt, tail = "PASS", ""
                    if strand:
                        filt, tail = indel_tail(F.depth(at), R.depth(at), F.insertions[pos].get(s, 0),
                                                R.insertions[pos].get(s, 0))
                    alt = "".join(ch if ch in _NUC + "N" else "N" for ch in s)
                    rec = (pos, ref[pos - 1], ref[pos - 1] + alt) if pos >= 1 else (1, ref[0], alt + ref[0])
                    out.append((rec[0], 2, 0, pos, rank, "%s\t%d\t.\t%s\t%s\t.\t%s\tINDEL;DP=%d;AO=%d;AF=%s%s" % (
                        nm, rec[0], rec[1], rec[2], filt, dpa, c, _af(c, dpa), tail)))
        for (rr, n), c in P.del_events.items():
            d = P.depth(rr)
            if not (c > a and _share(c, d) > r):
                continue
            if rr >= 1:
                rec = (rr, ref[rr - 1:rr + n], ref[rr - 1])
            elif n < L:
                rec = (1, ref[0:n + 1], ref[n])
            else:
                continue
            filt, tail = "PASS", ""
            if strand:
                filt, tail = indel_tail(F.depth(rr), R.depth(rr), F.del_events.get((rr, n), 0),
                                        R.del_events.get((rr, n), 0))
            out.append((rec[0], 1, n, 0, 0, "%s\t%d\t.\t%s\t%s\t.\t%s\tINDEL;DP=%d;AO=%d;AF=%s%s" % (
                nm, rec[0], rec[1], rec[2], filt, d, c, _af(c, d), tail)))
        out.sort(key=lambda x: x[:5])
        return [x[5] for x in out]

    def vcf(self, source, abs_threshold, rel_threshold, filters=(0, 0, 0), primers_name=None, reference=None,
            strand=False, max_sor=None, stats=None):
        """The whole VCF text.  source: the `##source` value; filters: (min_base_quality, min_mapq, exclude_flags) for
        the header; reference: None or (file name, {contig: reference text}); max_sor implies strand.  stats, a dict,
        counts the indel strand entries where some DP_s < AO_s ("clamp")."""
        strand = strand or max_sor is not None
        mbq, mapq, flags = filters
        lines = ["##fileformat=VCFv4.2", "##source=%s" % source,
                 "##kindelVariants=abs_threshold=%s;rel_threshold=%s;min_base_quality=%d;min_mapq=%d;exclude_flags=%s"
                 % (abs_threshold, rel_threshold, mbq, mapq, hex(flags))]
        if primers_name is not None:
            lines.append("##kindelPrimers=%s" % primers_name)
        if strand:
            lines.append("##kindelStrand=max_sor=%s" % ("." if max_sor is None else max_sor))
        if reference is not None:
            lines.append("##reference=%s" % reference[0])
        lines += ["##contig=<ID=%s,length=%d>" % c for c in self.contigs]
        lines.append('##INFO=<ID=DP,Number=1,Type=Integer,Description="Depth: A + C + G + T + N + deletions">')
        if reference is None:
            lines.append('##INFO=<ID=AD,Number=R,Type=Integer,Description="Count of REF (the most frequent allele) '
                         'and of each ALT allele">')
        else:
            lines.append('##INFO=<ID=AD,Number=R,Type=Integer,Description="Count of the REF base and of each ALT '
                         'base (SNVs)">')
        lines.append('##INFO=<ID=AF,Number=A,Type=Float,Description="Share of the depth of each ALT allele, rounded '
                     'to 4 decimals">')
        if reference is not None:
            lines += ['##INFO=<ID=INDEL,Number=0,Type=Flag,Description="The record is an insertion or a deletion">',
                      '##INFO=<ID=AO,Number=A,Type=Integer,Description="Count of the reads carrying the ALT allele">']
        if strand:
            lines += ['##INFO=<ID=ADF,Number=R,Type=Integer,Description="Forward-strand count of REF and of each ALT '
                      'allele">',
                      '##INFO=<ID=ADR,Number=R,Type=Integer,Description="Reverse-strand count of REF and of each ALT '
                      'allele">',
                      '##INFO=<ID=SOR,Number=A,Type=Float,Description="Strand odds ratio of each ALT allele against '
                      'REF">']
            if max_sor is not None:
                lines.append('##FILTER=<ID=sor,Description="The strand odds ratio of an ALT allele is above %s">'
                             % max_sor)
        lines.append("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO")
        for nm, L in self.contigs:
            if reference is None:
                lines += self._sites_lines(nm, L, abs_threshold, rel_threshold, strand, max_sor)
            else:
                lines += self._reference_lines(nm, reference[1][nm], abs_threshold, rel_threshold, strand, max_sor,
                                               stats)
        return "\n".join(lines) + "\n"
