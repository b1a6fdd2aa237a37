"""The VCF text of `kindel variants --vcf` (extensions, DESIGN.md §1): the one header and the one record writer.

One sample is the case S = 1 of several: every count the writer takes has a leading sample axis, INFO holds the
values summed over the samples, and a multi-sample VCF adds FORMAT DP:AD:AF with each sample's.  The strand fields
(ADF, ADR, SOR) and the quality fields (QUAL, BQ, AQ) are options of the writer, computed from the pooled values the
caller passes in; kindel.variants_vcf offers them with one sample only."""
from __future__ import annotations

import math

import numpy as np

_ALT = (0, 1, 2, 3, 5)  # the columns of the alleles without a reference: A, C, G, T, the deletion; N is not one
_LETTERS = "ACGTN*"     # the allele letter of each column
_ACGTN = str.maketrans({c: "N" for c in "=MRSVWYHKDB"})  # inserted bases: anything but A, C, G, T, N becomes N
QUAL_CAP = 3000
_EMASS_UNIT = 3.0 * 2.0 ** 32  # emass counts expected errors in units of 2^-32; a third of them hit one given base
_FORMAT = ['##FORMAT=<ID=DP,Number=1,Type=Integer,Description="The sample\'s depth: A + C + G + T + N + deletions '
           '(indels: the depth the allele is measured against)">',
           '##FORMAT=<ID=AD,Number=R,Type=Integer,Description="The sample\'s count of REF and of each ALT allele">',
           '##FORMAT=<ID=AF,Number=A,Type=Float,Description="The sample\'s share of DP of each ALT allele, rounded '
           'to 4 decimals">']


def check_number(value, name):
    """A filter threshold (`max_sor`, `min_qual`): None (no filter) or a float; NaN raises ValueError naming it."""
    if value is None:
        return None
    x = float(value)
    if math.isnan(x):
        raise ValueError("%s must be a number, got %r" % (name, value))
    return x


def header(contig_names, contig_len, abs_threshold, rel_threshold, filters, primers=None, mask_overlaps=False,
           reference_name=None, strand=False, max_sor=None, qual=False, min_qual=None, samples=None,
           normalise=None, dedup=False, left_align=False) -> list:
    """The header lines, the column line last.  filters: (min_base_quality, min_mapq, exclude_flags) or None; primers:
    the run's PrimerSet or None; samples: the FORMAT columns' names (a multi-sample VCF) or None; normalise: the
    --normalise cap N or None; dedup: the run went through --dedup; left_align: the indels were left-aligned against
    the reference (`##kindelLeftAlign` after `##reference`)."""
    from . import __version__

    mbq, mapq, flags = filters if filters is not None else (0, 0, 0)
    lines = ["##fileformat=VCFv4.2", "##source=kindel {}".format(__version__),
             "##kindelVariants=abs_threshold={};rel_threshold={};min_base_quality={};min_mapq={};exclude_flags={:#x}"
             .format(abs_threshold, rel_threshold, mbq, mapq, flags)]
    if primers is not None:
        lines.append("##kindelPrimers={}".format(primers.name))
    if dedup:
        lines.append("##kindelDedup=fragment ends, base-quality score")
    if normalise is not None:
        lines.append("##kindelNormalise={}".format(normalise))
    if mask_overlaps:
        lines.append("##kindelMateOverlaps=R2 masked where R1 covers")
    if strand:
        lines.append("##kindelStrand=max_sor={}".format("." if max_sor is None else max_sor))
    if qual:
        lines.append("##kindelQual=model=poisson;min_qual={}".format("." if min_qual is None else min_qual))
    if reference_name is not None:
        lines.append("##reference={}".format(reference_name))
        if left_align:
            lines.append("##kindelLeftAlign=leftmost against the reference")
    lines += ["##contig=<ID={},length={}>".format(name, int(L)) for name, L in zip(contig_names, contig_len)]
    lines += ['##INFO=<ID=DP,Number=1,Type=Integer,Description="Depth: A + C + G + T + N + deletions">',
              '##INFO=<ID=AD,Number=R,Type=Integer,Description="Count of REF (the most frequent allele) and of each '
              'ALT allele">' if reference_name is None else
              '##INFO=<ID=AD,Number=R,Type=Integer,Description="Count of the REF base and of each ALT base (SNVs)">',
              '##INFO=<ID=AF,Number=A,Type=Float,Description="Share of the depth of each ALT allele, rounded to 4 '
              'decimals">']
    if reference_name is not None:
        lines += ['##INFO=<ID=INDEL,Number=0,Type=Flag,Description="The record is an insertion or a deletion">',
                  '##INFO=<ID=AO,Number=A,Type=Integer,Description="Count of the reads carrying the ALT allele">']
    if strand:
        lines += ['##INFO=<ID=ADF,Number=R,Type=Integer,Description="Forward-strand count of REF and of each ALT '
                  'allele">',
                  '##INFO=<ID=ADR,Number=R,Type=Integer,Description="Reverse-strand count of REF and of each ALT '
                  'allele">',
                  '##INFO=<ID=SOR,Number=A,Type=Float,Description="Strand odds ratio of each ALT allele against REF">']
        if max_sor is not None:
            lines.append('##FILTER=<ID=sor,Description="The strand odds ratio of an ALT allele is above {}">'
                         .format(max_sor))
    if qual:
        lines += ['##INFO=<ID=BQ,Number=R,Type=Float,Description="Mean base quality of the counted bases of REF and of '
                  'each ALT allele">',
                  '##INFO=<ID=AQ,Number=A,Type=Integer,Description="Phred-scaled probability that sequencing errors '
                  'alone give the ALT base its count (Poisson model)">']
        if min_qual is not None:
            lines.append('##FILTER=<ID=lowqual,Description="QUAL is below {}">'.format(min_qual))
    columns = ["#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO"]
    if samples is not None:
        lines += _FORMAT + ["##kindelSamples=%d" % len(samples)]
        columns += ["FORMAT"] + list(samples)
    lines.append("\t".join(columns))
    return lines


def dpa_slots(layout, slot):
    """The slot each insertion at `slot` is measured against (DPa): the one before, the slot itself at a contig's
    first position."""
    contig_slot = np.asarray(layout.contig_slot, dtype=np.int64)
    p = slot - contig_slot[np.searchsorted(contig_slot, slot, side="right") - 1] if slot.size else slot
    return np.where(p >= 1, slot - 1, slot)


def records(layout, abs_threshold, rel_threshold, slot, mask, rows, ref_codes=None, dpa=None, strings_at=None,
            deletions=None, strand=None, max_sor=None, qual=None, min_qual=None, per_sample=False) -> list:
    """The data lines of S samples over `layout` (contig_names, contig_slot, contig_len).

    The sites: slot int64[n] ascending, mask uint8[n] (K6 / K6m bits 0-5 without a reference; K6r / K6m bits 0-3 and
    the insertion bit 6 with one) and rows int64 [S, 6, n], columns 0-5 of each sample at the sites.  With reference
    codes (uint8 per slot, reference.py) also: dpa int64 [S, n], each sample's DPa at the sites (None when no site has
    bit 6); strings_at(j, slot), sample j's {string: count} at a slot in first-seen order; deletions (slot int64[m],
    length int64[m], count int64 [S, m], depth int64 [S, m]), keys ascending (engine.deletion_union).

    Without a reference, per site: REF the pooled top allele's letter (N when it is N or a deletion, or at depth 0),
    ALT the variant alleles among A, C, G, T and the deletion (`*`), no record for N alone; AD the top allele's count,
    then each ALT's.  With one: SNV at p with a variant base: POS p + 1, REF the reference letter, ALT the variant
    bases in A, C, G, T order, AD the REF base's count (0 when the reference has no A, C, G or T) then each ALT's.
    Deletion (r, n), count c, D the depth at r: POS r, REF ref[r-1 .. r+n], ALT ref[r-1]; at r = 0 POS 1, REF
    ref[0 .. n], ALT ref[n] (no record for n = L).  Insertion of string s at slot p: POS p, REF ref[p-1], ALT ref[p-1]
    + s; at p = 0 POS 1, REF ref[0], ALT s + ref[0].  The strings of a slot: every sample's, in the order of the first
    sample that has the string, then its first-seen rank there; an empty one is skipped, and a string passes when its
    count exceeds abs_threshold and its share of DPa exceeds rel_threshold in some sample.  Indels carry INFO
    INDEL;DP;AO;AF.  INFO sums over the samples; AF is each ALT's share of DP rounded to 4 decimals (0 at DP 0).
    Order: contigs in slot order, then POS, then SNV < deletion < insertion, then deletion length, then insertion slot
    and rank.  per_sample: FORMAT DP:AD:AF and each sample's values (_sample_fields).

    strand: (rows int64 [6, n] of the reverse table at the sites, its DPa int64 [n] or None, the deletions' reverse
    counts and depths int64 [m] each or None, and rev_strings_at(slot), {string: reverse reads} at a slot) with
    max_sor: ;ADF;ADR;SOR and FILTER `sor` (strand_fields; an indel's _indel_strand).  qual: (qsum int64 [4, n],
    emass n ints) at the sites with min_qual: QUAL, ;BQ;AQ and FILTER `lowqual` of the site records (_qual_fields)."""
    contig_slot = np.asarray(layout.contig_slot, dtype=np.int64)
    contig_len = np.asarray(layout.contig_len, dtype=np.int64).tolist()
    names = layout.contig_names
    S = rows.shape[0]
    pooled = rows.sum(axis=0)                                    # [6, n]
    depth = pooled.sum(axis=0)
    with np.errstate(invalid="ignore", divide="ignore"):
        af = np.round(np.where(depth > 0, pooled / np.maximum(depth, 1), 0.0), 4).T.tolist()
    contig = np.searchsorted(contig_slot, slot, side="right") - 1
    t_of, d_of = pooled.T.tolist(), depth.tolist()
    starts = contig_slot.tolist()
    if ref_codes is None:
        ref_of = pooled.argmax(axis=0).tolist()                  # the top allele
    else:
        letters = np.frombuffer(b"ACGTN", dtype=np.uint8)[np.minimum(np.asarray(ref_codes), 4)].tobytes().decode()
        ref_of = np.asarray(ref_codes)[slot].astype(np.int64).tolist()  # the reference base
        da_of = dpa.T.tolist() if dpa is not None else None
    if per_sample:
        depth_s = rows.sum(axis=1)                               # [S, n]
    if strand is not None:
        rev_rows, rev_dpa, rev_dcnt, rev_ddepth, rev_strings_at = strand
        rev_of = rev_rows.T.tolist()
    if qual is not None:
        q_of, e_of = qual[0].T.tolist(), qual[1]
    recs = []  # (contig, POS, kind, deletion length, insertion slot, rank, line)
    for i, (s, m, c) in enumerate(zip(slot.tolist(), mask.tolist(), contig.tolist())):
        s0, name, t = starts[c], names[c], t_of[i]
        if ref_codes is None:
            alts = [k for k in _ALT if m >> k & 1]
            if not alts:
                continue  # N alone
            top = ref_of[i]
            ref_col = top if top < 4 and d_of[i] > 0 else None
            ks, ref = [top] + alts, "N" if ref_col is None else "ACGT"[top]
        elif m & 15:
            alts = [k for k in range(4) if m >> k & 1]
            ref_col = ref_of[i] if ref_of[i] < 4 else None
            ks, ref = [ref_col] + alts, letters[s]
        else:
            ks = None
        if ks is not None:  # a site record: AD's first column is REF's, None a reference base that is no base
            ad = [0 if k is None else t[k] for k in ks]
            alt = ",".join(_LETTERS[k] for k in alts)
            info = "DP={};AD={};AF={}".format(d_of[i], ",".join(map(str, ad)), ",".join(repr(af[i][k]) for k in alts))
            filt, score = "PASS", "."
            if strand is not None:
                adr = [0 if k is None else rev_of[i][k] for k in ks]
                filt, tail = strand_fields([a - b for a, b in zip(ad, adr)], adr, max_sor)
                info += tail
            if qual is not None:
                score, low, tail = _qual_fields(ref_col, alts, t, q_of[i], e_of[i], min_qual)
                filt = _filter(filt, low)
                info += tail
            fields = [name, str(s - s0 + 1), ".", ref, alt, score, filt, info]
            if per_sample:
                fields += _sample_fields(depth_s[:, i], np.stack(
                    [np.zeros(S, dtype=np.int64) if k is None else rows[:, k, i] for k in ks], axis=1))
            recs.append((c, s - s0 + 1, 0, 0, 0, 0, "\t".join(fields)))
        if m & 64:
            da = da_of[i]
            per = [strings_at(j, s) for j in range(S)]
            rank_of = {}
            for strings in per:
                for text in strings:
                    rank_of.setdefault(text, len(rank_of))
            rev_strings = rev_strings_at(s) if strand is not None else None
            for text, rank in rank_of.items():
                ao = [strings.get(text, 0) for strings in per]
                if not text or not any(cnt > abs_threshold and (cnt / dj if dj > 0 else 0.0) > rel_threshold
                                       for cnt, dj in zip(ao, da)):
                    continue
                anchored = _anchor(letters, s, s0, contig_len[c], "", text.translate(_ACGTN))
                if anchored is None:
                    continue
                line = _indel_line(name, anchored, sum(da), sum(ao),
                                   None if strand is None else (rev_dpa[i], rev_strings.get(text, 0)), max_sor,
                                   (np.asarray(da), np.asarray(ao)) if per_sample else None)
                recs.append((c, anchored[0], 2, 0, s, rank, line))

    if deletions is not None:
        d_slot, d_len, d_cnt, d_depth = deletions
        d_contig = np.searchsorted(contig_slot, d_slot, side="right") - 1
        cnt_of, dp_of = d_cnt.sum(axis=0).tolist(), d_depth.sum(axis=0).tolist()
        for i, (s, n, c) in enumerate(zip(d_slot.tolist(), d_len.tolist(), d_contig.tolist())):
            anchored = _anchor(letters, s, starts[c], contig_len[c], letters[s:s + n], "")
            if anchored is None:
                continue  # the whole contig deleted: no base is left to anchor the record
            line = _indel_line(names[c], anchored, dp_of[i], cnt_of[i],
                               None if strand is None else (rev_ddepth[i], rev_dcnt[i]), max_sor,
                               (d_depth[:, i], d_cnt[:, i]) if per_sample else None)
            recs.append((c, anchored[0], 1, n, 0, 0, line))
    if ref_codes is not None:  # the sites come in slot order; the indels' anchors and kinds need the sort
        recs.sort(key=lambda x: x[:6])
    return [x[6] for x in recs]


def _anchor(letters, s, s0, L, deleted, inserted):
    """(POS, REF, ALT) of an indel at slot s of a contig at slot s0 of length L that removes the reference bases
    `deleted` and adds the bases `inserted`: anchored on the base before it, or at the contig's first position on the
    first base after it; None when no base is left to anchor it."""
    if s > s0:
        return s - s0, letters[s - 1] + deleted, letters[s - 1] + inserted
    if len(deleted) >= L:
        return None
    after = letters[s0 + len(deleted)]
    return 1, deleted + after, inserted + after


def _indel_line(name, anchored, dp, ao, rev, max_sor, per_sample):
    """The line of an indel record: dp and ao summed over the samples, rev (its reverse DP and AO) or None,
    per_sample (each sample's dp and ao, int64 [S] arrays) or None."""
    pos, ref, alt = anchored
    info, filt = "INDEL;DP={};AO={};AF={}".format(dp, ao, _af(ao, dp)), "PASS"
    if rev is not None:
        filt, tail = _indel_strand(dp, int(rev[0]), ao, int(rev[1]), max_sor)
        info += tail
    fields = [name, str(pos), ".", ref, alt, ".", filt, info]
    if per_sample is not None:
        dp_s, ao_s = per_sample
        fields += _sample_fields(dp_s, np.stack([np.maximum(dp_s - ao_s, 0), ao_s], axis=1))
    return "\t".join(fields)


def _af(count, depth) -> str:
    """A share rounded to 4 decimals as `variants` prints it (0 at depth 0)."""
    return repr(float(np.round(np.float64(count / depth if depth > 0 else 0.0), 4)))


def _sample_fields(dp, ad) -> list:
    """The FORMAT column and the values DP:AD:AF of every sample: dp int64 [S], ad int64 [S, 1 + m] (REF, then each
    ALT); AF = each ALT's share of DP rounded to 4 decimals (0 at DP 0)."""
    dp = np.asarray(dp, dtype=np.int64)
    ad = np.asarray(ad, dtype=np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        af = np.round(np.where(dp[:, None] > 0, ad[:, 1:] / np.maximum(dp, 1)[:, None], 0.0), 4).tolist()
    return ["DP:AD:AF"] + ["%d:%s:%s" % (d, ",".join(map(str, a)), ",".join(map(repr, f)))
                           for d, a, f in zip(dp.tolist(), ad.tolist(), af)]


# ------------------------------------------------------------------------------------------------ strand
def strand_odds_ratio(f_ref, r_ref, f_alt, r_alt) -> float:
    """GATK's StrandOddsRatio of one ALT from the forward / reverse counts of REF and of the ALT, in float64."""
    t00, t01, t10, t11 = float(f_ref + 1), float(r_ref + 1), float(f_alt + 1), float(r_alt + 1)
    ratio = (t00 / t01) * (t11 / t10) + (t01 / t00) * (t10 / t11)
    return math.log(ratio) + math.log(min(t00, t01) / max(t00, t01)) - math.log(min(t10, t11) / max(t10, t11))


def strand_fields(adf, adr, max_sor):
    """(FILTER, INFO tail) of a record whose REF and ALTs have forward counts adf and reverse counts adr: the tail is
    ;ADF=..;ADR=..;SOR=.. (SOR per ALT, "%.3f"); FILTER is `sor` when max_sor is set and some ALT's SOR as written
    exceeds it, else PASS."""
    sor = ["%.3f" % strand_odds_ratio(adf[0], adr[0], adf[k], adr[k]) for k in range(1, len(adf))]
    filt = "sor" if max_sor is not None and any(float(x) > max_sor for x in sor) else "PASS"
    return filt, ";ADF={};ADR={};SOR={}".format(",".join(map(str, adf)), ",".join(map(str, adr)), ",".join(sor))


def _indel_strand(dp, dp_rev, ao, ao_rev, max_sor):
    """strand_fields of an indel record: DP and AO in total and on the reverse strand; forward = total - reverse;
    REF's entry on strand s is max(DP_s - AO_s, 0)."""
    dp_fwd, ao_fwd = dp - dp_rev, ao - ao_rev
    return strand_fields([max(dp_fwd - ao_fwd, 0), ao_fwd], [max(dp_rev - ao_rev, 0), ao_rev], max_sor)


# ------------------------------------------------------------------------------------------------ qual
def allele_quality(k: int, emass: int) -> int:
    """AQ of a base ALT with count k at a slot whose counted bases sum to emass (K11): with the expected number of
    errors that turn into this base, lambda = emass / (3 * 2^32), p = P(Poisson(lambda) >= k) =
    scipy.special.gammainc(k, lambda) -- the Poisson approximation to LoFreq's Poisson-binomial error model -- and AQ =
    -10 log10(p) rounded half up, clamped to [0, 3000], 3000 when p underflows to 0.  k = 0 gives 0."""
    from scipy.special import gammainc

    if k <= 0:
        return 0
    p = float(gammainc(float(k), float(emass) / _EMASS_UNIT))
    if p <= 0.0:
        return QUAL_CAP
    return min(max(int(math.floor(-10.0 * math.log10(p) + 0.5)), 0), QUAL_CAP)


def _qual_fields(ref_col, alt_cols, counts, qsum, emass, min_qual):
    """(QUAL, lowqual, INFO tail) of a record: ref_col / alt_cols the table columns of REF and of each ALT (0-3 a base,
    4 N, 5 the deletion, None a reference base that is no base), counts / qsum their counts and quality sums at the
    record's slot (columns 0-3), emass the slot's.  A record without a base ALT: (".", False, "")."""
    if not any(k is not None and k < 4 for k in alt_cols):
        return ".", False, ""

    def bq(k):
        return "." if k is None or k > 3 or counts[k] == 0 else "%.1f" % (qsum[k] / counts[k])

    aq = [allele_quality(int(counts[k]), emass) if k < 4 else None for k in alt_cols]
    q = max(a for a in aq if a is not None)
    tail = ";BQ={};AQ={}".format(",".join(bq(k) for k in [ref_col] + list(alt_cols)),
                                ",".join("." if a is None else str(a) for a in aq))
    return str(q), min_qual is not None and q < min_qual, tail


def _filter(strand_filter, lowqual):
    """FILTER from the strand filter (`sor` or PASS) and lowqual, in the order sor, lowqual."""
    failed = [f for f, on in (("sor", strand_filter == "sor"), ("lowqual", lowqual)) if on]
    return ";".join(failed) if failed else "PASS"
