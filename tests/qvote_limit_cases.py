"""Inputs at the limits of the quality vote (`consensus --quality-vote`) and the composed oracle it is checked against
(test infrastructure).

- A deep column (`deep_records`): DEEP_N simple reads over one slot of one 512-slot tile, so that K11w stages that
  tile's reads in more than three 1024-read chunks and a quarter-warp adds more than 671 Q93 reads to the slot (a
  uint32 sum of a quarter's partials over the whole tile, or a 32-bit fold of one chunk's partials, wraps there).  It
  comes as every base Q93, every base the BAM byte 254 (which weighs W[93] too) and a mix where a minority of Q40 G
  reads outweigh a majority of Q5 A reads.  A second stack straddles the edge of the next tile.
- A paired corpus with a quality on every read (`filled_case`): tests/pair_combo_cases.py's records, the mates with QUAL
  `*` filled with seeded qualities and every base of the "edge" contig at QV_EDGE set to Q1, plus a contig `qv` whose
  windows each hold one planted difference between the two votes:
    TO_OTHER      6 X at Q5, 4 Y at Q35: the count vote X, the quality vote Y (min_base_quality 20: both Y)
    TIE_TO_BASE   5 X at Q30, 5 Y at Q31: a count tie (N), the quality vote Y
    TO_N          3 X at Q0, 2 Y at Q1: the count vote X, no weight (N)
    MATES_FLIP    5 single X at Q15, two pairs with Y at Q40 in both mates: the count vote X both ways, the quality vote
                  Y, and X once the second mates' overlap is masked
    PRIMER_FLIP   5 X at Q10 over the primer, 2 Y at Q40 starting in it: the quality vote Y, and X once primers mask
    AT_INSERTION  TO_OTHER's column where the 6 X reads insert `GG` in front of it: an `I` call
    LAST          TO_OTHER's column at the contig's last position
  X is the reference base, Y another.  QV_EDGE lies in the span the `--realign` patch replaces once mates count once, so
  there the count vote keeps the reference base and the quality vote gives N.

The composed oracle (`QualityVotePiled`) is pair_combo_cases.PairedPiled (py_cvoracle.Composed or
py_moracle.ComposedMates, coracle, the host's CDR functions over the oracle's table) with the quality vote on top:
py_qvoracle's walk fed W[min(q, 93)] gives the masked weight sums, quality_vote_cases.restated_vote the calls and Q,
fqoracle.fastq the text with that Q, and the REPORT gains `- quality_vote: True` and `- quality-vote sites:`.
"""
from __future__ import annotations

import itertools

import numpy as np

import combo_cases as CC
import helpers as H
import pair_combo_cases as PC
import quality_vote_cases as QVC
from kindel_b200 import bamio
from kindel_b200.quality import WEIGHT
from oracle import coracle, fqoracle

DEEP_N = 4100            # reads over the deep slot (> 4 chunks of 1024)
DEEP_POS, DEEP_LEN = 100, 50
DEEP_SLOT = 120          # a slot every deep read covers
EDGE_N = 2100            # the second stack: reads from just before 512 into the next tile
DEEP_CONTIG = ("deep", 1536)
DEEP_VARIANTS = ("q93", "byte254", "minority")
MINORITY = (2700, 5, 1400, 40)  # (A reads, their Phred, G reads, their Phred): G wins by weight, A by count


def _deep_rows(rng):
    rows = [(DEEP_POS + int(rng.integers(0, 8)), DEEP_LEN) for _ in range(DEEP_N)]
    rows += [(int(rng.integers(470, 500)), 60) for _ in range(EDGE_N)]
    return sorted(rows)


def deep_records(variant, seed=11):
    """(contigs, records) of the deep column: every read all `G` at the variant's quality, or for `minority` the
    reads over the deep slot are MINORITY[0] A reads and MINORITY[2] G reads, interleaved."""
    rng = np.random.default_rng(seed)
    rows = _deep_rows(rng)
    q = {"q93": 93, "byte254": 254, "minority": 40}[variant]
    n_a, q_a, _, _ = MINORITY
    a_reads = set(rng.choice(DEEP_N, n_a, replace=False).tolist()) if variant == "minority" else set()
    recs, k_deep = [], 0
    for k, (pos, n) in enumerate(rows):
        base, qq = "G", q
        if pos < 470:  # a read of the deep stack
            if k_deep in a_reads:
                base, qq = "A", q_a
            k_deep += 1
        recs.append((0, pos, 0, [(n << 4) | 0], base * n, "d%d" % k, 60, bytes([qq] * n)))
    return [DEEP_CONTIG], recs


def write_deep(d, variant):
    """(SAM path or None, BAM path) of the deep column: SAM text stops at Q93, so `byte254` is BAM only."""
    contigs, recs = deep_records(variant)
    bam = str(d / ("deep_%s.bam" % variant))
    bamio.write_bam(bam, contigs, recs)
    sam = None
    if variant != "byte254":
        import qual_cases as QC

        sam = str(d / ("deep_%s.sam" % variant))
        QC.write_sam(sam, contigs, recs)
    return sam, bam


def deep_want(variant):
    """(A sum, G sum) at DEEP_SLOT, exactly."""
    if variant == "minority":
        n_a, q_a, n_g, q_g = MINORITY
        return n_a * WEIGHT[q_a], n_g * WEIGHT[q_g]
    return 0, DEEP_N * WEIGHT[93]


def check_deep_shape(batch, wsum):
    """The deep column reaches what it is built for: more than 3 * 1024 reads start in the tile of DEEP_SLOT, the G sum
    there passes 2^34 (Q93 variants), and the second stack's reads cross into the next tile."""
    start = np.asarray(batch.ref_start, dtype=np.int64)
    assert int((start // 512 == DEEP_SLOT // 512).sum()) > 3 * 1024
    assert int((start <= DEEP_SLOT).sum() - (start + np.asarray(batch.seq_len) <= DEEP_SLOT).sum()) == DEEP_N
    assert int(((start < 512) & (start + np.asarray(batch.seq_len) > 512)).sum()) == EDGE_N
    if wsum is not None:
        assert int(wsum[2, DEEP_SLOT]) > 2 ** 34


# ------------------------------------------------------------------------------------------- the filled paired corpus
QV_NAME, QV_LEN = "qv", 400
TO_OTHER, TIE_TO_BASE, TO_N, MATES_FLIP, PRIMER_FLIP, AT_INSERTION = 30, 60, 90, 120, 160, 200
LAST = QV_LEN - 1
QV_PRIMER = (QV_NAME, 158, 164)
QV_EDGE = range(PC.B1 + 4, PC.B1 + 7)  # "edge" positions whose every base is Q1


def _ref_positions(rec):
    """{query offset: reference position} of a record's M bases (the corpus's CIGARs: M, I, D, S)."""
    r, q, out = rec[1], 0, {}
    for i, w in enumerate(rec[3]):
        n, op = w >> 4, w & 15
        if op == 0:
            for k in range(n):
                out[q + k] = r + k
            r, q = r + n, q + n
        elif op == 1:
            q += n
        elif op == 2:
            r += n
        elif op == 4:
            q += n
            r += n if i else 0
    return out


def _qv_records(rng, ref, cid):
    out = []
    count = itertools.count()

    def rec(pos, cig, seq, qual, flag=0, name=None, mate=None):
        name = name or "qv_s%d" % next(count)
        nref, npos = (cid, mate) if mate is not None else (-1, -1)
        out.append((cid, pos, flag, bamio.parse_cigar_text(cig), seq, name, 60,
                    bytes(np.asarray(qual, dtype=np.uint8).tolist()), nref, npos))

    def planted(a, n, site, base, q):
        """(SEQ, QUAL) of n reference bases from a, `base` at Phred q on `site`, the others HIGH_Q."""
        seq = list(ref[a:a + n])
        seq[site - a] = base
        qual = rng.choice(PC.HIGH_Q, size=n).astype(np.uint8)
        qual[site - a] = q
        return "".join(seq), qual

    def column(p, xs, ys, lengths=(25, 27)):
        """xs / ys: (count, Phred) of reads with the reference base / another one at p."""
        x, y = ref[p], PC._other(ref, p)
        for (n, q), base, ln in ((xs, x, lengths[0]), (ys, y, lengths[1])):
            for k in range(n):
                a = max(0, min(p - 10 + k, QV_LEN - ln))
                rec(a, "%dM" % ln, *planted(a, ln, p, base, q))

    column(TO_OTHER, (6, 5), (4, 35))
    column(TIE_TO_BASE, (5, 30), (5, 31))
    column(TO_N, (3, 0), (2, 1))
    p = MATES_FLIP
    column(p, (5, 15), (0, 0))
    y = PC._other(ref, p)
    for k in range(2):
        name = "qv_p%d" % k
        s1, q1 = planted(p - 10 + k, 30, p, y, 40)
        s2, q2 = planted(p - 5 + k, 30, p, y, 40)
        rec(p - 10 + k, "30M", s1, q1, PC.FLAG_R1, name, p - 5 + k)
        rec(p - 5 + k, "30M", s2, q2, PC.FLAG_R2, name, p - 10 + k)
    p, (_, lo, _) = PRIMER_FLIP, QV_PRIMER
    for k in range(5):
        rec(lo - 13 + k, "30M", *planted(lo - 13 + k, 30, p, ref[p], 10))
    for k in range(2):
        rec(lo, "20M", *planted(lo, 20, p, PC._other(ref, p), 40))
    p = AT_INSERTION
    for k in range(6):  # 15M 2I 15M: the inserted GG sits in front of p, whose base is X at Q5
        s, q = planted(p - 15, 30, p, ref[p], 5)
        q = np.concatenate((q[:15], [35, 35], q[15:]))
        rec(p - 15, "15M2I15M", s[:15] + "GG" + s[15:], q)
    for k in range(4):
        rec(p - 14 + k, "28M", *planted(p - 14 + k, 28, p, PC._other(ref, p), 35))
    for k, (base, q) in enumerate([(ref[LAST], 5)] * 6 + [(PC._other(ref, LAST), 35)] * 4):
        n = 20 + k
        rec(QV_LEN - n, "%dM" % n, *planted(QV_LEN - n, n, LAST, base, q))
    return sorted(out, key=lambda r: r[1])


def filled_case(seed=1):
    """(contigs, records, primer rows): pair_combo_cases.pair_case's records with every QUAL `*` filled and QV_EDGE at
    Q1, then the `qv` contig's windows."""
    contigs, recs = PC.pair_case(seed)
    rng = np.random.default_rng(seed + 1000)
    out = []
    for r in recs:
        qual = r[7]
        if qual is None:
            qual = bytes(rng.choice(PC.HIGH_Q, size=len(r[4])).astype(np.uint8).tolist())
        if r[0] == PC.EDGE:
            q = bytearray(qual)
            for k, pos in _ref_positions(r).items():
                if pos in QV_EDGE:
                    q[k] = 1
            qual = bytes(q)
        out.append(r[:7] + (qual,) + r[8:])
    ref = "".join(rng.choice(list("ACGT"), size=QV_LEN))
    contigs = list(contigs) + [(QV_NAME, QV_LEN)]
    out += _qv_records(rng, ref, len(contigs) - 1)
    return contigs, out, list(PC.PRIMERS) + [QV_PRIMER]


def write_filled(d, seed=1):
    """dict(bam, sam, bed, rows, contigs, recs) of the filled corpus under directory d."""
    contigs, recs, rows = filled_case(seed)
    bam, sam, bed = str(d / "filled.bam"), str(d / "filled.sam"), d / "filled.bed"
    bamio.write_bam(bam, contigs, recs)
    with open(sam, "w") as fh:
        fh.write(PC.sam_text(contigs, recs))
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
    return dict(bam=bam, sam=sam, bed=str(bed), rows=rows, contigs=contigs, recs=recs)


def vote_matrix():
    """Rows of (min_base_quality, min_depth, realign, trim_ends, uppercase, fastq, (min_mapq, exclude_flags), primers,
    mask_overlaps) such that every pair of values of every two options occurs in some row (combo_cases' greedy
    method)."""
    levels = [(0, 20), (1, 3), (False, True), (False, True), (False, True), (False, True), ((0, 0), (30, 0x400)),
              (False, True), (False, True)]
    want = {(i, a, j, b) for i, j in itertools.combinations(range(len(levels)), 2)
            for a in range(len(levels[i])) for b in range(len(levels[j]))}
    rows = []
    while want:
        best = max(itertools.product(*[range(len(v)) for v in levels]), key=lambda r: len(CC._pairs(r) & want))
        want -= CC._pairs(best)
        rows.append(best)
    return [tuple(levels[i][v] for i, v in enumerate(r)) for r in rows]


# ------------------------------------------------------------------------------------------- composed oracle
def weight_sums(path, min_base_quality=0, min_mapq=0, exclude_flags=0, primer_rows=None, mates=False):
    """{contig: wsum [4][L]}: py_qvoracle.quality_sums (its records, filters and masks) with its walk adding
    W[min(q, 93)] in place of q."""
    from oracle import py_qvoracle as QV

    walk = QV.walk
    QV.walk = lambda L, rec, qual, masked, qsum, emass: walk(L, rec, [WEIGHT[min(q, 93)] for q in qual], masked,
                                                             qsum, emass)
    try:
        return {nm: v[0] for nm, v in QV.quality_sums(path, min_base_quality, min_mapq, exclude_flags, primer_rows,
                                                      mates).items()}
    finally:
        QV.walk = walk


class QualityVotePiled(PC.PairedPiled):
    """PairedPiled with the quality vote: the calls and Q of restated_vote over the oracle's table and its masked
    weight sums, the text of fqoracle.fastq with that Q, the REPORT with the quality-vote lines."""

    def __init__(self, path, layout, min_base_quality=0, min_mapq=0, exclude_flags=0, primer_rows=None, mates=False,
                 primers_name=None):
        super().__init__(path, layout, min_base_quality, min_mapq, exclude_flags, primer_rows, mates, primers_name)
        self.wsum = np.zeros((4, int(layout.n_slots)), dtype=object)
        for nm, w in weight_sums(path, min_base_quality, min_mapq, exclude_flags, primer_rows, mates).items():
            c = list(layout.contig_names).index(nm)
            s0 = int(layout.contig_slot[c])
            self.wsum[:, s0:s0 + len(w[0])] = np.array(w, dtype=object)
        self._votes = {}

    def vote(self, min_depth=1):
        """(calls, Q) uint8 [n_slots] of the quality vote."""
        if min_depth not in self._votes:
            self._votes[min_depth] = QVC.restated_vote(self.counts, self.wsum, int(np.ceil(min_depth)))
        return self._votes[min_depth]

    def calls(self, t=None, min_depth=1):
        assert t is None, "the quality vote has no IUPAC threshold"
        return self.vote(min_depth)[0]

    def sites(self, min_depth=1):
        """Slots whose quality-vote call byte differs from coracle.vote's."""
        return np.flatnonzero(self.calls(None, min_depth) != coracle.vote(self.counts, min_depth))

    def consensus(self, t=None, min_depth=1, realign=False, trim_ends=False, uppercase=False, min_overlap=9):
        calls, q = self.vote(min_depth)
        out = []
        for c, name, s0, L, ins_c in self.contigs():
            patches = self.patches(c, min_overlap) if realign else None
            seq, qual = fqoracle.fastq(self.counts, calls, s0, L, ins_c, patches, trim_ends, uppercase, qual=q)
            out.append((name, seq, CC._unpatched(H.calls_to_changes(calls[s0:s0 + L]), patches), qual, patches))
        return out

    def reports(self, bam_path, t=None, min_depth=1, realign=False, trim_ends=False, uppercase=False, min_overlap=9,
                clip_decay_threshold=0.1):
        """PairedPiled's REPORT with `- quality_vote: True` after the option lines and `- quality-vote sites:` (every
        position of the contig whose call differs from the count vote's, patched or not) after `- ambiguous
        sites:`."""
        sites = self.sites(min_depth)
        out = {}
        texts = super().reports(bam_path, None, min_depth, realign, trim_ends, uppercase, min_overlap,
                                clip_decay_threshold)
        for c, name, s0, L, _ in self.contigs():
            lines = texts[name].split("\n")
            lines.insert(lines.index("observations:"), "- quality_vote: True")
            at = next(k for k, x in enumerate(lines) if x.startswith("- ambiguous sites:"))
            mine = [str(s - s0 + 1) for s in sites.tolist() if s0 <= s < s0 + L]
            lines.insert(at + 1, "- quality-vote sites: %s" % ", ".join(mine))
            out[name] = "\n".join(lines)
        return out
