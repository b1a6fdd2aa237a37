"""A seeded paired-read corpus that reaches what `--mask-overlaps` and `--primers` change in a consensus, and the
composed oracle it is checked against (test infrastructure).

The corpus (`pair_case`) is a list of BAM-style records with RNEXT / PNEXT over three contigs, with real QUAL strings
(some mates QUAL `*`), written as BAM and as SAM text, plus a primer BED (`PRIMERS`).  Every shape below is planted in
its own window of "mix" or "edge", where nothing else covers it, so that the counts the comment states are exact:
- IUPAC sites (IUPAC_*): the minor allele in both mates of two pairs and the major one in five single reads (0.6:
  counting once turns a code into a base); R1 minor / R2 major (0.6: a base into a code); R1 major / R2 minor beside
  five single reads (0.99: a code into a base).
- THIN: two overlapping pairs alone, depth 4 off and 2 on (min_depth 3: `N`).
- Insertions: INS_STRING (R1s `GT` / R2s `GA`: the chosen string changes), INS_TIE_GONE (R1 `CC` / R2 `AA`: the tie
  goes away), INS_TIE_NEW (one pair `CC` beside one read `AA`: a tie appears), INS_CALL_GONE (both mates carry it, so
  R2's I op is dropped and the `I` call goes), INS_CALL_NEW (R1 only: R2's masked bases lower the depth, the call
  comes); low-quality inserted bases; an insertion at the contig's last position (hard reads, never paired).
- Deletions: DEL_GONE (both mates: R2's D is dropped and the `D` call goes), DEL_NEW (R1 only: the call comes).
- The documented exceptions of K10 (include/kindel_b200.h) in EXCEPTIONS: an R1 with a real N, an R1 base masked by
  quality and one masked by a primer where R2 fills in, a kept R2 deletion that starts outside R1, an R2 insertion
  beside an R1 end.
- Left alone by the pairing (LEFT_ALONE): an R1 dropped by min_mapq 30 and one by 0x400 (R2 becomes a single read),
  three records of one QNAME, a secondary record beside a proper pair.
- "edge": a replaced segment whose breakpoints soft-clip both mates of four pairs, across which ten pairs read the
  reference: counting the spanning pairs once makes the breakpoints clip-dominant and `--realign` patches them.
- "gone": only reads that min_mapq 30 or exclude_flags 0x400 drop; header order gone, mix, edge; file order edge,
  gone, mix.

The composed oracle (`PairedPiled`) is made of the existing restatements only: oracle/py_moracle.ComposedMates (mates
on) or oracle/py_cvoracle.Composed (off) for the 19 columns and the insertion dicts, coracle.vote / ioracle.vote_iupac,
and fqoracle.fastq with the host's CDR functions over the oracle's table for the `--realign` patches.  The REPORT is
written here, line by line, from the oracle's tables.
"""
from __future__ import annotations

import itertools

import numpy as np

import combo_cases as CC
import helpers as H
from kindel_b200 import bamio
from oracle import coracle, fqoracle, ioracle
from oracle import py_cvoracle as CV
from oracle import py_moracle as MO

CONTIGS = [("gone", 200), ("mix", 900), ("edge", 400)]
GONE, MIX, EDGE = 0, 1, 2
FLAG_R1, FLAG_R2 = 0x1 | 0x2 | 0x40 | 0x20, 0x1 | 0x2 | 0x80 | 0x10
HIGH_Q = (30, 35, 37, 40)
IUPAC_CODE_TO_BASE = (40, 50)    # at 0.6
IUPAC_BASE_TO_CODE = (110, 120)  # at 0.6
IUPAC_99 = (180, 190)            # at 0.99
THIN = (235, 270)                # [lo, hi): depth 4 off, 2 on
INS_STRING, INS_TIE_GONE, INS_TIE_NEW = 320, 390, 460
INS_CALL_GONE, INS_CALL_NEW = 530, 580
DEL_GONE, DEL_NEW = 640, 700
EXCEPTIONS = (740, 800)
LEFT_ALONE = (810, 850)
PRIMERS = [("mix", 758, 764), ("mix", 812, 818), ("edge", 20, 40), ("gone", 10, 30)]
B1, B2 = 150, 180                # the edge's replaced segment [B1, B2)


class _Writer:
    def __init__(self, rng, refs):
        self.rng, self.refs, self.out, self.n = rng, refs, [], 0

    def qual(self, n, low_frac=0.0):
        q = self.rng.choice(HIGH_Q, size=n)
        low = self.rng.random(n) < low_frac
        q[low] = self.rng.choice((5, 10, 19), size=int(low.sum()))
        return q.astype(np.uint8)

    def rec(self, c, pos0, flag, cig, seq, name, mapq=60, qual="auto", mate=None):
        if isinstance(qual, str):
            qual = self.qual(len(seq))
        q = None if qual is None else bytes(np.asarray(qual, dtype=np.uint8).tolist())
        nref, npos = (c, mate) if mate is not None else (-1, -1)
        self.out.append((c, pos0, flag, bamio.parse_cigar_text(cig), seq, name, mapq, q, nref, npos))

    def single(self, c, pos0, cig, seq, qual="auto", flag=None, mapq=60):
        self.n += 1
        flag = int(self.rng.choice([0, 16])) if flag is None else flag
        self.rec(c, pos0, flag, cig, seq, "%s_s%d" % (CONTIGS[c][0], self.n), mapq, qual)

    def pair(self, c, a, ca, sa, b, cb, sb, qa="auto", qb="auto", fa=FLAG_R1, fb=FLAG_R2, ma=60, mb=60, name=None):
        """R1 at a, R2 at b (0-based), each naming the other's start; R2 gets QUAL `*` one time in five."""
        self.n += 1
        name = name or "%s_p%d" % (CONTIGS[c][0], self.n)
        if isinstance(qb, str) and self.rng.random() < 0.2:
            qb = None
        self.rec(c, a, fa, ca, sa, name, ma, qa, b)
        self.rec(c, b, fb, cb, sb, name, mb, qb, a)

    def m(self, c, a, n, subs=None):
        """Reference bases [a, a + n) of contig c, with {position: letter} substituted."""
        s = list(self.refs[c][a:a + n])
        for p, x in (subs or {}).items():
            if a <= p < a + n:
                s[p - a] = x
        return "".join(s)


def _other(ref, p, k=1):
    return "ACGT"[("ACGT".index(ref[p]) + k) % 4]


def _mix(w):
    ref = w.refs[MIX]
    m = lambda a, n, subs=None: w.m(MIX, a, n, subs)  # noqa: E731
    # IUPAC 0.6, code -> base: five single X reads, two pairs with Y in both mates (off 5:4, on 5:2)
    y = {p: _other(ref, p) for p in IUPAC_CODE_TO_BASE}
    for k in range(5):
        w.single(MIX, 20 + k, "45M", m(20 + k, 45))
    for k in range(2):
        w.pair(MIX, 25 + k, "40M", m(25 + k, 40, y), 30 + k, "40M", m(30 + k, 40, y))
    # IUPAC 0.6, base -> code: two single X reads, two pairs R1 Y / R2 X (off 4:2, on 2:2)
    y = {p: _other(ref, p) for p in IUPAC_BASE_TO_CODE}
    for k in range(2):
        w.single(MIX, 90 + k, "48M", m(90 + k, 48))
        w.pair(MIX, 95 + k, "40M", m(95 + k, 40, y), 100 + k, "40M", m(100 + k, 40))
    # IUPAC 0.99, code -> base: five single X reads, one pair R1 X / R2 Y (off 6:1, on 6:0)
    y = {p: _other(ref, p) for p in IUPAC_99}
    for k in range(5):
        w.single(MIX, 160 + k, "45M", m(160 + k, 45))
    w.pair(MIX, 165, "40M", m(165, 40), 170, "35M", m(170, 35, y))
    # thin columns: two overlapping pairs alone
    lo, hi = THIN
    for k in range(2):
        w.pair(MIX, lo - 5, "%dM" % (hi - lo + 5), m(lo - 5, hi - lo + 5), lo, "%dM" % (hi - lo), m(lo, hi - lo))

    def ins_read(a, n_left, ins, n_right, low=()):
        """(CIGAR, SEQ, QUAL) of a read at a with `ins` after n_left bases; `low`: inserted offsets at Q10."""
        q = w.qual(n_left + len(ins) + n_right)
        for j in low:
            q[n_left + j] = 10
        return "%dM%dI%dM" % (n_left, len(ins), n_right), m(a, n_left) + ins + m(a + n_left, n_right), q

    def ins_pair(site, s1, s2, low1=(), d=20):
        a, b = site - d, site - d + 5
        c1, q1s, q1 = ins_read(a, site - a, s1, 20, low1)
        c2, q2s, q2 = ins_read(b, site - b, s2, 25) if s2 else ("%dM" % (site - b + 25), m(b, site - b + 25), "auto")
        w.pair(MIX, a, c1, q1s, b, c2, q2s, qa=q1, qb=q2)

    # the chosen string changes: R1s GT (one with a low-quality T) and R2s GA three times, both GA twice
    for k in range(3):
        ins_pair(INS_STRING, "GT", "GA", low1=(1,) if k == 0 else ())
    for k in range(2):
        ins_pair(INS_STRING, "GA", "GA")
    # the tie goes away (off CC 2 : AA 2, on CC 2) and appears (off CC 2 : AA 1, on CC 1 : AA 1)
    for k in range(2):
        ins_pair(INS_TIE_GONE, "CC", "AA")
    ins_pair(INS_TIE_NEW, "CC", "CC")
    cig, seq, q = ins_read(INS_TIE_NEW - 18, 18, "AA", 22, low=(0,))
    w.single(MIX, INS_TIE_NEW - 18, cig, seq, q)
    # the I call goes (both mates, three pairs beside four plain reads: off 6 of 10, on 3 of 7) and comes (R1 only,
    # three pairs beside two plain reads: off 3 of 8, on 3 of 5)
    for k in range(3):
        ins_pair(INS_CALL_GONE, "TT", "TT")
    for k in range(4):
        w.single(MIX, INS_CALL_GONE - 20 + k, "42M", m(INS_CALL_GONE - 20 + k, 42))
    for k in range(3):
        ins_pair(INS_CALL_NEW, "GG", None)
    for k in range(2):
        w.single(MIX, INS_CALL_NEW - 20 + k, "42M", m(INS_CALL_NEW - 20 + k, 42))

    def del_read(a, site, right, n=2):
        left = site - a
        return "%dM%dD%dM" % (left, n, right), m(a, left) + m(site + n, right)

    # the D call goes (both mates, two pairs beside five plain reads: off 4 > 5 / 2, on 2 of 5) and comes (R1 only,
    # two pairs beside three plain reads: off 2 of 5, on 2 of 3)
    for k in range(2):
        c1, s1 = del_read(DEL_GONE - 20, DEL_GONE, 20)
        c2, s2 = del_read(DEL_GONE - 15, DEL_GONE, 25)
        w.pair(MIX, DEL_GONE - 20, c1, s1, DEL_GONE - 15, c2, s2)
    for k in range(5):
        w.single(MIX, DEL_GONE - 20 + k, "42M", m(DEL_GONE - 20 + k, 42))
    for k in range(2):
        c1, s1 = del_read(DEL_NEW - 20, DEL_NEW, 20)
        w.pair(MIX, DEL_NEW - 20, c1, s1, DEL_NEW - 15, "40M", m(DEL_NEW - 15, 40))
    for k in range(3):
        w.single(MIX, DEL_NEW - 20 + k, "42M", m(DEL_NEW - 20 + k, 42))
    # the documented exceptions at the edges of R1's information
    s = m(740, 40)
    w.pair(MIX, 740, "40M", s[:10] + "N" + s[11:], 745, "40M", m(745, 40), name="nR1")
    q = w.qual(40)
    q[15:19] = 5
    w.pair(MIX, 740, "40M", m(740, 40), 745, "40M", m(745, 40), qa=q, name="lowR1")
    w.pair(MIX, 760, "40M", m(760, 40), 750, "45M", m(750, 45), name="primerR1")  # R1's 760..763: primer bases
    w.pair(MIX, 770, "30M", m(770, 30), 760, "8M4D26M", m(760, 8) + m(772, 26), name="delOutside")
    w.pair(MIX, 740, "30M", m(740, 30), 745, "25M2I20M", m(745, 25) + "CG" + m(770, 20), name="insBesideEnd")
    # left alone: R1 below MAPQ 30, R1 a duplicate, three records of one name, a secondary beside a proper pair
    lo = LEFT_ALONE[0]
    w.pair(MIX, lo + 2, "28M", m(lo + 2, 28), lo + 5, "30M", m(lo + 5, 30), ma=5, name="lowMapqR1")
    w.pair(MIX, lo + 2, "28M", m(lo + 2, 28), lo + 5, "30M", m(lo + 5, 30), fa=FLAG_R1 | 0x400, name="dupR1")
    w.pair(MIX, lo + 2, "28M", m(lo + 2, 28), lo + 5, "30M", m(lo + 5, 30), name="three")
    w.rec(MIX, lo + 5, FLAG_R2, "30M", m(lo + 5, 30), "three", mate=lo + 2)
    w.pair(MIX, lo + 2, "28M", m(lo + 2, 28), lo + 5, "30M", m(lo + 5, 30), name="withSecondary")
    w.rec(MIX, lo + 6, FLAG_R2 | 0x100, "20M", m(lo + 6, 20), "withSecondary", mate=lo + 2)
    # an insertion at the last position, partly masked (these reads reach the contig end: hard, never paired)
    L = CONTIGS[MIX][1]
    for k in range(5):
        n = 30 + 4 * k
        q = w.qual(n + 3)
        q[n:n + 2] = [[35, 35], [10, 35], [35, 10], [35, 35], [10, 10]][k]
        w.single(MIX, L - 1 - n, "%dM2I1M" % n, m(L - 1 - n, n) + "CA" + ref[L - 1], q, flag=0)
    w.pair(MIX, L - 41, "40M2I1M", m(L - 41, 40) + "CA" + ref[L - 1], L - 31, "30M2I1M",
           m(L - 31, 30) + "CA" + ref[L - 1], name="hardPair")


def _edge(w):
    ref = w.refs[EDGE]
    z = "".join(w.rng.choice(list("ACGT"), size=18))
    right = z + ref[B2:]
    left = ref[:B1] + z
    m = lambda a, n: w.m(EDGE, a, n)  # noqa: E731
    for k in range(4):  # both mates clipped at B1, and both at B2
        t1, t2 = right[:20 + k], right[:22 + k]
        w.pair(EDGE, B1 - 40 + k, "%dM%dS" % (40 - k, len(t1)), m(B1 - 40 + k, 40 - k) + t1,
               B1 - 30 + k, "%dM%dS" % (30 - k, len(t2)), m(B1 - 30 + k, 30 - k) + t2)
        h1, h2 = left[-(20 + k):], left[-(22 + k):]
        w.pair(EDGE, B2, "%dS%dM" % (len(h1), 40 - k), h1 + m(B2, 40 - k),
               B2, "%dS%dM" % (len(h2), 30 + k), h2 + m(B2, 30 + k))
    for k in range(10):  # pairs across the segment that read the reference
        w.pair(EDGE, B1 - 25 + k, "%dM" % (B2 - B1 + 50), m(B1 - 25 + k, B2 - B1 + 50),
               B1 - 20 + k, "%dM" % (B2 - B1 + 45), m(B1 - 20 + k, B2 - B1 + 45))
    for k in range(12):  # pairs and single reads elsewhere; positions 0..11 and L-12.. stay uncovered
        a = int(w.rng.integers(12, 90)) if k % 2 else int(w.rng.integers(B2 + 30, 330))
        if k % 3:
            w.pair(EDGE, a, "50M", m(a, 50), a + 8, "50M", m(a + 8, 50))
        else:
            w.single(EDGE, a, "55M", m(a, 55), w.qual(55, 0.1))


def _gone(w):
    for k in range(6):
        a = 10 + 20 * k
        if k % 2:
            w.pair(GONE, a, "40M", w.m(GONE, a, 40), a + 10, "40M", w.m(GONE, a + 10, 40), fa=FLAG_R1 | 0x400,
                   fb=FLAG_R2 | 0x400)
        else:
            w.pair(GONE, a, "40M", w.m(GONE, a, 40), a + 10, "40M", w.m(GONE, a + 10, 40), ma=5, mb=12)


def pair_case(seed):
    """(contigs, records): a record is (ref_id, pos0, flag, cigar words, SEQ, QNAME, MAPQ, QUAL bytes or None, RNEXT
    id, PNEXT 0-based), as bamio.write_bam takes it; file order edge, gone, mix."""
    rng = np.random.default_rng(seed)
    refs = ["".join(rng.choice(list("ACGT"), size=L)) for _, L in CONTIGS]
    parts = []
    for fill in (_edge, _gone, _mix):
        w = _Writer(rng, refs)
        fill(w)
        w.out.sort(key=lambda r: r[1])
        parts += w.out
    return list(CONTIGS), parts


def sam_text(contigs, records):
    lines = ["@HD\tVN:1.6\tSO:unsorted"] + ["@SQ\tSN:%s\tLN:%d" % c for c in contigs]
    for ref_id, pos, flag, cig, seq, name, mapq, qual, nref, npos in records:
        cig_text = "".join("%d%s" % (w >> 4, "MIDNSHP=X"[w & 15]) for w in cig)
        qtext = "*" if qual is None else "".join(chr(33 + x) for x in qual)
        rnext = "*" if nref < 0 else "="
        lines.append("\t".join([name, str(flag), contigs[ref_id][0], str(pos + 1), str(mapq), cig_text, rnext,
                                str(npos + 1), "0", seq, qtext]))
    return "\n".join(lines) + "\n"


def write(d, seed=1):
    """dict(bam, sam, bed, rows, contigs, recs) of the corpus under directory d."""
    contigs, recs = pair_case(seed)
    bam, sam, bed = str(d / "pairs.bam"), str(d / "pairs.sam"), d / "pairs.bed"
    bamio.write_bam(bam, contigs, recs)
    with open(sam, "w") as fh:
        fh.write(sam_text(contigs, recs))
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in PRIMERS))
    return dict(bam=bam, sam=sam, bed=str(bed), rows=list(PRIMERS), contigs=contigs, recs=recs)


def option_matrix():
    """Rows of (iupac_threshold, min_base_quality, min_depth, realign, trim_ends, uppercase, (min_mapq, exclude_flags),
    primers, mask_overlaps) such that every pair of values of every two options occurs in some row (combo_cases'
    greedy method)."""
    levels = [(None, 0.6, 0.99), (0, 20), (1, 3), (False, True), (False, True), (False, True), ((0, 0), (30, 0x400)),
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
class PairedPiled:
    """The oracle's table, insertion dicts and consensus of one file at one (min_base_quality, min_mapq,
    exclude_flags, primer rows, mates).  layout: any decode of the file's contigs (names, slots, lengths only)."""

    def __init__(self, path, layout, min_base_quality=0, min_mapq=0, exclude_flags=0, primer_rows=None, mates=False,
                 primers_name=None):
        self.path, self.layout, self.mates = path, layout, mates
        self.filters = (min_base_quality, min_mapq, exclude_flags)
        self.primers_name = primers_name
        if mates:
            self.oracle = MO.ComposedMates(path, min_base_quality, min_mapq, exclude_flags, primer_rows)
        else:
            self.oracle = CV.Composed(path, min_base_quality, min_mapq, exclude_flags, primer_rows)
        tables = self.oracle.tables(0)
        assert [nm for nm, _, _ in tables] == list(layout.contig_names)
        self.counts = np.zeros((19, int(layout.n_slots)), dtype=np.int32)
        self.ins = {}  # slot -> {string: count}, first-seen order
        for c, (nm, cols, dicts) in enumerate(tables):
            s0 = int(layout.contig_slot[c])
            self.counts[:, s0:s0 + len(cols[0])] = np.array(cols, dtype=np.int32)
            for p, d in enumerate(dicts):
                if d:
                    self.ins[s0 + p] = dict(d)

    @property
    def overlap_stats(self):
        return self.oracle.overlap_stats if self.mates else None

    def calls(self, t=None, min_depth=1):
        return coracle.vote(self.counts, min_depth) if t is None else ioracle.vote_iupac(self.counts, min_depth, t)

    def contigs(self):
        b = self.layout
        for c, name in enumerate(b.contig_names):
            s0, L = int(b.contig_slot[c]), int(b.contig_len[c])
            yield c, name, s0, L, {s - s0: d for s, d in self.ins.items() if s0 <= s <= s0 + L}

    def patches(self, c, min_overlap=9, clip_decay_threshold=0.1, mask_ends=50):
        """The merged CDR patches of contig c by the host's CDR functions over the oracle's table."""
        from kindel_b200 import kindel as K

        run = K.PileupRun.from_host_tables(self.layout, self.counts, coracle.derive(self.counts),
                                           np.zeros((0, 4), dtype=np.int32))
        aln = run.alignment(c)
        return K.merge_cdrps(K.cdrp_consensuses(aln.weights, aln.deletions, aln.clip_start_weights,
                                                aln.clip_end_weights, aln.clip_start_depth, aln.clip_end_depth,
                                                clip_decay_threshold, mask_ends), min_overlap)

    def consensus(self, t=None, min_depth=1, realign=False, trim_ends=False, uppercase=False, min_overlap=9):
        """[(name, sequence, changes, qualities, patches)] per contig."""
        calls = self.calls(t, min_depth)
        out = []
        for c, name, s0, L, ins_c in self.contigs():
            patches = self.patches(c, min_overlap) if realign else None
            seq, qual = fqoracle.fastq(self.counts, calls, s0, L, ins_c, patches, trim_ends, uppercase)
            out.append((name, seq, CC._unpatched(H.calls_to_changes(calls[s0:s0 + L]), patches), qual, patches))
        return out

    def reports(self, bam_path, t=None, min_depth=1, realign=False, trim_ends=False, uppercase=False, min_overlap=9,
                clip_decay_threshold=0.1):
        """{contig: REPORT text} as DESIGN.md section 1 words it: the reference's lines, the filter, primer, mate
        overlap and IUPAC option lines, and `- iupac sites:` (positions whose call holds two or more bases)."""
        calls = self.calls(t, min_depth)
        out = {}
        for (c, name, s0, L, _), (_, _, changes, _, patches) in zip(
                self.contigs(), self.consensus(t, min_depth, realign, trim_ends, uppercase, min_overlap)):
            acgt = self.counts[0:4, s0:s0 + L].astype(np.int64).sum(axis=0)
            sites = {k: [str(p + 1) for p, x in enumerate(changes) if x == k] for k in "NID"}
            lines = ["========================= REPORT ===========================", "reference: %s" % name,
                     "options:", "- bam_path: %s" % bam_path, "- min_depth: %s" % min_depth, "- realign: %s" % realign,
                     "    - min_overlap: %s" % min_overlap, "    - clip_decay_threshold: %s" % clip_decay_threshold,
                     "- trim_ends: %s" % trim_ends, "- uppercase: %s" % uppercase]
            if any(self.filters):
                lines += ["- min_base_quality: %d" % self.filters[0], "- min_mapq: %d" % self.filters[1],
                          "- exclude_flags: %#x" % self.filters[2]]
            if self.primers_name is not None:
                lines.append("- primers: %s" % self.primers_name)
            if self.mates:
                lines.append("- mate overlaps: %d pairs, %d bases, %d deletions, %d insertions masked"
                             % self.overlap_stats)
            if t is not None:
                lines.append("- iupac_threshold: %s" % t)
            lines += ["observations:", "- min, max observed depth: %d, %d" % (int(acgt.min()), int(acgt.max())),
                      "- ambiguous sites: %s" % ", ".join(sites["N"])]
            if t is not None:
                # multi-base calls (ioracle's 0x80) at the positions the walk emits: a patch replaces the ones it spans
                visited = CC._unpatched(list(range(1, L + 1)), patches)
                multi = [str(p + 1) for p in range(L) if int(calls[s0 + p]) & 0x80 and visited[p] is not None]
                lines.append("- iupac sites: %s" % ", ".join(multi))
            lines += ["- insertion sites: %s" % ", ".join(sites["I"]), "- deletion sites: %s" % ", ".join(sites["D"]),
                      "- clip-dominant regions: %s" % ", ".join("%d-%d: %s" % (r.start, r.end, r.seq)
                                                                for r in patches or [])]
            out[name] = "\n".join(lines) + "\n"
        return out

