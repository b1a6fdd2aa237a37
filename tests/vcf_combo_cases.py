"""A seeded corpus that turns every `variants --vcf` option on at once (test infrastructure): base and read filters,
primers, a reference FASTA and strand, checked against one composed oracle (oracle/py_cvoracle.py).

Contigs, in a header order unlike the read order (first-seen order: the tiny ones, one, two, lowmq, edge, main):
- "main" (513 bases): three tiled amplicons whose reads start and end in primers.  Amplicon 2's reads copy the
  reference at SITE, inside its left primer, where the sample differs; amplicon 1 reads through it.  Planted: a
  forward-only SNV, a reverse-only insertion and a forward-only deletion (amplicon 1), a balanced SNV (SOR ln 2) and an
  insertion written with an IUPAC letter, `GRT`, whose R is low-quality in some reads (amplicon 2), a reverse-only
  insertion whose anchor base is low-quality in every carrier (amplicon 3: with the quality mask its reverse depth is
  below its reverse count), an SNV that only primer bases carry (gone with primers) and one that only low-quality
  bases carry (gone with the quality mask).
- "edge" (150): a FASTA with N, IUPAC and lower-case letters; deletions at POS 1 (cursor 0 and cursor 1) and one that
  ends on the last base, insertions at p = 0 and p = L, soft clips with low-quality clip bases.
- "one" (1 base: insertions at p = 0 and p = L), "two" (2), a dozen tiny contigs that share one 512-slot tile, "lowmq"
  (every read below MAPQ 30) and "nohits" (a header line and no read at all).
Records carry both strands, QUAL `*` on some, low qualities on primer bases (masked twice, listed once), MAPQ values
below 30 and the flags 0x100 and 0x400.  With exotic=True one more read holds a low-quality `R` in an M op and a
low-quality `Y` in a soft clip: masked they raise nothing, unmasked the walk raises KeyError."""
from __future__ import annotations

import itertools

import numpy as np

from kindel_b200 import bamio

MAIN_L, EDGE_L = 513, 150
TINY = [("t%02d" % k, L) for k, L in enumerate((3, 5, 7, 9, 11, 13, 4, 6, 8, 10, 12, 14))]
READ_ORDER = [nm for nm, _ in TINY] + ["one", "two", "lowmq", "edge", "main"]
LENGTHS = dict(TINY, one=1, two=2, lowmq=80, edge=EDGE_L, main=MAIN_L, nohits=50)
AMPS = ((0, 200), (150, 360), (310, 513))
PRIMER = 20
SITE = 160                        # in amplicon 2's left primer [150, 170)
SNV_ONE, INS_ONE, DEL_ONE = 60, 100, 120
QLOW_SNV = 170                    # carried by low-quality bases only
SNV_BAL, IUPAC_INS = 250, 280
PRIMER_SNV, CLAMP_INS = 325, 420  # in amplicon 3's left primer / after an always-masked anchor
EDGE_ODD = {30: "N", 31: "R", 75: "Y", 76: "n"}
LOW_Q = (3, 11, 19)
HIGH_Q = (20, 27, 33, 38, 40)


def _other(b, k=1):
    return "ACGT"[("ACGT".index(b.upper()) + k) % 4]


class _Builder:
    def __init__(self, rng, header):
        self.rng, self.header, self.out = rng, header, []

    def read(self, contig, start, ops, sample, alt=None, flag=0, mapq=60, low=(), no_qual=False):
        """ops: ("M", n), ("I", text), ("D", n), ("S", text).  alt: {ref pos: base}; low: ref positions (M bases),
        ("I", k) (the k-th inserted base of the read) or ("S", k) (the k-th clipped base) with a low quality."""
        alt = alt or {}
        seq, q_of, cig, r, ins, clip = [], {}, [], start, [], []
        for op, x in ops:
            if op == "M":
                for p in range(r, r + x):
                    q_of[p] = len(seq)
                    seq.append(alt.get(p, sample[p]))
                r += x
                cig.append((x << 4) | 0)
            elif op == "D":
                r += x
                cig.append((x << 4) | 2)
            else:
                (ins if op == "I" else clip).extend(range(len(seq), len(seq) + len(x)))
                seq.extend(x)
                cig.append((len(x) << 4) | (1 if op == "I" else 4))
        qual = self.rng.choice(HIGH_Q, size=len(seq)).astype(np.uint8)
        for w in low:
            k = ins[w[1]] if isinstance(w, tuple) and w[0] == "I" else clip[w[1]] if isinstance(w, tuple) else q_of[w]
            qual[k] = self.rng.choice(LOW_Q)
        self.out.append((self.header.index(contig), start, flag, cig, "".join(seq), "r%d" % len(self.out), mapq,
                         None if no_qual else bytes(qual.tolist())))


def _fields(rng):
    """(extra flag, MAPQ) of an ordinary read: mostly kept, sometimes dropped by one of the two record filters."""
    return int(rng.choice([0, 0, 0, 0, 0x100, 0x400])), int(rng.choice([60, 60, 60, 60, 45, 29, 10, 0]))


def vcf_combo_case(seed=1, exotic=False):
    """(header contigs [(name, L)], records as bamio.write_bam takes them, {name: reference text}, primer rows)."""
    rng = np.random.default_rng(seed)
    header = list(LENGTHS)
    header = [header[i] for i in rng.permutation(len(header))]
    refs = {nm: "".join(rng.choice(list("ACGT"), size=L)) for nm, L in LENGTHS.items()}
    edge = list(refs["edge"])
    for p, ch in EDGE_ODD.items():
        edge[p] = ch
    edge[100:106] = [c.lower() for c in edge[100:106]]
    refs["edge"] = "".join(edge)
    B = _Builder(rng, header)

    def strand():
        return 16 * int(rng.integers(0, 2))

    # tiny contigs, one, two
    for nm, L in TINY:
        p = int(rng.integers(0, L))
        for j in range(6):
            a = int(rng.integers(0, L - 1))
            n = int(rng.integers(2, L - a + 1))
            f, mq = _fields(rng)
            B.read(nm, a, [("M", n)], refs[nm], {p: _other(refs[nm][p])} if j < 3 else None, f | strand(), mq,
                   no_qual=j == 5)
    for j in range(7):
        if j < 4:
            B.read("one", 0, [("M", 1), ("I", "G")], refs["one"], flag=16 * (j % 2), low=[("I", 0)] if j == 0 else ())
        else:
            B.read("one", 0, [("I", "T"), ("M", 1)], refs["one"], flag=16 * (j % 2))
    for j in range(6):
        B.read("two", 0, [("M", 2)], refs["two"], {1: _other(refs["two"][1])} if j < 3 else None, 16 * (j == 2))
    # lowmq: every read below MAPQ 30
    for j in range(10):
        a = int(rng.integers(0, 40))
        B.read("lowmq", a, [("M", 40)], refs["lowmq"], {40: _other(refs["lowmq"][40])} if j < 5 else None, strand(),
               int(rng.integers(0, 30)))
    # edge: the reads copy a sample without the reference's N / IUPAC letters
    s_edge = "".join(ch if ch in "ACGT" else "ACGT"[i % 4] for i, ch in enumerate(refs["edge"].upper()))
    L = EDGE_L
    for j in range(5):
        B.read("edge", 0, [("D", 3), ("M", 40)], s_edge, flag=16 * (j % 2))
    for j in range(4):
        B.read("edge", 0, [("M", 1), ("D", 2), ("M", 40)], s_edge, flag=16 * (j % 2), low=[0] if j == 0 else ())
        B.read("edge", 0, [("I", "TT"), ("M", 40)], s_edge, flag=16 * (j > 0))
        B.read("edge", L - 40, [("M", 40), ("I", "AC")], s_edge, flag=16 * (j % 2), low=[("I", 1)] if j == 1 else ())
        B.read("edge", L - 43, [("M", 40), ("D", 3)], s_edge, flag=16 * (j < 3))
    for j in range(3):
        B.read("edge", 20, [("S", "GATTAC"), ("M", 30)], s_edge, flag=strand(), low=[("S", 1), ("S", 4)])
        B.read("edge", L - 40, [("M", 30), ("S", "CCTGAG")], s_edge, flag=strand(), low=[("S", 0), 120])
    for j in range(30):
        a = int(rng.integers(0, L - 50))
        n = int(rng.integers(30, 50))
        alt = {p: _other(s_edge[p]) for p in (30, 31, 75, 101) if rng.random() < 0.4}
        if rng.random() < 0.1:
            alt[a + 3] = "N"
        f, mq = _fields(rng)
        low = [p for p in range(a, a + n) if rng.random() < 0.05]
        B.read("edge", a, [("M", n)], s_edge, alt, f | strand(), mq, low, no_qual=j % 7 == 6)
    if exotic:
        B.read("edge", 50, [("S", "AYC"), ("M", 40)], s_edge, {60: "R"}, 0, 60, low=[60, ("S", 1)])
    # main: three tiled amplicons
    ref = refs["main"]
    sample = ref[:SITE] + _other(ref[SITE], 2) + ref[SITE + 1:]
    primers = [(a, a + PRIMER) for a, b in AMPS] + [(b - PRIMER, b) for a, b in AMPS]

    def in_primer(p):
        return any(a <= p < b for a, b in primers)

    def amp_seq(k):
        """The sample with the amplicon's own primer bases copied from the reference (the oligo)."""
        a, b = AMPS[k]
        s = list(sample)
        s[a:a + PRIMER], s[b - PRIMER:b] = ref[a:a + PRIMER], ref[b - PRIMER:b]
        return "".join(s)

    def low_lattice(a, b, avoid=()):
        out = [p for p in range(a, b) if rng.random() < 0.03 and p not in avoid]
        if rng.random() < 0.5:  # low bases on primer bases: masked twice, listed once
            out += [p for p in (a + 2, a + 5, b - 3) if p not in out]
        return out

    s1 = amp_seq(0)
    for j in range(44):
        a, b = AMPS[0]
        if j % 4 == 3:
            a, b = a + int(rng.integers(1, 26)), b - int(rng.integers(1, 26))
        alt, ops, flag, mq = {}, [("M", b - a)], strand(), 60
        low = low_lattice(a, b, avoid=(QLOW_SNV,))
        if j < 10 or 26 <= j < 30:
            alt[SNV_ONE], flag = _other(s1[SNV_ONE]), 0x400 * (j >= 26)
            low = [p for p in low if p != SNV_ONE]
        elif j < 18:
            ops, flag = [("M", INS_ONE - a), ("I", "GT"), ("M", b - INS_ONE)], 16
            low += [("I", 0)] if j < 12 else []
        elif j < 26:
            ops, flag = [("M", DEL_ONE - a), ("D", 2), ("M", b - DEL_ONE - 2)], 0
        elif j < 34:
            flag, mq = _fields(rng)
            flag |= strand()
        if 34 <= j < 38:
            alt[QLOW_SNV] = _other(s1[QLOW_SNV])
            low.append(QLOW_SNV)
        if j >= 40:
            a = 10
            ops = [("S", "ACGTA"), ("M", b - a)] if j % 2 else [("M", b - a), ("S", "TTGCA")]
            low = [("S", 0), ("S", 3)] + [p for p in low if p >= a]
        B.read("main", a, ops, s1, alt, flag, mq, [p for p in low if not isinstance(p, int) or a <= p],
               no_qual=j % 9 == 8)
    s2 = amp_seq(1)
    for j in range(48):
        a, b = AMPS[1]
        alt, ops = {}, [("M", b - a)]
        if j < 12:
            alt[SNV_BAL] = _other(s2[SNV_BAL])
        low = low_lattice(a, b, avoid=(SNV_BAL,))
        if j in (13, 15, 17, 19, 21, 23):
            ops = [("M", IUPAC_INS - a), ("I", "GRT"), ("M", b - IUPAC_INS)]
            low += [("I", 1)] if j in (13, 15) else []
        B.read("main", a, ops, s2, alt, 16 * (j % 2), 60, low)
    s3 = amp_seq(2)
    for j in range(40):
        a, b = AMPS[2]
        alt, ops, flag, mq = {}, [("M", b - a)], 16 * (j % 2), 60
        low = low_lattice(a, b, avoid=(CLAMP_INS - 1, PRIMER_SNV))
        if j % 2:
            ops = [("M", CLAMP_INS - a), ("I", "CA"), ("M", b - CLAMP_INS)]
            low.append(CLAMP_INS - 1)
        else:
            f, mq = _fields(rng)
            flag |= f
        if j % 3 == 0:
            alt[PRIMER_SNV] = _other(s3[PRIMER_SNV])
        B.read("main", a, ops, s3, alt, flag, mq, low, no_qual=j % 11 == 10)
    assert in_primer(SITE) and in_primer(PRIMER_SNV)
    # file order: contig by contig in READ_ORDER, by position inside a contig
    recs = sorted(B.out, key=lambda r: (READ_ORDER.index(header[r[0]]), r[1]))
    rows = [("main", a, b) for a, b in primers] + [("main", 0, PRIMER)]  # a duplicate row
    rows += [("edge", 0, 12), ("t03", 0, 3), ("lowmq", 30, 50), ("elsewhere", 0, 5)]
    return [(nm, LENGTHS[nm]) for nm in header], recs, refs, rows


def write(d, seed=1, exotic=False):
    """(BAM, SAM, FASTA, BED paths, contigs, records, refs, rows) of the corpus, under directory d."""
    contigs, recs, refs, rows = vcf_combo_case(seed, exotic)
    tag = "%d%s" % (seed, "x" if exotic else "")
    bam, sam, fa, bed = (d / ("vc%s.%s" % (tag, ext)) for ext in ("bam", "sam", "fa", "bed"))
    bamio.write_bam(str(bam), contigs, recs)
    lines = ["@HD\tVN:1.6\tSO:unsorted"] + ["@SQ\tSN:%s\tLN:%d" % c for c in contigs]
    for ref_id, pos, flag, cig, seq, name, mapq, qual in recs:
        cig_text = "".join("%d%s" % (w >> 4, "MIDNSHP=X"[w & 15]) for w in cig)
        qtext = "*" if qual is None else "".join(chr(33 + x) for x in qual)
        lines.append("\t".join([name, str(flag), contigs[ref_id][0], str(pos + 1), str(mapq), cig_text, "*", "0", "0",
                                seq, qtext]))
    sam.write_text("\n".join(lines) + "\n")
    fa.write_text("".join(">%s some description\n%s\n" % (nm, "\n".join(refs[nm][i:i + 60] for i in
                                                                          range(0, len(refs[nm]), 60)))
                          for nm, _ in contigs))
    bed.write_text("track name=scheme\n" + "".join("%s\t%d\t%d\tp%d\t1\t+\n" % (r + (k,)) for k, r in enumerate(rows)))
    return bam, sam, fa, bed, contigs, recs, refs, rows


# ------------------------------------------------------------------------------------------------ option matrix
LEVELS = (("min_base_quality", (0, 20)), ("min_mapq", (0, 30)), ("exclude_flags", (0, 0x500)),
          ("primers", (False, True)), ("reference", (False, True)), ("strand", ("off", "on", 3.0)),
          ("thresholds", ((1, 0.01), (0, 0), (2, 0.2), (-1, -0.5))))


def _pairs(row):
    return {(i, row[i], j, row[j]) for i, j in itertools.combinations(range(len(row)), 2)}


def option_matrix():
    """Rows (one value per LEVELS entry) such that every pair of values of every two options occurs in some row."""
    sizes = [len(v) for _, v in LEVELS]
    want = set().union(*(_pairs(r) for r in itertools.product(*[range(n) for n in sizes])))
    rows = []
    while want:
        best = max(itertools.product(*[range(n) for n in sizes]), key=lambda r: len(_pairs(r) & want))
        want -= _pairs(best)
        rows.append(best)
    return [tuple(LEVELS[i][1][v] for i, v in enumerate(r)) for r in rows]


def masking_product():
    """Every combination of the four masking inputs, with reference, strand (max_sor 3) and (1, 0.01) on."""
    return [(bq, mq, ex, pr, True, 3.0, (1, 0.01)) for bq, mq, ex, pr in itertools.product((0, 20), (0, 30), (0, 0x500),
                                                                                          (False, True))]
