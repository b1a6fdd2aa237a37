"""Fixtures with base qualities for `variants --vcf --qual` (test infrastructure).

None of the fixtures under tests/golden/inputs/ has qualities, and the VCF combo corpus (vcf_combo_cases) has reads
with QUAL `*`.  `rewrite` writes such records again with seeded Phred values where they had none; `planted` builds a
truth set: a real 2 % allele at Q35 beside a 2 % allele made only of Q5 bases, a 20 % allele whose AQ hits the
underflow cap, a `*`-only site, and a strand-biased low-quality allele that fails both `sor` and `lowqual`."""
from __future__ import annotations

import numpy as np

from kindel_b200 import bamio

QUAL_LEN = 300
REF = "".join("ACGT"[(i * 7 + i // 5) % 4] for i in range(QUAL_LEN))
SITE_REAL, SITE_LOW, SITE_CAP, SITE_DEL, SITE_BIAS = 50, 100, 150, 200, 250


def _alt(b):
    return "ACGT"[("ACGT".index(b) + 1) % 4]


def write_sam(path, contigs, recs):
    """SAM text of records (ref_id, pos0, flag, cigar words, seq, name, mapq, qual or None[, next ref_id, next pos0]),
    as bamio.write_bam takes them: RNEXT / PNEXT `*` / 0 without a mate, CIGAR `*` without ops."""
    lines = ["@HD\tVN:1.6\tSO:unsorted"] + ["@SQ\tSN:%s\tLN:%d" % c for c in contigs]
    for rec in recs:
        ref_id, pos, flag, cig, seq, name, mapq, qual = rec[:8]
        nref, npos = rec[8:10] if len(rec) >= 10 else (-1, -1)
        cig_text = "".join("%d%s" % (w >> 4, "MIDNSHP=X"[w & 15]) for w in cig) or "*"
        qtext = "*" if qual is None else "".join(chr(33 + x) for x in qual)
        rnext = "*" if nref < 0 else ("=" if nref == ref_id else contigs[nref][0])
        lines.append("\t".join([name, str(flag), contigs[ref_id][0], str(pos + 1), str(mapq), cig_text, rnext,
                                str(npos + 1) if nref >= 0 else "0", "0", seq, qtext]))
    with open(path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


def rewrite(recs, seed=7):
    """The records with seeded Phred values (2..41) where they had none."""
    rng = np.random.default_rng(seed)
    out = []
    for ref_id, pos, flag, cig, seq, name, mapq, qual in recs:
        if qual is None:
            qual = bytes(rng.integers(2, 42, len(seq), dtype=np.uint8).tolist())
        out.append((ref_id, pos, flag, cig, seq, name, mapq, qual))
    return out


def planted(seed=3, depth=1000):
    """(contigs, records) of the truth set on one contig `q` of QUAL_LEN bases: `depth` 300-base reads of REF at Q35,
    where 2 % carry the ALT base at SITE_REAL (Q35); 2 % at SITE_LOW, a column of Q5 bases; 20 % at SITE_CAP; 3 % a
    deletion at SITE_DEL; and 2 % at SITE_BIAS, a column of Q10 bases, on reverse reads only."""
    rng = np.random.default_rng(seed)
    recs = []
    n_alt = depth // 50
    for j in range(depth):
        seq = list(REF)
        qual = [35] * QUAL_LEN
        cig = [(QUAL_LEN << 4) | 0]
        flag = 16 if j % 2 else 0
        if j < n_alt:
            seq[SITE_REAL] = _alt(REF[SITE_REAL])
        qual[SITE_LOW], qual[SITE_BIAS] = 5, 10
        if n_alt <= j < 2 * n_alt:
            seq[SITE_LOW] = _alt(REF[SITE_LOW])
        if j < depth // 5:
            seq[SITE_CAP] = _alt(REF[SITE_CAP])
        if 2 * n_alt <= j < 3 * n_alt:
            seq[SITE_BIAS] = _alt(REF[SITE_BIAS])
            flag = 16
        elif j >= 3 * n_alt:
            flag = 0 if j % 3 else flag
        if depth - 30 <= j:  # a deletion of SITE_DEL: `*` in the sites-only VCF
            del seq[SITE_DEL]
            del qual[SITE_DEL]
            cig = [(SITE_DEL << 4) | 0, (1 << 4) | 2, ((QUAL_LEN - SITE_DEL - 1) << 4) | 0]
        recs.append((0, 0, flag, cig, "".join(seq), "p%d" % j, 60, bytes(int(x) for x in qual)))
    rng.shuffle(recs)
    recs.sort(key=lambda r: r[1])
    return [("q", QUAL_LEN)], recs


def write(d, contigs, recs, tag):
    bam, sam = d / ("%s.bam" % tag), d / ("%s.sam" % tag)
    bamio.write_bam(str(bam), contigs, recs)
    write_sam(str(sam), contigs, recs)
    return str(bam), str(sam)
