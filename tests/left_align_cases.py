"""A truth set for `--left-align` (test infrastructure) that rests on no shared code: a reference with repeats and reads
that place one deletion and one insertion of a repeat unit at every offset of each repeat, and the expectation of
each placement by brute force over haplotype strings.

Contigs: "rep" with a homopolymer, a di- and a tri-nucleotide repeat and a G run split by an N; "head", whose first
bases are a repeat (the r = 0 and p = 0 placements, which without left-alignment become two records with one POS,
REF and ALT); "tail", whose last bases are a repeat (insertions at p = L).  Every placement has two reads, one on each
strand; the reads copy the reference elsewhere.  The expectation of a placement is its leftmost equivalent one:
moving one base left while the moved event still gives the same haplotype string, the base it crosses is A, C, G or
T, and (insertions) the string's last base is that base."""
from __future__ import annotations

from kindel_b200 import bamio

_FLANK = 8
# contig -> reference text; repeats: (contig, start, unit, copies)
REFS = {
    "rep": ("TGCATCGTCATGCATTCGAT" "AAAAAA" "CTGCTCATGGTCAGTACGTC" "ACACACAC" "TGTCATGCTCGATCGTACTG"
            "AGTAGTAGT" "CTGTCAGCTACGTCTAGCAT" "GGGNGGG" "TCATGCTACTCGTACTGCAT"),
    "head": "TTTTT" "GCAGTCAGCATGCATCGATGCATCAGCTAGCTAGCAGCTAC",
    "tail": "CTGACTGCATCGACTAGCATGCATCAGTCAGCTAGCAGCTTC" "GAGAGA",
}
_REP = REFS["rep"]
REPEATS = [("rep", _REP.index("AAAAAA"), "A", 6), ("rep", _REP.index("ACACACAC"), "AC", 4),
           ("rep", _REP.index("AGTAGTAGT"), "AGT", 3), ("rep", _REP.index("GGGN"), "G", 3),
           ("rep", _REP.index("NGGG") + 1, "G", 3), ("head", 0, "T", 5), ("tail", len(REFS["tail"]) - 6, "GA", 3)]
CONTIGS = [(nm, len(s)) for nm, s in REFS.items()]


def deletion_haplotype(ref, r, n):
    return ref[:r] + ref[r + n:]


def insertion_haplotype(ref, p, t):
    return ref[:p] + t + ref[p:]


def leftmost_deletion(ref, r, n):
    """The leftmost equivalent placement of a deletion (brute force over haplotype strings)."""
    hap = deletion_haplotype(ref, r, n)
    while r > 0 and ref[r - 1] in "ACGT" and deletion_haplotype(ref, r - 1, n) == hap:
        r -= 1
    return r


def leftmost_insertion(ref, p, t):
    """(p, t) of the leftmost equivalent placement of an insertion (brute force over haplotype strings)."""
    hap, m = insertion_haplotype(ref, p, t), len(t)
    while p > 0 and ref[p - 1] in "ACGT" and t[-1] == ref[p - 1]:
        q = p - 1
        s = hap[q:q + m]
        if insertion_haplotype(ref, q, s) != hap:
            break
        p, t = q, s
    return p, t


def placements():
    """[(repeat index, kind, contig, r or p, n or t)]: a deletion of one unit at every offset of each repeat and an
    insertion of one unit (rotated to the offset) at every offset, both ends included."""
    out = []
    for k, (nm, a, u, c) in enumerate(REPEATS):
        span = len(u) * c
        for r in range(a, a + span - len(u) + 1):
            out.append((k, "D", nm, r, len(u)))
        for p in range(a, a + span + 1):
            j = (p - a) % len(u)
            out.append((k, "I", nm, p, u[j:] + u[:j]))
    return out


def records(leftmost_only=False):
    """The BAM records ([(ref_id, pos, flag, cigar words, seq, name, mapq, qual)]): two reads per placement (only the
    placements that are already leftmost with leftmost_only)."""
    names = [nm for nm, _ in CONTIGS]
    out = []
    for k, kind, nm, at, x in placements():
        ref = REFS[nm]
        if leftmost_only and (at != (leftmost_deletion(ref, at, x) if kind == "D" else leftmost_insertion(ref, at, x)[0])):
            continue
        lo = max(0, at - _FLANK)
        if kind == "D":
            hi = min(len(ref), at + x + _FLANK)
            seq = ref[lo:at] + ref[at + x:hi]
            ops = [(at - lo, 0), (x, 2), (hi - at - x, 0)]
        else:
            hi = min(len(ref), at + _FLANK)
            seq = ref[lo:at] + x + ref[at:hi]
            ops = [(at - lo, 0), (len(x), 1), (hi - at, 0)]
        cig = [(n << 4) | op for n, op in ops if n > 0]
        for flag in (0, 16):
            out.append((names.index(nm), lo, flag, cig, seq, "la%d" % len(out), 60, bytes([35] * len(seq))))
    return out


def write(d, leftmost_only=False):
    """(BAM, FASTA) paths under directory d."""
    bam, fa = d / ("leftmost.bam" if leftmost_only else "left_align.bam"), d / "left_align.fa"
    bamio.write_bam(str(bam), CONTIGS, records(leftmost_only))
    fa.write_text("".join(">%s\n%s\n" % (nm, s) for nm, s in REFS.items()))
    return bam, fa


def expected():
    """{(kind, contig, leftmost r or p, n or t): reads} of every group the placements make."""
    out = {}
    for k, kind, nm, at, x in placements():
        ref = REFS[nm]
        key = (kind, nm, leftmost_deletion(ref, at, x), x) if kind == "D" else (kind, nm) + leftmost_insertion(ref, at, x)
        out[key] = out.get(key, 0) + 2
    return out
