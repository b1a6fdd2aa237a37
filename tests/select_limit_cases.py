"""Inputs for the read selection at the engine's limits -- `--dedup` (K14), the amplicon labels (K12) and
`--normalise N` (K13) -- (test infrastructure, no torch).

  planted      every limit group (limit_cases.GROUPS) with duplicates planted: for a seeded subset of its records a
               copy with a higher, the same and a lower QUAL sum, the same 5' end reached by a longer soft clip and by
               a hard clip, the other strand (never a duplicate), secondary and supplementary copies (left alone),
               a copy with QUAL `*` (score 0); read pairs made of the subset's neighbours with a better copy, an
               R1/R2-swapped copy, a copy whose R2 the read filters take out (MAPQ 0 or FLAG 0x400), and a mate
               that is KDL_HARD wherever the group has one; and on the first contig long enough, the `template`
               below, whose ends include u < 0 (a leading clip at POS 1) and u >= L (a reverse read whose trailing
               clip runs past the contig's end)
  many         `template` at the same positions on each of 2 500 contigs, in header order or shuffled
               (qual_limit_cases.many_contigs_sam): the same ends on every contig, so nothing may be removed across
               contigs; `twin` is the smallest such file, two identical contigs
  interleaved  a name-sorted paired file over three contigs first seen in an order unlike the header, the first
               record of the first contig a duplicate the dedup removes, and singles of one amplicon for the cap

Every file has a named tiled scheme (synth.tiled_scheme through amplicon_cases) dense enough that most reads get an
amplicon.  Records are bamio.write_bam tuples (ref_id, pos0, flag, cigar words, seq, qname, mapq, qual bytes or None,
next ref_id, next pos0); everything is seeded."""
from __future__ import annotations

import random
import zlib

import numpy as np

import amplicon_cases as AC
import limit_cases as LC
import qual_cases as QC
import qual_limit_cases as QL
from kindel_b200 import bamio, synth

_S, _H = 4, 5
_REF = (0, 2, 3, 7, 8)
_ALIGNED = (0, 7, 8)
N_MANY = 2500
TEMPLATE_LEN = 160
SPACING, OVERLAP = 50, 20  # the tiled scheme: a left primer every 50 bases, an insert between every pair


def _ops(cig):
    return [(w >> 4, w & 15) for w in cig]


def _words(ops):
    return [(n << 4) | op for n, op in ops if n > 0]


def _q(n, q):
    return bytes([q]) * n


def _clipped(r, hard):
    """A copy of r with the same 5' end (u, strand) and one more base clipped at its 5' side, or None."""
    rid, pos0, flag, cig, seq, name, mapq, qual = r[:8]
    ops = _ops(cig)
    at = [k for k, (_, op) in enumerate(ops) if op in _REF]
    if not at:
        return None
    rev = bool(flag & 0x10)
    k = at[-1] if rev else at[0]
    n, op = ops[k]
    outer = ops[k + 1:] if rev else ops[:k]
    if op not in _ALIGNED or n < 2 or any(o not in (_S, _H) for _, o in outer) or (hard and outer):
        return None
    if rev:  # the last aligned base becomes a clip: the span shrinks by one, the trailing clip grows by one
        if hard:
            new, seq, qual = ops[:k] + [(n - 1, op), (1, _H)], seq[:-1], None if qual is None else qual[:-1]
        elif outer and outer[0][1] == _S:
            new = ops[:k] + [(n - 1, op), (outer[0][0] + 1, _S)] + outer[1:]
        else:
            new = ops[:k] + [(n - 1, op), (1, _S)] + outer
        return (rid, pos0, flag, _words(new), seq, name + ("_hc" if hard else "_sc"), mapq, qual, -1, -1)
    if hard:
        new, seq, qual = [(1, _H), (n - 1, op)] + ops[k + 1:], seq[1:], None if qual is None else qual[1:]
    elif outer and outer[-1][1] == _S:
        new = outer[:-1] + [(outer[-1][0] + 1, _S), (n - 1, op)] + ops[k + 1:]
    else:
        new = outer + [(1, _S), (n - 1, op)] + ops[k + 1:]
    return (rid, pos0 + 1, flag, _words(new), seq, name + ("_hc" if hard else "_sc"), mapq, qual, -1, -1)


def copies(r):
    """The planted copies of one single record r (see the module docstring)."""
    rid, pos0, flag, cig, seq, name, mapq, qual = r[:8]
    n = len(seq)
    out = [(rid, pos0, flag, cig, seq, name + "_hi", mapq, _q(n, 41), -1, -1),
           (rid, pos0, flag, cig, seq, name + "_eq", mapq, qual, -1, -1),
           (rid, pos0, flag, cig, seq, name + "_lo", mapq, _q(n, 14), -1, -1),
           (rid, pos0, flag ^ 0x10, cig, seq, name + "_fl", mapq, _q(n, 41), -1, -1),
           (rid, pos0, flag | 0x100, cig, seq, name + "_2nd", mapq, _q(n, 60), -1, -1),
           (rid, pos0, flag | 0x800, cig, seq, name + "_sup", mapq, _q(n, 60), -1, -1),
           (rid, pos0, flag, cig, seq, name + "_nq", mapq, None, -1, -1)]
    return out + [c for c in (_clipped(r, False), _clipped(r, True)) if c is not None]


def pair(a, b, name, q=None, swap=False, r2_mapq=None, r2_flag=0):
    """Records a (forward) and b (reverse) as one proper pair called `name`: a is R1 unless `swap`.  q: one Phred value
    for every base (None: their own qualities); r2_mapq / r2_flag: the R2's MAPQ and extra FLAG bits."""
    fa, fb = (0x1 | 0x20, 0x1 | 0x10)
    fa |= 0x80 if swap else 0x40
    fb |= 0x40 if swap else 0x80
    ra = [a[0], a[1], fa, a[3], a[4], name, a[6], a[7] if q is None else _q(len(a[4]), q), b[0], b[1]]
    rb = [b[0], b[1], fb, b[3], b[4], name, b[6], b[7] if q is None else _q(len(b[4]), q), a[0], a[1]]
    r2 = ra if swap else rb
    if r2_mapq is not None:
        r2[6] = r2_mapq
    r2[2] |= r2_flag
    return [tuple(ra), tuple(rb)]


def template(rid, L, tag):
    """The same planted records on every contig of length L >= TEMPLATE_LEN (see the module docstring)."""
    assert L >= TEMPLATE_LEN
    rng = random.Random(17)
    seq = lambda n: "".join(rng.choice("ACGT") for _ in range(n))  # noqa: E731
    w = bamio.parse_cigar_text
    s_neg, s_mid, s_end, s_p1, s_p2 = seq(35), seq(40), seq(36), seq(40), seq(40)
    recs = [
        # u = -5: a leading soft clip at POS 1, its duplicates, the same u through a longer and a hard clip
        (rid, 0, 0, w("5S30M"), s_neg, tag + "n0", 60, _q(35, 30), -1, -1),
        (rid, 0, 0, w("5S30M"), s_neg, tag + "n1", 60, _q(35, 33), -1, -1),
        (rid, 0, 0, w("5S30M"), s_neg, tag + "n2", 60, _q(35, 33), -1, -1),
        (rid, 2, 0, w("7S28M"), s_neg, tag + "n3", 60, _q(35, 33), -1, -1),
        (rid, 2, 0, w("7H28M"), s_neg[7:], tag + "n4", 60, _q(28, 41), -1, -1),
        (rid, 0, 0x10, w("5S30M"), s_neg, tag + "n5", 60, _q(35, 41), -1, -1),  # the other strand: u = 29
        (rid, 0, 0x100, w("5S30M"), s_neg, tag + "n6", 60, _q(35, 60), -1, -1),
        # u = L + 5: a reverse read whose trailing clip runs past the contig's end
        (rid, L - 30, 0x10, w("30M6S"), s_end, tag + "e0", 60, _q(36, 20), -1, -1),
        (rid, L - 30, 0x10, w("28M8S"), s_end, tag + "e1", 60, _q(36, 25), -1, -1),
        (rid, L - 30, 0x10, w("30M6S"), s_end, tag + "e2", 60, None, -1, -1),
        (rid, L - 30, 0x810, w("30M6S"), s_end, tag + "e3", 60, _q(36, 60), -1, -1),
        # a plain stack: the best score is the third record
        (rid, 60, 0, w("40M"), s_mid, tag + "m0", 60, _q(40, 25), -1, -1),
        (rid, 60, 0, w("40M"), s_mid, tag + "m1", 60, _q(40, 25), -1, -1),
        (rid, 60, 0, w("40M"), s_mid, tag + "m2", 60, _q(40, 35), -1, -1),
        # a single on a pair mate's end (shadowed)
        (rid, 20, 0, w("40M"), s_p1, tag + "s0", 60, _q(40, 60), -1, -1),
    ]
    a = (rid, 20, 0, w("40M"), s_p1, "", 60, _q(40, 30))
    b = (rid, 90, 0, w("40M"), s_p2, "", 60, _q(40, 30))
    hard = (rid, 0, 0, w("5S30M"), s_neg, "", 60, _q(35, 30))
    recs += pair(a, b, tag + "p0")
    recs += pair(a, b, tag + "p1", q=35)               # the best of the fragment
    recs += pair(a, b, tag + "p2", swap=True)          # R1 / R2 swapped: the same fragment
    recs += pair(a, b, tag + "p3", r2_mapq=0)          # the R2 filtered out under min_mapq: R1 a single
    recs += pair(a, b, tag + "p4", r2_flag=0x400)      # ... under exclude_flags 0x400
    recs += pair(hard, b, tag + "p5")                  # R1 KDL_HARD: no pair, two singles
    c = (rid, 100, 0, w("40M"), s_mid, "", 60, _q(40, 36))
    d = (rid, 110, 0, w("40M"), s_p2, "", 60, _q(40, 36))
    recs += pair(c, d, tag + "p6", swap=True)          # a tie: the swapped pair's smaller index (its R2) wins
    recs += pair(c, d, tag + "p7")
    return recs


def _seed(name):
    return zlib.crc32(name.encode())


def planted(name):
    """(contigs, records) of limit group `name` with duplicates planted, coordinate-sorted (stable)."""
    contigs, recs = QL.parse_sam(LC.sam_text(name))
    recs = [r + (-1, -1) for r in recs]
    rng = random.Random(_seed(name))
    with_ref = [k for k, r in enumerate(recs) if any(op in _REF for _, op in _ops(r[3]))]
    pick = sorted(set(rng.sample(with_ref, min(8, len(with_ref))) + [with_ref[0], with_ref[-1]]))
    out = list(recs)
    for k in pick:
        out += copies(recs[k])
    for i, (k, j) in enumerate(zip(pick, pick[1:])):
        a, b = recs[k], recs[j]
        if a[0] != b[0]:
            continue
        nm = "%s_pair%d" % (name, i)
        out += pair(a, b, nm) + pair(a, b, nm + "_dp", q=41) + pair(a, b, nm + "_sw", swap=True)
        out += pair(a, b, nm + "_mq", r2_mapq=0) + pair(a, b, nm + "_dx", r2_flag=0x400)
    hard = [r for r in recs if r[5].endswith("_h")]
    simple = [r for r in recs if r[5].endswith("_s")]
    if hard and simple:
        h = hard[0]
        s = min((r for r in simple if r[0] == h[0]), key=lambda r: abs(r[1] - h[1]), default=None)
        if s is not None:
            out += pair(h, s, "%s_hardmate" % name) + pair(h, s, "%s_hardmate_dp" % name, q=41)
    long_enough = [k for k, (_, L) in enumerate(contigs) if L >= TEMPLATE_LEN]
    if long_enough:
        out += template(long_enough[0], contigs[long_enough[0]][1], name + "_t_")
    out.sort(key=lambda r: (r[0], r[1]))
    return contigs, out


def scheme_rows(contigs):
    """The named tiled scheme over contigs [(name, L)]: rows (chrom, start, end, amplicon, side)."""
    names = [c for c, _ in contigs]
    return AC.tiled_rows(synth.tiled_scheme(_seed("".join(names[:3])), names, [L for _, L in contigs],
                                            spacing=SPACING, overlap=OVERLAP))


def many(n_contigs=N_MANY, shuffled=False):
    """(contigs, records) of `template` on each of n_contigs contigs of TEMPLATE_LEN bases, one block per contig in
    the header's order or shuffled (qual_limit_cases.many_contigs_sam's order)."""
    contigs = [("c%04d" % k, TEMPLATE_LEN) for k in range(n_contigs)]
    plan = template(0, TEMPLATE_LEN, "")
    reads = {nm: [(r[1], "%dM" % len(r[4]), r[4]) for r in plan] for nm, _ in contigs}
    _, placed = QL.parse_sam(QL.many_contigs_sam(contigs, reads, shuffled, 7))
    out, at = [], {}
    for rid, *_ in placed:  # the k-th record of a contig's block is the template's k-th
        k = at.get(rid, 0)
        at[rid] = k + 1
        r = plan[k]
        nx = -1 if r[8] < 0 else rid
        out.append((rid, r[1], r[2], r[3], r[4], "c%04d_%s" % (rid, r[5]), r[6], r[7], nx, r[9]))
    return contigs, out


def twin():
    """(contigs, records): `template` on two identical contigs, in header order."""
    return many(2)


def interleaved():
    """(contigs, records) of a name-sorted paired file over x0, x1, x2 (header order), first seen x2, x0, x1: the
    first record of the file, on x2, is the worse copy of a pair the dedup removes; four singles per contig start in
    one left primer, so the cap drops some.  The cap cannot remove a contig's first record (the first read of its
    group always stays)."""
    contigs = [("x0", TEMPLATE_LEN), ("x1", TEMPLATE_LEN), ("x2", TEMPLATE_LEN)]
    rng = random.Random(23)
    seq = lambda n: "".join(rng.choice("ACGT") for _ in range(n))  # noqa: E731
    w = bamio.parse_cigar_text
    ends = {c: ((c, 2 + c, 0, w("40M"), seq(40), "", 60, _q(40, 30)),
                (c, 80 + c, 0, w("40M"), seq(40), "", 60, _q(40, 30))) for c in range(3)}
    plan = [(2, 20), (0, 30), (2, 35), (1, 30), (0, 30), (1, 41), (2, 30), (0, 25), (1, 30), (2, 30)]
    out = []
    for k, (c, q) in enumerate(plan):
        a, b = ends[c]
        out += pair(a, b, "q%03d" % k, q=q)
    for k in range(12):  # singles of one amplicon and strand, each its own end: the cap drops all but the first ones
        c = k % 3
        out.append((c, 5 + k, 0, w("40M"), seq(40), "s%03d" % k, 60, _q(40, 30), -1, -1))
    return contigs, out  # (written in this order: names ascending, mates together)


def write(d, stem, contigs, recs, sam=True):
    """(BAM path, SAM path or None) of the records under directory d."""
    bam = str(d / (stem + ".bam"))
    bamio.write_bam(bam, contigs, recs)
    path = None
    if sam:
        path = str(d / (stem + ".sam"))
        QC.write_sam(path, contigs, recs)
    return bam, path


# ------------------------------------------------------------------------------------------ K14 lists by hand
def hand_batch(starts, reverse, score, n_contig_len):
    """A one-contig batch of 40M reads at `starts`, strands and duplicate scores set by hand."""
    n = len(starts)
    b = synth.simple_reads(5, [400], 1, read_len=40)
    return bamio.finalize(b.contig_names, np.array([n_contig_len], dtype=np.int64), [0, n], np.asarray(starts),
                          np.arange(n) * 5, np.full(n, 40), np.arange(n + 1), np.full(n, 40 << 4),
                          np.tile(b.seq4[:5], n), n_records=n, reverse=np.asarray(reverse, dtype=np.uint8),
                          dup_score=np.asarray(score, dtype=np.int32))


CHUNK = 256 * 256  # entries of K14s-c's chunk: 256 CTAs of 256 entries
MODES = ("before", "on", "after", "long")


def carry_runs(m, rng, mode):
    """(run id of each of m sorted entries, head flags).  before / on / after: a head one entry before, on or one
    entry after every CTA boundary (multiples of 256, chunk boundaries among them), so that a run crosses every
    boundary but with `on`; long: a run from the middle of every chunk into the next one, short runs between them.
    Random heads elsewhere, never on a boundary."""
    head = np.zeros(m, dtype=bool)
    head[0] = True
    extra = rng.integers(1, m, m // 100) if m > 1 else np.zeros(0, dtype=np.int64)
    if mode == "long":
        for c in range(0, m, CHUNK):
            if c + 30_000 < m:
                head[c + 30_000] = True
        extra = extra[(extra % CHUNK >= 10_000) & (extra % CHUNK < 30_000)]
    else:
        off = {"before": -1, "on": 0, "after": 1}[mode]
        for b in range(256, m, 256):
            if b + off < m:
                head[b + off] = True
    head[extra[extra % 256 != 0]] = True
    if mode == "on":
        assert head[::256].all()
    else:  # a run crosses CTA boundaries, and the chunk boundary when there is one
        crossing = ~head[256::256]
        assert crossing.all() if mode != "long" else crossing.any()
        assert m <= CHUNK or not head[CHUNK]
    return np.cumsum(head) - 1, head


def placeholders(recs, removed):
    """The records with every record of a file index in `removed` turned into an unmapped placeholder: FLAG | 0x4,
    RNAME kept, so it counts for the first-seen order of contigs and for nothing else."""
    return [r if k not in removed else (r[0], r[1], r[2] | 0x4) + tuple(r[3:]) for k, r in enumerate(recs)]
