"""Multi-sample inputs for the `variants --vcf a.bam b.bam ...` tests (test_cohort.py, test_gpu_cohort.py).

- stacked tables: S samples' count tables over one shared layout with planted counts in the slot behind each contig
  and in the padding, a sample lacking a contig, and pooled counts above 2^31;
- the VCF combo corpus split into samples (by read, one sample without a contig, one the whole corpus), as BAM or SAM;
- a truth set of planted multi-sample cases: a fixed difference, a minority allele in one sample only, a deletion
  and an insertion that pass in one sample and stay below the threshold in another, a sample without a contig."""
from __future__ import annotations

import dataclasses
import itertools
import sys

import numpy as np

import vcf_combo_cases as VC
from kindel_b200 import bamio
from oracle import py_msoracle as MS

LENS = [700, 7, 0, 400, 1]


def layout(rng):
    """(contig_slot, contig_len, n_slots) with gaps of padding between contigs; n_slots % 4 == 0, not a multiple of
    the 1024-slot CTA span."""
    slots, s = [], 0
    for L in LENS:
        slots.append(s)
        s = (s + L + 1 + 3) // 4 * 4 + 4 * int(rng.integers(0, 3))
    return np.array(slots, dtype=np.int64), np.array(LENS, dtype=np.int64), s + 4


def stacked(seed, S):
    """(T int32 [S, 7, n_slots], contig_slot, contig_len, ref codes uint8 [n_slots], lacking {sample: contig})."""
    rng = np.random.default_rng(seed)
    cs, cl, n = layout(rng)
    T = np.zeros((S, 7, n), dtype=np.int64)
    T[:, 0:7] = rng.integers(0, 6, size=(S, 7, n))
    T[:, 0:7][:, :, rng.random(n) < 0.1] = 0                                 # zero depth in every sample
    for i in range(S):
        big = rng.random(n) < 0.08
        T[i][0:6][:, big] = rng.integers((1 << 31) - 8, 1 << 31, size=(6, int(big.sum())))  # pooled sums above 2^31
        lone = rng.random(n) < 0.05
        T[i, int(rng.integers(0, 6)), lone] = 40                             # a sample-specific allele
    is_pos = np.zeros(n, dtype=bool)
    for s0, L in zip(cs, cl):
        is_pos[s0:s0 + L] = True
    T[:, 0:6, ~is_pos] = np.array([[100], [50], [40], [30], [20], [10]])      # slot L and padding
    lacking = {}
    if S > 1:  # the last sample lacks contig 3: zeros there
        lacking[S - 1] = 3
        T[S - 1, :, cs[3]:cs[3] + cl[3] + 1] = 0
    ref = rng.integers(0, 5, size=n).astype(np.uint8)
    ref[~is_pos] = 4
    return T.astype(np.int32), cs, cl, ref, lacking


def oracle_samples(T, cs, cl, lacking):
    names = ["c%d" % c for c in range(len(cl))]
    out = []
    for i in range(T.shape[0]):
        keep = [c for c in range(len(cl)) if lacking.get(i) != c]
        out.append(MS.Sample.from_table([names[c] for c in keep], cl[keep], cs[keep], T[i]))
    return names, out


def ref_texts(ref, cs, cl):
    return {"c%d" % c: "".join("ACGTN"[x] for x in ref[s0:s0 + L].tolist()) for c, (s0, L) in
            enumerate(zip(cs.tolist(), cl.tolist()))}


# --------------------------------------------------------------------------------------------- alignment files
def write_sam(path, contigs, recs):
    lines = ["@HD\tVN:1.6\tSO:unsorted"] + ["@SQ\tSN:%s\tLN:%d" % c for c in contigs]
    for r in recs:
        ref_id, pos, flag, cig, seq, name, mapq, qual = r[:8]
        cig_text = "".join("%d%s" % (w >> 4, "MIDNSHP=X"[w & 15]) for w in cig)
        qtext = "*" if qual is None else "".join(chr(33 + x) for x in qual)
        lines.append("\t".join([name, str(flag), contigs[ref_id][0], str(pos + 1), str(mapq), cig_text, "*", "0", "0",
                                seq, qtext]))
    path.write_text("\n".join(lines) + "\n")
    return path


def split_corpus(d, sam=False):
    """(paths, fa, bed, rows) of the VCF combo corpus as three samples: the even records, the odd records without
    contig `edge`, and the whole corpus -- in that order, so sample 2 shows contigs sample 1 lacks."""
    bam, _, fa, bed, contigs, recs, refs, rows = VC.write(d)
    edge = [nm for nm, _ in contigs].index("edge")
    parts = [recs[0::2], [r for r in recs[1::2] if r[0] != edge], recs]
    paths = []
    for k, part in enumerate(parts):
        p = d / ("s%d.%s" % (k, "sam" if sam and k == 1 else "bam"))
        if p.suffix == ".sam":
            write_sam(p, contigs, part)
        else:
            bamio.write_bam(str(p), contigs, part)
        paths.append(str(p))
    return paths, str(fa), str(bed), rows, refs


def covering_rows(n_factors=6):
    """Rows of 0/1 (one per factor) in which every pair of values of every two factors occurs: each factor's column
    is a distinct weight-3 subset of rows 1..5 (two such subsets always meet and always differ; row 0 is all zero)."""
    cols = list(itertools.combinations(range(1, 6), 3))[:n_factors]
    return [tuple(int(r in c) for c in cols) for r in range(6)]


# --------------------------------------------------------------------------------------------- truth set
REF = "ACGTACGTAC" * 6  # 60 bases
FIXED, MINOR, DEL, INS = 10, 20, 35, 45  # 0-based positions


def _read(ref_id, pos, cig, seq, name):
    return (ref_id, pos, 0, [(n << 4) | "MIDNSHP=X".index(op) for n, op in cig], seq, name, 60, None)


def truth_set(d):
    """(paths, fa) of three samples over contigs `a` (60 bases) and `b` (60 bases):
    sample x: 20 reads over a, each with T at FIXED, 2 of them G at MINOR, 3 with a 2-base deletion at DEL and 3 with
              an insertion `GG` behind DEL + 10; 10 reads over b
    sample y: 20 reads over a with C at FIXED, 1 with the deletion and 1 with the insertion (below abs 1); none on b
    sample z: 10 reads over b only."""
    contigs = [("a", 60), ("b", 60)]
    fa = d / "truth.fa"
    fa.write_text(">a\n%s\n>b\n%s\n" % (REF, REF))

    def full(base_at_fixed, k, dele, ins, minor):
        seq = list(REF)
        seq[FIXED] = base_at_fixed
        if minor:
            seq[MINOR] = "G" if REF[MINOR] != "G" else "T"
        if dele:
            return _read(0, 0, [(DEL, "M"), (2, "D"), (60 - DEL - 2, "M")], "".join(seq[:DEL] + seq[DEL + 2:]), k)
        if ins:
            return _read(0, 0, [(INS, "M"), (2, "I"), (60 - INS, "M")], "".join(seq[:INS] + ["G", "G"] + seq[INS:]), k)
        return _read(0, 0, [(60, "M")], "".join(seq), k)

    x = [full("T", "x%d" % k, k < 3, 3 <= k < 6, 6 <= k < 8) for k in range(20)]
    x += [_read(1, 0, [(60, "M")], REF, "xb%d" % k) for k in range(10)]
    y = [full("C", "y%d" % k, k == 0, k == 1, False) for k in range(20)]
    z = [_read(1, 0, [(60, "M")], REF, "zb%d" % k) for k in range(10)]
    paths = []
    for nm, recs in (("x", x), ("y", y), ("z", z)):
        p = d / ("%s.bam" % nm)
        bamio.write_bam(str(p), contigs, recs)
        paths.append(str(p))
    return paths, str(fa)


# --------------------------------------------------------------------------------------------- synthetic samples
def plant(batch, pos, code, frac, seed):
    """The batch (simple reads of one contig) with the base at 0-based position `pos` set to nibble `code` in a share
    `frac` of the reads that cover it: a sample-specific allele."""
    rng = np.random.default_rng(seed)
    start = np.asarray(batch.ref_start, dtype=np.int64)
    ln = np.asarray(batch.l_seq, dtype=np.int64)
    reads = np.flatnonzero((start <= pos) & (pos < start + ln))
    reads = reads[rng.random(reads.size) < frac]
    q = pos - start[reads]
    seq4 = np.array(batch.seq4, dtype=np.uint32, copy=True)
    word = np.asarray(batch.seq_off, dtype=np.int64)[reads] + (q >> 3)
    shift = (28 - 4 * (q & 7)).astype(np.uint32)
    seq4[word] = (seq4[word] & ~(np.uint32(0xF) << shift)) | (np.uint32(code) << shift)
    return dataclasses.replace(batch, seq4=seq4)


def synthetic_samples(d, n_samples, length, depth, seed=4, progress=False):
    """n_samples BAMs of one contig (the same bases for all, `seed`), each with reads of its own and, at positions of
    its own, a planted allele in 30 % of the reads.  [(path, batch)]."""
    from kindel_b200 import synth

    out = []
    for i in range(n_samples):
        batch = synth.simple_reads(seed, [length], depth, read_seed=1000 + i)
        for k in range(4):
            batch = plant(batch, 500 + 7919 * (4 * i + k) % (length - 1000), 1 << (k % 4), 0.3, 77 * i + k)
        path = str(d / ("sample%02d.bam" % i))
        synth.write_simple_bam(path, batch)
        out.append((path, batch))
        if progress:
            print("sample %d of %d written" % (i + 1, n_samples), file=sys.stderr, flush=True)
    return out
