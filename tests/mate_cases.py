"""Paired-read inputs of the `--mask-overlaps` tests (tests/test_mates.py, tests/test_gpu_mates.py) and the emulated
K10 chain they share."""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

import emu_harness as E
from kindel_b200 import _ffi, engine, synth

FLAG_R1, FLAG_R2 = 0x1 | 0x2 | 0x40 | 0x20, 0x1 | 0x2 | 0x80 | 0x10
L = 400
PRIMERS = [("c0", 225, 245)]  # the lattice's one primer: the tail of `primerR1`'s first mate


def lattice_sam(path):
    """A SAM file of planted pairs on one contig of L bases (`c0`), and one on a second contig (`c1`): disjoint,
    abutting, partially overlapping, contained and identical spans; D and I in R1, in R2 and in both inside the
    overlap; a deletion of R2 that starts inside R1 and runs past it; R1 bases that are N or of low quality; clipped
    ends; and the cases the pairing must leave alone (three records of one name, a supplementary, two first mates,
    PNEXT off by one, mates on two contigs, a hard read, a lone mate)."""
    rng = np.random.default_rng(5)
    ref = "".join("ACGT"[x] for x in rng.integers(0, 4, L))
    rows = []

    def rec(name, flag, pos0, cigar, seq, pnext0, rnext="=", qual=None, contig="c0"):
        rows.append("\t".join((name, str(flag), contig, str(pos0 + 1), "60", cigar, rnext, str(pnext0 + 1), "0", seq,
                               qual or "*")))

    def ref_seq(a, n):
        return ref[a:a + n]

    def pair(name, a, ca, sa, b, cb, sb, swap=False, fa=FLAG_R1, fb=FLAG_R2, qa=None):
        recs = [(name, fa, a, ca, sa, b, "=", qa), (name, fb, b, cb, sb, a, "=", None)]
        for r in (recs[::-1] if swap else recs):
            rec(*r)

    m = lambda a, n: ref_seq(a, n)  # noqa: E731
    pair("disjoint", 10, "30M", m(10, 30), 60, "30M", m(60, 30))
    pair("abut", 10, "30M", m(10, 30), 40, "30M", m(40, 30))
    pair("partial", 20, "40M", m(20, 40), 40, "40M", m(40, 40), swap=True)
    pair("contained", 30, "50M", m(30, 50), 40, "20M", m(40, 20))
    pair("same", 50, "30M", m(50, 30), 50, "30M", m(50, 30))
    pair("r2left", 90, "30M", m(90, 30), 70, "30M", m(70, 30))
    # D in R1, in R2, in both; an R2 deletion that runs past R1's end
    pair("delR1", 100, "10M3D17M", m(100, 10) + m(113, 17), 105, "25M", m(105, 25))
    pair("delR2", 100, "30M", m(100, 30), 105, "10M3D12M", m(105, 10) + m(118, 12))
    pair("delBoth", 100, "10M3D17M", m(100, 10) + m(113, 17), 105, "5M3D17M", m(105, 5) + m(113, 17))
    pair("delPast", 140, "20M", m(140, 20), 150, "8M6D10M", m(150, 8) + m(164, 10))
    # I in R1, in R2, in both
    pair("insR1", 170, "10M2I15M", m(170, 10) + "GG" + m(180, 15), 175, "20M", m(175, 20))
    pair("insR2", 170, "25M", m(170, 25), 175, "5M3I12M", m(175, 5) + "TTT" + m(180, 12))
    pair("insBoth", 170, "10M2I15M", m(170, 10) + "CC" + m(180, 15), 175, "5M2I12M", m(175, 5) + "CA" + m(180, 12))
    # R1 with an N and with low-quality bases; clipped ends
    s = m(200, 30)
    pair("nR1", 200, "30M", s[:5] + "N" + s[6:], 205, "30M", m(205, 30))
    pair("lowR1", 240, "30M", m(240, 30), 250, "30M", m(250, 30), qa="I" * 20 + "#" * 10)
    pair("clips", 280, "4S26M", "ACGT" + m(280, 26), 290, "20M5S", m(290, 20) + "TTTTT")
    # left alone: three of one name, a supplementary, two first mates, PNEXT off by one, a hard read, a lone mate
    rec("three", FLAG_R1, 300, "20M", m(300, 20), 305)
    rec("three", FLAG_R2, 305, "20M", m(305, 20), 300)
    rec("three", FLAG_R2, 305, "20M", m(305, 20), 300)
    rec("supp", FLAG_R1, 300, "20M", m(300, 20), 305)
    rec("supp", FLAG_R2, 305, "20M", m(305, 20), 300)
    rec("supp", FLAG_R2 | 0x800, 306, "10M", m(306, 10), 300)
    pair("twoR1", 320, "20M", m(320, 20), 325, "20M", m(325, 20), fb=FLAG_R1)
    rec("offby1", FLAG_R1, 340, "20M", m(340, 20), 346)
    rec("offby1", FLAG_R2, 345, "20M", m(345, 20), 340)
    pair("hard", 5, "30M", m(5, 30), 0, "2S30M", "AA" + m(0, 30))  # a left clip before base 1: hard
    rec("lone", FLAG_R1, 360, "20M", m(360, 20), 365)
    rec("lowmapq", FLAG_R1, 360, "20M", m(360, 20), 365)
    rows.append("\t".join(("lowmapq", str(FLAG_R2), "c0", "366", "5", "20M", "=", "361", "0", m(365, 20), "*")))
    # the first mate's overlap bases lie in a primer (PRIMERS): masked by K9 first, they cover nothing
    pair("primerR1", 210, "30M", m(210, 30), 220, "30M", m(220, 30))
    # a mate flagged unmapped (0x8), a secondary (0x100): no role, so no pair; a second pair written R2 first
    rec("mateUnmapped", FLAG_R1 | 0x8, 330, "20M", m(330, 20), 335)
    rec("mateUnmapped", FLAG_R2, 335, "20M", m(335, 20), 330)
    rec("secondary", FLAG_R1, 350, "20M", m(350, 20), 355)
    rec("secondary", FLAG_R2 | 0x100, 355, "20M", m(355, 20), 350)
    pair("insR2swap", 170, "25M", m(170, 25), 176, "4M2I12M", m(176, 4) + "AC" + m(180, 12), swap=True)
    rec("twoContigs", FLAG_R1, 370, "20M", m(370, 20), 10, rnext="c1")
    rec("twoContigs", FLAG_R2, 10, "20M", "A" * 20, 370, rnext="c0", contig="c1")
    head = "@HD\tVN:1.6\tSO:unsorted\n@SQ\tSN:c0\tLN:%d\n@SQ\tSN:c1\tLN:100\n" % L
    with open(path, "w") as fh:
        fh.write(head + "\n".join(rows) + "\n")
    return path


def emu_overlaps(batch, order=None, mate=None):
    """K10p (unless `mate` is given) and K10 under the emulator over a host ReadBatch with mates: (the masked batch
    -- merged mask list, R2 nibbles --, drop rows int32 [m, 4], totals, mate).  order: the sorted eligible reads
    (default: a numpy argsort of the hashes)."""
    lib = E.load()
    lib.emu_set_sm_count(E.SM_COUNT)
    st, keep = engine.host_struct(batch)
    n = batch.n_reads
    if mate is None:
        if order is None:
            idx = np.flatnonzero(batch.pair_role)
            order = idx[np.argsort(batch.name_hash[idx], kind="stable")]
        order = np.ascontiguousarray(order, dtype=np.int32)
        mate = np.full(max(n, 1), 7, dtype=np.int32)
        h = np.ascontiguousarray(batch.name_hash, dtype=np.uint64)
        ms = np.ascontiguousarray(batch.mate_start, dtype=np.int32)
        ro = np.ascontiguousarray(batch.pair_role, dtype=np.uint8)
        E._check(lib.kdl_mates_pair(C.byref(st), h.ctypes.data, ms.ctypes.data, ro.ctypes.data,
                                    order.ctypes.data if order.size else None, order.size, mate.ctypes.data, None),
                 "kdl_mates_pair")
        mate = mate[:n]
    mate = np.ascontiguousarray(mate, dtype=np.int32)
    qm, qkeep = engine.host_qmask(batch)
    qp = C.byref(qm) if qm is not None else None
    scratch = np.full(int(lib.kdl_overlap_scratch_words(n)), 0xDEADBEEF, dtype=np.uint32)
    args = (C.byref(st), qp, mate.ctypes.data if n else None, scratch.ctypes.data)
    E._check(lib.kdl_overlap_count(*args, None), "kdl_overlap_count")
    tot = scratch[-8:].astype(np.int64)
    n_mr, n_mb, n_d = int(tot[0]), int(tot[1]), int(tot[2])
    seq4 = np.array(batch.seq4, dtype=np.uint32, copy=True)
    out = dict(mask_read=np.full(n_mr + 1, 7, np.uint32), mask_off=np.full(n_mr + 2, 7, np.uint32),
               mask_qpos=np.full(n_mb + 1, 7, np.uint32))
    om = _ffi.KdlQmask()
    om.n_reads, om.n_bases = n_mr, n_mb
    om.read_idx, om.off, om.qpos = (out[f].ctypes.data for f in ("mask_read", "mask_off", "mask_qpos"))
    drops = np.full((n_d + 1, 4), -7, dtype=np.int32)
    E._check(lib.kdl_overlap_apply(*args, seq4.ctypes.data, C.byref(om) if n_mr else None, drops.ctypes.data, n_d,
                                   None), "kdl_overlap_apply")
    assert (drops[n_d] == -7).all() and out["mask_qpos"][n_mb] == 7 and out["mask_read"][n_mr] == 7, "K10 overran"
    del keep, qkeep
    masked = dataclasses.replace(batch, seq4=seq4, mask_read=out["mask_read"][:n_mr] if n_mr else None,
                                 mask_off=out["mask_off"][:n_mr + 1] if n_mr else None,
                                 mask_qpos=out["mask_qpos"][:n_mb] if n_mr else None)
    return masked, drops[:n_d], tot, mate


def untake(drops, counts):
    """K10u under the emulator over a host table (in place)."""
    lib = E.load()
    d = np.ascontiguousarray(drops, dtype=np.int32)
    E._check(lib.kdl_overlap_untake(d.ctypes.data if d.size else None, d.shape[0], counts.ctypes.data,
                                    counts.shape[1], None), "kdl_overlap_untake")
    return counts


def emu_tables(batch, order=None):
    """The whole emulated chain: K10p, K10, the pileup, K1q, K10u.  (counts, events without the dropped rows, drops,
    totals, mate)."""
    masked, drops, tot, mate = emu_overlaps(batch, order)
    counts, events = E.pileup_pipeline(masked)
    E.unmask(masked, counts)
    untake(drops, counts)
    gone = np.sort(drops[drops[:, 3] >= 0, 3])
    return counts, np.delete(events, gone, axis=0), drops, tot, mate, masked


def mask_lists(batch):
    """Per read, its entries in the batch's mask list."""
    out = [[] for _ in range(batch.n_reads)]
    for j in range(batch.n_mask_reads):
        out[int(batch.mask_read[j])] = batch.mask_qpos[batch.mask_off[j]:batch.mask_off[j + 1]].tolist()
    return out


def paired_bam(path, seed=1, contig_lens=(3000,), depth=30, read_len=100, insert_mean=170, indel_frac=0.15):
    b, flag, frag = synth.paired_reads(seed, list(contig_lens), depth, read_len=read_len, insert_mean=insert_mean,
                                       insert_sd=40, indel_frac=indel_frac)
    synth.write_paired_bam(path, b, flag, frag)
    return path


def combo_files(d, seed=3):
    """A paired corpus for the option matrix: two contigs of synth.paired_reads (with indels), random qualities (some
    below 20), MAPQ 5 / 40 / 60, a few duplicates (0x400), as BAM and as SAM; a tiled primer BED; the contigs' FASTA.
    Returns dict(bam, sam, bed, fa, rows, refs)."""
    from kindel_b200 import bamio

    refs = {}
    b, flag, frag = synth.paired_reads(seed, [2400, 1700], 25, read_len=100, insert_mean=170, insert_sd=40,
                                       indel_frac=0.15, refs=refs)
    contigs, recs = synth.paired_records(b, flag, frag)
    rng = np.random.default_rng(seed)
    out = []
    for r in recs:
        qual = bytes(int(q) for q in rng.choice([8, 30, 38], len(r[4]), p=[.08, .42, .5]))
        fl = r[2] | (0x400 if rng.random() < 0.03 else 0)
        out.append((r[0], r[1], fl, r[3], r[4], r[5], int(rng.choice([5, 40, 60])), qual, r[8], r[9]))
    bam, sam = str(d / "combo.bam"), str(d / "combo.sam")
    bamio.write_bam(bam, contigs, out)
    with open(sam, "w") as fh:
        fh.write("@HD\tVN:1.6\n" + "".join("@SQ\tSN:%s\tLN:%d\n" % c for c in contigs))
        for ref_id, pos0, fl, words, seq, qn, mq, qual, nref, npos in out:
            cig = "".join("%d%s" % (w >> 4, "MIDNSHP=X"[w & 15]) for w in words)
            fh.write("\t".join((qn, str(fl), contigs[ref_id][0], str(pos0 + 1), str(mq), cig, "=", str(npos + 1), "0",
                                seq, "".join(chr(33 + q) for q in qual))) + "\n")
    rows = synth.tiled_scheme(1, [c[0] for c in contigs], [c[1] for c in contigs], spacing=150, overlap=40)
    bed = d / "combo.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
    fa = d / "combo.fa"
    fa.write_text("".join(">%s\n%s\n" % (nm, refs[nm]) for nm, _ in contigs))
    return dict(bam=bam, sam=sam, bed=str(bed), fa=str(fa), rows=rows, refs=refs)


def mates_matrix():
    """(min_base_quality, min_mapq, exclude_flags, primers, reference, strand, (abs, rel)) rows with mask_overlaps
    on: a pairwise-covering set over the four options, and everything at once."""
    return [(0, 0, 0, False, False, False, (1, 0.01)), (20, 0, 0, True, False, True, (0, 0.0)),
            (0, 30, 0x400, True, True, False, (1, 0.05)), (20, 30, 0, False, True, True, (0, 0.0)),
            (20, 0, 0x400, False, True, False, (2, 0.1)), (0, 30, 0, True, False, True, (1, 0.01)),
            (20, 30, 0x400, True, True, True, (0, 0.0))]
