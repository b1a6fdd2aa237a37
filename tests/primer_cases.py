"""Amplicon primer masking (`--primers`, an extension) -- test infrastructure: primer schemes, K9 under the kernel
emulator, and a planted truth set.

The truth set is a 2 kb contig tiled by five overlapping amplicons.  The sample differs from the reference at SITE,
inside the left primer of amplicon 2: amplicon 2's reads start in that primer and copy its (reference) base there,
while amplicon 1 reads through the site with the sample's base.  Amplicon 2 has more reads, so without primer
masking the consensus shows the primer's base; with it, only amplicon 1's reads count there and the consensus shows
the sample's.  A few reads carry an insertion, a deletion or soft clips, so columns 5-18 and the insertion events are
exercised too."""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

import emu_harness as E
from kindel_b200 import bamio, engine
from kindel_b200 import primers as P

OPS = "MIDNSHP=X"
L = 2000
AMPLICONS = [(30, 480), (380, 830), (730, 1180), (1080, 1530), (1430, 1880)]
PRIMER_LEN = (24, 22, 26, 23, 25)
SITE = 390                        # 0-based; inside amplicon 2's left primer [380, 402)
N_READS = (8, 30, 10, 10, 10)     # per amplicon
REL = 0.5                         # `variants -r`: amplicon 1's share at SITE without masking is below it


def scheme_rows(name="t"):
    """[(chrom, start, end, name, pool, strand)]: both primers of every amplicon, ARTIC style."""
    rows = []
    for k, ((a, b), n) in enumerate(zip(AMPLICONS, PRIMER_LEN)):
        rows.append((name, a, a + n, "amp%d_LEFT" % (k + 1), 1 + k % 2, "+"))
        rows.append((name, b - n, b, "amp%d_RIGHT" % (k + 1), 1 + k % 2, "-"))
    return rows


def truth_set(seed=7):
    """(reference text, sample text, records [(pos0, ops, seq, reverse)])."""
    rng = np.random.default_rng(seed)
    ref = "".join("ACGT"[i] for i in rng.integers(0, 4, L))
    alt = "ACGT"[("ACGT".index(ref[SITE]) + 2) % 4]
    sample = ref[:SITE] + alt + ref[SITE + 1:]
    reads = []
    for k, ((a, b), n) in enumerate(zip(AMPLICONS, N_READS)):
        for j in range(n):
            # the primer's bases come from the oligo (the reference), the rest from the sample
            seq = list(sample[a:b])
            for lo, hi in ((a, a + PRIMER_LEN[k]), (b - PRIMER_LEN[k], b)):
                seq[lo - a:hi - a] = ref[lo:hi]
            seq = "".join(seq)
            ops = [(b - a, "M")]
            if j == 1:    # an insertion in the middle
                mid = (b - a) // 2
                seq = seq[:mid] + "TT" + seq[mid:]
                ops = [(mid, "M"), (2, "I"), (b - a - mid, "M")]
            elif j == 2:  # a deletion
                mid = (b - a) // 3
                seq = seq[:mid] + seq[mid + 3:]
                ops = [(mid, "M"), (3, "D"), (b - a - mid - 3, "M")]
            elif j == 3:  # soft clips at both ends (the clipped bases are adapter, not primer)
                seq = "GGGG" + seq + "CCC"
                ops = [(4, "S"), (b - a, "M"), (3, "S")]
            reads.append((a, ops, seq, j % 2))
    reads.sort(key=lambda r: r[0])
    return ref, sample, reads


def write(tmp_path, seed=7):
    """(BAM, BED, FASTA, ref, sample) of the truth set."""
    ref, sample, reads = truth_set(seed)
    bam, bed, fa = tmp_path / "amp.bam", tmp_path / "scheme.primer.bed", tmp_path / "ref.fa"
    bamio.write_bam(str(bam), [("t", L)],
                    [(0, p, 16 * rv, [(n << 4) | OPS.index(o) for n, o in ops], seq) for p, ops, seq, rv in reads])
    bed.write_text("".join("%s\t%d\t%d\t%s\t%d\t%s\n" % r for r in scheme_rows()))
    fa.write_text(">t\n" + "\n".join(ref[i:i + 60] for i in range(0, L, 60)) + "\n")
    return bam, bed, fa, ref, sample


def random_rows(rng, contigs, n_max=8):
    """Random, overlapping and duplicated intervals over contigs [(name, L)] -- at 0 and ending at L included -- plus
    rows of a contig the alignment does not have."""
    rows = []
    for name, Lc in contigs:
        if Lc < 1:
            continue
        for _ in range(int(rng.integers(0, n_max + 1))):
            a = int(rng.integers(0, Lc))
            b = int(rng.integers(a + 1, min(Lc, a + 12) + 1))
            rows.append((name, a, b))
        if rng.random() < 0.5:
            rows.append((name, 0, int(rng.integers(1, Lc + 1))))
        if rng.random() < 0.5:
            rows.append((name, int(rng.integers(0, Lc)), Lc))
        if rows and rng.random() < 0.3:
            rows.append(rows[-1])
    rows.append(("elsewhere", 0, 5))
    return rows


def primer_set(rows, name="scheme.bed") -> P.PrimerSet:
    return P.read_bed("".join("%s\t%d\t%d\n" % r[:3] for r in rows).encode(), name)


def arrays_for(batch, rows) -> P.PrimerArrays:
    return P.primer_arrays(primer_set(rows), batch.contig_names, batch.contig_len)


def emu_primers(batch, arrays):
    """K9 (kdl_primers_count, one read of the totals record, kdl_primers_apply) under the emulator, in place on a copy
    of the batch's seq4 as the engine runs it.  Returns (masked batch: the copy's seq4 and the merged mask list,
    totals [4])."""
    lib = E.load()
    struct, hold = engine.host_struct(batch)
    seq4 = np.array(batch.seq4, dtype=np.uint32, copy=True)
    struct.seq4 = seq4.ctypes.data
    qmask, qhold = engine.host_qmask(batch)
    qp = C.byref(qmask) if qmask is not None else None
    keep = {f: np.ascontiguousarray(getattr(arrays, f)) for f in ("contig_off", "start_sorted", "end_max", "end_sorted",
                                                                  "start_min")}
    p = engine.primers_struct(arrays, {f: (a.ctypes.data if a.size else None) for f, a in keep.items()})
    scratch = np.full(int(lib.kdl_primers_scratch_words(batch.n_reads)), 0xDEADBEEF, dtype=np.uint32)
    E._check(lib.kdl_primers_count(C.byref(struct), qp, C.byref(p), scratch.ctypes.data, None), "kdl_primers_count")
    tot = scratch[-8:].astype(np.int64)
    assert (tot[4:] == 0).all()
    n_mr, n_mb = int(tot[0]), int(tot[1])
    # one element more than announced, poisoned: the scatter must write exactly the announced ones
    out = dict(mask_read=np.full(n_mr + 1, 7, np.uint32), mask_off=np.full(n_mr + 2, 7, np.uint32),
               mask_qpos=np.full(n_mb + 1, 7, np.uint32))
    om = None
    if n_mr:
        om = C.byref(engine.make_qmask(_Counts(n_mr, n_mb), {f: out[f].ctypes.data for f in out}))
    E._check(lib.kdl_primers_apply(C.byref(struct), qp, C.byref(p), scratch.ctypes.data, seq4.ctypes.data, om, None),
             "kdl_primers_apply")
    sizes = dict(mask_read=n_mr, mask_off=n_mr + 1 if n_mr else 0, mask_qpos=n_mb)
    for f, k in sizes.items():
        assert (out[f][k:] == 7).all(), "K9 wrote past %s" % f
    del hold, qhold, keep
    masked = dataclasses.replace(batch, seq4=seq4, mask_read=out["mask_read"][:n_mr] if n_mr else None,
                                 mask_off=out["mask_off"][:n_mr + 1] if n_mr else None,
                                 mask_qpos=out["mask_qpos"][:n_mb] if n_mr else None)
    return masked, tot[:4]


@dataclasses.dataclass
class _Counts:
    n_mask_reads: int
    n_masked: int


def mask_lists(batch):
    """Per read, its sorted masked query offsets (from the batch's mask list)."""
    out = [[] for _ in range(batch.n_reads)]
    if batch.n_masked:
        for j, r in enumerate(np.asarray(batch.mask_read).tolist()):
            out[r] = np.asarray(batch.mask_qpos[int(batch.mask_off[j]):int(batch.mask_off[j + 1])]).tolist()
    return out


def nibbles(batch, r):
    """The nibbles of read r's bases."""
    base, n = int(batch.seq_off[r]), int(batch.seq_len[r])
    return [(int(batch.seq4[base + (q >> 3)]) >> (28 - 4 * (q & 7))) & 0xF for q in range(n)]
