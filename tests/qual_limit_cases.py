"""Base-quality plans over the limit corpus, and a many-contig corpus, for `variants --vcf --qual` (test infrastructure).

K11 / K11g (kindel_b200/csrc/quality.cu) sum each counted base's Phred value and EPS[min(q, 93)].  The limit corpus
(limit_cases.py) puts reads on every capacity of the tile path, with a Q2 / Q40 lattice; the plans here give the same
reads other qualities, seeded and deterministic:

  lattice     the groups' own Q2 / Q40 lattice, unchanged
  uniform     per-base seeded values 0..93 (SAM and BAM)
  bam_wide    per-base seeded bytes 0..254 with every value 94..254 present (BAM only: SAM text stops at Q93), so
              that emass clamps at EPS[93] while qsum adds the raw byte
  const<q>    every base q, q in {0, 41, 93}

`many_contigs` builds a file of many contigs from SAM text, in the way limit_cases._Group does: lengths from a
fixed set around the tile size and uniform 1..400, contigs without reads (which leave the batch), a run of 60
consecutive contigs of 1..12 bases with reads (each owns L + 1 slots, so dozens share one 512-slot tile),
simple, clipped + inserting and deleting reads, and hard reads that wrap (SAM POS 0), run a right clip past the
contig's end, or have a soft clip between two M ops.  The reads copy a seeded reference with a few mismatches and
N bases.  The file holds one block of reads per contig, in the header's order or shuffled; `check_shapes`
asserts that a batch of it reaches what it is built for."""
from __future__ import annotations

import random
import zlib

import numpy as np

import limit_cases as LC
import qual_cases as QC
from kindel_b200 import bamio

PLANS = ("lattice", "uniform", "bam_wide", "const0", "const41", "const93")
SAM_PLANS = tuple(p for p in PLANS if p != "bam_wide")
CONST = {"const0": 0, "const41": 41, "const93": 93}
MAX_SAM_Q = 93
WIDE_LO, WIDE_HI = 94, 254  # (255 = 0xff in the first byte means "no qualities")


def parse_sam(text):
    """(contigs [(name, L)], records as bamio.write_bam takes them: (ref_id, pos0, flag, cigar words, seq, qname,
    mapq, qual bytes or None)) of SAM text, in the file's order."""
    contigs, recs = [], []
    ids = {}
    for line in text.splitlines():
        f = line.split("\t")
        if line.startswith("@SQ"):
            kv = dict(x.split(":", 1) for x in f[1:])
            ids[kv["SN"]] = len(contigs)
            contigs.append((kv["SN"], int(kv["LN"])))
            continue
        if line.startswith("@") or len(f) < 11:
            continue
        qual = None if f[10] == "*" else bytes(ord(c) - 33 for c in f[10])
        recs.append((ids.get(f[2], -1), int(f[3]) - 1, int(f[1]), bamio.parse_cigar_text(f[5]), f[9], f[0], int(f[4]),
                     qual))
    return contigs, recs


def plan_qualities(plan, lengths, seed):
    """One bytes object per read (`lengths` bases each) for a plan other than `lattice`."""
    total = int(sum(lengths))
    if plan in CONST:
        flat = np.full(total, CONST[plan], dtype=np.uint8)
    else:
        rng = np.random.default_rng(seed)
        hi = MAX_SAM_Q if plan == "uniform" else WIDE_HI
        flat = rng.integers(0, hi + 1, total, dtype=np.int64).astype(np.uint8)
        if plan == "bam_wide":
            wide = np.arange(WIDE_LO, WIDE_HI + 1, dtype=np.uint8)
            at = rng.choice(total, wide.size, replace=False)  # every value 94..254 somewhere
            flat[at] = wide
            assert set(range(WIDE_LO, WIDE_HI + 1)) <= set(np.unique(flat).tolist())
    out, k = [], 0
    for n in lengths:
        out.append(flat[k:k + n].tobytes())
        k += n
    return out


def with_plan(contigs, recs, plan, seed):
    """The records with the plan's qualities (`lattice`: unchanged)."""
    if plan == "lattice":
        return list(recs)
    quals = plan_qualities(plan, [len(r[4]) for r in recs], seed)
    return [r[:7] + (q,) for r, q in zip(recs, quals)]


def _seed(name):
    return zlib.crc32(name.encode())


def write_limit_group(d, name, plan):
    """(SAM path or None, BAM path) of limit group `name` with the plan's qualities under directory d."""
    contigs, recs = parse_sam(LC.sam_text(name))
    recs = with_plan(contigs, recs, plan, _seed(name + plan))
    stem = "%s_%s" % (name, plan)
    bam = str(d / (stem + ".bam"))
    bamio.write_bam(bam, contigs, recs)
    sam = None
    if plan in SAM_PLANS:  # (SAM text holds Q0..93)
        sam = str(d / (stem + ".sam"))
        QC.write_sam(sam, contigs, recs)
    return sam, bam


# ---------------------------------------------------------------------------------------------------- many contigs
LENGTH_SET = (1, 2, 3, 7, 40, 150, 300, 511, 512, 513, 700)
RUN = 60          # consecutive tiny contigs, each with reads
TINY = (1, 12)    # their lengths


def _mutate(rng, ref):
    out = []
    for b in ref:
        x = rng.random()
        out.append("N" if x < 0.01 else "ACGT"[("ACGT".index(b) + 1 + rng.randrange(3)) % 4] if x < 0.04 else b)
    return "".join(out)


def _reads_for(rng, ref):
    """(pos0, cigar, seq) of the reads of one contig with reference text `ref`."""
    L = len(ref)
    out = []
    if L == 1:  # (a read of one base is dropped): two-base reads whose second base is clipped or inserted
        return [(0, "1M1S", _mutate(rng, ref) + "A"), (0, "1S1M", "C" + _mutate(rng, ref)), (0, "1M1I", "GT")]
    for _ in range(1 + L // 30):
        kind = rng.random()
        if kind < 0.5 or L < 6:
            n = rng.randint(2, min(L, 150))
            pos = rng.randint(0, L - n)
            out.append((pos, "%dM" % n, _mutate(rng, ref[pos:pos + n])))
        elif kind < 0.65:  # clipped + inserting
            m1, m2 = rng.randint(1, min(60, L // 2)), rng.randint(1, min(60, L // 2))
            pos = rng.randint(0, L - m1 - m2)
            a, i, c = rng.randint(1, 6), rng.randint(1, 9), rng.randint(0, 5)
            seq = "".join(rng.choice("ACGT") for _ in range(a)) + _mutate(rng, ref[pos:pos + m1]) + \
                "".join(rng.choice("ACGT") for _ in range(i)) + _mutate(rng, ref[pos + m1:pos + m1 + m2]) + \
                "".join(rng.choice("ACGT") for _ in range(c))
            out.append((pos, "%dS%dM%dI%dM" % (a, m1, i, m2) + ("%dS" % c if c else ""), seq))
        elif kind < 0.8:  # deleting
            m1, dl = rng.randint(1, min(60, L // 3)), rng.randint(1, min(20, L // 3))
            m2 = rng.randint(1, min(60, L - m1 - dl))
            pos = rng.randint(0, L - m1 - dl - m2)
            out.append((pos, "%dM%dD%dM" % (m1, dl, m2),
                        _mutate(rng, ref[pos:pos + m1] + ref[pos + m1 + dl:pos + m1 + dl + m2])))
        elif kind < 0.87:  # SAM POS 0: the first base lands on the contig's last position (weights[-1])
            n = rng.randint(2, min(L, 30))
            out.append((-1, "%dM" % n, _mutate(rng, ref[-1] + ref[:n - 1])))
        elif kind < 0.94:  # a right clip that runs past the contig's end
            m = rng.randint(1, min(L - 1, 40))
            c = rng.randint(1, 8)
            pos = L - m - rng.randint(0, min(c - 1, L - m))
            out.append((pos, "%dM%dS" % (m, c), _mutate(rng, ref[pos:pos + m]) +
                        "".join(rng.choice("ACGT") for _ in range(c))))
        else:  # at POS 1 (hard), a soft clip between two M ops: the clip advances both cursors
            m1, c = rng.randint(1, min(20, L // 3)), rng.randint(1, min(6, L // 3))
            m2 = rng.randint(1, min(20, L - m1 - c))
            seq = _mutate(rng, ref[:m1]) + "".join(rng.choice("ACGT") for _ in range(c)) + \
                _mutate(rng, ref[m1 + c:m1 + c + m2])
            out.append((0, "%dM%dS%dM" % (m1, c, m2), seq))
    return sorted(out, key=lambda x: x[0])


def many_contigs(n_contigs, seed):
    """(contigs [(name, L)] in header order, {name: reference text}, {name: [(pos0, cigar, seq)]}).  About one contig
    in eight has no reads; contigs [n // 3, n // 3 + RUN) are the run of tiny contigs with reads."""
    assert n_contigs >= RUN + 10
    rng = random.Random(seed)
    contigs, refs, reads = [], {}, {}
    run0 = n_contigs // 3
    for k in range(n_contigs):
        tiny = run0 <= k < run0 + RUN
        if tiny:
            L = rng.randint(*TINY)
        elif rng.random() < 0.5:
            L = rng.choice(LENGTH_SET)
        else:
            L = rng.randint(1, 400)
        nm = "c%04d" % k
        contigs.append((nm, L))
        refs[nm] = "".join(rng.choice("ACGT") for _ in range(L))
        if tiny or rng.random() >= 0.125:
            reads[nm] = _reads_for(rng, refs[nm])
    return contigs, refs, reads


def many_contigs_sam(contigs, reads, shuffled, seed):
    """SAM text: one block of reads per contig, blocks in the header's order or shuffled; every quality `I` (Q40)
    until a plan replaces it."""
    order = [nm for nm, _ in contigs if nm in reads]
    if shuffled:  # the run of tiny contigs stays one run (shuffled inside), or nothing would put dozens in one tile
        rng = random.Random(seed ^ 0x5EED)
        run0 = len(contigs) // 3
        run = [nm for nm, _ in contigs[run0:run0 + RUN]]
        rng.shuffle(run)
        units = [[nm] for nm in order if nm not in set(run)] + [run]
        rng.shuffle(units)
        order = [nm for u in units for nm in u]
    lines = ["@HD\tVN:1.6\tSO:unsorted"] + ["@SQ\tSN:%s\tLN:%d" % c for c in contigs]
    k = 0
    for nm in order:
        for pos0, cigar, seq in reads[nm]:
            lines.append("m%d\t0\t%s\t%d\t60\t%s\t*\t0\t0\t%s\t%s" % (k, nm, pos0 + 1, cigar, seq, "I" * len(seq)))
            k += 1
    return "\n".join(lines) + "\n"


def write_many_contigs(d, n_contigs, seed, shuffled, plan="uniform"):
    """(SAM path or None, BAM path, FASTA path, {name: reference text}) of the many-contig corpus under directory d."""
    contigs, refs, reads = many_contigs(n_contigs, seed)
    hdr, recs = parse_sam(many_contigs_sam(contigs, reads, shuffled, seed))
    recs = with_plan(hdr, recs, plan, seed + 17)
    stem = "many_%d_%d_%s_%s" % (n_contigs, seed, "shuffled" if shuffled else "header", plan)
    bam, fa = str(d / (stem + ".bam")), str(d / (stem + ".fa"))
    bamio.write_bam(bam, hdr, recs)
    sam = None
    if plan in SAM_PLANS:
        sam = str(d / (stem + ".sam"))
        QC.write_sam(sam, hdr, recs)
    with open(fa, "w") as fh:
        fh.write("".join(">%s\n%s\n" % (nm, refs[nm]) for nm, _ in contigs))
    return sam, bam, fa, refs


def tile_contigs(batch):
    """Per 512-slot tile, the number of the batch's contigs whose first slot lies in it."""
    n_tiles = int(batch.n_slots) // LC.KDL_TILE
    return np.bincount(np.asarray(batch.contig_slot, dtype=np.int64) // LC.KDL_TILE, minlength=n_tiles)


def check_shapes(batch, n_header, shuffled):
    """The many-contig batch reaches what it is built for: a 512-slot tile holds >= 24 contigs, the reads of one tile
    come from >= 24 contigs, contigs without reads left the batch, hard and tile-eligible complex reads are there;
    shuffled, the batch's contig order (first seen in the file) is not the header's."""
    assert tile_contigs(batch).max() >= 24
    contig_of = np.repeat(np.arange(batch.n_contigs), np.diff(np.asarray(batch.contig_read_off, dtype=np.int64)))
    start = np.asarray(batch.contig_slot, dtype=np.int64)[contig_of] + np.asarray(batch.ref_start, dtype=np.int64)
    per_tile = {}
    for t, c in zip((start // LC.KDL_TILE).tolist(), contig_of.tolist()):
        per_tile.setdefault(t, set()).add(c)
    assert max(len(v) for v in per_tile.values()) >= 24
    assert batch.n_contigs < n_header
    assert batch.n_hard > 0 and batch.n_complex > batch.n_hard and batch.reads_sorted
    names = list(batch.contig_names)
    assert (names != sorted(names)) == shuffled
