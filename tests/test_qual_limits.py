"""K11 + K11g (`variants --vcf --qual`) at the engine's limits, without a GPU: every kdl_* call runs on the kernel
emulator, against oracle/py_qvoracle.py.

- Every limit group (tests/limit_cases.py) under every quality plan (tests/qual_limit_cases.py), in three thread
  orders and with 1 SM (K11g's grid-stride loop then runs more than once), into outputs that start as garbage.
- The two branches of kdl_quality_pileup give the same bits: the sorted batch (K0 + K11 + K11g over the hard reads)
  and the same reads unsorted (a zeroing pass + K11g over every read).
- With one quality q on every base, qsum is q times the pileup's columns A, C, G, T (coracle) and emass EPS[min(q, 93)]
  times their sum; on the limit lattice masked at MASK_QUAL, the counted bases are py_cvoracle's.
- The decoders lay out the qualities at the byte edges (0..254), and a first quality byte 0xff means "no qualities".
- A many-contig corpus, in the header's order and shuffled, through the pileup, K11 and the VCF.
- Sharded runs of `variants_vcf(qual=True)`, the ranks emulated in process, equal the oracle and one device."""
from __future__ import annotations

import itertools
import os

import numpy as np
import pytest

import emu_harness as E
import limit_cases as LC
import mate_cases as MC
import qual_limit_cases as QL
from kindel_b200 import bamio, distributed
from kindel_b200 import kindel as K
from oracle import coracle, py_cvoracle as CV, py_qvoracle as QV, samdecode
from test_consensus_combined import _emulated_ranks
from test_quality_filters import same_arrays
from test_variant_qual import _oracle, assert_sums, corpus, emu_quality, laid_out  # noqa: F401
from test_vcf_combined import SOURCE, on_the_emulator

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers for the kernel emulator")
GROUPS = list(LC.GROUPS)
MANY = 150  # contigs of the CPU's many-contig corpus (the device takes thousands)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """{(group, plan): (SAM path or None, BAM path)} and a cache of oracle sums."""
    d = tmp_path_factory.mktemp("qual_limits")
    out = {(name, plan): QL.write_limit_group(d, name, plan) for name in GROUPS for plan in QL.PLANS}
    return dict(paths=out, dir=d, sums={})


def sums_of(files, path, batch):
    if path not in files["sums"]:
        files["sums"][path] = QV.quality_sums(path)
    return laid_out(batch, files["sums"][path])


def k11(batch, qual8, schedule, sm, monkeypatch):
    """test_variant_qual.emu_quality (outputs poisoned first) with `sm` emulated SMs."""
    monkeypatch.setattr(E, "SM_COUNT", sm)
    try:
        return emu_quality(batch, qual8, schedule)
    finally:
        E.set_schedule("forward")


def per_read_quals(batch):
    """The reads' qualities out of a batch's qual8, concatenated in read order."""
    lens = batch.seq_len.astype(np.int64)
    idx = np.repeat(8 * batch.seq_off.astype(np.int64) - (np.cumsum(lens) - lens), lens) + np.arange(int(lens.sum()))
    return batch.qual8[idx]


def permuted(batch, seed):
    """(the batch's reads in a seeded random order, kept grouped by contig as bamio.select_reads keeps them; its
    qual8 with every read's qualities moved along)."""
    perm = np.random.default_rng(seed).permutation(batch.n_reads)
    perm = perm[np.argsort(np.searchsorted(batch.contig_read_off, perm, side="right"), kind="stable")]
    ub = bamio.select_reads(batch, perm)
    quals = per_read_quals(batch)
    at = np.concatenate(([0], np.cumsum(batch.seq_len.astype(np.int64))))
    return ub, bamio.qual_layout(ub, np.concatenate([quals[at[r]:at[r + 1]] for r in perm]))


def tiled(batch):
    """kdl_quality_pileup's test for its K0 + K11 branch (E._host_batch always supplies the tile index)."""
    return E.tileable(batch)


# ------------------------------------------------------------------------------------------- K11 + K11g on the groups
@needs_emu
@pytest.mark.parametrize("name", GROUPS)
def test_k11_on_every_limit_group(files, name, monkeypatch):
    """Each plan against py_qvoracle; over the plans, forward, reverse and random thread order with E.SM_COUNT SMs and
    with 1.  The SAM decode of a plan gives the same qual8 as the BAM's."""
    orders = list(itertools.product(("forward", "reverse", "random"), (E.SM_COUNT, 1)))
    for k, plan in enumerate(QL.PLANS):
        sam, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        assert tiled(batch)
        if sam is not None:
            np.testing.assert_array_equal(bamio.read_alignment(sam, qual=True).qual8, batch.qual8)
        want = sums_of(files, bam, batch)
        schedule, sm = orders[k % len(orders)]  # six plans, six orders: each once per group
        assert_sums(k11(batch, batch.qual8, schedule, sm, monkeypatch), want, "%s %s %s sm=%d" % (name, plan, schedule,
                                                                                                   sm))


@needs_emu
@pytest.mark.parametrize("name", GROUPS)
def test_both_dispatch_branches_agree(files, name, monkeypatch):
    """The sorted batch runs K0 + K11 + K11g over hard_idx, the same reads permuted (bamio.select_reads) a zeroing pass +
    K11g over every read: equal bit for bit, and equal to the oracle."""
    for plan in (("uniform", "bam_wide")[GROUPS.index(name) % 2],):  # (the groups alternate the two plans)
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        want = sums_of(files, bam, batch)
        ub, uq8 = permuted(batch, len(name))
        assert tiled(batch) and not ub.reads_sorted and not tiled(ub)
        a = k11(batch, batch.qual8, "random", 1, monkeypatch)
        b = k11(ub, uq8, "random", 1, monkeypatch)
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[1], b[1])
        assert_sums(a, want, "%s %s" % (name, plan))


# ------------------------------------------------------------------------------------------- invariants
@needs_emu
@pytest.mark.parametrize("name", GROUPS)
def test_constant_quality_against_the_pileup(files, name, monkeypatch):
    """With one quality q on every base: qsum == q * coracle's columns A, C, G, T and emass == EPS[q] * their sum.  The
    lattice decoded with min_base_quality=MASK_QUAL counts only Q40 bases: qsum == 40 * py_cvoracle's columns."""
    counts = None
    for plan, q in QL.CONST.items():
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        if counts is None:
            counts = coracle.pileup(batch)[0][0:4].astype(np.int64)
        qsum, emass = k11(batch, batch.qual8, "random", E.SM_COUNT, monkeypatch)
        np.testing.assert_array_equal(qsum.astype(np.int64), q * counts, err_msg=plan)
        np.testing.assert_array_equal(emass.astype(object), QV.EPS[q] * counts.sum(axis=0).astype(object), err_msg=plan)
    _, bam = files["paths"][(name, "lattice")]
    masked = bamio.read_alignment(bam, qual=True, min_base_quality=LC.MASK_QUAL)
    assert masked.n_masked > 0
    want = np.zeros((4, int(masked.n_slots)), dtype=np.int64)
    for c, (nm, cols, _) in enumerate(CV.Composed(bam, LC.MASK_QUAL, 0, 0, None).tables()):
        assert nm == masked.contig_names[c]
        s0, L = int(masked.contig_slot[c]), int(masked.contig_len[c])
        want[:, s0:s0 + L] = np.array([x[:L] for x in cols[0:4]], dtype=np.int64)
    qsum, emass = k11(masked, masked.qual8, "reverse", 1, monkeypatch)
    np.testing.assert_array_equal(qsum.astype(np.int64), 40 * want)
    np.testing.assert_array_equal(emass.astype(object), QV.EPS[40] * want.sum(axis=0).astype(object))


# ------------------------------------------------------------------------------------------- decoding
def _file_quals(path, batch):
    """samdecode's qualities of the kept records, in the batch's read order."""
    _, records = samdecode.read_alignment_file(path)
    by_contig = {}
    for rec in records:
        if rec.rname != "*" and not rec.flag & 4 and len(rec.seq) > 1:
            by_contig.setdefault(rec.rname, []).append(bytes(rec.qual))
    return np.frombuffer(b"".join(q for nm in batch.contig_names for q in by_contig[nm]), dtype=np.uint8)


@pytest.mark.parametrize("name", GROUPS)
def test_qual8_at_the_byte_edges(files, name):
    """kdl_bam_fill_qual's qual8 of every BAM plan is bamio.qual_layout of samdecode's qualities, byte for byte."""
    for plan in QL.PLANS:
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        quals = _file_quals(bam, batch)
        np.testing.assert_array_equal(batch.qual8, bamio.qual_layout(batch, quals), err_msg=plan)
        if plan == "bam_wide":
            assert set(range(QL.WIDE_LO, QL.WIDE_HI + 1)) <= set(np.unique(quals).tolist())


@needs_emu
def test_a_first_quality_byte_of_0xff_means_no_qualities(tmp_path, monkeypatch):
    """A read whose first quality byte is 0xff is a read without qualities (the decoder and samdecode agree), whatever
    its other bytes; a 0xff anywhere else is a quality of 255: qsum adds 255, emass EPS[93]."""
    contigs = [("f", 400)]
    good = bytes(range(60, 90))
    for first_ff in (True, False):
        odd = (b"\xff" + good[1:]) if first_ff else (good[:5] + b"\xff" + good[6:])
        recs = [(0, 10 * k, 0, [(30 << 4) | 0], "ACGT" * 7 + "AC", "r%d" % k, 60, good) for k in range(20)]
        recs[7] = recs[7][:7] + (odd,)
        path = str(tmp_path / ("ff%d.bam" % first_ff))
        bamio.write_bam(path, contigs, recs)
        _, records = samdecode.read_alignment_file(path)
        assert (records[7].qual is None) == first_ff
        if first_ff:
            with pytest.raises(ValueError, match="without base qualities"):
                bamio.read_alignment(path, qual=True)
            with pytest.raises(ValueError, match="without qualities"):
                QV.quality_sums(path)
            assert bamio.read_alignment(path).n_reads == 20  # without --qual nothing changes
            continue
        batch = bamio.read_alignment(path, qual=True)
        assert batch.qual8[8 * int(batch.seq_off[7]) + 5] == 0xFF
        want = laid_out(batch, QV.quality_sums(path))
        qsum, emass = k11(batch, batch.qual8, "forward", E.SM_COUNT, monkeypatch)
        assert_sums((qsum, emass), want)
        assert want[0][:, 75].sum() >= 255


# ------------------------------------------------------------------------------------------- many contigs
@pytest.fixture(scope="module")
def many(tmp_path_factory):
    d = tmp_path_factory.mktemp("many_contigs")
    return {sh: QL.write_many_contigs(d, MANY, 3, sh) for sh in (False, True)}


@needs_emu
@pytest.mark.parametrize("shuffled,fmt", [(False, "bam"), (True, "sam")], ids=["header_order-bam", "shuffled-sam"])
def test_many_contigs(many, shuffled, fmt, monkeypatch):
    """Dozens of contigs per tile, contigs without reads, in the header's order and shuffled: the SAM and BAM decodes
    agree, the pileup equals coracle, K11 (both branches) py_qvoracle, and variants_vcf(qual=True, reference=...) the
    composed oracle."""
    sam, bam, fa, refs = many[shuffled]
    path = sam if fmt == "sam" else bam
    batch = bamio.read_alignment(path, qual=True)
    other = bamio.read_alignment(bam if fmt == "sam" else sam, qual=True)
    same_arrays(other, batch)
    np.testing.assert_array_equal(other.qual8, batch.qual8)
    QL.check_shapes(batch, MANY, shuffled)
    counts, events = E.pileup_pipeline(batch)
    want_c, want_e = coracle.pileup(batch)
    np.testing.assert_array_equal(counts, want_c)
    np.testing.assert_array_equal(events, want_e)
    want = laid_out(batch, QV.quality_sums(bam))
    assert_sums(k11(batch, batch.qual8, "random", E.SM_COUNT, monkeypatch), want, "sorted")
    ub, uq8 = permuted(batch, 5)
    assert not tiled(ub)
    assert_sums(k11(ub, uq8, "forward", 1, monkeypatch), want, "permuted")
    on_the_emulator(monkeypatch)
    got = K.variants_vcf(path, 0, 0.0, qual=True, reference=fa, min_qual=20.0)
    oracle = QV.with_quality(CV.Composed(bam).vcf(SOURCE, 0, 0.0, (0, 0, 0), None, (os.path.basename(fa), refs)),
                             QV.quality_sums(bam), 20.0)
    assert got == oracle
    assert sum(not x.startswith("#") for x in got.splitlines()) > 100 and ";AQ=" in got


# ------------------------------------------------------------------------------------------- sharded runs
@pytest.fixture(scope="module")
def mixed(tmp_path_factory):
    """The `mixed` limit group (tile-eligible and hard reads) with seeded 0..93 qualities, a reference and primers."""
    d = tmp_path_factory.mktemp("qual_mixed")
    sam, bam = QL.write_limit_group(d, "mixed", "uniform")
    contigs, _ = QL.parse_sam(LC.sam_text("mixed"))
    nm, L = contigs[0]
    rng = np.random.default_rng(9)
    refs = {nm: "".join(rng.choice(list("ACGT"), L))}
    fa, bed = d / "mixed.fa", d / "mixed.bed"
    fa.write_text(">%s\n%s\n" % (nm, refs[nm]))
    rows = [(nm, a, a + 25) for a in range(1150, L - 200, 1333)]
    bed.write_text("".join("%s\t%d\t%d\tp%d\t1\t+\n" % (r + (k,)) for k, r in enumerate(rows)))
    return dict(bam=bam, sam=sam, fa=str(fa), bed=str(bed), refs=refs, rows=rows)


# every pair of the five options takes all four on / off combinations (checked below)
SHARD_ROWS = [  # (filters, primers, mates, reference, strand + max_sor)
    (0, 0, 0, 0, 0), (1, 1, 0, 0, 1), (1, 0, 1, 0, 1), (1, 0, 0, 1, 0), (0, 1, 1, 1, 1), (0, 1, 1, 1, 0),
]


def test_shard_rows_cover_every_pair():
    for i, j in itertools.combinations(range(5), 2):
        assert {(r[i], r[j]) for r in SHARD_ROWS} == {(0, 0), (0, 1), (1, 0), (1, 1)}, (i, j)


def _vcf_kwargs(inp, row):
    flt, pr, mates, ref, strand = row
    return dict(min_base_quality=20 if flt else 0, min_mapq=30 if flt else 0, exclude_flags=0x500 if flt else 0,
                primers=inp["bed"] if pr else None, mask_overlaps=bool(mates), reference=inp["fa"] if ref else None,
                strand=bool(strand), max_sor=3.0 if strand else None)


@pytest.fixture(scope="module")
def pairs(tmp_path_factory):
    """Overlapping read pairs (FLAG 0x1, RNEXT / PNEXT set) with qualities, a reference and primers: the input of the
    rows with mates on, where the second mates' overlap bases must be masked again before K11."""
    return MC.combo_files(tmp_path_factory.mktemp("qual_pairs"))


@needs_emu
def test_mates_change_the_paired_input(pairs, monkeypatch):
    """The mates rows are not vacuous: on the paired input, mask_overlaps changes the K11 sums (the overlap bases of
    the second mates leave them) and the VCF text."""
    on_the_emulator(monkeypatch)
    off, _ = K.pileup_run(pairs["bam"], qual=True)
    on, _ = K.pileup_run(pairs["bam"], qual=True, mask_overlaps=True)
    q_off, q_on = (r.quality_table()[0].numpy().view(np.uint32).astype(np.int64) for r in (off, on))
    assert on.overlap_stats[0] > 100 and on.overlap_stats[1] > 1000  # (pairs, masked bases)
    assert (q_on <= q_off).all() and int((q_off - q_on).sum()) > 1000 * 8
    kw = dict(qual=True, reference=pairs["fa"])
    assert K.variants_vcf(pairs["bam"], **kw) != K.variants_vcf(pairs["bam"], mask_overlaps=True, **kw)


_single = {}  # row -> (single-device text, oracle text): the same for every world and plan


@needs_emu
@pytest.mark.parametrize("plan", ["reads", "contigs"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_qual_equals_the_oracle_and_one_device(corpus, mixed, pairs, world, plan, monkeypatch):
    """variants_vcf(qual=True, devices=2 / 3): the ranks pile their shards on the emulated engine, the reduced table
    and the re-uploaded batch (its primers and mates masked again) feed K11; the text equals the oracle and the
    single-device text.  The rows with mates on read overlapping pairs; the others the qual combo corpus and the
    `mixed` limit group.  Each input is read as BAM in one world and as SAM in the other."""
    on_the_emulator(monkeypatch)
    monkeypatch.setattr(distributed, "run_sharded", _emulated_ranks(plan))
    inputs = [corpus, mixed, pairs, corpus, pairs, pairs]
    for k, row in enumerate(SHARD_ROWS):
        inp, fmt = inputs[k], ("bam", "sam")[(k + world) % 2]
        assert (inp is pairs) == bool(row[2])
        kw = _vcf_kwargs(inp, row)
        min_qual = (None, 30.0, 20.0)[k % 3]
        got = K.variants_vcf(inp[fmt], qual=True, min_qual=min_qual, devices=world, **kw)
        if k not in _single:
            ref = (os.path.basename(inp["fa"]), inp["refs"]) if row[3] else None
            _single[k] = (K.variants_vcf(inp[fmt], qual=True, min_qual=min_qual, devices=1, **kw),
                          _oracle(inp, inp["bam"], kw["min_base_quality"], kw["min_mapq"], kw["exclude_flags"],
                                  bool(row[1]), ref, kw["strand"], kw["max_sor"], bool(row[2]), min_qual))
        one, want = _single[k]
        assert got == want, (row, world, plan, fmt)
        assert one == got
        assert ";AQ=" in got
