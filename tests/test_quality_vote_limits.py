"""The quality vote (`consensus --quality-vote`) at the engine's limits, without a GPU: every kdl_* call runs on the
kernel emulator, against py_qvoracle's walk fed W[min(q, 93)] and the composed oracle of tests/qvote_limit_cases.py.

- K11w + K11g-w on every limit group under every quality plan, in three thread orders and with 1 SM, into outputs
  preset to garbage; the sorted and the permuted dispatch branch give the same bits.
- With one quality on every base, wsum is W[q] times the pileup's columns, and K2w is the count vote where it can be.
- A column of 4100 reads (more than four 1024-read chunks of one tile), as Q93, as the BAM byte 254 and as a minority
  that wins by weight, with its exact sums.
- A 150-contig corpus through K11w and `bam_to_consensus(quality_vote=True, qualities=True)`.
- A pairwise option matrix (filters, min_depth, realign, trim, uppercase, FASTQ, primers, mates) on a paired corpus
  with a quality on every read, and sharded runs with the ranks emulated in process.
- Reads without qualities: dropped ones are fine, kept ones are an error naming the file."""
from __future__ import annotations

import itertools
import os
import re

import numpy as np
import pytest

import emu_harness as E
import limit_cases as LC
import qual_limit_cases as QL
import qvote_limit_cases as QVL
from kindel_b200 import bamio, distributed
from kindel_b200 import kindel as K
from kindel_b200.quality import WEIGHT
from oracle import coracle, fqoracle, py_cvoracle as CV
from test_consensus_combined import _emulated_ranks, same_as_oracle, same_reports
from test_qual_limits import SHARD_ROWS, files, mixed, pairs, permuted, tiled  # noqa: F401
from test_quality_vote import assert_wsum, emu_vote_quality, emu_weights, weight_oracle
from test_vcf_combined import on_the_emulator

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers for the kernel emulator")
GROUPS = list(LC.GROUPS)
MANY = 150


def k11w(batch, qual8, schedule, sm, monkeypatch):
    """test_quality_vote.emu_weights (outputs poisoned first) with `sm` emulated SMs."""
    monkeypatch.setattr(E, "SM_COUNT", sm)
    try:
        return emu_weights(batch, qual8, schedule)
    finally:
        E.set_schedule("forward")


def wsums_of(files, path, batch, *args):
    """The oracle's weight sums of a file laid out on the batch's slots (cached per file and options)."""
    key = ("w", path) + args
    if key not in files["sums"]:
        files["sums"][key] = QVL.weight_sums(path, *args)
    want = np.zeros((4, int(batch.n_slots)), dtype=object)
    want[:] = 0
    for c, nm in enumerate(batch.contig_names):
        s0 = int(batch.contig_slot[c])
        w = files["sums"][key].get(nm)
        if w is not None:
            want[:, s0:s0 + len(w[0])] = np.array(w, dtype=object)
    return want


# ------------------------------------------------------------------------------------------- K11w on the groups
@needs_emu
@pytest.mark.parametrize("name", GROUPS)
def test_k11w_on_every_limit_group(files, name, monkeypatch):
    """Each plan against py_qvoracle fed weights; over the plans, forward, reverse and random thread order with
    E.SM_COUNT SMs and with 1.  The SAM decode gives the same sums."""
    orders = list(itertools.product(("forward", "reverse", "random"), (E.SM_COUNT, 1)))
    for k, plan in enumerate(QL.PLANS):
        sam, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        assert tiled(batch)
        want = wsums_of(files, bam, batch)
        schedule, sm = orders[k % len(orders)]
        got = k11w(batch, batch.qual8, schedule, sm, monkeypatch)
        assert_wsum(got, want, "%s %s %s sm=%d" % (name, plan, schedule, sm))
        if sam is not None:
            sb = bamio.read_alignment(sam, qual=True)
            assert_wsum(k11w(sb, sb.qual8, "random", E.SM_COUNT, monkeypatch), want, "%s %s sam" % (name, plan))


@needs_emu
@pytest.mark.parametrize("name", GROUPS)
def test_both_dispatch_branches_agree(files, name, monkeypatch):
    """The sorted batch (K0 + K11w + K11g-w over the hard reads) and the same reads permuted (a zeroing pass + K11g-w
    over every read): equal bit for bit, and equal to the oracle."""
    plan = ("uniform", "bam_wide")[GROUPS.index(name) % 2]
    _, bam = files["paths"][(name, plan)]
    batch = bamio.read_alignment(bam, qual=True)
    ub, uq8 = permuted(batch, len(name))
    assert tiled(batch) and not ub.reads_sorted and not tiled(ub)
    a = k11w(batch, batch.qual8, "random", 1, monkeypatch)
    b = k11w(ub, uq8, "reverse", E.SM_COUNT, monkeypatch)
    np.testing.assert_array_equal(a, b)
    assert_wsum(a, wsums_of(files, bam, batch), "%s %s" % (name, plan))


# ------------------------------------------------------------------------------------------- invariants
@needs_emu
@pytest.mark.parametrize("name", GROUPS)
def test_constant_quality_invariants(files, name, monkeypatch):
    """wsum == W[q] * coracle's columns A, C, G, T for q in {0, 41, 93}; K2w under Q0 emits N at Q0 everywhere with
    kdl_vote's change bits, under Q41 / Q93 it equals kdl_vote wherever the N count is below the largest base count.
    The lattice masked at MASK_QUAL counts only its Q40 bases: wsum == W[40] * py_cvoracle's columns."""
    counts = None
    for plan, q in QL.CONST.items():
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        if counts is None:
            counts = coracle.pileup(batch)[0]
        wsum = k11w(batch, batch.qual8, "random", E.SM_COUNT, monkeypatch)
        np.testing.assert_array_equal(wsum.astype(object), WEIGHT[q] * counts[0:4].astype(object), err_msg=plan)
        for md in (1, 3):
            calls, qual = emu_vote_quality(counts, wsum, md)
            base = E.vote(counts, md)
            np.testing.assert_array_equal(calls >> 4, base >> 4, err_msg=plan)
            if q == 0:
                assert ((calls & 0x0F) == 4).all() and not qual.any(), plan
            else:
                live = counts[4] < counts[0:4].max(axis=0)
                assert live.sum() > 100
                np.testing.assert_array_equal(calls[live], base[live], err_msg="%s md=%d" % (plan, md))
    _, bam = files["paths"][(name, "lattice")]
    masked = bamio.read_alignment(bam, qual=True, min_base_quality=LC.MASK_QUAL)
    assert masked.n_masked > 0
    want = np.zeros((4, int(masked.n_slots)), dtype=np.int64)
    for c, (nm, cols, _) in enumerate(CV.Composed(bam, LC.MASK_QUAL, 0, 0, None).tables()):
        s0, L = int(masked.contig_slot[c]), int(masked.contig_len[c])
        want[:, s0:s0 + L] = np.array([x[:L] for x in cols[0:4]], dtype=np.int64)
    wsum = k11w(masked, masked.qual8, "reverse", 1, monkeypatch)
    np.testing.assert_array_equal(wsum.astype(object), WEIGHT[40] * want.astype(object))


# ------------------------------------------------------------------------------------------- the deep column
@pytest.fixture(scope="module")
def deep(tmp_path_factory):
    d = tmp_path_factory.mktemp("qvote_deep")
    return {v: QVL.write_deep(d, v) for v in QVL.DEEP_VARIANTS}


@needs_emu
@pytest.mark.parametrize("variant", QVL.DEEP_VARIANTS)
def test_the_deep_column(deep, variant, monkeypatch):
    """More than 3 * 1024 reads start in one tile and 4100 cover one slot: K11w's uint32 partials are folded once per
    chunk.  Both dispatch branches equal the oracle, the slot's sums are exact (n * W[q]), and the byte 254 weighs
    what Q93 does."""
    sam, bam = deep[variant]
    batch = bamio.read_alignment(bam, qual=True)
    assert tiled(batch) and batch.n_complex == 0
    got = k11w(batch, batch.qual8, "random", E.SM_COUNT, monkeypatch)
    QVL.check_deep_shape(batch, got if variant != "minority" else None)
    want = weight_oracle(batch, per_read(batch))
    assert_wsum(got, want, variant)
    a, g = QVL.deep_want(variant)
    assert (int(got[0, QVL.DEEP_SLOT]), int(got[2, QVL.DEEP_SLOT])) == (a, g)
    ub, uq8 = permuted(batch, 4)
    assert not tiled(ub)
    np.testing.assert_array_equal(k11w(ub, uq8, "forward", 1, monkeypatch), got)
    if variant == "byte254":
        q93 = bamio.read_alignment(deep["q93"][1], qual=True)
        np.testing.assert_array_equal(k11w(q93, q93.qual8, "reverse", 1, monkeypatch), got)
    if variant == "minority":  # the count vote takes A, the quality vote G
        counts = coracle.pileup(batch)[0]
        assert E.vote(counts)[QVL.DEEP_SLOT] == 0
        assert emu_vote_quality(counts, got)[0][QVL.DEEP_SLOT] == 2
    if sam is not None:
        sb = bamio.read_alignment(sam, qual=True)
        np.testing.assert_array_equal(sb.qual8, batch.qual8)


def per_read(batch):
    """The reads' qualities out of a batch's qual8, in read order."""
    lens = batch.seq_len.astype(np.int64)
    idx = np.repeat(8 * batch.seq_off.astype(np.int64) - (np.cumsum(lens) - lens), lens) + np.arange(int(lens.sum()))
    return batch.qual8[idx]


# ------------------------------------------------------------------------------------------- many contigs
@pytest.fixture(scope="module")
def many(tmp_path_factory):
    d = tmp_path_factory.mktemp("qvote_many")
    return {sh: QL.write_many_contigs(d, MANY, 3, sh) for sh in (False, True)}


def check_vote_consensus(got, p, path, md=1, realign=False, trim=False, upper=False, fastq=True, what=""):
    want = p.consensus(None, md, realign, trim, upper)
    if not fastq:
        want = [(n, s, c, None, pt) for n, s, c, _, pt in want]
    same_as_oracle(got, want, what)
    same_reports(got, p.reports(path, None, md, realign, trim, upper), what)


@needs_emu
@pytest.mark.parametrize("shuffled,fmt", [(False, "bam"), (True, "sam")], ids=["header_order-bam", "shuffled-sam"])
def test_many_contigs(many, shuffled, fmt, monkeypatch):
    """Dozens of contigs per tile, 1-base contigs, contigs without reads, in the header's order and shuffled: K11w
    (both branches) equals the oracle, and bam_to_consensus(quality_vote=True, qualities=True) the composed oracle on
    every contig's sequence, qualities and REPORT."""
    sam, bam, _, _ = many[shuffled]
    path = sam if fmt == "sam" else bam
    batch = bamio.read_alignment(path, qual=True)
    QL.check_shapes(batch, MANY, shuffled)
    want = wsums_of({"sums": {}}, bam, batch)
    assert_wsum(k11w(batch, batch.qual8, "random", E.SM_COUNT, monkeypatch), want, "sorted")
    ub, uq8 = permuted(batch, 5)
    assert_wsum(k11w(ub, uq8, "forward", 1, monkeypatch), want, "permuted")
    on_the_emulator(monkeypatch)
    got = K.bam_to_consensus(path, quality_vote=True, qualities=True)
    p = QVL.QualityVotePiled(bam, batch)
    check_vote_consensus(got, p, path, what=path)
    assert len(got.consensuses) == batch.n_contigs < MANY and 1 in set(batch.contig_len.tolist())
    assert len(p.sites()) > 10


# ------------------------------------------------------------------------------------------- the consensus matrix
@pytest.fixture(scope="module")
def filled(tmp_path_factory):
    d = tmp_path_factory.mktemp("qvote_filled")
    out = QVL.write_filled(d)
    out.update(dir=d, layout=bamio.read_alignment(out["bam"], qual=True), piled={})
    return out


def vpiled(inp, bq=0, mq=0, ex=0, primers=False, mates=False):
    key = (bq, mq, ex, primers, mates)
    if key not in inp["piled"]:
        inp["piled"][key] = QVL.QualityVotePiled(inp["bam"], inp["layout"], bq, mq, ex,
                                                 inp["rows"] if primers else None, mates,
                                                 os.path.basename(inp["bed"]) if primers else None)
    return inp["piled"][key]


def test_vote_matrix_covers_every_pair():
    rows = QVL.vote_matrix()
    assert len(rows) <= 10
    for i, j in itertools.combinations(range(9), 2):
        assert {(r[i], r[j]) for r in rows} == {(a, b) for a in {r[i] for r in rows} for b in {r[j] for r in rows}}


def test_shard_rows_cover_every_pair():
    for i, j in itertools.combinations(range(5), 2):
        assert {(r[i], r[j]) for r in SHARD_ROWS} == {(0, 0), (0, 1), (1, 0), (1, 1)}, (i, j)


def test_corpus_has_what_it_is_for(filled):
    """Every planted window of the filled corpus is reached in the oracle: the two votes differ each way, mates and
    primers flip the quality vote, min_base_quality 20 brings the votes together, a `--realign` patch covers a site,
    and sites sit at an insertion and at a contig's last position.  Every record has its qualities."""
    assert all(r[7] is not None for r in filled["recs"])
    lay = filled["layout"]
    q0 = int(lay.contig_slot[lay.contig_names.index(QVL.QV_NAME)])
    plain, mates, primed, bq20 = vpiled(filled), vpiled(filled, mates=True), vpiled(filled, primers=True), \
        vpiled(filled, 20)
    cv, qv = coracle.vote(plain.counts, 1), plain.calls()
    at = lambda calls, p: int(calls[q0 + p])  # noqa: E731
    a, b = at(cv, QVL.TO_OTHER), at(qv, QVL.TO_OTHER)
    assert a & 7 < 4 and b & 7 < 4 and a != b
    assert at(cv, QVL.TIE_TO_BASE) & 7 == 4 and at(qv, QVL.TIE_TO_BASE) & 7 < 4
    assert at(cv, QVL.TO_N) & 7 < 4 and at(qv, QVL.TO_N) == 4
    assert (plain.vote()[1][q0 + QVL.TO_N], plain.vote()[1][q0 + QVL.TO_OTHER]) == (0, 60)
    for p, other in ((QVL.MATES_FLIP, mates), (QVL.PRIMER_FLIP, primed)):
        assert at(qv, p) != at(cv, p) == at(coracle.vote(other.counts, 1), p) == at(other.calls(), p), p
    assert at(coracle.vote(bq20.counts, 1), QVL.TO_OTHER) == at(bq20.calls(), QVL.TO_OTHER) == at(qv, QVL.TO_OTHER)
    assert q0 + QVL.TO_OTHER not in set(bq20.sites().tolist())
    ins = at(qv, QVL.AT_INSERTION)
    assert ins >> 4 == 3 and at(cv, QVL.AT_INSERTION) >> 4 == 3 and ins != at(cv, QVL.AT_INSERTION)
    last = q0 + QVL.QV_LEN - 1
    assert last in set(plain.sites().tolist())
    e = lay.contig_names.index("edge")
    e0 = int(lay.contig_slot[e])
    patched = {e0 + x for r in mates.patches(e) if r.seq for x in range(r.start, r.end)}
    assert patched & set(mates.sites().tolist())
    assert not any(r.seq for r in plain.patches(e))
    # the quality vote differs from the count vote outside the planted contig too (other windows, other Q)
    assert len(plain.sites()) > len([s for s in plain.sites() if s >= q0])


def test_fastq_oracle_default_q_is_its_own_rule(filled):
    """fqoracle.fastq without `qual` is fqoracle.fastq with qual(counts, calls): every existing caller is unchanged."""
    p = vpiled(filled, mates=True)
    calls = coracle.vote(p.counts, 1)
    own = fqoracle.qual(p.counts, calls)
    n = 0
    for c, name, s0, L, ins_c in p.contigs():
        for realign in (False, True):
            patches = p.patches(c) if realign else None
            a = fqoracle.fastq(p.counts, calls, s0, L, ins_c, patches, realign, not realign)
            assert a == fqoracle.fastq(p.counts, calls, s0, L, ins_c, patches, realign, not realign, qual=own)
            n += len(a[0])
        q = np.full(p.counts.shape[1], 7, dtype=np.uint8)
        _, quals = fqoracle.fastq(p.counts, calls, s0, L, ins_c, qual=q)  # one "(" per position that emits a base
        assert quals.count("(") >= int((((calls[s0:s0 + L] >> 4) & 3) != 1).sum())
    assert n > 3000


def vote_kwargs(inp, row):
    bq, md, realign, trim, upper, fastq, (mq, ex), pr, mates = row
    return dict(min_base_quality=bq, min_depth=md, realign=realign, trim_ends=trim, uppercase=upper, qualities=fastq,
                min_mapq=mq, exclude_flags=ex, primers=inp["bed"] if pr else None, mask_overlaps=mates,
                quality_vote=True)


def check_row(inp, row, got, path):
    bq, md, realign, trim, upper, fastq, (mq, ex), pr, mates = row
    check_vote_consensus(got, vpiled(inp, bq, mq, ex, pr, mates), path, md, realign, trim, upper, fastq, row)


@needs_emu
def test_vote_matrix_emulated(filled, monkeypatch):
    """bam_to_consensus(quality_vote=True) over the pairwise option matrix, from BAM and from SAM: sequence, qualities,
    change lists and REPORT equal the oracle."""
    on_the_emulator(monkeypatch)
    n_sites = 0
    for k, row in enumerate(QVL.vote_matrix()):
        for path in (filled["bam"], filled["sam"]):
            got = K.bam_to_consensus(path, **vote_kwargs(filled, row))
            check_row(filled, row, got, path)
        n_sites += sum(bool(re.search(r"- quality-vote sites: \d", r)) for r in got.refs_reports.values())
    assert n_sites > 10


# ------------------------------------------------------------------------------------------- sharded runs
def shard_kwargs(inp, row):
    flt, pr, mates, fastq, realign = row
    return dict(min_base_quality=20 if flt else 0, min_mapq=30 if flt else 0, exclude_flags=0x400 if flt else 0,
                primers=inp["bed"] if pr else None, mask_overlaps=bool(mates), qualities=bool(fastq),
                realign=bool(realign), quality_vote=True)


def shard_oracle(inp, row):
    kw = shard_kwargs(inp, row)
    inp.setdefault("piled", {})
    if "layout" not in inp:
        inp["layout"] = bamio.read_alignment(inp["bam"], qual=True)
    return vpiled(inp, kw["min_base_quality"], kw["min_mapq"], kw["exclude_flags"], bool(row[1]), bool(row[2]))


_single = {}  # row -> single-device result


@needs_emu
@pytest.mark.parametrize("plan", ["reads", "contigs"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_vote_equals_the_oracle_and_one_device(filled, mixed, pairs, world, plan, monkeypatch):
    """bam_to_consensus(quality_vote=True, devices=2 / 3): the ranks' majority calls are dropped, the reduced table and
    the re-uploaded batch (its primers and mates masked again) feed K11w and K2w.  The rows pairwise-cover filters,
    primers, mates, FASTQ and realign; the rows with mates read overlapping pairs.  Each equals the oracle and the
    one-device result, read as BAM in one world and as SAM in the other."""
    on_the_emulator(monkeypatch)
    monkeypatch.setattr(distributed, "run_sharded", _emulated_ranks(plan))
    inputs = [filled, mixed, pairs, mixed, pairs, filled]
    for k, row in enumerate(SHARD_ROWS):
        inp, fmt = inputs[k], ("bam", "sam")[(k + world) % 2]
        assert not (inp is mixed and row[2])
        kw = shard_kwargs(inp, row)
        got = K.bam_to_consensus(inp[fmt], devices=world, **kw)
        if (k, fmt) not in _single:
            _single[k, fmt] = K.bam_to_consensus(inp[fmt], devices=1, **kw)
        one = _single[k, fmt]
        check_vote_consensus(got, shard_oracle(inp, row), inp[fmt], 1, bool(row[4]), False, False, bool(row[3]),
                             (row, world, plan, fmt))
        assert [(r.name, r.sequence, r.qualities) for r in got.consensuses] == \
            [(r.name, r.sequence, r.qualities) for r in one.consensuses]
        assert got.refs_reports == one.refs_reports


# ------------------------------------------------------------------------------------------- qualities missing
def _noqual_file(d, fmt, dropped):
    """One contig of 30 reads with qualities and one without; `dropped`: how the filters see that read (its flag and
    MAPQ make exclude_flags 0x400, min_mapq 30 or being unmapped drop it), or "kept"."""
    import qual_cases as QC

    rng = np.random.default_rng(3)
    ref = "".join(rng.choice(list("ACGT"), 300))
    recs = [(0, 5 * k, 0, [(40 << 4) | 0], ref[5 * k:5 * k + 40], "r%d" % k, 60,
             bytes(rng.integers(2, 41, 40, dtype=np.int64).astype(np.uint8).tolist())) for k in range(30)]
    flag, mapq = {"dup": (0x400, 60), "mapq": (0, 5), "unmapped": (4, 0), "kept": (0, 60)}[dropped]
    recs.insert(10, (0, 52, flag, [(40 << 4) | 0], ref[52:92], "noq", mapq, None))
    base = d / ("noq_%s" % dropped)
    if fmt == "bam":
        path = str(base) + ".bam"
        bamio.write_bam(path, [("c", 300)], recs)
    else:
        path = str(base) + ".sam"
        QC.write_sam(path, [("c", 300)], recs)
    return path


@needs_emu
@pytest.mark.parametrize("fmt", ["bam", "sam"])
def test_reads_without_qualities(tmp_path, fmt, monkeypatch):
    """A read with QUAL `*` that exclude_flags or min_mapq drops, or that is unmapped, does not stop the vote (the
    result is the oracle's); a kept one is a ValueError naming the file and both options."""
    on_the_emulator(monkeypatch)
    for dropped, kw in (("dup", dict(exclude_flags=0x400)), ("mapq", dict(min_mapq=30)), ("unmapped", {})):
        path = _noqual_file(tmp_path, fmt, dropped)
        got = K.bam_to_consensus(path, quality_vote=True, qualities=True, **kw)
        layout = bamio.read_alignment(path, qual=True, **kw)
        p = QVL.QualityVotePiled(path, layout, 0, kw.get("min_mapq", 0), kw.get("exclude_flags", 0))
        check_vote_consensus(got, p, path, what=dropped)
        if kw:
            with pytest.raises(ValueError, match="without base qualities"):
                K.bam_to_consensus(path, quality_vote=True)
    path = _noqual_file(tmp_path, fmt, "kept")
    for kw in (dict(), dict(min_mapq=30, exclude_flags=0x400), dict(qualities=True, mask_overlaps=True)):
        with pytest.raises(ValueError, match=os.path.basename(path)) as e:
            K.bam_to_consensus(path, quality_vote=True, **kw)
        assert "without base qualities" in str(e.value) and "--quality-vote" in str(e.value)


def test_the_paired_corpus_without_filling_is_refused(tmp_path):
    """pair_combo_cases.write leaves some mates with QUAL `*`: under the vote that is the error, with mates on or
    off."""
    import pair_combo_cases as PC

    raw = PC.write(tmp_path)
    for path in (raw["bam"], raw["sam"]):
        for mates in (False, True):
            with pytest.raises(ValueError, match=os.path.basename(path)):
                K.bam_to_consensus(path, quality_vote=True, mask_overlaps=mates)


@needs_emu
def test_a_0xff_after_the_first_byte_weighs_w93(tmp_path, monkeypatch):
    """A 0xff that is not a read's first quality byte is a quality of 255, which weighs W[93]."""
    good = bytes(range(60, 90))
    recs = [(0, 10 * k, 0, [(30 << 4) | 0], "ACGT" * 7 + "AC", "r%d" % k, 60, good) for k in range(20)]
    recs[7] = recs[7][:7] + (good[:5] + b"\xff" + good[6:],)
    path = str(tmp_path / "ff.bam")
    bamio.write_bam(path, [("f", 400)], recs)
    batch = bamio.read_alignment(path, qual=True)
    got = k11w(batch, batch.qual8, "forward", E.SM_COUNT, monkeypatch)
    assert_wsum(got, wsums_of({"sums": {}}, path, batch))
    # slot 75 = read 7's base 5; reads 5 and 6 cover it too, with their own bases and qualities
    want = [0] * 4
    for k in (5, 6, 7):
        d = 75 - 10 * k
        want["ACGT".index(recs[k][4][d])] += WEIGHT[min(recs[k][7][d], 93)]
    assert [int(x) for x in got[:, 75]] == want and want[1] >= WEIGHT[93]


def test_oracle_does_not_read_the_engine():
    """The composed oracle never imports the engine nor reads a product batch's mask list or masked bases."""
    import helpers as H

    src = open(os.path.join(H.ROOT, "tests", "qvote_limit_cases.py")).read()
    oracle = src[src.index("composed oracle\n"):]
    for word in ("engine", "mask_read", "mask_off", "mask_qpos", "seq4", "n_masked", "read_alignment", "qual8",
                 "kindel_b200.kindel", "PileupRun"):
        assert word not in oracle, word
    assert "import engine" not in src and "engine." not in src and "kdl_" not in src
