"""The quality vote (`consensus --quality-vote`): the weight table, K11w + K11g-w and K2w under the kernel emulator, and
the product's bam_to_consensus with every engine call emulated, against tests/quality_vote_cases.py and
oracle/py_qvoracle.py's walk over the weights."""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np
import pytest

import emu_harness as E
import quality_vote_cases as QVC
import qual_cases as QC
import vcf_combo_cases as VC
from kindel_b200 import bamio, cli, synth
from kindel_b200 import kindel as K
from kindel_b200.quality import WEIGHT
from oracle import py_qvoracle as QV
from test_variant_qual import batch_oracle, laid_out
from test_vcf_combined import on_the_emulator

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers for the kernel emulator")
W = np.array(WEIGHT, dtype=np.int64)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """The VCF combo corpus (filters, primers, mates) with a quality on every read, and the truth set."""
    d = tmp_path_factory.mktemp("qvote")
    contigs, recs, _, rows = VC.vcf_combo_case(1)
    bam, sam = QC.write(d, contigs, QC.rewrite(recs), "qv")
    bed = d / "qv.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
    tc, trecs = QVC.records()
    tbam, tsam = QC.write(d, tc, trecs, "truth")
    return dict(bam=bam, sam=sam, bed=str(bed), rows=rows, tbam=tbam, tsam=tsam)


# ------------------------------------------------------------------------------------------------ helpers
def emu_weights(batch, qual8, schedule="forward"):
    """kdl_quality_weights (K0 + K11w + K11g-w) on the emulator: wsum uint64 [4, n], preset to garbage."""
    lib = E.load()
    E.set_schedule(schedule, 5)
    lib.emu_set_sm_count(E.SM_COUNT)
    st, keep = E._host_batch(batch)
    n = int(batch.n_slots)
    wsum = np.full((4, n), 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)
    q8 = np.ascontiguousarray(qual8 if qual8.size else np.zeros(8, np.uint8), dtype=np.uint8)
    rc = lib.kdl_quality_weights(C.byref(st), q8.ctypes.data, wsum.ctypes.data, n, None)
    assert rc == 0, lib.kdl_status_string(rc)
    del keep
    return wsum


def emu_vote_quality(counts, wsum, min_depth=1, with_qual=True):
    """kdl_vote_quality (K2w) on the emulator: (calls, qual) uint8 [n], preset to garbage."""
    lib = E.load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    wsum = np.ascontiguousarray(wsum, dtype=np.uint64)
    n = counts.shape[1]
    calls = np.full(n, 0xEE, dtype=np.uint8)
    qual = np.full(n, 0xEE, dtype=np.uint8)
    rc = lib.kdl_vote_quality(counts.ctypes.data, wsum.ctypes.data, n, int(math.ceil(min_depth)), calls.ctypes.data,
                              qual.ctypes.data if with_qual else None, None)
    assert rc == 0, lib.kdl_status_string(rc)
    return calls, qual


def weight_oracle(batch, qual):
    """py_qvoracle's walk with every quality replaced by its weight: wsum int64 [4, n_slots]."""
    return batch_oracle(batch, W[np.minimum(np.asarray(qual, dtype=np.int64), 93)])[0]


def weight_sums(monkeypatch, path, *args, **kw):
    """py_qvoracle.quality_sums (its records, filters and masks) with the walk adding weights: {contig: wsum [4][L]}."""
    walk = QV.walk
    monkeypatch.setattr(QV, "walk", lambda L, rec, qual, masked, qsum, emass: walk(
        L, rec, [WEIGHT[min(q, 93)] for q in qual], masked, qsum, emass))
    try:
        return {nm: (v[0], v[1]) for nm, v in QV.quality_sums(path, *args, **kw).items()}
    finally:
        monkeypatch.setattr(QV, "walk", walk)


def assert_wsum(got, want, what=""):
    assert [[int(x) for x in row] for row in got.tolist()] == [[int(x) for x in row] for row in want.tolist()], what


# ------------------------------------------------------------------------------------------------ the table
def test_weight_table_is_the_exact_rounding():
    from decimal import Decimal, getcontext

    getcontext().prec = 80
    for q in range(94):
        e = min(Decimal(10) ** (Decimal(-q) / 10), Decimal(3) / 4)
        x = Decimal(2) ** 16 * 10 * (3 * (1 - e) / e).log10()
        assert abs(Decimal(WEIGHT[q]) - x) <= Decimal("0.5"), q
        assert q < 2 or abs(abs(x - int(x)) - Decimal("0.5")) > Decimal("1e-6"), q  # no tie to round
    assert WEIGHT[0] == WEIGHT[1] == 0
    assert [WEIGHT[q] for q in (2, 10, 20, 30, 40, 93)] == [160037, 938059, 1620546, 2278481, 2934098, 6407534]
    assert 256 * WEIGHT[93] < 2 ** 32  # a chunk's uint32 partial sum is exact
    src = open(os.path.join(E.ROOT, "kindel_b200", "csrc", "quality.cu")).read()
    body = src[src.index("kQualWeight[kEpsMax + 1] = {"):]
    body = body[body.index("{") + 1:body.index("};")]
    assert tuple(int(v.strip().rstrip("u")) for v in body.replace("\n", " ").split(",") if v.strip()) == WEIGHT


# ------------------------------------------------------------------------------------------------ K11w + K11g-w
@needs_emu
@pytest.mark.parametrize("schedule", ["forward", "random"])
def test_k11w_equals_the_oracle_on_the_corpus(corpus, monkeypatch, schedule):
    for kw in (dict(), dict(min_base_quality=20, min_mapq=30, exclude_flags=0x500)):
        batch = bamio.read_alignment(corpus["bam"], qual=True, **kw)
        want = laid_out(batch, weight_sums(monkeypatch, corpus["bam"], kw.get("min_base_quality", 0),
                                           kw.get("min_mapq", 0), kw.get("exclude_flags", 0)))[0]
        assert_wsum(emu_weights(batch, batch.qual8, schedule), want, str(kw))


@needs_emu
@pytest.mark.parametrize("schedule", ["forward", "reverse"])
def test_k11w_on_complex_and_hard_reads_sorted_and_shuffled(schedule):
    for seed in (1, 2):
        batch = synth.complex_reads(seed, 3000, 30)
        assert batch.n_hard > 0 and batch.n_complex > batch.n_hard and batch.reads_sorted
        qual = synth.qualities(seed, batch.seq_len)
        want = weight_oracle(batch, qual)
        assert_wsum(emu_weights(batch, bamio.qual_layout(batch, qual), schedule), want, "sorted %d" % seed)
        perm = np.random.default_rng(seed).permutation(batch.n_reads)
        ub = bamio.select_reads(batch, perm)
        at = np.concatenate(([0], np.cumsum(batch.seq_len.astype(np.int64))))
        uq = np.concatenate([qual[at[r]:at[r + 1]] for r in perm])
        assert_wsum(emu_weights(ub, bamio.qual_layout(ub, uq), schedule), want, "shuffled %d" % seed)


@needs_emu
def test_k11w_across_tile_edges_with_a_deep_tile_of_q93(tmp_path):
    """Simple reads around tile edges, more than 1024 of them in the first tile (several chunks), every quality
    0..93 and a column of Q93 bases deep enough that a chunk's partial sums of all four quarters pass 2^32."""
    rng = np.random.default_rng(5)
    rows = []
    for c, L in enumerate((1536, 1100)):
        for _ in range(1500 if c == 0 else 300):
            n = int(rng.integers(2, 300))
            edge = int(rng.choice([0, 512, 1024]))
            rows.append((c, int(np.clip(edge + rng.integers(-n - 2, 10), 0, L - n)), n, None))
    rows += [(0, 100, 50, 93)] * 800  # 800 * W[93] > 2^32 at slots 100..149
    rows.sort(key=lambda r: r[:3])
    contigs = [("t0", 1536), ("t1", 1100)]
    recs = [(c, pos, 0, [(n << 4) | 0], "".join(rng.choice(list("ACGTN"), n)) if q is None else "G" * n, "x", 60,
             bytes(rng.integers(0, 94, n, dtype=np.uint8).tolist()) if q is None else bytes([q] * n))
            for c, pos, n, q in rows]
    path = str(tmp_path / "edges.sam")
    QC.write_sam(path, contigs, recs)
    batch = bamio.read_alignment(path, qual=True)
    assert batch.n_complex == 0 and batch.reads_sorted
    got = emu_weights(batch, batch.qual8)
    want = weight_oracle(batch, np.frombuffer(b"".join(r[7] for r in recs), dtype=np.uint8))
    assert_wsum(got, want)
    assert int(got[2, 120]) > 2 ** 32


@needs_emu
def test_constant_quality_gives_w_times_the_pileup_columns_and_the_count_vote():
    """wsum[k] == n_k * W[q]; the quality vote then equals kdl_vote wherever N is below the largest base count."""
    batch = synth.complex_reads(3, 3000, 30)
    counts, _ = E.pileup_pipeline(batch)
    for q in (2, 20, 41, 93):
        wsum = emu_weights(batch, bamio.qual_layout(batch, np.full(int(batch.seq_len.sum()), q, np.uint8)))
        np.testing.assert_array_equal(wsum.astype(object), WEIGHT[q] * counts[0:4].astype(object))
        for md in (1, 3):
            calls, _ = emu_vote_quality(counts, wsum, md)
            base = E.vote(counts, md)
            np.testing.assert_array_equal(calls >> 4, base >> 4)
            live = counts[4] < counts[0:4].max(axis=0)
            np.testing.assert_array_equal(calls[live], base[live], err_msg="q=%d md=%d" % (q, md))


# ------------------------------------------------------------------------------------------------ K2w
def planted_table(rng, n):
    counts = np.zeros((19, n), dtype=np.int32)
    counts[0:5] = rng.integers(0, 6, (5, n))
    counts[5] = rng.integers(0, 4, n) * (rng.random(n) < 0.2)
    counts[6] = rng.integers(0, 6, n) * (rng.random(n) < 0.2)
    counts[:, n - 8:] = 0  # the slot behind the contig and the padding
    wsum = rng.integers(0, 1 << 40, (4, n), dtype=np.int64).astype(np.uint64)
    kind = rng.integers(0, 6, n)
    wsum[:, kind == 0] = 0                                  # no weight
    top = wsum.max(axis=0)
    tie = kind == 1
    wsum[1, tie] = top[tie]                                 # two bases share the largest sum
    wsum[3, tie] = top[tie]
    near = kind == 2
    wsum[0, near] = wsum[2, near] + rng.integers(0, 1 << 18, int(near.sum())).astype(np.uint64)
    counts[4, kind == 3] = 50                               # an N count above every base
    wsum[:, kind == 4] = rng.integers(0, 1 << 20, (4, int((kind == 4).sum()))).astype(np.uint64)
    wsum[2, kind == 5] = np.uint64(3) << np.uint64(60)      # far above 2^32
    wsum[:, n - 8:] = 0
    return counts, wsum


@needs_emu
def test_k2w_equals_the_restatement_on_planted_tables():
    rng = np.random.default_rng(9)
    for n, md in ((4096, 1), (1024, 3), (8, 1)):
        counts, wsum = planted_table(rng, n)
        want = QVC.restated_vote(counts, wsum.astype(object), md)
        got = emu_vote_quality(counts, wsum, md)
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])
        assert not (got[0] & 0x80).any()
        np.testing.assert_array_equal(got[0] >> 4, E.vote(counts, md) >> 4)  # the change bits are kdl_vote's
        np.testing.assert_array_equal(emu_vote_quality(counts, wsum, md, with_qual=False)[0], got[0])


# ------------------------------------------------------------------------------------------------ the product
@needs_emu
@pytest.mark.parametrize("sam", [False, True])
@pytest.mark.parametrize("bq,trim,upper,realign,fastq", [
    (0, False, False, False, True), (10, True, False, True, True), (0, True, True, False, False),
    (10, False, True, False, False), (0, False, False, True, False), (10, False, False, False, True)])
def test_truth_set_through_bam_to_consensus(corpus, monkeypatch, sam, bq, trim, upper, realign, fastq):
    on_the_emulator(monkeypatch)
    path = corpus["tsam" if sam else "tbam"]
    count, text, quals, sites, n_sites = QVC.expected(bq)
    res = K.bam_to_consensus(path, realign=realign, trim_ends=trim, uppercase=upper, min_base_quality=bq,
                             qualities=fastq, quality_vote=True)
    rec = res.consensuses[0]
    want, qtext = text, "".join(chr(33 + q) for q in quals)
    if trim:
        lo, hi = len(want) - len(want.lstrip("N")), len(want.rstrip("N"))
        want, qtext = want[lo:hi], qtext[lo:hi]
    assert rec.sequence == want
    assert rec.qualities == (qtext if fastq else None)
    report = res.refs_reports["v"].split("\n")
    assert "- quality_vote: True" in report
    at = report.index("- ambiguous sites: %s" % ", ".join(map(str, n_sites)))
    assert report[at + 1] == "- quality-vote sites: %s" % ", ".join(map(str, sites))
    # off: the count vote, and no extra line
    off = K.bam_to_consensus(path, realign=realign, trim_ends=trim, uppercase=upper, min_base_quality=bq)
    cw = count.strip("N") if trim else count
    assert off.consensuses[0].sequence == cw
    assert not any("quality" in x for x in off.refs_reports["v"].split("\n") if "min_base_quality" not in x)


def test_the_truth_set_holds_the_issue_table():
    count, text, quals, _, _ = QVC.expected()
    for p, c, v, q in ((4, "A", "G", 60), (12, "A", "G", 6), (20, "N", "C", 5), (28, "A", "N", 0),
                       (36, "N", "A", 60), (44, "T", "T", 60), (52, "N", "N", 0)):
        assert (count[p], text[p], quals[p]) == (c, v, q), p


@needs_emu
@pytest.mark.parametrize("primers,mates,bq", [(False, False, 0), (True, False, 20), (False, True, 0),
                                              (True, True, 20)])
def test_vote_with_primers_and_mates_equals_the_restatement(corpus, monkeypatch, primers, mates, bq):
    """K11w over the masked batch (primer bases, mate overlaps and low-quality bases are N nibbles), then K2w, equal
    the restated vote over the pileup's table and py_qvoracle's masked weight sums."""
    rows = corpus["rows"] if primers else None
    want = weight_sums(monkeypatch, corpus["bam"], bq, 0, 0, rows, mates)
    on_the_emulator(monkeypatch)
    run, _ = K.pileup_run(corpus["bam"], min_base_quality=bq, primers=corpus["bed"] if primers else None,
                          mask_overlaps=mates, qual=True)
    wsum = laid_out(run.batch, want)[0]
    assert_wsum(run.quality_weights().numpy().view(np.uint64), wsum)
    calls = run.vote(1, quality=True)
    rc, rq = QVC.restated_vote(run.host_counts, wsum.astype(object), 1)
    np.testing.assert_array_equal(calls, rc)
    np.testing.assert_array_equal(run.vote_qual.numpy(), rq)


@needs_emu
def test_two_rank_host_tables_equal_one_rank(corpus, monkeypatch):
    """A run from host tables (as a multi-GPU job leaves it) votes from device_tables() and equals the one-device
    run, the REPORT included."""
    on_the_emulator(monkeypatch)
    kw = dict(min_base_quality=20, primers=corpus["bed"], mask_overlaps=True, qualities=True, quality_vote=True)
    one = K.bam_to_consensus(corpus["bam"], **kw)
    real = K.pileup_run

    def sharded(path, devices=None, min_depth=1, *filters, **opts):
        run, _ = real(path, 1, min_depth, *filters, **opts)
        host = K.PileupRun.from_host_tables(run.batch, run.host_counts, run.host_derived, run.events.numpy(),
                                            primers=run.primers, mask_overlaps=run.mask_overlaps,
                                            dropped_events=K.engine.dropped_event_rows(run.dbatch),
                                            overlap_stats=run.overlap_stats)
        return host, np.zeros(run.batch.n_slots, np.uint8)  # the ranks' majority calls: discarded

    monkeypatch.setattr(K, "pileup_run", sharded)
    two = K.bam_to_consensus(corpus["bam"], **kw)
    assert [(r.name, r.sequence, r.qualities) for r in two.consensuses] == \
        [(r.name, r.sequence, r.qualities) for r in one.consensuses]
    assert two.refs_reports == one.refs_reports


# ------------------------------------------------------------------------------------------------ errors and CLI
def test_errors(corpus, tmp_path):
    with pytest.raises(ValueError, match="iupac_threshold"):
        K.bam_to_consensus(corpus["tbam"], iupac_threshold=0.5, quality_vote=True)
    contigs, recs, _, _ = VC.vcf_combo_case(1)
    bam, sam = QC.write(tmp_path, contigs, recs, "noq")
    for path in (bam, sam):
        with pytest.raises(ValueError, match=os.path.basename(path)):
            K.bam_to_consensus(path, quality_vote=True)
    run = K.PileupRun.from_host_tables(bamio.read_alignment(bam), np.zeros((19, 4), np.int32),
                                       np.zeros((5, 4), np.int32), np.zeros((0, 4), np.int32))
    with pytest.raises(ValueError, match="quality_vote"):
        K.consensus_from_run(run, np.zeros(4, np.uint8), bam, quality_vote=True)


def test_cli_refuses_quality_vote_with_iupac(corpus, capsys):
    with pytest.raises(SystemExit) as e:
        cli.main(["consensus", "--quality-vote", "--iupac-threshold", "0.5", corpus["tbam"]])
    assert e.value.code == 2
    assert "--quality-vote cannot be combined" in capsys.readouterr().err


@needs_emu
def test_cli_quality_vote(corpus, monkeypatch, capsys):
    on_the_emulator(monkeypatch)
    _, text, quals, _, _ = QVC.expected()
    assert cli.main(["consensus", "--quality-vote", "--fastq", corpus["tbam"]]) in (0, None)
    out = capsys.readouterr()
    assert out.out == "@v_cns\n%s\n+\n%s\n" % (text, "".join(chr(33 + q) for q in quals))
    assert "- quality_vote: True" in out.err
    assert cli.main(["consensus", "--quality-vote", corpus["tsam"]]) in (0, None)
    assert capsys.readouterr().out == ">v_cns\n%s\n" % text
