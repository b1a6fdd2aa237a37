"""Duplicate removal (`--dedup`, an extension) on the GPU: K10p + K14k + the sort + K14s through the real library
against the oracle (oracle/py_doracle.py) on the golden inputs, the truth set and synthetic pairs; the metamorphic rule
-- every command with `--dedup` on a file equals the same command without it on a file that holds only the oracle's
kept records, apart from the lines naming the option and the path; `--dedup` with `--normalise`, `--primers` and
`--mask-overlaps`; a duplicate-free file; `amplicons --dedup`; and two GPUs against one."""
import os
import subprocess
import sys

import numpy as np
import pytest

import amplicon_cases as AC
import dedup_cases as D
from kindel_b200 import bamio, engine, synth
from kindel_b200 import kindel as K
from oracle import py_doracle as DO

pytestmark = pytest.mark.gpu

GOLDEN = ["bact_tiny.bam", "bwa_1_1.bam", "mm2_multi.bam", "ext_2_bc63.sam"]
MARKS = ("- bam_path:", "- duplicates:", "##kindelDedup")


def _device_keep(path, **decode):
    b = bamio.read_alignment(path, strand=True, mates=True, dup=True, **decode)
    keep, stats = engine.dedup(engine.upload(b))
    return b, keep.cpu().numpy(), stats


@pytest.mark.parametrize("name", GOLDEN)
def test_keep_bytes_on_golden_inputs(name):
    path = os.path.join(os.path.dirname(__file__), "golden", "inputs", name)
    for filters in (dict(), dict(min_mapq=20, exclude_flags=0x400)):
        b, keep, stats = _device_keep(path, **filters)
        want, totals, gone = DO.keep_by_record(path, b.contig_names, filters.get("min_mapq", 0),
                                               filters.get("exclude_flags", 0))
        assert keep.tolist() == want.tolist() and stats == totals
        run, _ = K.pileup_run(path, dedup=True, **filters)
        assert run.deduplicated == (totals[0], totals[1], b.n_reads - len(gone), b.n_reads)
        assert run.batch.n_reads == b.n_reads - len(gone)
        assert run.batch.reverse is None and run.batch.mates is None and run.batch.dup_score is None


def test_keep_bytes_on_the_truth_set(tmp_path):
    p = tmp_path / "t.sam"
    p.write_text(D.sam_text())
    b, keep, stats = _device_keep(str(p))
    assert keep.tolist() == D.engine_order(D.KEEP) and stats == D.TOTALS


@pytest.mark.parametrize("amplicons", [False, True])
def test_keep_bytes_on_synthetic_pairs(amplicons):
    rows = synth.tiled_scheme(5, ["ctg0"], [200_000]) if amplicons else None
    b, flag, frag, _ = synth.dup_pairs(5, 200_000, 100, amplicons=rows)
    keep, stats = engine.dedup(engine.upload(b))
    mate = _mates_by_fragment(b, frag)
    u, alone = _ends(b)
    want, totals = DO.keep_vectorised(np.zeros(b.n_reads), u, b.reverse, alone, b.dup_score, mate)
    assert keep.cpu().numpy().tolist() == want.tolist() and stats == totals and totals[0] > 1000


def _mates_by_fragment(b, frag):
    """The oracle's pairing of dup_pairs' reads: the two reads of each fragment, R2 -> R1, neither KDL_HARD."""
    order = np.argsort(frag, kind="stable")
    a, c = order[0::2], order[1::2]
    r1 = np.where(b.pair_role[a] == 1, a, c)
    r2 = np.where(b.pair_role[a] == 1, c, a)
    hard = (b.l_seq.view(np.uint32) & 0x40000000) != 0
    ok = ~hard[r1] & ~hard[r2]
    mate = np.full(b.n_reads, -1, dtype=np.int64)
    mate[r2[ok]] = r1[ok]
    return mate


def _ends(b):
    """(u, left alone) of every read of a batch of one- and two-op reads (dup_pairs'), vectorised."""
    co = b.cig_off.astype(np.int64)
    first, last = b.cigar[co[:-1]], b.cigar[co[1:] - 1]
    lead = np.where((first & 15) == 4, first >> 4, 0).astype(np.int64)
    trail = np.where(((last & 15) == 4) & (co[1:] - co[:-1] > 1), last >> 4, 0).astype(np.int64)
    span = b.seq_len.astype(np.int64) - lead - trail
    start = b.ref_start.astype(np.int64)
    u = np.where(b.reverse == 1, start + span - 1 + trail, start - lead)
    return u, b.dup_score < 0


def _pair_records(seed, contig_len=6_000, depth=60, amplicons=False):
    """(contigs, write_bam records with QNAME, MAPQ, qualities, RNEXT and PNEXT, scheme rows or None) of synthetic
    pairs with planted duplicates, a twentieth of the records left out (their mates are singles)."""
    rows = synth.tiled_scheme(seed, ["ctg0"], [contig_len]) if amplicons else None
    batch, flag, frag, qual = synth.dup_pairs(seed, contig_len, depth, dup_frac=0.4, amplicons=rows, want_qual=True)
    contigs, recs = synth.paired_records(batch, flag, frag)
    at = np.concatenate(([0], np.cumsum(batch.seq_len.astype(np.int64))))
    gone = np.random.default_rng(seed).random(len(recs)) < 0.05
    out = [r[:7] + (qual[at[k]:at[k + 1]].tobytes(),) + tuple(r[8:]) for k, r in enumerate(recs) if not gone[k]]
    return contigs, out, None if rows is None else AC.tiled_rows(rows)


def _files(tmp_path, seed, amplicons=False):
    """(full BAM, BAM of the oracle's kept records, scheme BED or None, reference FASTA, removed file indices)."""
    contigs, recs, rows = _pair_records(seed, amplicons=amplicons)
    full, sub = tmp_path / ("full%d.bam" % seed), tmp_path / ("kept%d.bam" % seed)
    bamio.write_bam(str(full), contigs, recs)
    _, _, gone = DO.keep_by_record(str(full), [c for c, _ in contigs])
    bamio.write_bam(str(sub), contigs, [r for k, r in enumerate(recs) if k not in gone])
    bed = None
    if rows is not None:
        bed = tmp_path / "scheme.bed"
        bed.write_text(AC.bed_text(rows))
        bed = str(bed)
    ref = K.bam_to_consensus(str(full), uppercase=True).consensuses[0].sequence.replace("N", "A")
    fa = tmp_path / "ref.fa"
    fa.write_text(">%s\n%s\n" % (contigs[0][0], ref))
    return str(full), str(sub), bed, str(fa), gone


def _without(text, *marks):
    return [ln for ln in text.splitlines() if not any(m in ln for m in marks)]


def _same_consensus(a, b):
    assert [(r.name, r.sequence, r.qualities) for r in a.consensuses] == \
        [(r.name, r.sequence, r.qualities) for r in b.consensuses]
    assert a.refs_changes == b.refs_changes
    for k in a.refs_reports:
        assert _without(a.refs_reports[k], *MARKS) == _without(b.refs_reports[k], *MARKS)


def _every_output(full, sub, n_gone, n_reads, **opts):
    for kw in (dict(), dict(qualities=True), dict(iupac_threshold=0.6), dict(quality_vote=True, qualities=True),
               dict(realign=True)):
        on = K.bam_to_consensus(full, dedup=True, **opts, **kw)
        off = K.bam_to_consensus(sub, **opts, **kw)
        _same_consensus(on, off)
        report = next(iter(on.refs_reports.values()))
        line = [ln for ln in report.splitlines() if ln.startswith("- duplicates:")]
        assert len(line) == 1 and line[0].endswith("%d of %d reads kept" % (n_reads - n_gone, n_reads))
    assert K.weights(full, dedup=True, **opts).equals(K.weights(sub, **opts))
    assert K.features(full, dedup=True, **opts).equals(K.features(sub, **opts))
    assert K.variants(full, dedup=True, **opts).equals(K.variants(sub, **opts))


def test_every_output_equals_the_file_of_the_kept_records(tmp_path):
    full, sub, _, fa, gone = _files(tmp_path, 7)
    n = bamio.read_alignment(full).n_reads
    assert len(gone) > 100
    _every_output(full, sub, len(gone), n)
    for kw in (dict(), dict(reference=fa), dict(strand=True), dict(qual=True), dict(reference=fa, strand=True, qual=True)):
        on = K.variants_vcf(full, dedup=True, **kw)
        off = K.variants_vcf(sub, **kw)
        assert "##kindelDedup=fragment ends, base-quality score" in on.splitlines()
        assert _without(on, "##kindelDedup") == off.splitlines()
    cohort_on = K.variants_vcf([full, full], dedup=True, samples=["a", "b"])
    cohort_off = K.variants_vcf([sub, sub], samples=["a", "b"])
    assert _without(cohort_on, "##kindelDedup") == cohort_off.splitlines()


def test_dedup_with_normalise_primers_and_mate_overlaps(tmp_path):
    full, sub, bed, fa, gone = _files(tmp_path, 9, amplicons=True)
    n = bamio.read_alignment(full).n_reads
    assert len(gone) > 100
    _every_output(full, sub, len(gone), n, primers=bed, mask_overlaps=True)
    for cap in (5, 40):
        on = K.bam_to_consensus(full, dedup=True, primers=bed, mask_overlaps=True, normalise=cap, qualities=True)
        off = K.bam_to_consensus(sub, primers=bed, mask_overlaps=True, normalise=cap, qualities=True)
        _same_consensus(on, off)
        lines = next(iter(on.refs_reports.values())).splitlines()
        k = [i for i, ln in enumerate(lines) if ln.startswith("- primers:")][0]
        assert lines[k + 1].startswith("- duplicates:") and lines[k + 2].startswith("- normalise:")
        on = K.variants_vcf(full, dedup=True, primers=bed, mask_overlaps=True, normalise=cap, reference=fa,
                            strand=True, qual=True)
        off = K.variants_vcf(sub, primers=bed, mask_overlaps=True, normalise=cap, reference=fa, strand=True, qual=True)
        assert _without(on, "##kindelDedup") == off.splitlines()
        head = on.splitlines()
        assert head.index("##kindelDedup=fragment ends, base-quality score") == head.index("##kindelNormalise=%d" % cap) - 1


def test_cli_equals_the_file_of_the_kept_records(tmp_path):
    full, sub, _, fa, gone = _files(tmp_path, 11)
    run = lambda *a: subprocess.run([sys.executable, "-m", "kindel_b200", *a], capture_output=True, text=True,  # noqa
                                    check=True)
    for cmd in (["consensus", "--fastq"], ["variants", "--vcf", "--reference", fa, "--strand", "--qual"]):
        on = run(*cmd, full, "--dedup")
        off = run(*cmd, sub)
        assert _without(on.stdout, "##kindelDedup") == off.stdout.splitlines()
        assert _without(on.stderr, *MARKS) == _without(off.stderr, *MARKS)
    assert "single reads removed" in run("consensus", full, "--dedup").stderr


def test_a_duplicate_free_file_changes_nothing_but_the_lines(tmp_path):
    _, sub, _, fa, _ = _files(tmp_path, 13)
    for kw in (dict(qualities=True), dict(quality_vote=True, qualities=True), dict(mask_overlaps=True)):
        on, off = K.bam_to_consensus(sub, dedup=True, **kw), K.bam_to_consensus(sub, **kw)
        assert [(r.sequence, r.qualities) for r in on.consensuses] == [(r.sequence, r.qualities) for r in off.consensuses]
        for k in on.refs_reports:
            assert _without(on.refs_reports[k], "- duplicates:") == off.refs_reports[k].splitlines()
            n = bamio.read_alignment(sub).n_reads
            assert "- duplicates: 0 pairs and 0 single reads removed, %d of %d reads kept" % (n, n) in on.refs_reports[k]
    assert K.weights(sub, dedup=True).to_csv() == K.weights(sub).to_csv()
    on = K.variants_vcf(sub, dedup=True, reference=fa, strand=True, qual=True)
    assert _without(on, "##kindelDedup") == K.variants_vcf(sub, reference=fa, strand=True, qual=True).splitlines()


def test_amplicons_describe_the_kept_reads(tmp_path):
    full, sub, bed, _, gone = _files(tmp_path, 17, amplicons=True)
    on = K.amplicons(full, bed, 5, dedup=True)
    off = K.amplicons(sub, bed, 5)
    cols = [c for c in K.AMPLICON_COLUMNS if c != "sample"]
    assert on[cols].equals(off[cols])
    name = on["sample"].iloc[0]
    assert on.attrs["duplicates"] == {name: len(gone)} and "duplicates" not in off.attrs
    res = subprocess.run([sys.executable, "-m", "kindel_b200", "amplicons", "--primers", bed, "--dedup",
                          "--min-depth", "5", full], capture_output=True, text=True, check=True)
    assert res.stderr.strip().endswith("; %d duplicate reads removed" % len(gone))


def test_two_gpus_equal_one(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    batch, flag, frag, qual = synth.dup_pairs(6, 200_000, 50, clip_frac=0.0, want_qual=True)
    path = tmp_path / "a.bam"
    synth.write_simple_bam(str(path), batch, names=synth.pair_names(frag), flag=flag, next_pos=batch.mate_start,
                           qual=qual)
    for kw in (dict(), dict(mask_overlaps=True)):
        one = K.bam_to_consensus(str(path), devices=1, dedup=True, **kw)
        two = K.bam_to_consensus(str(path), devices=2, dedup=True, **kw)
        assert [r.sequence for r in one.consensuses] == [r.sequence for r in two.consensuses]
        assert one.refs_reports == two.refs_reports
    assert K.variants_vcf(str(path), devices=1, dedup=True) == K.variants_vcf(str(path), devices=2, dedup=True)
