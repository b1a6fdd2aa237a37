"""Depth normalisation (`--normalise N`, an extension) on the GPU: K12 + K13's keep bytes through the real library
against the per-record oracle (oracle/py_noracle.py) on the golden inputs and on synthetic amplicon reads and pairs;
the metamorphic rule -- every command with `--normalise N` on a file equals the same command without it on a file that
holds only the oracle's kept records, apart from the lines naming the option and the path; the idempotent case
byte for byte; `amplicons --normalise`; and two GPUs against one."""
import os
import subprocess
import sys

import numpy as np
import pytest

import amplicon_cases as AC
from kindel_b200 import bamio, engine, synth
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from oracle import py_aoracle as AO
from oracle import py_noracle as NO

pytestmark = pytest.mark.gpu

GOLDEN = ["bwa_1_1.bam", "bwa_4_1.bam", "ext_2_bc63.sam"]


def _device_keep(path, bed, cap, **decode):
    b = bamio.read_alignment(path, strand=True, **decode)
    scheme = P.load_scheme(bed)
    arr = P.amplicon_arrays(scheme, b.contig_names, b.contig_len)
    db = engine.upload(b)
    label = engine.assign_amplicons(db, arr)
    import torch

    keep, total, dropped = engine.normalise(label, torch.from_numpy(b.reverse).to(db.device), arr.n_amplicons, cap)
    return b, label.cpu().numpy(), keep.cpu().numpy(), total.cpu().numpy(), int(dropped.item())


@pytest.mark.parametrize("name", GOLDEN)
def test_keep_bytes_on_golden_inputs(tmp_path, name):
    path = os.path.join(os.path.dirname(__file__), "golden", "inputs", name)
    b0 = bamio.read_alignment(path)
    rng = np.random.default_rng(len(name))
    contigs = list(zip(b0.contig_names, b0.contig_len.tolist()))
    span = [min(n, 100_000) for n in b0.contig_len.tolist()]
    rows = AC.tiled_rows(synth.tiled_scheme(3, b0.contig_names, span)) + AC.random_scheme_rows(rng, contigs, 12)
    bed = tmp_path / "scheme.bed"
    bed.write_text(AC.bed_text(rows))
    for cap in (1, 3, 50):
        b, label, keep, total, dropped = _device_keep(path, str(bed), cap)
        if b.n_reads < 20_000:
            want, gone = NO.keep_by_record(path, b.contig_names, rows, cap)
            assert len(gone) == dropped
        else:
            want = NO.keep_vectorised(AO.labels_of_batch(b, rows), b.reverse, cap)
        assert keep.tolist() == want.tolist() and dropped == int((want == 0).sum())
        assert total.tolist() == NO.totals(label, b.reverse, total.shape[0] // 2).tolist()
        run, _ = K.pileup_run(path, primers=str(bed), normalise=cap)
        assert run.normalised == (cap, dropped, b.n_reads - dropped) and run.batch.n_reads == b.n_reads - dropped
        assert run.batch.reverse is None  # (strand was not asked for)


def _amplicon_records(seed, contig_len=6_000, depth=60, pairs=False):
    """(contigs, write_bam records with QNAME, MAPQ and qualities, scheme rows) of synthetic amplicon reads with
    seeded strands, or amplicon read pairs."""
    if pairs:
        batch, flag, frag, trows = synth.amplicon_pairs(seed, contig_len, depth)
        contigs, recs = synth.paired_records(batch, flag, frag)
    else:
        batch, trows = synth.amplicon_reads(seed, contig_len, depth)
        contigs, recs = synth.to_records(synth.with_strands(batch, seed))
        recs = [r + ("r%d" % k, 60) for k, r in enumerate(recs)]
    qual = synth.qualities(seed, [len(r[4]) for r in recs])
    at = np.concatenate(([0], np.cumsum([len(r[4]) for r in recs])))
    out = [r[:7] + (qual[at[k]:at[k + 1]].tobytes(),) + tuple(r[8:]) for k, r in enumerate(recs)]
    return contigs, out, AC.tiled_rows(trows)


def _pair(tmp_path, seed, cap, pairs=False):
    """(full BAM, BAM of the oracle's kept records, scheme BED, reference FASTA, dropped) of one synthetic case."""
    contigs, recs, rows = _amplicon_records(seed, pairs=pairs)
    full, sub = tmp_path / ("full%d.bam" % seed), tmp_path / ("kept%d.bam" % seed)
    bamio.write_bam(str(full), contigs, recs)
    bed = tmp_path / "scheme.bed"
    bed.write_text(AC.bed_text(rows))
    _, dropped = NO.keep_by_record(str(full), [c for c, _ in contigs], rows, cap)
    bamio.write_bam(str(sub), contigs, [r for k, r in enumerate(recs) if k not in dropped])
    ref = K.bam_to_consensus(str(full), uppercase=True).consensuses[0].sequence.replace("N", "A")
    fa = tmp_path / "ref.fa"
    fa.write_text(">%s\n%s\n" % (contigs[0][0], ref))
    return str(full), str(sub), str(bed), str(fa), dropped


def _without(text, *marks):
    return [ln for ln in text.splitlines() if not any(m in ln for m in marks)]


def _same_consensus(a, b):
    assert [(r.name, r.sequence, r.qualities) for r in a.consensuses] == \
        [(r.name, r.sequence, r.qualities) for r in b.consensuses]
    assert a.refs_changes == b.refs_changes
    for k in a.refs_reports:
        assert _without(a.refs_reports[k], "- bam_path:", "- normalise:") == \
            _without(b.refs_reports[k], "- bam_path:", "- normalise:")


@pytest.mark.parametrize("pairs", [False, True])
def test_every_output_equals_the_file_of_the_kept_records(tmp_path, pairs):
    cap = 20
    full, sub, bed, fa, dropped = _pair(tmp_path, 7 + pairs, cap, pairs)
    assert len(dropped) > 100
    overlaps = dict(mask_overlaps=True) if pairs else {}
    opts = dict(primers=bed, **overlaps)
    for kw in (dict(), dict(qualities=True), dict(iupac_threshold=0.6), dict(quality_vote=True, qualities=True),
               dict(realign=True)):
        on = K.bam_to_consensus(full, normalise=cap, **opts, **kw)
        off = K.bam_to_consensus(sub, **opts, **kw)
        _same_consensus(on, off)
        report = next(iter(on.refs_reports.values()))
        line = [ln for ln in report.splitlines() if ln.startswith("- normalise:")]
        assert line == ["- normalise: %d per amplicon and strand, %d of %d reads dropped"
                        % (cap, len(dropped), bamio.read_alignment(full).n_reads)]
    assert K.weights(full, normalise=cap, **opts).equals(K.weights(sub, **opts))
    assert K.features(full, normalise=cap, **opts).equals(K.features(sub, **opts))
    assert K.variants(full, normalise=cap, **opts).equals(K.variants(sub, **opts))
    for kw in (dict(), dict(reference=fa), dict(strand=True), dict(qual=True), dict(reference=fa, strand=True, qual=True)):
        on = K.variants_vcf(full, normalise=cap, **opts, **kw)
        off = K.variants_vcf(sub, **opts, **kw)
        assert "##kindelNormalise=%d" % cap in on.splitlines()
        assert _without(on, "##kindelNormalise") == off.splitlines()
    cohort_on = K.variants_vcf([full, full], normalise=cap, samples=["a", "b"], **opts)
    cohort_off = K.variants_vcf([sub, sub], samples=["a", "b"], **opts)
    assert _without(cohort_on, "##kindelNormalise") == cohort_off.splitlines()


def test_cli_equals_the_file_of_the_kept_records(tmp_path):
    cap = 15
    full, sub, bed, fa, _ = _pair(tmp_path, 11, cap)
    run = lambda *a: subprocess.run([sys.executable, "-m", "kindel_b200", *a], capture_output=True, text=True,  # noqa
                                    check=True)
    for cmd in (["consensus", "--fastq"], ["variants", "--vcf", "--reference", fa, "--strand", "--qual"]):
        on = run(*cmd, full, "--primers", bed, "--normalise", str(cap))
        off = run(*cmd, sub, "--primers", bed)
        assert _without(on.stdout, "##kindelNormalise") == off.stdout.splitlines()
        assert _without(on.stderr, "- bam_path:", "- normalise:") == _without(off.stderr, "- bam_path:")


def test_a_cap_above_every_group_changes_nothing(tmp_path):
    contigs, recs, rows = _amplicon_records(13, pairs=True)
    full = tmp_path / "full.bam"
    bamio.write_bam(str(full), contigs, recs)
    bed = tmp_path / "scheme.bed"
    bed.write_text(AC.bed_text(rows))
    full, bed = str(full), str(bed)
    big = (1 << 31) - 1
    opts = dict(primers=bed, mask_overlaps=True)
    for kw in (dict(qualities=True), dict(quality_vote=True, qualities=True), dict(iupac_threshold=0.7)):
        on, off = K.bam_to_consensus(full, normalise=big, **opts, **kw), K.bam_to_consensus(full, **opts, **kw)
        assert [(r.sequence, r.qualities) for r in on.consensuses] == [(r.sequence, r.qualities) for r in off.consensuses]
        for k in on.refs_reports:
            assert _without(on.refs_reports[k], "- normalise:") == off.refs_reports[k].splitlines()
            assert "- normalise: %d per amplicon and strand, 0 of %d reads dropped" % (big, len(recs)) \
                in on.refs_reports[k]
    assert K.weights(full, normalise=big, **opts).to_csv() == K.weights(full, **opts).to_csv()
    assert K.features(full, normalise=big, **opts).to_csv() == K.features(full, **opts).to_csv()
    on = K.variants_vcf(full, normalise=big, strand=True, qual=True, **opts)
    assert _without(on, "##kindelNormalise") == K.variants_vcf(full, strand=True, qual=True, **opts).splitlines()


def test_amplicons_describe_the_kept_reads(tmp_path):
    cap = 10
    full, sub, bed, _, dropped = _pair(tmp_path, 17, cap)
    on = K.amplicons(full, bed, 5, normalise=cap)
    off = K.amplicons(sub, bed, 5)
    cols = [c for c in K.AMPLICON_COLUMNS if c != "sample"]
    assert on[cols].equals(off[cols])
    assert (on["reads"] <= 2 * cap).all() and (on["reads"] == 2 * cap).any()
    name = on["sample"].iloc[0]
    assert on.attrs["dropped"] == {name: len(dropped)} and "dropped" not in off.attrs
    res = subprocess.run([sys.executable, "-m", "kindel_b200", "amplicons", "--primers", bed, "--normalise", str(cap),
                          "--min-depth", "5", full], capture_output=True, text=True, check=True)
    assert res.stderr.strip().endswith("; %d reads over the normalise cap dropped" % len(dropped))


def test_two_gpus_equal_one(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    batch, trows = synth.amplicon_reads(6, 200_000, 50)
    path = tmp_path / "a.bam"
    synth.write_simple_bam(str(path), synth.with_strands(batch, 6))
    bed = tmp_path / "scheme.bed"
    bed.write_text(synth.named_scheme_bed(trows))
    for kw in (dict(), dict(mask_overlaps=True)):
        one = K.bam_to_consensus(str(path), devices=1, primers=str(bed), normalise=30, **kw)
        two = K.bam_to_consensus(str(path), devices=2, primers=str(bed), normalise=30, **kw)
        assert [r.sequence for r in one.consensuses] == [r.sequence for r in two.consensuses]
        assert one.refs_reports == two.refs_reports
    one = K.variants_vcf(str(path), devices=1, primers=str(bed), normalise=30)
    assert one == K.variants_vcf(str(path), devices=2, primers=str(bed), normalise=30)
