"""Per-amplicon reads and depth (`kindel amplicons`, an extension) on the GPU: K12's labels, the per-amplicon read
counts and K12d's insert statistics through the real library against the per-record oracle (oracle/py_aoracle.py) on
the golden inputs and on synthetic amplicon reads and pairs, under the read and base filters; the depths against
weights(..., primers=); a dropout; the CLI; and two GPUs against one."""
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

pytestmark = pytest.mark.gpu

GOLDEN = ["bwa_1_1.bam", "bwa_4_1.bam", "ext_2_bc63.sam"]


def _bed(tmp_path, rows, name="scheme.bed"):
    p = tmp_path / name
    p.write_text(AC.bed_text(rows))
    return p


def _check(path, bed, rows, min_depth=20, **filters):
    """kindel.amplicons of one file against the oracle: labels (K12 on the run's device batch), per-amplicon reads,
    and the insert statistics against A+C+G+T of weights(..., primers=) under the same filters."""
    mapq, flags = filters.get("min_mapq", 0), filters.get("exclude_flags", 0)
    df = K.amplicons(str(path), str(bed), min_depth, **filters)
    run, _ = K.pileup_run(str(path), None, 1, filters.get("min_base_quality", 0), mapq, flags,
                          primers=P.load_scheme(bed).primers, mask_overlaps=filters.get("mask_overlaps", False))
    arr = P.amplicon_arrays(P.load_scheme(bed), run.batch.contig_names, run.batch.contig_len)
    labels = engine.assign_amplicons(run.device_tables()[1], arr).cpu().numpy()
    names = list(run.batch.contig_names)
    if run.batch.n_reads < 20_000:
        want = AO.labels_by_read(str(path), names, rows, mapq, flags)
    else:
        want = AO.labels_of_batch(run.batch, rows)
    assert labels.tolist() == want.tolist()
    table = AO.amplicon_table(rows, names)
    assert df["amplicon"].tolist() == [t[1] for t in table]
    assert df["reads"].tolist() == [int((want == k).sum()) for k in range(len(table))]
    kept, assigned, unprimed, mispaired, ambiguous = df.attrs["reads"][df["sample"].iloc[0]] if len(df) else (0,) * 5
    if len(df):
        assert (kept, unprimed, mispaired, ambiguous) == (len(want), int((want == -1).sum()), int((want == -2).sum()),
                                                          int((want == -3).sum()))
        assert assigned == int((want >= 0).sum())
    w = K.weights(str(path), primers=str(bed), **filters)
    acgt = w[["A", "C", "G", "T"]].sum(axis=1).to_numpy()
    first = {c: int(np.flatnonzero(w["chrom"].to_numpy() == c)[0]) for c in names}
    mean, lowest, covered = [], [], []
    for c, _, _, _, i0, i1 in table:
        d = acgt[first[c] + i0:first[c] + i1]
        mean.append(d.sum() / (i1 - i0))
        lowest.append(d.min())
        covered.append((d >= min_depth).mean())
    assert np.allclose(df["mean_depth"], mean, rtol=0, atol=1e-9) and df["lowest_depth"].tolist() == lowest
    assert np.allclose(df["covered"], covered, rtol=0, atol=1e-12)
    assert df["status"].tolist() == ["dropout" if m < min_depth else "PASS" for m in mean]
    stats = AO.insert_stats(run.host_counts, run.batch.contig_slot, names, table, min_depth)
    assert [(int(round(r.mean_depth * (t[5] - t[4]))), r.lowest_depth) for r, t in
            zip(df.itertuples(index=False), table)] == [(s[0], s[1]) for s in stats]
    return df, want


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_inputs_with_synthetic_schemes(tmp_path, name):
    path = os.path.join(os.path.dirname(__file__), "golden", "inputs", name)
    b = bamio.read_alignment(path)
    rng = np.random.default_rng(len(name))
    contigs = list(zip(b.contig_names, b.contig_len.tolist()))
    # a tiled scheme over each contig's first 100 kb, and random amplicons whose primers overlap its own
    span = [min(n, 100_000) for n in b.contig_len.tolist()]
    rows = AC.tiled_rows(synth.tiled_scheme(3, b.contig_names, span)) + AC.random_scheme_rows(rng, contigs, 12)
    bed = _bed(tmp_path, rows)
    _check(path, bed, rows, min_depth=5)
    if name.endswith(".bam"):
        _check(path, bed, rows, min_depth=5, min_base_quality=20, min_mapq=10, exclude_flags=0x10)


def test_synthetic_amplicon_reads_under_filters(tmp_path):
    batch, trows = synth.amplicon_reads(3, 60_000, 40)
    path = tmp_path / "amp.bam"
    synth.write_simple_bam(str(path), batch)
    rows = AC.tiled_rows(trows)
    bed = tmp_path / "scheme.bed"
    bed.write_text(synth.named_scheme_bed(trows))
    df, want = _check(path, bed, rows)
    assert (want >= 0).all() and (df["status"] == "PASS").mean() > 0.5
    _check(path, bed, rows, min_depth=30, min_mapq=1, exclude_flags=0x400)


def test_synthetic_amplicon_pairs_with_mask_overlaps(tmp_path):
    batch, flag, frag, trows = synth.amplicon_pairs(5, 20_000, 60)
    path = tmp_path / "pairs.bam"
    contigs, recs = synth.paired_records(batch, flag, frag)
    bamio.write_bam(str(path), contigs, recs)
    rows = AC.tiled_rows(trows)
    bed = tmp_path / "scheme.bed"
    bed.write_text(synth.named_scheme_bed(trows))
    on, _ = _check(path, bed, rows, mask_overlaps=True)
    off, _ = _check(path, bed, rows)
    assert on["reads"].tolist() == off["reads"].tolist()  # the labels do not depend on the masking
    assert (on["mean_depth"] <= off["mean_depth"]).all() and (on["mean_depth"] < off["mean_depth"]).any()


def test_an_amplicon_without_reads_is_a_dropout(tmp_path):
    batch, trows = synth.amplicon_reads(2, 20_000, 30)
    path = tmp_path / "amp.bam"
    rows = AC.tiled_rows(trows)
    # every read of the tiled contig starts or ends at an amplicon: take away every read near amplicon 3
    a3 = [r for r in rows if r[3] == "amp_3"]
    start = np.asarray(batch.ref_start, dtype=np.int64)
    keep = (start < a3[0][1] - 200) | (start > a3[1][2] + 200)
    synth.write_simple_bam(str(path), bamio.select_reads(batch, np.flatnonzero(keep)))
    bed = tmp_path / "scheme.bed"
    bed.write_text(synth.named_scheme_bed(trows))
    df, _ = _check(path, bed, rows)
    row = df[df["amplicon"] == "amp_3"].iloc[0]
    assert row.reads == 0 and row.mean_depth == 0 and row.lowest_depth == 0 and row.covered == 0
    assert row.status == "dropout"


def test_cli_end_to_end(tmp_path):
    batch, trows = synth.amplicon_reads(4, 10_000, 30)
    paths = []
    for k in range(2):
        p = tmp_path / ("s%d.bam" % k)
        synth.write_simple_bam(str(p), batch)
        paths.append(str(p))
    bed = tmp_path / "scheme.bed"
    bed.write_text(synth.named_scheme_bed(trows))
    res = subprocess.run([sys.executable, "-m", "kindel_b200", "amplicons", "--primers", str(bed), *paths],
                         capture_output=True, text=True, check=True)
    lines = res.stdout.splitlines()
    assert lines[0].split("\t") == K.AMPLICON_COLUMNS
    n = len(trows) // 2
    assert [ln.split("\t")[0] for ln in lines[1:]] == ["s0.bam"] * n + ["s1.bam"] * n
    assert lines[1:n + 1] == [ln.replace("s1.bam", "s0.bam", 1) for ln in lines[n + 1:]]
    assert res.stderr.count("reads kept") == 2


def test_two_gpus_equal_one(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    batch, trows = synth.amplicon_reads(6, 200_000, 50)
    path = tmp_path / "a.bam"
    synth.write_simple_bam(str(path), batch)
    bed = tmp_path / "scheme.bed"
    bed.write_text(synth.named_scheme_bed(trows))
    one = K.amplicons(str(path), str(bed), devices=1)
    two = K.amplicons(str(path), str(bed), devices=2)
    assert one.to_csv(sep="\t") == two.to_csv(sep="\t") and one.attrs == two.attrs
