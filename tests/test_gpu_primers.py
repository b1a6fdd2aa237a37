"""Amplicon primer masking (`--primers`, an extension) on the GPU: K9 through the real library against the per-record
oracle (oracle/py_poracle.py), a tenth of config 4 against the oracle's table, the strand split of a masked run, the
planted truth set through the CLI, and several GPUs against one."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
import primer_cases as PC
from fuzz_cases import random_case
from kindel_b200 import bamio, synth
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from oracle import py_poracle as PO

pytestmark = pytest.mark.gpu


def _sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _device_lists(db):
    n = int(db.struct.n_reads)
    out = [[] for _ in range(n)]
    if db.qmask is not None:
        mr = db.tensors["mask_read"].cpu().numpy().view(np.uint32)
        mo = db.tensors["mask_off"].cpu().numpy().view(np.uint32)
        mq = db.tensors["mask_qpos"].cpu().numpy().view(np.uint32)
        for j, r in enumerate(mr.tolist()):
            out[r] = mq[mo[j]:mo[j + 1]].tolist()
    return out


def test_k9_fuzz_and_edge_cases_against_the_oracle(tmp_path):
    rng = np.random.default_rng(3)
    n_checked = n_raised = 0
    for seed in range(40):
        p = tmp_path / ("f%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            b = bamio.read_alignment(p)
        except (ValueError, KeyError):
            continue
        rows = PC.random_rows(rng, list(zip(b.contig_names, b.contig_len.tolist())))
        prim = PO.masked_by_read(str(p), b.contig_names, rows)
        try:
            want, _ = PO.pileup(b, prim)
        except (IndexError, KeyError) as exc:
            with pytest.raises(type(exc)):
                K.PileupRun(b, primers=PC.primer_set(rows))
            n_raised += 1
            continue
        run = K.PileupRun(b, primers=PC.primer_set(rows))
        assert _device_lists(run.dbatch) == [list(x) for x in prim], seed
        assert np.array_equal(run.counts.cpu().numpy(), want), seed
        assert run.dbatch.primer_masked == (sum(1 for x in prim if x), sum(len(x) for x in prim))
        n_checked += 1
    assert n_checked >= 5 and n_checked + n_raised > 20  # (most fuzz cases raise, as the reference does)


def test_k9_on_a_tenth_of_config4_equals_the_oracle():
    plain = synth.mixed_reads(4, [500_000], 200, 0.01)
    batch, qual = synth.with_qualities(plain, 5)  # bases below Q20 masked as the decoders mask them
    rows = synth.tiled_scheme(1, batch.contig_names, batch.contig_len)
    prim = PO.masked_by_batch(plain, rows)
    for b, q, mbq in ((plain, None, 0), (batch, qual, 20)):
        run = K.PileupRun(b, primers=PC.primer_set(rows))
        assert run.dbatch.primer_masked[1] == sum(len(x) for x in prim) > 0
        want, _ = PO.pileup(plain, prim, q, mbq)  # (the oracle masks the unmasked bases itself)
        assert _sha(run.counts.cpu().numpy()) == _sha(want), mbq


def test_no_primers_empty_and_foreign_beds_are_the_plain_table(tmp_path):
    b = bamio.read_alignment(os.path.join(H.ROOT, "tests", "golden", "inputs", "mm2_multi.bam"))
    plain = K.PileupRun(b).counts.cpu().numpy()
    (tmp_path / "e.bed").write_text("# nothing\n")
    (tmp_path / "f.bed").write_text("chrZ\t0\t10\n")
    for primers in (None, str(tmp_path / "e.bed"), str(tmp_path / "f.bed")):
        run = K.PileupRun(b, primers=P.as_primer_set(primers))
        assert np.array_equal(run.counts.cpu().numpy(), plain)
        assert run.dbatch.primer_masked == (0, 0)


def test_reverse_table_of_a_masked_run_is_the_masked_sub_batch():
    batch, rows = synth.amplicon_reads(2, 60_000, 100)
    batch = synth.with_strands(batch, 4)
    ps = PC.primer_set(rows)
    run = K.PileupRun(batch, primers=ps)
    rev = run.reverse_table()[0].cpu().numpy()
    sub = bamio.select_reads(batch, np.flatnonzero(batch.reverse))
    want = K.PileupRun(sub, primers=ps).counts.cpu().numpy()
    assert np.array_equal(rev, want)
    unmasked_rev = K.PileupRun(sub).counts.cpu().numpy()
    assert not np.array_equal(rev[0:5], unmasked_rev[0:5]) and np.array_equal(rev[5:], unmasked_rev[5:])


def _cli(*args):
    res = subprocess.run([sys.executable, "-m", "kindel_b200", *args], capture_output=True, text=True, cwd=H.ROOT)
    assert res.returncode == 0, res.stderr
    return res


def test_planted_truth_set_through_the_cli(tmp_path):
    bam, bed, fa, ref, sample = PC.write(tmp_path)
    site = PC.SITE
    off = _cli("consensus", str(bam))
    on = _cli("consensus", "--primers", str(bed), str(bam))
    seq_off, seq_on = off.stdout.splitlines()[1], on.stdout.splitlines()[1]
    assert seq_off[site] == ref[site] and seq_on[site] == sample[site] != ref[site]
    assert "- primers: scheme.primer.bed" in on.stderr and "- primers:" not in off.stderr
    vcf_args = ("variants", "--vcf", "--reference", str(fa), "-r", str(PC.REL))
    v_off = _cli(*vcf_args, str(bam)).stdout.splitlines()
    v_on = _cli(*vcf_args, "--primers", str(bed), str(bam)).stdout.splitlines()
    assert not [ln for ln in v_off if ln.startswith("t\t%d\t" % (site + 1))]
    snv = [ln.split("\t") for ln in v_on if ln.startswith("t\t%d\t" % (site + 1))]
    assert len(snv) == 1 and snv[0][3:5] == [ref[site], sample[site]]
    assert "##kindelPrimers=scheme.primer.bed" in v_on and v_on.index("##kindelPrimers=scheme.primer.bed") == 3
    assert not any(ln.startswith("##kindelPrimers") for ln in v_off)
    # columns 5-18 and the insertion events are the same with and without primers
    a, b = K.pileup_run(str(bam))[0], K.pileup_run(str(bam), primers=str(bed))[0]
    assert np.array_equal(a.host_counts[5:], b.host_counts[5:])
    assert np.array_equal(a.events.cpu().numpy(), b.events.cpu().numpy())
    for cmd in ("weights", "features"):
        assert _cli(cmd, "--primers", str(bed), str(bam)).stdout.count("\n") > 2000
    _cli("variants", "--vcf", "--strand", "--primers", str(bed), str(bam))


def test_two_gpus_equal_one(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    batch, rows = synth.amplicon_reads(6, 200_000, 50)
    path = tmp_path / "a.bam"
    synth.write_simple_bam(str(path), batch)
    bed = tmp_path / "s.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
    one = K.bam_to_consensus(str(path), devices=1, primers=str(bed))
    two = K.bam_to_consensus(str(path), devices=2, primers=str(bed))
    assert [r.sequence for r in one.consensuses] == [r.sequence for r in two.consensuses]
    assert one.refs_reports == two.refs_reports
    r1, _ = K.pileup_run(str(path), devices=1, primers=str(bed))
    r2, _ = K.pileup_run(str(path), devices=2, primers=str(bed))
    assert np.array_equal(r1.host_counts, r2.host_counts)
