"""`variants --vcf --qual` on the device: K11 + K11g against oracle/py_qvoracle.py and the constant-quality invariant
against engine.pileup, and the VCF equal to the oracle byte for byte."""
from __future__ import annotations

import os

import numpy as np
import pytest
import torch

import qual_cases as QC
from kindel_b200 import bamio, engine, synth
from kindel_b200 import kindel as K
from oracle import py_qvoracle as QV
from test_variant_qual import MATRIX, _oracle, assert_sums, batch_oracle, corpus, laid_out  # noqa: F401

pytestmark = pytest.mark.gpu


def device_sums(batch, qual8):
    dev = torch.device("cuda", 0)
    db = engine.upload(batch, dev)
    qsum, emass = engine.quality_sums(db, torch.from_numpy(qual8).to(dev))
    torch.cuda.synchronize()
    return qsum.cpu().numpy().view(np.uint32), emass.cpu().numpy().view(np.uint64), db


def test_k11_equals_the_oracle_on_the_corpus(corpus):
    for kw in (dict(), dict(min_base_quality=20, min_mapq=30, exclude_flags=0x500)):
        batch = bamio.read_alignment(corpus["bam"], qual=True, **kw)
        want = laid_out(batch, QV.quality_sums(corpus["bam"], kw.get("min_base_quality", 0), kw.get("min_mapq", 0),
                                               kw.get("exclude_flags", 0)))
        qs, em, _ = device_sums(batch, batch.qual8)
        assert_sums((qs, em), want, str(kw))


def test_k11_with_primers_and_mates_through_the_run(corpus):
    for pr, mates in ((True, False), (False, True), (True, True)):
        run = K.pileup_run(corpus["bam"], primers=corpus["bed"] if pr else None, mask_overlaps=mates, qual=True)[0]
        qsum, emass = run.quality_table()
        want = laid_out(run.batch, QV.quality_sums(corpus["bam"], 0, 0, 0, corpus["rows"] if pr else None, mates))
        assert_sums((qsum.cpu().numpy().view(np.uint32), emass.cpu().numpy().view(np.uint64)), want, (pr, mates))


def test_k11_on_synthetic_reads_with_hard_reads():
    batch = synth.complex_reads(5, 20000, 40)
    qual = synth.qualities(5, batch.seq_len)
    qs, em, _ = device_sums(batch, bamio.qual_layout(batch, qual))
    assert_sums((qs, em), batch_oracle(batch, qual))


def test_constant_quality_on_a_tenth_of_config_4():
    """Config 4's shape at a tenth of its depth (mixed reads, 1 % complex): with every quality q, qsum == q * the
    pileup's columns 0-3 and emass == EPS[q] * their sum; with seeded qualities, the masked batch counts no base the
    pileup does not."""
    batch = synth.mixed_reads(4, [5_000_000], 20, 0.01)
    dev = torch.device("cuda", 0)
    db = engine.upload(batch, dev)
    counts, _ = engine.pileup(db)
    c = counts[0:4].cpu().numpy().astype(np.int64)
    for q in (30, 93):
        qual8 = bamio.qual_layout(batch, np.full(int(batch.seq_len.sum()), q, dtype=np.uint8))
        qsum, emass = engine.quality_sums(db, torch.from_numpy(qual8).to(dev))
        np.testing.assert_array_equal(qsum.cpu().numpy().view(np.uint32).astype(np.int64), q * c)
        np.testing.assert_array_equal(emass.cpu().numpy().view(np.uint64).astype(np.int64), QV.EPS[q] * c.sum(axis=0))
    masked, qual = synth.with_qualities(batch, 4, 20)
    dm = engine.upload(masked, dev)
    mc, _ = engine.pileup(dm)
    qsum, _ = engine.quality_sums(dm, torch.from_numpy(bamio.qual_layout(masked, qual)).to(dev))
    qs = qsum.cpu().numpy().view(np.uint32).astype(np.int64)
    mc = mc[0:4].cpu().numpy().astype(np.int64)
    assert ((qs >= 20 * mc) & (qs <= 41 * mc)).all()


def test_variants_vcf_qual_equals_the_oracle(corpus):
    for bq, mq, ex, pr, ref, strand, max_sor, mates, min_qual, sam in MATRIX:
        kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, primers=corpus["bed"] if pr else None,
                  reference=corpus["fa"] if ref else None, strand=strand, max_sor=max_sor, mask_overlaps=mates)
        got = K.variants_vcf(corpus["sam"] if sam else corpus["bam"], qual=True, min_qual=min_qual, **kw)
        want = _oracle(corpus, corpus["bam"], bq, mq, ex, pr, (os.path.basename(corpus["fa"]), corpus["refs"])
                       if ref else None, strand, max_sor, mates, min_qual)
        assert got == want


def test_cli_on_the_planted_truth_set(corpus, capsys):
    from kindel_b200 import cli

    cli.main(["variants", "--vcf", "--reference", corpus["pfa"], "--qual", "--min-qual", "30", corpus["pbam"]])
    out = capsys.readouterr().out
    recs = {int(x.split("\t")[1]) - 1: x.split("\t") for x in out.splitlines() if not x.startswith("#")}
    assert recs[QC.SITE_REAL][6] == "PASS" and recs[QC.SITE_LOW][6] == "lowqual"
    cli.main(["variants", "--vcf", "--reference", corpus["pfa"], corpus["pbam"]])
    plain = capsys.readouterr().out
    assert plain == K.variants_vcf(corpus["pbam"], reference=corpus["pfa"]) and "##kindelQual" not in plain
