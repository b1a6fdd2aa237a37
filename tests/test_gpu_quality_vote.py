"""The quality vote (`consensus --quality-vote`) on the device: K11w + K11g-w against py_qvoracle's walk over weights,
K2w against the per-slot restatement, the truth set through bam_to_consensus and the CLI, a tenth of config 4 by
sha256, and two GPUs."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import quality_vote_cases as QVC
from kindel_b200 import bamio, engine, synth
from kindel_b200 import kindel as K
from test_quality_vote import corpus, laid_out, planted_table, weight_oracle, weight_sums  # noqa: F401
from test_quality_vote import test_truth_set_through_bam_to_consensus as _truth_matrix

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def device_weights(batch, qual8):
    dev = torch.device("cuda", 0)
    db = engine.upload(batch, dev)
    torch.cuda.synchronize()
    wsum = engine.quality_weights(db, torch.from_numpy(qual8).to(dev))
    torch.cuda.synchronize()
    return wsum.cpu().numpy().view(np.uint64)


def test_k11w_on_the_corpus_and_on_complex_reads(corpus, monkeypatch):
    for kw in (dict(), dict(min_base_quality=20, min_mapq=30, exclude_flags=0x500)):
        batch = bamio.read_alignment(corpus["bam"], qual=True, **kw)
        want = laid_out(batch, weight_sums(monkeypatch, corpus["bam"], kw.get("min_base_quality", 0),
                                           kw.get("min_mapq", 0), kw.get("exclude_flags", 0)))[0]
        np.testing.assert_array_equal(device_weights(batch, batch.qual8).astype(object), want.astype(object))
    for seed in (1, 2):
        batch = synth.complex_reads(seed, 3000, 30)
        qual = synth.qualities(seed, batch.seq_len)
        want = weight_oracle(batch, qual)
        np.testing.assert_array_equal(device_weights(batch, bamio.qual_layout(batch, qual)).astype(object),
                                      want.astype(object))
        perm = np.random.default_rng(seed).permutation(batch.n_reads)
        ub = bamio.select_reads(batch, perm)
        at = np.concatenate(([0], np.cumsum(batch.seq_len.astype(np.int64))))
        uq = np.concatenate([qual[at[r]:at[r + 1]] for r in perm])
        np.testing.assert_array_equal(device_weights(ub, bamio.qual_layout(ub, uq)).astype(object),
                                      want.astype(object))


def test_a_deep_q93_column_passes_2_to_the_32(tmp_path):
    """720 reads of Q93 G over one column: the uint64 sum passes 2^32, exactly 720 * W[93]."""
    recs = [(0, 40, 0, [(60 << 4) | 0], "G" * 60, "d%d" % j, 60, bytes([93] * 60)) for j in range(720)]
    path = str(tmp_path / "deep.bam")
    bamio.write_bam(path, [("d", 1024)], recs)
    batch = bamio.read_alignment(path, qual=True)
    wsum = device_weights(batch, batch.qual8)
    assert int(wsum[2, 70]) == 720 * 6407534 > 2 ** 32
    assert int(wsum[[0, 1, 3]].sum()) == 0


def test_k2w_against_the_restatement():
    rng = np.random.default_rng(9)
    dev = torch.device("cuda", 0)
    for n, md in ((1 << 16, 1), (4096, 3)):
        counts, wsum = planted_table(rng, n)
        c = torch.from_numpy(counts).to(dev)
        w = torch.from_numpy(wsum.view(np.int64)).to(dev)
        calls, qual = engine.vote_quality(c, w, md)
        want = QVC.restated_vote(counts, wsum.astype(object), md)
        np.testing.assert_array_equal(calls.cpu().numpy(), want[0])
        np.testing.assert_array_equal(qual.cpu().numpy(), want[1])
        np.testing.assert_array_equal(calls.cpu().numpy() >> 4, engine.vote(c, md).cpu().numpy() >> 4)


@pytest.mark.parametrize("sam", [False, True])
@pytest.mark.parametrize("bq,trim,upper,realign,fastq", [
    (0, False, False, False, True), (10, True, False, True, True), (0, True, True, False, False)])
def test_truth_set_on_the_device(corpus, monkeypatch, sam, bq, trim, upper, realign, fastq):
    import test_quality_vote as T

    monkeypatch.setattr(T, "on_the_emulator", lambda mp: None)  # the same checks, on the device
    _truth_matrix(corpus, monkeypatch, sam, bq, trim, upper, realign, fastq)


def test_cli_with_every_flag(corpus):
    _, text, quals, sites, _ = QVC.expected(10)
    args = [sys.executable, "-m", "kindel_b200", "consensus", "--quality-vote", "--fastq", "--min-depth", "1",
            "--min-base-quality", "10", "--min-mapq", "0", "--mask-overlaps", "-t", "-u", corpus["tbam"]]
    res = subprocess.run(args, capture_output=True, text=True, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    lo, hi = len(text) - len(text.lstrip("N")), len(text.rstrip("N"))
    q = "".join(chr(33 + x) for x in quals)
    assert res.stdout == "@v_cns\n%s\n+\n%s\n" % (text[lo:hi], q[lo:hi])
    assert "- quality-vote sites: %s" % ", ".join(map(str, sites)) in res.stderr.split("\n")


def test_a_tenth_of_config_4_by_sha256():
    import bench_quality_vote as B

    batch = synth.mixed_reads(4, [500_000], 200, 0.01)
    qual = synth.qualities(7, batch.seq_len)
    dev = torch.device("cuda", 0)
    db = engine.upload(batch, dev)
    counts, _ = engine.pileup(db)
    wsum = engine.quality_weights(db, torch.from_numpy(bamio.qual_layout(batch, qual)).to(dev))
    calls, qv = engine.vote_quality(counts, wsum, 1)
    torch.cuda.synchronize()
    want_w = B.oracle_weights(batch, qual)
    want_c, want_q = B.oracle_vote(counts.cpu().numpy(), want_w)
    sha = lambda *a: hashlib.sha256(b"".join(np.ascontiguousarray(x).tobytes() for x in a)).hexdigest()
    assert sha(wsum.cpu().numpy().view(np.uint64), calls.cpu().numpy(), qv.cpu().numpy()) == \
        sha(want_w, want_c, want_q)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus_equal_one(corpus):
    kw = dict(min_base_quality=20, primers=corpus["bed"], mask_overlaps=True, qualities=True, quality_vote=True)
    one = K.bam_to_consensus(corpus["bam"], devices=1, **kw)
    two = K.bam_to_consensus(corpus["bam"], devices=2, **kw)
    assert [(r.sequence, r.qualities) for r in two.consensuses] == [(r.sequence, r.qualities) for r in one.consensuses]
    assert two.refs_reports == one.refs_reports
