"""Per-base consensus qualities (`qualities=True`, `--fastq`; extension) on the GPU: K2q equals the C oracle after both
votes on fuzz, adversarial and the full config-4 table; bam_to_consensus(qualities=True) keeps the sequence, changes
and reports of qualities=False and its qualities equal the C oracle's walk over oracle tables; the CLI writes FASTQ;
the launch count rises by exactly K2q + K5q; two GPUs equal one."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
from conftest import golden_input
from fuzz_cases import random_case
from kindel_b200 import _ffi, bamio, synth
from kindel_b200 import kindel as K
from oracle import coracle, fqoracle, ioracle
from test_fastq import _boundary_tables
from test_gpu_iupac import _shuffled_two_haplotypes
from test_iupac import MIN_DEPTHS, _adversarial, _contigs, _two_haplotypes

pytestmark = pytest.mark.gpu


def _device_qual(table, calls):
    import torch

    from kindel_b200 import engine

    t = torch.from_numpy(np.ascontiguousarray(table)).cuda()
    c = torch.from_numpy(np.ascontiguousarray(calls)).cuda()
    return engine.consensus_qual(t, c).cpu().numpy()


def _votes(table, md):
    yield coracle.vote(table, md)
    for t in (0.0, 0.6, 0.99):
        yield ioracle.vote_iupac(table, md, t)


def test_k2q_equals_oracle_on_fuzz_and_adversarial_tables(tmp_path):
    tables = _adversarial(3) + _adversarial(4) + [_boundary_tables()[0]]
    for s in range(400):
        p = tmp_path / ("fuzz%d.sam" % s)
        p.write_text(random_case(s))
        try:
            tables.append(coracle.pileup(bamio.read_alignment(p))[0])
        except (ValueError, KeyError, IndexError):
            continue
    big = np.concatenate([t[:, : t.shape[1] // 4 * 4] for t in tables], axis=1)  # one launch over all of them too
    for md in MIN_DEPTHS:
        for calls in _votes(big, md):
            np.testing.assert_array_equal(_device_qual(big, calls), fqoracle.qual(big, calls))
        for tab in tables[:7]:
            for calls in _votes(tab, md):
                np.testing.assert_array_equal(_device_qual(tab, calls), fqoracle.qual(tab, calls))


def test_k2q_on_the_full_config4_table():
    """cfg 4 (5 Mb x 200x, 1 % substitutions, ~1 % indel / clip reads), after the device's own votes."""
    import torch

    from kindel_b200 import engine

    batch = synth.mixed_reads(4, [5_000_000], 200, 0.01)
    counts, _ = engine.pileup(engine.upload(batch))
    host = counts.cpu().numpy()
    for t in (None, 0.99):
        calls = engine.vote(counts, 1, iupac_threshold=t)
        got = engine.consensus_qual(counts, calls).cpu().numpy()
        torch.cuda.synchronize()
        want = fqoracle.qual(host, calls.cpu().numpy())
        np.testing.assert_array_equal(got, want)
        assert got.max() >= 20 and np.count_nonzero(got == 0) > 0


def _host_qualities(path, t=None, **kw):
    """The C oracle's walk over the oracle's tables and calls, with the host code's patches: (texts, qualities)."""
    batch = bamio.read_alignment(path)
    counts, events = coracle.pileup(batch)
    md = kw.get("min_depth", 1)
    calls = coracle.vote(counts, md) if t is None else ioracle.vote_iupac(counts, md, t)
    run = K.PileupRun.from_host_tables(batch, counts, coracle.derive(counts), events)
    out = []
    for c, (s0, L, ins_c) in enumerate(_contigs(batch, counts, events)):
        patches = None
        if kw.get("realign"):
            aln = run.alignment(c)
            patches = K.merge_cdrps(K.cdrp_consensuses(
                aln.weights, aln.deletions, aln.clip_start_weights, aln.clip_end_weights, aln.clip_start_depth,
                aln.clip_end_depth, kw.get("clip_decay_threshold", 0.1), kw.get("mask_ends", 50)),
                kw.get("min_overlap", 9))
        out.append(fqoracle.fastq(counts, calls, s0, L, ins_c, patches, kw.get("trim_ends", False),
                                  kw.get("uppercase", False)))
    return out


def _same(got, want):
    assert [s.sequence for s in got.consensuses] == [s.sequence for s in want.consensuses]
    assert [s.name for s in got.consensuses] == [s.name for s in want.consensuses]
    assert {k: list(v) for k, v in got.refs_changes.items()} == {k: list(v) for k, v in want.refs_changes.items()}
    assert got.refs_reports == want.refs_reports


def test_bam_to_consensus_qualities(manifest, tmp_path):
    """Device path (K2q + K5 + K5q, or K2q + the host assembly with --realign) == the C oracle's walk; the sequence,
    changes and reports equal qualities=False's; qualities=False leaves `.qualities` None."""
    from clip_cases import clip_case

    mix = str(tmp_path / "mix.bam")
    _two_haplotypes(mix)
    shuffled = str(tmp_path / "shuffled.bam")
    _shuffled_two_haplotypes(shuffled)
    paths = [golden_input(e) for e in manifest["files"].values()] + [mix, shuffled]
    for seed in range(0, 96, 8):
        p = tmp_path / ("clip%d.sam" % seed)
        p.write_text(clip_case(seed))
        paths.append(str(p))
    options = [dict(), dict(realign=True), dict(trim_ends=True, uppercase=True), dict(min_depth=7),
               dict(realign=True, min_overlap=7, trim_ends=True)]
    n = 0
    for k, path in enumerate(paths):
        for j, t in enumerate((None, 0.6)):
            kw = options[(k + j) % len(options)]
            if path in (mix, shuffled) and j == 0:
                kw = dict(realign=True, min_overlap=7)
            got = K.bam_to_consensus(path, iupac_threshold=t, qualities=True, **kw)
            plain = K.bam_to_consensus(path, iupac_threshold=t, **kw)
            _same(got, plain)
            assert all(r.qualities is None for r in plain.consensuses)
            want = _host_qualities(path, t, **kw)
            assert [(r.sequence, r.qualities) for r in got.consensuses] == want, (path, t, kw)
            for r in got.consensuses:
                assert len(r.qualities) == len(r.sequence)
                n += len(r.qualities)
    assert n > 10_000


def test_launch_count(manifest):
    """qualities=True adds exactly K2q and K5q (and K2q alone with --realign); qualities=False adds nothing."""
    lib = _ffi.load()
    path = golden_input(next(iter(manifest["files"].values())))

    def launches(**kw):
        K.bam_to_consensus(path, **kw)  # warm
        n0 = lib.kdl_launch_count()
        K.bam_to_consensus(path, **kw)
        return lib.kdl_launch_count() - n0

    base = launches()
    assert launches(qualities=True) == base + 2
    assert launches(realign=True, qualities=True) == launches(realign=True) + 1
    assert launches(qualities=False) == base


def test_cli_fastq(tmp_path):
    path = str(tmp_path / "mix.bam")
    _two_haplotypes(path)
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    fasta = subprocess.run([sys.executable, "-m", "kindel", "consensus", path], capture_output=True, text=True, env=env,
                           timeout=900)
    fq = subprocess.run([sys.executable, "-m", "kindel", "consensus", "--fastq", path], capture_output=True, text=True,
                        env=env, timeout=900)
    assert fasta.returncode == 0 and fq.returncode == 0, fq.stderr[-2000:]
    assert fq.stderr == fasta.stderr  # the REPORT is unchanged
    lines = fq.stdout.splitlines()
    assert len(lines) % 4 == 0
    fa = fasta.stdout.splitlines()
    want = _host_qualities(path)
    for r in range(len(lines) // 4):
        name, seq, plus, qual = lines[4 * r: 4 * r + 4]
        assert name.startswith("@") and plus == "+" and len(qual) == len(seq)
        assert all(33 <= ord(ch) <= 93 for ch in qual)
        assert fa[2 * r] == ">" + name[1:] and fa[2 * r + 1] == seq  # the FASTA's sequence, byte for byte
        assert (seq, qual) == want[r]


def test_two_gpus_equal_one(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    path = str(tmp_path / "mix.bam")
    _two_haplotypes(path)
    for t in (None, 0.7):
        for realign in (False, True):
            one = K.bam_to_consensus(path, iupac_threshold=t, realign=realign, devices=1, qualities=True)
            two = K.bam_to_consensus(path, iupac_threshold=t, realign=realign, devices=2, qualities=True)
            _same(two, one)
            assert [r.qualities for r in two.consensuses] == [r.qualities for r in one.consensuses]
    # K2q over each exchange mode's reduced table and gathered calls equals K2q over one GPU's
    from kindel_b200 import distributed as D

    batch = synth.mixed_reads(21, [60_000], 100, 0.1)
    table = coracle.pileup(batch)[0]
    for t in (None, 0.7):
        want = fqoracle.qual(table, coracle.vote(table, 1) if t is None else ioracle.vote_iupac(table, 1, t))
        for mode in ("fused", "allreduce"):
            calls, counts, _, _ = D.run_sharded(batch, 2, 1, mode=mode, iupac_threshold=t)
            np.testing.assert_array_equal(_device_qual(counts, calls), want, err_msg=mode)
