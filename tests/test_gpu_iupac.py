"""The IUPAC vote (`iupac_threshold`, extension) on the GPU: K2 with the IUPAC vote is bit-identical to the C oracle's
vote on fuzz, adversarial and full config-4 tables; bam_to_consensus (device vote + K5, or the host assembly for
--realign) equals consensus_from_run over oracle tables and oracle calls; the CLI; two GPUs equal one."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
from conftest import golden_input
from fuzz_cases import random_case
from kindel_b200 import bamio, synth
from kindel_b200 import kindel as K
from oracle import coracle, ioracle
from test_iupac import MIN_DEPTHS, THRESHOLDS, _adversarial, _two_haplotypes

pytestmark = pytest.mark.gpu


def _device_vote(table, md, t):
    import torch

    from kindel_b200 import engine

    calls = engine.vote(torch.from_numpy(np.ascontiguousarray(table)).cuda(), md, iupac_threshold=t)
    return calls.cpu().numpy()


def test_vote_equals_oracle_on_fuzz_and_adversarial_tables(tmp_path):
    tables = _adversarial(3) + _adversarial(4)
    for s in range(400):
        p = tmp_path / ("fuzz%d.sam" % s)
        p.write_text(random_case(s))
        try:
            tables.append(coracle.pileup(bamio.read_alignment(p))[0])
        except (ValueError, KeyError, IndexError):
            continue
    big = np.concatenate([t[:, : t.shape[1] // 4 * 4] for t in tables], axis=1)  # one launch over all of them too
    for md in MIN_DEPTHS:
        for t in THRESHOLDS:
            np.testing.assert_array_equal(_device_vote(big, md, t), ioracle.vote_iupac(big, md, t))
            for tab in tables[:6]:
                np.testing.assert_array_equal(_device_vote(tab, md, t), ioracle.vote_iupac(tab, md, t))


def test_vote_on_the_full_config4_table():
    """cfg 4 (5 Mb x 200x, 1 % substitutions, ~1 % indel / clip reads) at t = 0.99: many mixed sites."""
    import torch

    from kindel_b200 import engine

    batch = synth.mixed_reads(4, [5_000_000], 200, 0.01)
    counts, _ = engine.pileup(engine.upload(batch))
    host = counts.cpu().numpy()
    got = engine.vote(counts, 1, iupac_threshold=0.99).cpu().numpy()
    torch.cuda.synchronize()
    want = ioracle.vote_iupac(host, 1, 0.99)
    np.testing.assert_array_equal(got, want)
    assert np.count_nonzero(got & 0x80) > 100_000
    # the default vote is untouched on the same table
    np.testing.assert_array_equal(engine.vote(counts, 1).cpu().numpy(), coracle.vote(host, 1))


def _host_result(path, t, **kw):
    batch = bamio.read_alignment(path)
    counts, events = coracle.pileup(batch)
    run = K.PileupRun.from_host_tables(batch, counts, coracle.derive(counts), events)
    calls = ioracle.vote_iupac(counts, kw.get("min_depth", 1), t)
    return K.consensus_from_run(run, calls, path, iupac_threshold=t, **kw)


def _same(got, want):
    assert [s.sequence for s in got.consensuses] == [s.sequence for s in want.consensuses]
    assert [s.name for s in got.consensuses] == [s.name for s in want.consensuses]
    assert {k: list(v) for k, v in got.refs_changes.items()} == {k: list(v) for k, v in want.refs_changes.items()}
    assert got.refs_reports == want.refs_reports


def _shuffled_two_haplotypes(path, seed=9):
    rng = np.random.default_rng(seed)
    sorted_path = path + ".sorted.bam"
    ref, _ = _two_haplotypes(sorted_path, seed=seed)
    batch = bamio.read_alignment(sorted_path)
    records = []
    for r in rng.permutation(batch.n_reads).tolist():
        seq = H.event_string(batch, r, 0, int(batch.seq_len[r]))
        cig = batch.cigar[int(batch.cig_off[r]):int(batch.cig_off[r + 1])].tolist()
        records.append((0, int(batch.ref_start[r]), 0, cig, seq))
    bamio.write_bam(path, [("hap", len(ref))], records)


def test_bam_to_consensus_equals_host_assembly(manifest, tmp_path):
    """Device path (K2-IUPAC + K5, or the host assembly with --realign) == oracle tables + oracle IUPAC calls through
    consensus_from_run: FASTA, changes and REPORT."""
    mix = str(tmp_path / "mix.bam")
    _two_haplotypes(mix)
    shuffled = str(tmp_path / "shuffled.bam")
    _shuffled_two_haplotypes(shuffled)
    assert not bamio.read_alignment(shuffled).reads_sorted
    paths = [golden_input(e) for e in manifest["files"].values()] + [mix, shuffled]
    options = [dict(), dict(realign=True), dict(trim_ends=True, uppercase=True), dict(min_depth=7),
               dict(realign=True, min_overlap=7, trim_ends=True)]
    n = 0
    for k, path in enumerate(paths):
        for j, t in enumerate((0.0, 0.6, 0.99)):
            kw = options[(k + j) % len(options)]
            got = K.bam_to_consensus(path, iupac_threshold=t, **kw)
            _same(got, _host_result(path, t, **kw))
            n += sum(1 for r in got.refs_reports.values() if "- iupac sites: \n" not in r)
        # off: byte-identical to the default call
        plain = K.bam_to_consensus(path)
        assert all("iupac" not in r for r in plain.refs_reports.values())
    assert n > 10


def test_cli_iupac_threshold(tmp_path):
    path = str(tmp_path / "mix.bam")
    _two_haplotypes(path)
    want = _host_result(path, 0.6, min_overlap=7)
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    res = subprocess.run([sys.executable, "-m", "kindel", "consensus", "--iupac-threshold", "0.6", path],
                         capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout == "".join(">%s\n%s\n" % (s.name, s.sequence) for s in want.consensuses)
    assert res.stderr == "\n".join(want.refs_reports.values()) + "\n"
    assert "- iupac_threshold: 0.6" in res.stderr and any(ch in res.stdout for ch in "MRWSYK")
    bad = subprocess.run([sys.executable, "-m", "kindel", "consensus", "--iupac-threshold", "1.5", path],
                         capture_output=True, text=True, env=env, timeout=900)
    assert bad.returncode == 2 and "iupac" in bad.stderr


def test_two_gpus_equal_one(tmp_path):
    import torch

    from kindel_b200 import distributed as D

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    path = str(tmp_path / "mix.bam")
    _two_haplotypes(path)
    batch = synth.mixed_reads(21, [60_000], 100, 0.1)
    for t in (0.0, 0.7):
        one = K.bam_to_consensus(path, iupac_threshold=t, devices=1)
        two = K.bam_to_consensus(path, iupac_threshold=t, devices=2)
        _same(two, one)
        want = ioracle.vote_iupac(coracle.pileup(batch)[0], 1, t)
        for mode in ("fused", "allreduce"):
            calls = D.run_sharded(batch, 2, 1, mode=mode, iupac_threshold=t)[0]
            np.testing.assert_array_equal(calls, want, err_msg=mode)
