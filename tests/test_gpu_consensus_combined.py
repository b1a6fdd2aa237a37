"""The consensus with `--primers` and `--mask-overlaps` together on the GPU, against the composed oracle of
tests/pair_combo_cases.py: the option matrix through the real library, the full `consensus --fastq` command,
ShardedConsensus with primers= and drops= over many epochs in one process, two GPUs, and config 4's shape as amplicon
pairs by sha256."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import helpers as H
import pair_combo_cases as PC
import test_gpu_sharded_epochs as SE
from kindel_b200 import bamio, synth
from kindel_b200 import distributed as D
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from oracle import fqoracle, ioracle
from oracle import py_moracle as MO
from oracle import py_poracle as PO
from test_consensus_combined import _merged_pre, check_consensus, consensus_kwargs, piled
from test_mates import _reverse_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("gpu_pair_combo")
    out = PC.write(d)
    out.update(dir=d, layout=bamio.read_alignment(out["bam"]), piled={})
    return out


@pytest.mark.parametrize("k", range(len(PC.option_matrix())))
def test_option_matrix_on_the_device(corpus, k):
    """bam_to_consensus with qualities on equals the oracle: sequence, qualities, changes and REPORT lines."""
    row = PC.option_matrix()[k]
    path = corpus["sam"] if k % 3 == 2 else corpus["bam"]
    check_consensus(corpus, row, K.bam_to_consensus(path, qualities=True, **consensus_kwargs(corpus, row)), path)


def test_cli_with_every_flag(corpus):
    """`consensus --fastq` with every filter, primers, mates, min_depth, -t and -u prints the oracle's FASTQ; without
    --fastq the same sequences as FASTA; the REPORT on stderr is the API's."""
    path = corpus["bam"]
    args = ["--iupac-threshold", "0.6", "--min-base-quality", "20", "--min-mapq", "30", "--exclude-flags", "0x400",
            "--primers", corpus["bed"], "--mask-overlaps", "--min-depth", "3", "-t", "-u", path]
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    run = lambda extra: subprocess.run([sys.executable, "-m", "kindel", "consensus"] + extra + args,  # noqa: E731
                                       capture_output=True, text=True, cwd=H.ROOT, env=env)
    fq, fa = run(["--fastq"]), run([])
    assert fq.returncode == 0 and fa.returncode == 0, fq.stderr + fa.stderr
    row = (0.6, 20, 3, False, True, True, (30, 0x400), True, True)
    want = piled(corpus, 20, 30, 0x400, True, True).consensus(0.6, 3, False, True, True, min_overlap=7)
    assert fq.stdout == "".join("@%s_cns\n%s\n+\n%s\n" % (n, s, q) for n, s, _, q, _ in want)
    assert fa.stdout == "".join(">%s_cns\n%s\n" % (n, s) for n, s, _, _, _ in want)
    api = K.bam_to_consensus(path, min_overlap=7, qualities=True, **consensus_kwargs(corpus, row))
    assert fq.stderr.endswith("\n".join(api.refs_reports.values()) + "\n")
    assert "- mate overlaps: %d pairs" % piled(corpus, 20, 30, 0x400, True, True).overlap_stats[0] in fq.stderr


@pytest.mark.skipif(torch.cuda.device_count() < 2,
                    reason="needs two GPUs: the sharded branch runs one process per GPU")
def test_two_gpus_against_the_oracle(corpus):
    for row in ((0.6, 20, 3, True, False, False, (30, 0x400), True, True),
                (0.99, 0, 1, True, True, True, (0, 0), False, True)):
        got = K.bam_to_consensus(corpus["bam"], devices=2, qualities=True, **consensus_kwargs(corpus, row))
        check_consensus(corpus, row, got, corpus["bam"])


# ------------------------------------------------------------------------------------------- ShardedConsensus
class _MaskedRanks(D.ShardedConsensus):
    """A rank of _Lockstep's job built with its primer arrays or its rows of K10's drop list."""

    extra = {}  # rank -> dict(primers=..., drops=...)

    def __init__(self, shard, device, mode="fused", group=None):
        super().__init__(shard, device, mode=mode, group=group, **self.extra.get(group.rank, {}))


def _lockstep(monkeypatch, corpus, world, mates):
    path = corpus["bam"]
    batch = bamio.read_alignment(path, min_base_quality=20, mates=mates)
    plain = bamio.read_alignment(path)
    names = plain.contig_names
    pre = _merged_pre(path, names, 20, 0, 0, corpus["rows"])
    extra = {}
    if mates:  # the parent masks once (K9, K10p, K10); every rank takes back its own drop rows
        shards, drops, _ = K._masked_for_shards(batch, P.load_primers(corpus["bed"]), True)
        o = MO.Masked(path, names, pre_masked=pre)
        want_ev = PO.pileup(plain, o.masked())[1]  # (every row: the ranks write the dropped ones too)
        want = o.pileup(plain, dict(zip(names, plain.contig_slot.tolist())))[0]
    else:  # every rank masks its own primer bases
        shards = batch
        arrays = P.primer_arrays(P.load_primers(corpus["bed"]), names, batch.contig_len)
        want, want_ev = PO.pileup(plain, pre)
    idx = [D.shard_indices(batch, r, world, "reads") for r in range(world)]
    for r in range(world):
        extra[r] = dict(drops=D.shard_drops(drops, idx[r])) if mates else dict(primers=arrays)
    monkeypatch.setattr(_MaskedRanks, "extra", extra)
    monkeypatch.setattr(D, "ShardedConsensus", _MaskedRanks)
    drv = SE._Lockstep(monkeypatch, batch, world, "fused", masked=shards)
    drv.want, drv.want_ev = want, want_ev
    if mates:
        drv.shard_want = [_reverse_oracle(o, plain, i, path) for i in idx]
    else:
        drv.shard_want = [PO.pileup(bamio.select_reads(plain, i), [pre[k] for k in i])[0] for i in idx]
    return drv


@pytest.mark.parametrize("mates", [True, False], ids=["drops", "primers"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_epochs_with_primers_and_drops(monkeypatch, corpus, world, mates):
    """Every epoch's calls (majority and IUPAC) equal the oracle vote of the whole masked table, each rank's table the
    oracle table of its shard's reads with the same masks and drops, and the dirty map covers every non-zero sector."""
    _lockstep(monkeypatch, corpus, world, mates).run(SE._iupac_on_odd_epochs)


# ------------------------------------------------------------------------------------------- config 4's shape
def _sha(x) -> str:
    return hashlib.sha256(x.encode() if isinstance(x, str) else np.ascontiguousarray(x).tobytes()).hexdigest()


def test_config4_shape_as_amplicon_pairs(tmp_path):
    """Config 4's depth and read length (200x of 2 x 150 bp) as tiled amplicon pairs over 100 kb, primers and mates
    on, IUPAC 0.6: the consensus text and qualities against the oracle's by sha256.  The oracle table is the C walk
    fed py_moracle.Masked's merged mask lists."""
    b, flag, frag, rows = synth.amplicon_pairs(6, 100_000, 200, read_len=150)
    path = str(tmp_path / "amp.bam")
    synth.write_paired_bam(path, b, flag, frag)
    bed = tmp_path / "amp.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
    got = K.bam_to_consensus(path, iupac_threshold=0.6, qualities=True, primers=str(bed), mask_overlaps=True)
    plain = bamio.read_alignment(path)
    counts, qpos = PO.masked_arrays(plain, rows)
    ends = np.cumsum(counts)
    pre = [qpos[e - n:e].tolist() for n, e in zip(counts.tolist(), ends.tolist())]
    o = MO.Masked(path, plain.contig_names, pre_masked=pre)
    table, events = o.pileup(plain, dict(zip(plain.contig_names, plain.contig_slot.tolist())))
    assert o.stats()[0] > 50_000
    calls = ioracle.vote_iupac(table, 1, 0.6)
    ins = H.events_to_dicts(plain, events)
    s0, L = int(plain.contig_slot[0]), int(plain.contig_len[0])
    seq, qual = fqoracle.fastq(table, calls, s0, L, {s - s0: d for s, d in ins.items()})
    r = got.consensuses[0]
    assert (_sha(r.sequence), _sha(r.qualities)) == (_sha(seq), _sha(qual))
    assert got.refs_reports["ctg0"].count("- mate overlaps: %d pairs" % o.stats()[0]) == 1
