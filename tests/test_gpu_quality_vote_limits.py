"""The quality vote (`consensus --quality-vote`) at the engine's limits on the device: K11w + K11g-w on every limit
group under every plan, both dispatch branches and the deep column, into outputs preset to two patterns and through
engine.quality_weights; K2w over those sums against the restatement; thousands of contigs and a deep tile of long
reads; the consensus matrix; the CLI; and two GPUs against one."""
from __future__ import annotations

import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

import helpers as H
import limit_cases as LC
import qual_limit_cases as QL
import quality_vote_cases as QVC
import qvote_limit_cases as QVL
from kindel_b200 import _ffi, bamio, engine
from kindel_b200 import kindel as K
from test_qual_limits import files, pairs, permuted, tiled  # noqa: F401
from test_quality_vote import assert_wsum, weight_oracle
from test_quality_vote_limits import check_row, check_vote_consensus, deep, filled, per_read, vote_kwargs  # noqa: F401
from test_quality_vote_limits import vpiled, wsums_of

pytestmark = pytest.mark.gpu
GROUPS = list(LC.GROUPS)
POISON = (0xA5A5A5A5A5A5A5A5, 0x0F0F0F0F0F0F0F0F)


def device_weights(batch, qual8, poison=0):
    """kdl_quality_weights (K0 + K11w + K11g-w) on the device into wsum preset to a pattern, so that a slot the kernels
    leave unwritten shows.  (wsum uint64 [4, n_slots], the DeviceBatch)."""
    dev = torch.device("cuda", 0)
    db = engine.upload(batch, dev)
    n = int(db.n_slots)
    with torch.cuda.device(dev):
        wsum = torch.from_numpy(np.full((4, n), POISON[poison], dtype=np.uint64).view(np.int64)).to(dev)
        q = torch.from_numpy(qual8).to(dev)
        rc = _ffi.load().kdl_quality_weights(C.byref(db.struct), q.data_ptr(), wsum.data_ptr(), n,
                                             engine._stream_ptr(dev))
        _ffi.check(rc, "kdl_quality_weights")
    torch.cuda.synchronize()
    return wsum.cpu().numpy().view(np.uint64), db


def twice(batch, qual8):
    """K11w + K11g-w into outputs preset to two patterns, and once through engine.quality_weights: the same bits.  K2w
    over the sums equals restated_vote."""
    a, db = device_weights(batch, qual8, 0)
    b, _ = device_weights(batch, qual8, 1)
    w = engine.quality_weights(db, torch.from_numpy(qual8).to(db.device))
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(a, w.cpu().numpy().view(np.uint64))
    counts, _ = engine.pileup(db)
    calls, qual = engine.vote_quality(counts, w, 1)
    want = QVC.restated_vote(counts.cpu().numpy(), a.astype(object), 1)
    np.testing.assert_array_equal(calls.cpu().numpy(), want[0])
    np.testing.assert_array_equal(qual.cpu().numpy(), want[1])
    return a


@pytest.mark.parametrize("name", GROUPS)
def test_k11w_on_every_limit_group(files, name):
    for plan in QL.PLANS:
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        assert_wsum(twice(batch, batch.qual8), wsums_of(files, bam, batch), "%s %s" % (name, plan))


@pytest.mark.parametrize("name", GROUPS)
def test_sorted_and_permuted_branches(files, name):
    for plan in ("uniform", "bam_wide"):
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        ub, uq8 = permuted(batch, len(name))
        assert tiled(batch) and not tiled(ub)
        a = twice(batch, batch.qual8)
        np.testing.assert_array_equal(a, twice(ub, uq8))
        assert_wsum(a, wsums_of(files, bam, batch), "%s %s" % (name, plan))


@pytest.mark.parametrize("variant", QVL.DEEP_VARIANTS)
def test_the_deep_column(deep, variant):
    _, bam = deep[variant]
    batch = bamio.read_alignment(bam, qual=True)
    got = twice(batch, batch.qual8)
    QVL.check_deep_shape(batch, got if variant != "minority" else None)
    assert (int(got[0, QVL.DEEP_SLOT]), int(got[2, QVL.DEEP_SLOT])) == QVL.deep_want(variant)
    assert_wsum(got, weight_oracle(batch, per_read(batch)), variant)
    ub, uq8 = permuted(batch, 4)
    np.testing.assert_array_equal(twice(ub, uq8), got)


# ------------------------------------------------------------------------------------------- thousands of contigs
@pytest.fixture(scope="module")
def many(tmp_path_factory):
    d = tmp_path_factory.mktemp("qvote_many_gpu")
    return {sh: QL.write_many_contigs(d, 2500, 4, sh) for sh in (False, True)}


@pytest.mark.parametrize("shuffled", [False, True], ids=["header_order", "shuffled"])
def test_thousands_of_contigs(many, shuffled):
    sam, bam, _, _ = many[shuffled]
    for path in (bam, sam):
        batch = bamio.read_alignment(path, qual=True)
        QL.check_shapes(batch, 2500, shuffled)
        assert batch.n_contigs >= 2000
        want = wsums_of({"sums": {}}, bam, batch)
        assert_wsum(twice(batch, batch.qual8), want, path)
        ub, uq8 = permuted(batch, 6)
        assert_wsum(twice(ub, uq8), want, "permuted " + path)
    path = sam if shuffled else bam
    got = K.bam_to_consensus(path, quality_vote=True, qualities=True)
    check_vote_consensus(got, QVL.QualityVotePiled(bam, bamio.read_alignment(path, qual=True)), path, what=path)


def test_a_deep_tile_of_long_reads(tmp_path):
    """3600 reads start inside one 512-slot tile, with lengths up to 8192, beside a background that reaches the tile
    from the left: K11w stages the tile in four chunks, through K11w and through bam_to_consensus."""
    rng = random.Random(12)
    L, t0 = 30000, 8192
    rows = []
    for _ in range(3600):
        n = rng.randint(2, 8192) if rng.random() < 0.3 else rng.randint(2, 300)
        rows.append((t0 + rng.randrange(512), n))
    for _ in range(400):
        rows.append((rng.randrange(0, t0), rng.randint(2, 8192)))
    rows = sorted((min(p, L - n), n) for p, n in rows)
    qrng = np.random.default_rng(12)
    recs = [(0, p, 0, [(n << 4) | 0], "".join(rng.choice("ACGTN") for _ in range(n)), "d%d" % k, 60,
             qrng.integers(0, 94, n, dtype=np.int64).astype(np.uint8).tobytes()) for k, (p, n) in enumerate(rows)]
    path = str(tmp_path / "deep.bam")
    bamio.write_bam(path, [("deep", L)], recs)
    batch = bamio.read_alignment(path, qual=True)
    assert tiled(batch) and batch.n_complex == 0
    start = batch.ref_start.astype(np.int64)
    assert int(((start >= t0) & (start < t0 + 512)).sum()) >= 3 * 1024 and int(batch.seq_len.max()) > 8000
    want = wsums_of({"sums": {}}, path, batch)
    assert_wsum(twice(batch, batch.qual8), want)
    ub, uq8 = permuted(batch, 3)
    assert_wsum(twice(ub, uq8), want, "permuted")
    got = K.bam_to_consensus(path, quality_vote=True, qualities=True)
    check_vote_consensus(got, QVL.QualityVotePiled(path, batch), path)


# ------------------------------------------------------------------------------------------- the consensus
@pytest.mark.parametrize("k", range(len(QVL.vote_matrix())))
def test_vote_matrix_on_the_device(filled, k):
    row = QVL.vote_matrix()[k]
    for path in (filled["bam"], filled["sam"]):
        check_row(filled, row, K.bam_to_consensus(path, **vote_kwargs(filled, row)), path)


def test_cli_with_primers_mates_and_filters(filled):
    """`consensus --quality-vote --fastq` with primers, mates, filters, min_depth, -t and -u prints the oracle's FASTQ,
    and its stderr REPORT is the oracle's."""
    path = filled["bam"]
    args = [sys.executable, "-m", "kindel_b200", "consensus", "--quality-vote", "--fastq", "--min-base-quality", "20",
            "--min-mapq", "30", "--exclude-flags", "0x400", "--primers", filled["bed"], "--mask-overlaps",
            "--min-depth", "3", "-t", "-u", path]
    res = subprocess.run(args, capture_output=True, text=True, cwd=H.ROOT, env=dict(os.environ, PYTHONPATH=H.ROOT))
    assert res.returncode == 0, res.stderr
    p = vpiled(filled, 20, 30, 0x400, True, True)
    want = p.consensus(None, 3, False, True, True)
    assert res.stdout == "".join("@%s_cns\n%s\n+\n%s\n" % (n, s, q) for n, s, _, q, _ in want)
    assert res.stderr.endswith("\n".join(p.reports(path, None, 3, False, True, True, min_overlap=7).values()) + "\n")
    assert "- quality-vote sites: " in res.stderr


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus_equal_one(filled, pairs):
    for inp in (filled, pairs):
        kw = dict(min_base_quality=20, primers=inp["bed"], mask_overlaps=True, qualities=True, quality_vote=True,
                  realign=True)
        one = K.bam_to_consensus(inp["bam"], devices=1, **kw)
        two = K.bam_to_consensus(inp["bam"], devices=2, **kw)
        assert [(r.sequence, r.qualities) for r in two.consensuses] == \
            [(r.sequence, r.qualities) for r in one.consensuses]
        assert two.refs_reports == one.refs_reports
        inp.setdefault("piled", {})
        inp.setdefault("layout", bamio.read_alignment(inp["bam"], qual=True))
        check_vote_consensus(two, vpiled(inp, 20, 0, 0, True, True), inp["bam"], realign=True)
