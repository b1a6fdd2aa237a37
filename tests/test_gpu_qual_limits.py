"""K11 + K11g (`variants --vcf --qual`) at the engine's limits on the device, against oracle/py_qvoracle.py: every limit
group under every quality plan (into outputs preset to two patterns, and through engine.quality_sums: integer sums,
so the same bits every time, and every slot written), the sorted and the permuted branch, the
constant-quality invariant against engine.pileup, thousands of contigs, a tile of several 1024-read chunks with reads
of up to 8192 bases, and a real two-GPU `variants_vcf(qual=True)`."""
from __future__ import annotations

import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

import limit_cases as LC
import qual_limit_cases as QL
from kindel_b200 import _ffi, bamio, engine
from kindel_b200 import kindel as K
from oracle import coracle, py_cvoracle as CV, py_qvoracle as QV
from test_qual_limits import (SHARD_ROWS, _vcf_kwargs, files, mixed, pairs, permuted, sums_of,  # noqa: F401
                              tiled)
from test_variant_qual import _oracle, assert_sums, corpus, laid_out  # noqa: F401
from test_vcf_combined import SOURCE

pytestmark = pytest.mark.gpu
GROUPS = list(LC.GROUPS)
POISON = ((0xA5A5A5A5, 0x5A5A5A5A5A5A5A5A), (0x3C3C3C3C, 0x0F0F0F0F0F0F0F0F))


def device_sums(batch, qual8, poison=0):
    """kdl_quality_pileup (K0 + K11 + K11g) on the device into outputs preset to a pattern, so that a slot the kernels
    leave unwritten shows (engine.quality_sums allocates them with torch.empty, which may hand back memory that still
    holds an earlier run's sums).  (qsum uint32 [4, n_slots], emass uint64 [n_slots], the DeviceBatch)."""
    dev = torch.device("cuda", 0)
    db = engine.upload(batch, dev)
    n = int(db.n_slots)
    pq, pe = POISON[poison]
    with torch.cuda.device(dev):
        qsum = torch.from_numpy(np.full((4, n), pq, dtype=np.uint32).view(np.int32)).to(dev)
        emass = torch.from_numpy(np.full(n, pe, dtype=np.uint64).view(np.int64)).to(dev)
        q = torch.from_numpy(qual8).to(dev)
        rc = _ffi.load().kdl_quality_pileup(C.byref(db.struct), q.data_ptr(), qsum.data_ptr(), emass.data_ptr(), n,
                                            engine._stream_ptr(dev))
        _ffi.check(rc, "kdl_quality_pileup")
    torch.cuda.synchronize()
    return qsum.cpu().numpy().view(np.uint32), emass.cpu().numpy().view(np.uint64), db


def twice(batch, qual8):
    """K11 + K11g on the device into outputs preset to two different patterns, and once through the product's
    engine.quality_sums: the three results are the same bits."""
    a = device_sums(batch, qual8, 0)
    b = device_sums(batch, qual8, 1)
    qs, em = engine.quality_sums(a[2], torch.from_numpy(qual8).to(a[2].device))
    for x in (b[:2], (qs.cpu().numpy().view(np.uint32), em.cpu().numpy().view(np.uint64))):
        np.testing.assert_array_equal(a[0], x[0])
        np.testing.assert_array_equal(a[1], x[1])
    return a[:2]


@pytest.mark.parametrize("name", GROUPS)
def test_k11_on_every_limit_group(files, name):
    for plan in QL.PLANS:
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        assert_sums(twice(batch, batch.qual8), sums_of(files, bam, batch), "%s %s" % (name, plan))


@pytest.mark.parametrize("name", GROUPS)
def test_sorted_and_permuted_branches(files, name):
    for plan in ("uniform", "bam_wide"):
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        ub, uq8 = permuted(batch, len(name))
        assert tiled(batch) and not tiled(ub)
        a, b = twice(batch, batch.qual8), twice(ub, uq8)
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[1], b[1])
        assert_sums(a, sums_of(files, bam, batch), "%s %s" % (name, plan))


@pytest.mark.parametrize("name", GROUPS)
def test_constant_quality_against_the_pileup(files, name):
    for plan, q in QL.CONST.items():
        _, bam = files["paths"][(name, plan)]
        batch = bamio.read_alignment(bam, qual=True)
        qs, em, db = device_sums(batch, batch.qual8)
        counts = engine.pileup(db)[0][0:4].cpu().numpy().astype(np.int64)
        np.testing.assert_array_equal(counts, coracle.pileup(batch)[0][0:4])
        np.testing.assert_array_equal(qs.astype(np.int64), q * counts, err_msg=plan)
        np.testing.assert_array_equal(em.astype(object), QV.EPS[q] * counts.sum(axis=0).astype(object), err_msg=plan)


# ------------------------------------------------------------------------------------------- thousands of contigs
@pytest.fixture(scope="module")
def many(tmp_path_factory):
    d = tmp_path_factory.mktemp("many_contigs_gpu")
    return {sh: QL.write_many_contigs(d, 2500, 4, sh) for sh in (False, True)}


@pytest.mark.parametrize("shuffled", [False, True], ids=["header_order", "shuffled"])
def test_thousands_of_contigs(many, shuffled):
    sam, bam, fa, refs = many[shuffled]
    for path in (bam, sam):
        batch = bamio.read_alignment(path, qual=True)
        QL.check_shapes(batch, 2500, shuffled)
        assert batch.n_contigs >= 2000
        want = laid_out(batch, QV.quality_sums(bam))
        qs, em, db = device_sums(batch, batch.qual8)
        assert_sums((qs, em), want, path)
        counts, _ = engine.pileup(db)
        np.testing.assert_array_equal(counts.cpu().numpy(), coracle.pileup(batch)[0])
        ub, uq8 = permuted(batch, 6)
        assert_sums(device_sums(ub, uq8)[:2], want, "permuted " + path)
    got = K.variants_vcf(sam if shuffled else bam, 0, 0.0, qual=True, reference=fa, min_qual=20.0)
    want = QV.with_quality(CV.Composed(bam).vcf(SOURCE, 0, 0.0, (0, 0, 0), None, (os.path.basename(fa), refs)),
                           QV.quality_sums(bam), 20.0)
    assert got == want


# ------------------------------------------------------------------------------------------- a deep tile
def test_a_deep_tile_of_long_reads(tmp_path):
    """3600 reads start inside one 512-slot tile at random offsets, with lengths up to 8192 (so reads from far left
    of later tiles reach them too): K11 stages each tile's reads in four chunks of 1024, whose boundaries fall inside
    the warps' search windows."""
    rng = random.Random(12)
    L, t0 = 30000, 8192
    rows = []
    for _ in range(3600):
        n = rng.randint(2, 8192) if rng.random() < 0.3 else rng.randint(2, 300)
        rows.append((t0 + rng.randrange(512), n))
    for _ in range(400):  # a background that reaches the tile from the left
        n = rng.randint(2, 8192)
        rows.append((rng.randrange(0, t0), n))
    rows = sorted((min(p, L - n), n) for p, n in rows)
    qrng = np.random.default_rng(12)
    recs = [(0, p, 0, [(n << 4) | 0], "".join(rng.choice("ACGTN") for _ in range(n)), "d%d" % k, 60,
             qrng.integers(0, 94, n, dtype=np.int64).astype(np.uint8).tobytes()) for k, (p, n) in enumerate(rows)]
    path = str(tmp_path / "deep.bam")
    bamio.write_bam(path, [("deep", L)], recs)
    batch = bamio.read_alignment(path, qual=True)
    assert tiled(batch) and batch.n_complex == 0
    start = batch.ref_start.astype(np.int64)
    assert int(((start >= t0) & (start < t0 + 512)).sum()) >= 3 * 1024
    assert int(batch.seq_len.max()) > 8000
    want = laid_out(batch, QV.quality_sums(path))
    assert_sums(twice(batch, batch.qual8), want)
    ub, uq8 = permuted(batch, 3)
    assert_sums(device_sums(ub, uq8)[:2], want, "permuted")


# ------------------------------------------------------------------------------------------- two GPUs
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_variants_vcf_qual_on_two_gpus(corpus, mixed, pairs):
    inputs = [corpus, mixed, pairs, corpus, pairs, pairs]  # (the rows with mates on read overlapping pairs)
    for k, row in enumerate(SHARD_ROWS):
        inp = inputs[k]
        kw = _vcf_kwargs(inp, row)
        min_qual = (None, 30.0, 20.0)[k % 3]
        for fmt in ("bam", "sam"):
            got = K.variants_vcf(inp[fmt], qual=True, min_qual=min_qual, devices=2, **kw)
            ref = (os.path.basename(inp["fa"]), inp["refs"]) if row[3] else None
            assert got == _oracle(inp, inp["bam"], kw["min_base_quality"], kw["min_mapq"], kw["exclude_flags"],
                                  bool(row[1]), ref, kw["strand"], kw["max_sor"], bool(row[2]), min_qual), (row, fmt)
            assert got == K.variants_vcf(inp[fmt], qual=True, min_qual=min_qual, devices=1, **kw)
