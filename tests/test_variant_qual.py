"""`variants --vcf --qual`: the qualities beside the bases (decode), K11 + K11g under the kernel emulator, the QUAL model
and the product's VCF against oracle/py_qvoracle.py.  Every kdl_* call of the product path runs on the emulator."""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np
import pytest

import emu_harness as E
import qual_cases as QC
import vcf_combo_cases as VC
from kindel_b200 import bamio, cli, synth
from kindel_b200 import kindel as K
from oracle import py_cvoracle as CV
from oracle import py_moracle as MO
from oracle import py_oracle, py_qvoracle as QV, samdecode
from test_vcf_combined import SOURCE, on_the_emulator

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers for the kernel emulator")


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """The VCF combo corpus (filters, primers, reference, strand shapes) with a quality on every read."""
    d = tmp_path_factory.mktemp("qual_combo")
    contigs, recs, refs, rows = VC.vcf_combo_case(1)
    recs = QC.rewrite(recs)
    bam, sam = QC.write(d, contigs, recs, "vcq")
    fa, bed = d / "vcq.fa", d / "vcq.bed"
    fa.write_text("".join(">%s\n%s\n" % (nm, refs[nm]) for nm, _ in contigs))
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
    pc, precs = QC.planted()
    pbam, psam = QC.write(d, pc, precs, "planted")
    pfa = d / "planted.fa"
    pfa.write_text(">q\n%s\n" % QC.REF)
    return dict(bam=bam, sam=sam, fa=str(fa), bed=str(bed), refs=refs, rows=rows, contigs=contigs, recs=recs,
                pbam=pbam, psam=psam, pfa=str(pfa))


# ------------------------------------------------------------------------------------------------ helpers
def emu_quality(batch, qual8, schedule="forward"):
    """kdl_quality_pileup (K0 + K11 + K11g) on the emulator over a host batch: (qsum uint32 [4, n], emass uint64 [n]).
    The outputs start as garbage: every slot must be written."""
    lib = E.load()
    E.set_schedule(schedule, 5)
    lib.emu_set_sm_count(E.SM_COUNT)
    st, keep = E._host_batch(batch)
    n = int(batch.n_slots)
    qsum = np.full((4, n), 0xA5A5A5A5, dtype=np.uint32)
    emass = np.full(n, 0x5A5A5A5A5A5A5A5A, dtype=np.uint64)
    q8 = np.ascontiguousarray(qual8 if qual8.size else np.zeros(8, np.uint8), dtype=np.uint8)
    rc = lib.kdl_quality_pileup(C.byref(st), q8.ctypes.data, qsum.ctypes.data, emass.ctypes.data, n, None)
    assert rc == 0, lib.kdl_status_string(rc)
    del keep
    return qsum, emass


def batch_oracle(batch, qual):
    """py_qvoracle's walk over the reads of a host batch (py_oracle.records_of), qual concatenated in read order; the
    batch's N nibbles are what is masked.  (qsum int64 [4, n_slots], emass list of ints)."""
    recs = py_oracle.records_of(batch)
    qs = np.zeros((4, int(batch.n_slots)), dtype=np.int64)
    em = [0] * int(batch.n_slots)
    at = np.concatenate(([0], np.cumsum(batch.seq_len.astype(np.int64))))
    for c in range(batch.n_contigs):
        L, s0 = int(batch.contig_len[c]), int(batch.contig_slot[c])
        q4, e = [[0] * L for _ in range(4)], [0] * L
        for r in range(int(batch.contig_read_off[c]), int(batch.contig_read_off[c + 1])):
            QV.walk(L, recs[r], qual[at[r]:at[r + 1]].tolist(), set(), q4, e)
        qs[:, s0:s0 + L] = np.array(q4, dtype=np.int64).reshape(4, L)
        em[s0:s0 + L] = e
    return qs, em


def laid_out(batch, sums):
    qs = np.zeros((4, int(batch.n_slots)), dtype=np.int64)
    em = [0] * int(batch.n_slots)
    for c, nm in enumerate(batch.contig_names):
        s0, L = int(batch.contig_slot[c]), int(batch.contig_len[c])
        qs[:, s0:s0 + L] = np.array(sums[nm][0], dtype=np.int64).reshape(4, L)
        em[s0:s0 + L] = sums[nm][1]
    return qs, em


def assert_sums(got, want, what=""):
    qs, em = got
    np.testing.assert_array_equal(qs.astype(np.int64), want[0], err_msg=what)
    assert [int(x) for x in em.tolist()] == [int(x) for x in want[1]], what


# ------------------------------------------------------------------------------------------------ EPS and the model
def test_eps_table_is_the_exact_rounding():
    from decimal import Decimal, getcontext

    getcontext().prec = 80
    for q in range(94):
        x = Decimal(2) ** 32 * Decimal(10) ** (Decimal(-q) / 10)
        assert abs(Decimal(QV.EPS[q]) - x) <= Decimal("0.5"), q
        assert abs(abs(x - int(x)) - Decimal("0.5")) > Decimal("1e-6"), q  # no tie: round-half-even is safe
    src = open(os.path.join(os.path.dirname(E.EMU_DIR), "..", "kindel_b200", "csrc", "quality.cu")).read()
    body = src[src.index("kQualEps[kEpsMax + 1] = {"):]
    body = body[body.index("{") + 1:body.index("};")]
    assert [int(v.strip().rstrip("ul")) for v in body.replace("\n", " ").split(",") if v.strip()] == QV.EPS


@needs_emu
def test_eps_per_quality_on_the_device_walk(tmp_path):
    """One 8-base read per quality 0..99 on slots of its own: emass at each of its slots is EPS[min(q, 93)], qsum q."""
    contigs = [("e", 1200)]
    recs = [(0, 12 * q, 0, [(8 << 4) | 0], "ACGTACGT", "r%d" % q, 60, bytes([q] * 8)) for q in range(100)]
    path = str(tmp_path / "eps.bam")  # (SAM text stops at Q93)
    bamio.write_bam(path, contigs, recs)
    batch = bamio.read_alignment(path, qual=True)
    qsum, emass = emu_quality(batch, batch.qual8)
    for q in range(100):
        s = 12 * q
        assert emass[s:s + 8].tolist() == [QV.EPS[min(q, 93)]] * 8
        assert qsum[:, s:s + 8].sum(axis=0).tolist() == [q] * 8


def _lgamma_tail(k, lam):
    """log P(Poisson(lam) >= k) as a log-sum of lgamma terms."""
    if lam == 0.0:
        return -math.inf
    terms, j = [], k
    while True:
        t = j * math.log(lam) - lam - math.lgamma(j + 1)
        terms.append(t)
        if j > lam and t < max(terms) - 50:
            break
        j += 1
    m = max(terms)
    return m + math.log(sum(math.exp(t - m) for t in terms))


def test_allele_quality_against_a_log_space_restatement():
    unit = 3.0 * 2.0 ** 32
    n = 0
    for k in list(range(1, 40)) + [50, 100, 300, 1000, 5000]:
        for lam in (1e-6, 0.001, 0.01, 0.1, 0.5, 1.0, 2.0, 5.0, 10.0, 33.0, 100.0, 500.0, 2000.0):
            got = K.allele_quality(k, int(lam * unit))
            lt = _lgamma_tail(k, int(lam * unit) / unit)
            x = -10.0 * lt / math.log(10.0)
            if abs(x - math.floor(x) - 0.5) < 1e-6:
                continue
            want = 3000 if x >= 3000.5 else max(0, int(math.floor(x + 0.5)))
            assert got == want, (k, lam, got, x)
            assert got == QV.allele_quality(k, int(lam * unit))
            n += 1
    assert n > 400
    assert K.allele_quality(0, 12345) == 0
    assert K.allele_quality(5, 0) == K.QUAL_CAP  # no error mass: p == 0


# ------------------------------------------------------------------------------------------------ decode
def _layout_of(batch, recs_by_order):
    return bamio.qual_layout(batch, np.frombuffer(b"".join(recs_by_order), dtype=np.uint8))


def test_decoders_lay_the_qualities_beside_the_bases(corpus):
    """kdl_bam_fill_qual (BAM and the C++ SAM converter) and the Python SAM reader give the same qual8, and it holds
    samdecode's qualities of the kept records at 8 * seq_off + k, 0xff elsewhere."""
    b = bamio.read_alignment(corpus["bam"], qual=True)
    s = bamio.read_alignment(corpus["sam"], qual=True)
    p = bamio.read_sam(corpus["sam"], qual=True)
    np.testing.assert_array_equal(b.seq_off, p.seq_off)
    np.testing.assert_array_equal(b.qual8, s.qual8)
    np.testing.assert_array_equal(b.qual8, p.qual8)
    _, records = samdecode.read_alignment_file(corpus["bam"])
    by_contig = {}
    for rec in records:
        if rec.rname != "*" and not rec.flag & 4 and len(rec.seq) > 1:
            by_contig.setdefault(rec.rname, []).append(bytes(rec.qual))
    want = _layout_of(b, [q for nm in b.contig_names for q in by_contig[nm]])
    np.testing.assert_array_equal(b.qual8, want)
    assert b.qual8.shape[0] == 8 * b.seq4.shape[0]
    assert (b.qual8 == 0xFF).sum() > 0
    # with a filter: the layout follows the kept reads
    f = bamio.read_alignment(corpus["bam"], qual=True, min_mapq=30, exclude_flags=0x500, min_base_quality=20)
    g = bamio.read_sam(corpus["sam"], qual=True, min_mapq=30, exclude_flags=0x500, min_base_quality=20)
    np.testing.assert_array_equal(f.qual8, g.qual8)
    assert bamio.read_alignment(corpus["bam"]).qual8 is None


def test_a_read_without_qualities_is_an_error(tmp_path):
    contigs, recs, _, _ = VC.vcf_combo_case(1)
    bam, sam = QC.write(tmp_path, contigs, recs, "noq")
    for path in (bam, sam):
        with pytest.raises(ValueError, match="without base qualities"):
            bamio.read_alignment(path, qual=True)
        with pytest.raises(ValueError, match=os.path.basename(path)):
            bamio.read_alignment(path, qual=True)
    with pytest.raises(ValueError, match="without base qualities"):
        bamio.read_sam(sam, qual=True)
    assert bamio.read_alignment(bam).n_reads > 0  # without --qual nothing changes


# ------------------------------------------------------------------------------------------------ K11 + K11g
@needs_emu
@pytest.mark.parametrize("schedule", ["forward", "random"])
def test_k11_equals_the_oracle_on_the_corpus(corpus, schedule):
    for kw in (dict(), dict(min_base_quality=20, min_mapq=30, exclude_flags=0x500)):
        batch = bamio.read_alignment(corpus["bam"], qual=True, **kw)
        want = laid_out(batch, QV.quality_sums(corpus["bam"], kw.get("min_base_quality", 0), kw.get("min_mapq", 0),
                                               kw.get("exclude_flags", 0)))
        assert_sums(emu_quality(batch, batch.qual8, schedule), want, str(kw))


@needs_emu
@pytest.mark.parametrize("schedule", ["forward", "random"])
def test_k11_on_synthetic_reads_with_hard_reads_and_unsorted(schedule):
    """Complex reads with clips, indels and hard reads that wrap (POS 0) or stall, then the same reads unsorted."""
    for seed in (1, 2):
        batch = synth.complex_reads(seed, 3000, 30)
        assert batch.n_hard > 0 and batch.n_complex > batch.n_hard and batch.reads_sorted
        qual = synth.qualities(seed, batch.seq_len)
        want = batch_oracle(batch, qual)
        assert_sums(emu_quality(batch, bamio.qual_layout(batch, qual), schedule), want, "sorted %d" % seed)
        perm = np.random.default_rng(seed).permutation(batch.n_reads)
        ub = bamio.select_reads(batch, perm)
        assert not ub.reads_sorted
        lens = batch.seq_len.astype(np.int64)
        at = np.concatenate(([0], np.cumsum(lens)))
        uq = np.concatenate([qual[at[r]:at[r + 1]] for r in perm])
        assert_sums(emu_quality(ub, bamio.qual_layout(ub, uq), schedule), want, "unsorted %d" % seed)


@needs_emu
def test_k11_on_reads_across_tile_edges():
    """Simple reads of many lengths starting on every offset around tile edges, with a deep tile (several chunks of
    1024 reads), on two contigs."""
    rng = np.random.default_rng(11)
    rows = []
    for c, L in enumerate((1536, 1100)):
        for _ in range(1500 if c == 0 else 300):
            n = int(rng.integers(2, 300))
            edge = int(rng.choice([0, 512, 1024]))
            pos = int(np.clip(edge + rng.integers(-n - 2, 10), 0, L - n))
            rows.append((c, pos, n))
    rows.sort()
    contigs = [("t0", 1536), ("t1", 1100)]
    recs = [(c, pos, 0, [(n << 4) | 0], "".join(rng.choice(list("ACGTN"), n)), "x", 60,
             bytes(rng.integers(0, 94, n, dtype=np.uint8).tolist())) for c, pos, n in rows]  # (SAM: at most Q93)
    import tempfile

    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "edges.sam")
        QC.write_sam(path, contigs, recs)
        batch = bamio.read_alignment(path, qual=True)
        want = laid_out(batch, QV.quality_sums(path))
    assert batch.n_complex == 0 and batch.reads_sorted
    assert_sums(emu_quality(batch, batch.qual8), want)


@needs_emu
def test_constant_quality_gives_q_times_the_pileup_columns():
    batch = synth.complex_reads(3, 3000, 30)
    for q in (0, 7, 41, 93, 120):
        qual = np.full(int(batch.seq_len.sum()), q, dtype=np.uint8)
        qsum, emass = emu_quality(batch, bamio.qual_layout(batch, qual))
        counts, _ = E.pileup_pipeline(batch)
        np.testing.assert_array_equal(qsum.astype(np.int64), q * counts[0:4].astype(np.int64))
        np.testing.assert_array_equal(emass.astype(object), QV.EPS[min(q, 93)] * counts[0:4].sum(axis=0).astype(object))


# ------------------------------------------------------------------------------------------------ the VCF
def _oracle(corpus, bam, bq=0, mq=0, ex=0, pr=False, ref=None, strand=False, max_sor=None, mates=False,
            min_qual=None, a=1, r=0.01):
    cls = MO.ComposedMates if mates else CV.Composed
    rows = corpus["rows"] if pr else None
    text = cls(bam, bq, mq, ex, rows).vcf(SOURCE, a, r, (bq, mq, ex), os.path.basename(corpus["bed"]) if pr else None,
                                          ref, strand, max_sor)
    return QV.with_quality(text, QV.quality_sums(bam, bq, mq, ex, rows, mates), min_qual)


MATRIX = [  # (min_base_quality, min_mapq, exclude_flags, primers, reference, strand, max_sor, mates, min_qual, sam)
    (0, 0, 0, False, False, False, None, False, None, False),
    (20, 30, 0x500, True, True, True, 3.0, False, 30.0, True),
    (0, 0, 0, False, True, False, None, True, 20.0, False),
    (20, 0, 0, True, False, True, None, True, None, False),
    (0, 30, 0x500, False, False, False, 3.0, False, 1e9, True),
    (20, 0, 0, False, True, True, None, False, None, False),
]


@needs_emu
def test_variants_vcf_qual_on_the_emulator_equals_the_oracle(corpus, monkeypatch):
    on_the_emulator(monkeypatch)
    for bq, mq, ex, pr, ref, strand, max_sor, mates, min_qual, sam in MATRIX:
        kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, primers=corpus["bed"] if pr else None,
                  reference=corpus["fa"] if ref else None, strand=strand, max_sor=max_sor, mask_overlaps=mates)
        got = K.variants_vcf(corpus["sam"] if sam else corpus["bam"], qual=True, min_qual=min_qual, **kw)
        want = _oracle(corpus, corpus["bam"], bq, mq, ex, pr, (os.path.basename(corpus["fa"]), corpus["refs"])
                       if ref else None, strand, max_sor, mates, min_qual)
        assert got == want, (bq, mq, ex, pr, ref, strand, max_sor, mates, min_qual)
        assert "QUAL" in got and ";AQ=" in got
        off = K.variants_vcf(corpus["bam"], **kw)
        assert "##kindelQual" not in off and ";BQ=" not in off


@needs_emu
def test_planted_truth_set(corpus, monkeypatch):
    """The Q35 2 % allele passes --min-qual 30, the 2 % allele of a Q5 column is lowqual, the 20 % allele hits the
    cap, the `*`-only site has no QUAL, and the reverse-only allele of a Q10 column fails both sor and lowqual."""
    on_the_emulator(monkeypatch)
    for ref in (None, corpus["pfa"]):
        text = K.variants_vcf(corpus["pbam"], qual=True, min_qual=30, max_sor=3.0, reference=ref)
        want = _oracle(corpus, corpus["pbam"], ref=("planted.fa", {"q": QC.REF}) if ref else None, strand=True,
                       max_sor=3.0, min_qual=30.0)
        assert text == want
        recs = {int(x.split("\t")[1]) - 1: x.split("\t") for x in text.splitlines() if not x.startswith("#")}
        assert recs[QC.SITE_REAL][6] == "PASS" and int(recs[QC.SITE_REAL][5]) >= 30
        assert recs[QC.SITE_LOW][6] == "lowqual" and int(recs[QC.SITE_LOW][5]) < 30
        assert recs[QC.SITE_CAP][5] == str(K.QUAL_CAP)
        assert recs[QC.SITE_BIAS][6] == "sor;lowqual"
        if ref is None:
            assert recs[QC.SITE_DEL][4] == "*" and recs[QC.SITE_DEL][5] == "." and ";BQ=" not in recs[QC.SITE_DEL][7]
        else:  # the deletion is an INDEL record: no QUAL
            assert all(x[5] == "." for x in recs.values() if x[7].startswith("INDEL"))


def test_api_and_cli_errors(corpus, capsys):
    with pytest.raises(ValueError, match="several samples"):
        K.variants_vcf([corpus["bam"], corpus["sam"]], qual=True)
    with pytest.raises(ValueError, match="min_qual"):
        K.variants_vcf(corpus["bam"], min_qual=float("nan"))
    for argv in (["variants", corpus["bam"], "--qual"], ["variants", corpus["bam"], "--min-qual", "20"],
                 ["variants", "--vcf", "--qual", corpus["bam"], corpus["sam"]],
                 ["variants", "--vcf", "--min-qual", "nan", corpus["bam"]]):
        with pytest.raises(SystemExit):
            cli.main(argv)
    err = capsys.readouterr().err
    assert "--qual and --min-qual need --vcf" in err and "take one alignment file" in err
