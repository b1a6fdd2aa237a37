"""Amplicon primer masking (`--primers`, an extension) without a GPU: the BED loader and the per-contig arrays, K9 from
its CUDA source under the kernel emulator against the per-record oracle (oracle/py_poracle.py) on the fuzz and limit
corpora and on hand-made edge cases, the emulated pileup + K1q of the masked batch against the oracle's table, the
planted truth set, and the CLI / REPORT / VCF header plumbing."""
import gzip
import os

import numpy as np
import pytest

import emu_harness as E
import limit_cases as LC
import primer_cases as PC
from fuzz_cases import random_case
from kindel_b200 import bamio, cli
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from oracle import py_poracle as PO

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")


# ------------------------------------------------------------------------------------------------ BED
def _load(tmp_path, text, name="s.bed", gz=False):
    p = tmp_path / name
    data = text.encode()
    p.write_bytes(gzip.compress(data) if gz else data)
    return P.load_primers(p)


def test_bed_rows_headers_crlf_gzip(tmp_path):
    text = ("track name=primers\r\nbrowser position t:1-10\r\n# a comment\r\n\r\n"
            "t\t10\t34\tamp1_LEFT\t1\t+\r\nt\t400\t424\r\n  \nother\t5\t9\tx\t2\t-\n")
    for gz in (False, True):
        ps = _load(tmp_path, text, "s.bed.gz" if gz else "s.bed", gz)
        assert ps.name == ("s.bed.gz" if gz else "s.bed")
        assert ps.chrom == ("t", "t", "other")
        assert ps.start.tolist() == [10, 400, 5] and ps.end.tolist() == [34, 424, 9]
        assert ps.line.tolist() == [5, 6, 8]
    # space-separated rows are read too; a contig the alignment lacks is ignored
    ps = _load(tmp_path, "t 3 7\nchrZ 0 99999\n")
    arr = P.primer_arrays(ps, ["t"], [50])
    assert arr.n_intervals == 1 and arr.contig_off.tolist() == [0, 1]


@pytest.mark.parametrize("text, line, what", [
    ("t\t1\t5\nt\t7\n", 2, "needs chrom, start and end"),
    ("#h\nt\tx\t5\n", 2, "must be integers"),
    ("t\t1\t5.5\n", 1, "must be integers"),
])
def test_bed_parse_errors_name_the_line(tmp_path, text, line, what):
    with pytest.raises(ValueError, match=r"s\.bed line %d: .*%s" % (line, what)):
        _load(tmp_path, text)


@pytest.mark.parametrize("row", ["t\t-1\t5", "t\t5\t5", "t\t9\t5", "t\t40\t51"])
def test_bed_interval_errors_name_the_line(tmp_path, row):
    ps = _load(tmp_path, "t\t1\t5\n" + row + "\nu\t-5\t-9\n")  # (rows of other contigs are not checked)
    with pytest.raises(ValueError, match=r"s\.bed line 2: interval"):
        P.primer_arrays(ps, ["t"], [50])


def test_bed_end_at_contig_length_is_allowed(tmp_path):
    arr = P.primer_arrays(_load(tmp_path, "t\t0\t50\nt\t0\t50\n"), ["t"], [50])
    assert arr.n_intervals == 2


def _plain_window(intervals, s, e):
    left = [b for a, b in intervals if a <= s < b]
    right = [a for a, b in intervals if a <= e < b]
    return (max(left) if left else s), (min(right) if right else e + 1)


def test_arrays_match_the_plain_interval_loop():
    rng = np.random.default_rng(5)
    for trial in range(40):
        contigs = [("c%d" % k, int(rng.integers(1, 300))) for k in range(int(rng.integers(1, 4)))]
        rows = PC.random_rows(rng, contigs, n_max=30)
        arr = P.primer_arrays(PC.primer_set(rows), [c for c, _ in contigs], [n for _, n in contigs])
        assert arr.n_contigs == len(contigs)
        for c, (name, Lc) in enumerate(contigs):
            iv = PO.contig_intervals(rows, name)
            assert int(arr.contig_off[c + 1] - arr.contig_off[c]) == len(iv)
            for _ in range(60):
                s = int(rng.integers(-2, Lc + 2))
                e = s + int(rng.integers(0, 40))
                assert P.window(arr, c, s, e) == _plain_window(iv, s, e), (trial, name, s, e)


# ------------------------------------------------------------------------------------------------ K9
def _random_quals(text, seed):
    """The SAM text with random qualities (a few below 20) on every record with a SEQ."""
    rng = np.random.default_rng(seed)
    out = []
    for line in text.splitlines():
        f = line.split("\t")
        if not line.startswith("@") and len(f) >= 11 and f[9] != "*":
            f[10] = "".join(chr(33 + int(q)) for q in rng.choice([5, 15, 30, 40], len(f[9]), p=[.1, .1, .4, .4]))
        out.append("\t".join(f))
    return "\n".join(out) + "\n"


def _sam_quals(path, contig_names):
    """Qualities of the kept reads in read order (0xff for QUAL `*`)."""
    groups = {}
    with open(path) as fh:
        for line in fh:
            f = line.rstrip("\n").split("\t")
            if line.startswith("@") or len(f) < 11 or (int(f[1]) & 4) or len(f[9]) <= 1:
                continue
            groups.setdefault(f[2], []).append(b"\xff" * len(f[9]) if f[10] == "*" else
                                               bytes(ord(c) - 33 for c in f[10]))
    return np.frombuffer(b"".join(b"".join(groups.get(n, [])) for n in contig_names), dtype=np.uint8)


def _check_case(path, rows, mbq, what):
    """K9 under the emulator on the file's batch (masked below mbq at decode) against the oracle: the mask list, the
    nibbles, the totals, and the pileup + K1q table."""
    plain = bamio.read_alignment(path)
    batch = bamio.read_alignment(path, min_base_quality=mbq) if mbq else plain
    qual = _sam_quals(path, plain.contig_names) if mbq else None
    arrays = P.primer_arrays(PC.primer_set(rows), batch.contig_names, batch.contig_len)
    masked, tot = PC.emu_primers(batch, arrays)
    prim = PO.masked_by_read(path, batch.contig_names, rows)
    assert len(prim) == batch.n_reads, what
    assert PC.mask_lists(masked) == PO.merged_mask(prim, qual, batch.seq_len, mbq), what
    assert tot[2:].tolist() == [sum(1 for x in prim if x), sum(len(x) for x in prim)], what
    for r in range(batch.n_reads):
        want = PC.nibbles(batch, r)
        for q in prim[r]:
            want[q] = 15
        assert PC.nibbles(masked, r) == want, (what, r)
    try:
        want_t, want_ev = PO.pileup(plain, prim, qual, mbq)
    except (IndexError, KeyError) as exc:
        with pytest.raises(type(exc)):
            E.pileup_pipeline(masked)
        return tot
    got, ev = E.pileup_pipeline(masked)
    E.unmask(masked, got)
    assert np.array_equal(got, want_t), what
    assert np.array_equal(ev, want_ev), what
    return tot


@needs_emu
@pytest.mark.parametrize("mbq", [0, 20])
def test_k9_fuzz_cases_against_the_oracle(tmp_path, mbq):
    rng = np.random.default_rng(11 + mbq)
    n_masked = 0
    for seed in range(60):
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(_random_quals(random_case(seed), seed))
        try:
            b = bamio.read_alignment(p, min_base_quality=mbq)
        except (ValueError, KeyError):
            continue
        rows = PC.random_rows(rng, list(zip(b.contig_names, b.contig_len.tolist())))
        n_masked += int(_check_case(str(p), rows, mbq, "fuzz%d" % seed)[3])
    assert n_masked > 100  # the corpus does mask


@needs_emu
@pytest.mark.parametrize("name", sorted(LC.GROUPS))
def test_k9_limit_cases_against_the_oracle(tmp_path, name):
    p = tmp_path / ("limit_%s.sam" % name)
    p.write_text(LC.sam_text(name))
    b = bamio.read_alignment(p)
    rng = np.random.default_rng(len(name))
    rows = []
    for c, Lc in zip(b.contig_names, b.contig_len.tolist()):  # a tiled scheme: ~25 bp primers every ~200 bp
        for a in range(0, max(Lc - 30, 1), 200):
            n = int(rng.integers(22, 31))
            rows += [(c, a, min(a + n, Lc)), (c, max(a + 200 - n, 0), min(a + 200, Lc))]
        rows.append((c, max(Lc - 25, 0), Lc))
    for mbq in (0, LC.MASK_QUAL):
        _check_case(str(p), [r for r in rows if r[1] < r[2]], mbq, name)


EDGE_SAM = """@SQ\tSN:c0\tLN:40
@SQ\tSN:c1\tLN:30
pos0\t0\tc0\t0\t60\t6M\t*\t0\t0\tACGTAC\t*
leadD\t0\tc0\t2\t60\t3D6M\t*\t0\t0\tACGTAC\t*
leadI\t0\tc0\t2\t60\t2I6M\t*\t0\t0\tGGACGTAC\t*
noM\t0\tc0\t3\t60\t6S\t*\t0\t0\tACGTAC\t*
insOnly\t0\tc0\t3\t60\t4I\t*\t0\t0\tACGT\t*
inside\t0\tc0\t22\t60\t5M\t*\t0\t0\tACGTA\t*
clipped\t0\tc0\t4\t60\t3S6M2I4M2S\t*\t0\t0\tTTTACGTACGGACGTAA\t*
midS\t0\tc0\t12\t60\t3M2S3M\t*\t0\t0\tACGTACGT\t*
tail\t16\tc0\t33\t60\t5M3S\t*\t0\t0\tACGTAGGG\t*
exotic\t0\tc0\t21\t60\t4M1D4M\t*\t0\t0\tARGTACGT\t*
whole\t0\tc1\t1\t60\t30M\t*\t0\t0\tACGTACGTACGTACGTACGTACGTACGTAC\t*
"""
EDGE_ROWS = [("c0", 0, 6), ("c0", 0, 3), ("c0", 20, 30), ("c0", 24, 28), ("c0", 34, 40), ("c0", 3, 9),
             ("c1", 0, 30), ("nowhere", 1, 2)]


@needs_emu
def test_k9_edge_cases(tmp_path):
    p = tmp_path / "edge.sam"
    p.write_text(EDGE_SAM)
    tot = _check_case(str(p), EDGE_ROWS, 0, "edge")
    prim = PO.masked_by_read(str(p), ["c0", "c1"], EDGE_ROWS)
    b = bamio.read_alignment(p)
    # read order: c0's reads in file order, then c1's
    got = dict(zip([ln.split("\t")[0] for ln in EDGE_SAM.splitlines()[2:]], prim))
    assert got["pos0"] == [1, 2, 3, 4, 5]         # s = -1 is in no primer; e = 4 lies in [0, 6) and [3, 9)
    assert got["leadD"] == [0, 1, 2, 3, 4]        # s = 4 in [0, 6) and [3, 9): up to 9; e = 9 in none
    assert got["leadI"] == [2, 3, 4, 5, 6, 7]     # the inserted bases are never masked
    assert got["noM"] == [] and got["insOnly"] == []
    assert got["inside"] == [0, 1, 2, 3, 4]       # both ends in [20, 30)
    assert got["clipped"] == [3, 4, 5, 6, 7, 8]   # s = 3 in [3, 9); clipped and inserted bases stay
    assert got["midS"] == []                      # cursors 11..13 and 16..18: in no primer
    assert got["tail"] == [2, 3, 4]               # e = 36 in [34, 40); the right clip stays
    assert got["exotic"] == list(range(8))        # the R is masked: no KeyError
    assert got["whole"] == list(range(30))
    assert int(tot[3]) == sum(len(x) for x in prim)
    assert b.n_reads == 11


@needs_emu
def test_k9_with_no_primer_on_the_batch_changes_nothing(tmp_path):
    p = tmp_path / "edge.sam"
    p.write_text(EDGE_SAM)
    b = bamio.read_alignment(p)
    for rows in ([], [("nowhere", 0, 10), ("c9", 3, 4)]):
        arrays = PC.arrays_for(b, rows)
        assert arrays.n_intervals == 0
        masked, tot = PC.emu_primers(b, arrays)
        assert tot.tolist() == [0, 0, 0, 0] and masked.n_masked == 0
        assert np.array_equal(masked.seq4, b.seq4)
    # an empty BED file loads, and so does one with headers only
    (tmp_path / "e.bed").write_text("")
    (tmp_path / "h.bed").write_text("track x\n# y\n")
    for f in ("e.bed", "h.bed"):
        assert P.primer_arrays(P.load_primers(tmp_path / f), b.contig_names, b.contig_len).n_intervals == 0


@needs_emu
def test_k9_keeps_quality_masked_reads_without_primer_bases(tmp_path):
    p = tmp_path / "q.sam"
    p.write_text(_random_quals(EDGE_SAM, 3))
    b = bamio.read_alignment(p, min_base_quality=20)
    assert b.n_masked > 0
    masked, tot = PC.emu_primers(b, PC.arrays_for(b, [("c0", 24, 28)]))  # primes only the `inside` read's end
    assert PC.mask_lists(masked)[:5] == PC.mask_lists(b)[:5]
    assert int(tot[2]) == 1


# ------------------------------------------------------------------------------------------------ truth set
@needs_emu
def test_planted_truth_set_emulated(tmp_path):
    bam, bed, fa, ref, sample = PC.write(tmp_path)
    plain = bamio.read_alignment(bam)
    arrays = P.primer_arrays(P.load_primers(bed), plain.contig_names, plain.contig_len)
    masked, tot = PC.emu_primers(plain, arrays)
    assert int(tot[2]) == plain.n_reads  # every read starts and ends in a primer
    t0, ev0 = E.pileup_pipeline(plain)
    t1, ev1 = E.pileup_pipeline(masked)
    E.unmask(masked, t1)
    assert np.array_equal(t0[5:], t1[5:]) and np.array_equal(ev0, ev1)  # only columns 0-4 change
    c0, c1 = E.vote(t0), E.vote(t1)
    assert "ACGT"[c0[PC.SITE] & 7] == ref[PC.SITE] != sample[PC.SITE]
    assert "ACGT"[c1[PC.SITE] & 7] == sample[PC.SITE]
    prim = PO.masked_by_read(str(bam), plain.contig_names, PO.read_bed_rows(str(bed)))
    want, _ = PO.pileup(plain, prim)
    assert np.array_equal(t1, want)


# ------------------------------------------------------------------------------------------------ interface
def test_cli_takes_primers_on_every_pileup_command():
    parser = cli.build_parser()
    for cmd in (["consensus"], ["weights"], ["features"], ["variants"], ["variants", "--vcf"]):
        a = parser.parse_args(cmd + ["x.bam", "--primers", "s.bed"])
        assert cli._filters(a)["primers"] == "s.bed"
        assert "primers" not in cli._filters(parser.parse_args(cmd + ["x.bam"]))


def test_report_and_vcf_header_lines():
    args = ("t", K.DepthRange(0, 3), [None] * 3, None, "a.bam", False, 1, 9, 0.1, False, False)
    plain = K.build_report(*args)
    with_p = K.build_report(*args, filters=(20, 0, 0), primers="scheme.bed").splitlines()
    assert "- primers: scheme.bed" not in plain
    at = with_p.index("- primers: scheme.bed")
    assert with_p[at - 1].startswith("- exclude_flags:") and with_p[at + 1] == "observations:"
    assert K.build_report(*args, primers="s.bed").splitlines()[10] == "- primers: s.bed"

    class Run:
        batch = bamio.ReadBatch(contig_names=["t"], contig_len=np.array([5], np.int32),
                                contig_read_off=np.zeros(2, np.int64), contig_slot=np.zeros(1, np.int64), n_slots=512,
                                ref_start=np.zeros(0, np.int32), seq_off=np.zeros(0, np.uint32),
                                l_seq=np.zeros(0, np.int32), seq_len=np.zeros(0, np.int32),
                                cig_off=np.zeros(1, np.uint32), cigar=np.zeros(0, np.uint32),
                                seq4=np.zeros(0, np.uint32))
        primers = P.PrimerSet("scheme.bed", (), np.zeros(0), np.zeros(0), np.zeros(0))

    lines = K._vcf_header(Run(), 1, 0.01, None, strand=True)
    assert lines[3] == "##kindelPrimers=scheme.bed" and lines[2].startswith("##kindelVariants=")
    Run.primers = None
    assert not any(x.startswith("##kindelPrimers") for x in K._vcf_header(Run(), 1, 0.01, None))


def test_primer_arrays_travel_through_a_file(tmp_path):
    rng = np.random.default_rng(2)
    contigs = [("a", 100), ("b", 50)]
    arr = P.primer_arrays(PC.primer_set(PC.random_rows(rng, contigs)), ["a", "b"], [100, 50])
    P.save_arrays(str(tmp_path / "p.npz"), arr)
    back = P.load_arrays(str(tmp_path / "p.npz"))
    for f in ("contig_off", "start_sorted", "end_max", "end_sorted", "start_min"):
        assert np.array_equal(getattr(back, f), getattr(arr, f)) and getattr(back, f).dtype == getattr(arr, f).dtype


def test_primers_path_or_set():
    assert P.as_primer_set(None) is None
    ps = PC.primer_set([("t", 1, 2)])
    assert P.as_primer_set(ps) is ps
    assert os.path.basename(ps.name) == "scheme.bed"


@needs_emu
def test_scaled_oracle_and_amplicon_batches_under_the_emulator():
    """py_poracle.masked_by_batch (the oracle's vectorised form for the large GPU checks) and the synthetic amplicon
    batch, against K9 under the emulator."""
    from kindel_b200 import synth

    plain = synth.mixed_reads(3, [6_000], 30, 0.05)
    rows = synth.tiled_scheme(2, plain.contig_names, plain.contig_len)
    masked, tot = PC.emu_primers(plain, PC.arrays_for(plain, rows))
    want = PO.masked_by_batch(plain, rows)
    assert PC.mask_lists(masked) == [x.tolist() for x in want] and int(tot[3]) > 0
    amp, arows = synth.amplicon_reads(1, 4_000, 20)
    masked, tot = PC.emu_primers(amp, PC.arrays_for(amp, arows))
    assert int(tot[2]) == amp.n_reads  # every read begins or ends in a primer
    assert PC.mask_lists(masked) == [x.tolist() for x in PO.masked_by_batch(amp, arows)]
