"""Per-amplicon reads and depth (`kindel amplicons`, an extension) without a GPU: the named-scheme reader and its
segment arrays, K12 and K12d from their CUDA source under the kernel emulator against the per-record oracle
(oracle/py_aoracle.py) on the fuzz and limit corpora and on hand-made edges, and the API / CLI plumbing."""
import gzip

import numpy as np
import pandas as pd
import pytest

import amplicon_cases as AC
import emu_harness as E
import limit_cases as LC
import primer_cases as PC
from fuzz_cases import random_case
from kindel_b200 import bamio, cli
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from oracle import py_aoracle as AO
from oracle import py_poracle as PO

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")


# ------------------------------------------------------------------------------------------------ scheme
ARTIC = ("track name=scheme\r\n"
         "MN908947.3\t30\t54\tnCoV-2019_1_LEFT\t1\t+\r\n"
         "MN908947.3\t385\t410\tnCoV-2019_1_RIGHT\t1\t-\r\n"
         "MN908947.3\t320\t342\tnCoV-2019_2_LEFT\tnCoV-2019_2\t+\r\n"
         "MN908947.3\t315\t337\tnCoV-2019_2_LEFT_alt0\tnCoV-2019_2\t+\r\n"
         "MN908947.3\t704\t726\tnCoV-2019_2_RIGHT\tnCoV-2019_2\t-\r\n"
         "MN908947.3\t642\t664\tnCoV-2019_3_LEFT\t1\n"
         "MN908947.3\t1004\t1028\tnCoV-2019_3_RIGHT\t1\t-\tGGCATTTCTAAAGCAAGGAACC\n")


def _write(tmp_path, text, name="s.bed", gz=False):
    p = tmp_path / name
    p.write_bytes(gzip.compress(text.encode()) if gz else text.encode())
    return p


@pytest.mark.parametrize("gz", [False, True])
def test_scheme_artic_columns_alt_gzip_crlf(tmp_path, gz):
    s = P.load_scheme(_write(tmp_path, ARTIC, "s.bed.gz" if gz else "s.bed", gz))
    assert s.name == ("s.bed.gz" if gz else "s.bed")
    assert s.names == ("nCoV-2019_1", "nCoV-2019_2", "nCoV-2019_3")
    assert s.pool == ("1", "nCoV-2019_2", "1")
    assert s.start.tolist() == [30, 315, 642] and s.end.tolist() == [410, 726, 1028]
    assert s.insert_start.tolist() == [54, 342, 664] and s.insert_end.tolist() == [385, 704, 1004]
    assert s.primers.line.tolist() == [2, 3, 4, 5, 6, 7, 8]
    assert s.row_left.tolist() == [True, False, True, True, False, True, False]
    # the rows are the ones load_primers reads
    ps = P.load_primers(tmp_path / ("s.bed.gz" if gz else "s.bed"))
    assert ps.chrom == s.primers.chrom and (ps.start == s.primers.start).all() and (ps.end == s.primers.end).all()


def test_scheme_without_pool_column_writes_a_dot(tmp_path):
    s = P.load_scheme(_write(tmp_path, "c\t0\t5\tx_LEFT\nc\t20\t25\tx_RIGHT\n"))
    assert s.pool == (".",) and s.names == ("x",)


@pytest.mark.parametrize("text, what", [
    ("c\t0\t5\tx_LEFT\nc\t20\t25\n", r"s\.bed line 2: .*primer name in column 4"),
    ("c\t0\t5\tx_LEFT\nc\t20\t25\tx_R\n", r"s\.bed line 2: primer name 'x_R' has neither"),
    ("c\t0\t5\tx_LEFT\nc\tq\t25\tx_RIGHT\n", r"s\.bed line 2: start and end must be integers"),
    ("c\t-1\t5\tx_LEFT\nc\t20\t25\tx_RIGHT\n", r"s\.bed line 1: interval \[-1, 5\)"),
    ("c\t0\t5\tx_LEFT\nc\t25\t25\tx_RIGHT\n", r"s\.bed line 2: interval \[25, 25\)"),
    ("c\t0\t5\tx_LEFT\t1\nc\t20\t25\tx_RIGHT\t2\n", r"s\.bed line 2: amplicon 'x' is in pool '2' here"),
    ("c\t0\t5\tx_LEFT\n", r"s\.bed: amplicon 'x' on 'c' has no right primer"),
    ("c\t20\t25\tx_RIGHT\n", r"s\.bed: amplicon 'x' on 'c' has no left primer"),
    ("c\t0\t22\tx_LEFT\nc\t20\t25\tx_RIGHT\n", r"s\.bed: amplicon 'x' on 'c' leaves no insert"),
])
def test_scheme_errors_name_their_line_or_amplicon(tmp_path, text, what):
    with pytest.raises(ValueError, match=what):
        P.load_scheme(_write(tmp_path, text))


def test_three_column_bed_loads_as_primers_and_is_refused_as_a_scheme(tmp_path):
    p = _write(tmp_path, "c\t0\t5\nc\t20\t25\n")
    assert P.load_primers(p).start.tolist() == [0, 20]
    with pytest.raises(ValueError, match=r"line 1: .*column 4"):
        P.load_scheme(p)


def test_arrays_check_intervals_against_the_contigs_and_ignore_other_contigs(tmp_path):
    s = P.load_scheme(_write(tmp_path, "c\t0\t5\tx_LEFT\nc\t20\t31\tx_RIGHT\nz\t0\t5\ty_LEFT\nz\t9\t99\ty_RIGHT\n"))
    with pytest.raises(ValueError, match=r"s\.bed line 2: interval \[20, 31\) of 'c'"):
        P.amplicon_arrays(s, ["c"], [30])
    arr = P.amplicon_arrays(s, ["c"], [31])
    assert arr.n_amplicons == 1 and arr.amplicon.tolist() == [0]


def _plain_labels(rows, c, L, side, index):
    """Per position of [0, L] the label of one side's primers, one position at a time."""
    out = []
    for x in range(L + 1):
        amps = {index[r[3]] for r in rows if r[0] == c and r[4] == side and r[1] <= x < r[2]}
        out.append(-1 if not amps else (amps.pop() if len(amps) == 1 else -3))
    return out


def test_segment_arrays_match_a_plain_per_position_loop():
    rng = np.random.default_rng(3)
    n_ambiguous = 0
    for trial in range(30):
        contigs = [("c%d" % k, int(rng.integers(12, 500))) for k in range(int(rng.integers(1, 4)))]
        rows = AC.random_scheme_rows(rng, contigs, n_max=8)
        s = AC.scheme(rows)
        names = [c for c, _ in contigs]
        arr = P.amplicon_arrays(s, names, [n for _, n in contigs])
        table = AO.amplicon_table(rows, names)
        assert [s.names[j] for j in arr.amplicon.tolist()] == [t[1] for t in table]
        assert arr.insert_start.tolist() == [t[4] for t in table]
        assert arr.insert_end.tolist() == [t[5] for t in table]
        for c, (name, Lc) in enumerate(contigs):
            index = {t[1]: k for k, t in enumerate(table) if t[0] == name}
            for side, off, at, lab in (("L", arr.left_off, arr.left_at, arr.left_label),
                                       ("R", arr.right_off, arr.right_at, arr.right_label)):
                want = _plain_labels(rows, name, Lc, side, index)
                got = [P.segment_label(off, at, lab, c, x) for x in range(Lc + 1)]
                assert got == want, (trial, name, side)
                n_ambiguous += want.count(-3)
    assert n_ambiguous > 0  # overlapping primers of different amplicons occur


# ------------------------------------------------------------------------------------------------ K12 / K12d
def _check_case(path, rows, what, mbq=0):
    """K12 under the emulator against the oracle's labels; with the pileup of the primer-masked batch (emulated, K9 +
    K1 + K1q, equal to the oracle's own table without a quality mask), K12d against the oracle's sums over that
    table.  Returns the labels."""
    batch = bamio.read_alignment(path, min_base_quality=mbq) if mbq else bamio.read_alignment(path)
    s = AC.scheme(rows)
    arr = P.amplicon_arrays(s, batch.contig_names, batch.contig_len)
    got = AC.emu_assign(batch, arr)
    want = AO.labels_by_read(path, batch.contig_names, rows)
    assert got.tolist() == want.tolist(), what
    assert AO.labels_of_batch(batch, rows).tolist() == want.tolist(), what
    plain_rows = [r[:3] for r in rows]
    masked, _ = PC.emu_primers(batch, P.primer_arrays(s.primers, batch.contig_names, batch.contig_len))
    prim = PO.masked_by_read(path, batch.contig_names, plain_rows)
    try:
        want_t, _ = PO.pileup(bamio.read_alignment(path), prim)
    except (IndexError, KeyError):
        return got
    table, _ = E.pileup_pipeline(masked)
    E.unmask(masked, table)
    if not mbq:  # (with a quality mask the table is test_primers.py's to check)
        assert np.array_equal(table, want_t), what
    amp_table = AO.amplicon_table(rows, list(batch.contig_names))
    for md in (1, 3):
        stats = AC.emu_depth(table, batch, arr, md)
        assert stats.tolist() == [list(x) for x in AO.insert_stats(table, batch.contig_slot, list(batch.contig_names),
                                                                   amp_table, md)], (what, md)
    return got


@needs_emu
def test_k12_fuzz_cases_against_the_oracle(tmp_path):
    rng = np.random.default_rng(21)
    seen = set()
    for seed in range(60):
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            b = bamio.read_alignment(p)
        except (ValueError, KeyError):
            continue
        rows = AC.random_scheme_rows(rng, list(zip(b.contig_names, b.contig_len.tolist())))
        seen |= set(_check_case(str(p), rows, "fuzz%d" % seed).tolist())
    assert {-1, 0}.issubset(seen)


@needs_emu
@pytest.mark.parametrize("name", sorted(LC.GROUPS))
def test_k12_limit_cases_against_the_oracle(tmp_path, name):
    p = tmp_path / ("limit_%s.sam" % name)
    p.write_text(LC.sam_text(name))
    b = bamio.read_alignment(p)
    rows = []
    for c, Lc in zip(b.contig_names, b.contig_len.tolist()):  # a tiled scheme: ~25 bp primers every ~200 bp
        for k, a in enumerate(range(0, max(Lc - 250, 0) + 1, 200)):
            if a + 250 <= Lc:
                rows += [(c, a, a + 25, "%s_%d" % (c, k), "L"), (c, a + 225, a + 250, "%s_%d" % (c, k), "R")]
        if Lc >= 60:
            rows += [(c, Lc - 60, Lc - 35, c + "_end", "L"), (c, Lc - 25, Lc, c + "_end", "R")]
    _check_case(str(p), rows, name)
    _check_case(str(p), rows, name, mbq=LC.MASK_QUAL)


EDGE_SAM = """@SQ\tSN:c0\tLN:80
@SQ\tSN:c1\tLN:40
s_first\t0\tc0\t6\t60\t10M\t*\t0\t0\tACGTACGTAC\t*
s_last\t0\tc0\t10\t60\t10M\t*\t0\t0\tACGTACGTAC\t*
s_past\t0\tc0\t11\t60\t10M\t*\t0\t0\tACGTACGTAC\t*
lead_soft\t0\tc0\t6\t60\t3S10M\t*\t0\t0\tGGGACGTACGTAC\t*
lead_del\t0\tc0\t4\t60\t2D10M\t*\t0\t0\tACGTACGTAC\t*
lead_ins\t0\tc0\t6\t60\t2I8M\t*\t0\t0\tACGTACGTAC\t*
no_m\t0\tc0\t3\t60\t6S\t*\t0\t0\tACGTAC\t*
ins_only\t0\tc0\t3\t60\t4I\t*\t0\t0\tACGT\t*
right_only\t0\tc0\t28\t60\t8M\t*\t0\t0\tACGTACGT\t*
same\t0\tc0\t6\t60\t30M\t*\t0\t0\tACGTACGTACGTACGTACGTACGTACGTAC\t*
mispaired\t0\tc0\t6\t60\t60M\t*\t0\t0\tACGTACGTACGTACGTACGTACGTACGTACACGTACGTACGTACGTACGTACGTACGTAC\t*
ambiguous\t0\tc0\t23\t60\t10M\t*\t0\t0\tACGTACGTAC\t*
amp_b\t16\tc0\t21\t60\t2S45M3S\t*\t0\t0\tTTACGTACGTACGTACGTACGTACGTACGTACACGTACGTACGTACGTAGGG\t*
pos0\t0\tc0\t0\t60\t6M\t*\t0\t0\tACGTAC\t*
mid_s\t0\tc0\t11\t60\t10M10S4M\t*\t0\t0\tACGTACGTACGTACGTACGTACGT\t*
whole\t0\tc1\t1\t60\t40M\t*\t0\t0\tACGTACGTACGTACGTACGTACGTACGTACGTACGTACGT\t*
tail\t0\tc1\t31\t60\t10M4S\t*\t0\t0\tACGTACGTACGGGG\t*
"""
EDGE_ROWS = [("c0", 5, 10, "A", "L"), ("c0", 30, 35, "A", "R"),
             ("c0", 20, 25, "B", "L"), ("c0", 60, 65, "B", "R"),
             ("c0", 22, 27, "D", "L"), ("c0", 70, 75, "D", "R"),
             ("c1", 0, 4, "C", "L"), ("c1", 36, 40, "C", "R"), ("c1", 37, 40, "C", "R"),
             ("nowhere", 1, 2, "Z", "L"), ("nowhere", 5, 9, "Z", "R")]


@needs_emu
def test_k12_edge_cases(tmp_path):
    p = tmp_path / "edge.sam"
    p.write_text(EDGE_SAM)
    got = _check_case(str(p), EDGE_ROWS, "edge")
    names = [ln.split("\t")[0] for ln in EDGE_SAM.splitlines()[2:]]
    lab = dict(zip(names, got.tolist()))
    A, B, C_ = 0, 1, 3  # contig order, then start (D, starting at 22, is 2)
    assert lab["s_first"] == A and lab["s_last"] == A and lab["s_past"] == -1
    assert lab["lead_soft"] == A and lab["lead_del"] == A  # a leading clip does not move s; a deletion does
    assert lab["lead_ins"] == A
    assert lab["no_m"] == -1 and lab["ins_only"] == -1
    assert lab["right_only"] == A and lab["same"] == A
    assert lab["mispaired"] == -2 and lab["ambiguous"] == -3 and lab["amp_b"] == B
    assert lab["pos0"] == -1      # s = -1 lies outside the contig; e = 4 in no right primer
    assert lab["mid_s"] == A      # the later S advances the cursor: e = 33, in A's right primer
    assert lab["whole"] == C_ and lab["tail"] == C_  # an amplicon at the contig's end; an alt right primer


HARD_SAM = """@SQ\tSN:c0\tLN:80
past_l\t0\tc0\t72\t60\t10M\t*\t0\t0\tACGTACGTAC\t*
below0\t0\tc0\t0\t60\t2M4S\t*\t0\t0\tACGTAC\t*
clip_end\t0\tc0\t59\t60\t4M20S\t*\t0\t0\tACGTACGTACGTACGTACGTACGT\t*
late_s\t0\tc0\t60\t60\t2M30S4M\t*\t0\t0\tACGTACGTACGTACGTACGTACGTACGTACGTACGT\t*
"""


@needs_emu
def test_k12_hard_reads_with_cursors_outside_the_contig(tmp_path):
    """KDL_HARD reads whose walk runs below 0 or past L (the pileup would raise or wrap): K12 reads only their ends."""
    p = tmp_path / "hard.sam"
    p.write_text(HARD_SAM)
    b = bamio.read_alignment(p)
    assert b.n_hard >= 2
    rows = [("c0", 0, 3, "H", "L"), ("c0", 20, 25, "H", "R"), ("c0", 70, 74, "E", "L"), ("c0", 77, 80, "E", "R"),
            ("c0", 58, 62, "F", "L"), ("c0", 66, 72, "F", "R")]
    arr = P.amplicon_arrays(AC.scheme(rows), b.contig_names, b.contig_len)
    got = AC.emu_assign(b, arr)
    assert got.tolist() == AO.labels_by_read(str(p), b.contig_names, rows).tolist()
    F, E_ = 1, 2  # (H, starting at 0, is 0)
    # past_l: s = 71 in E's left primer, e = 80 = L in none; below0: s = -1 is outside the contig (not wrapped to L - 1),
    # e = 0 in no right primer; clip_end / late_s: s = 58 / 59 in F's left primer, late_s's e past L after its S stops
    assert got.tolist() == [E_, -1, F, F]


@needs_emu
def test_k12_many_contigs(tmp_path):
    n = 300
    head = "".join("@SQ\tSN:k%d\tLN:%d\n" % (c, 100 + c) for c in range(n))
    body, rows = [], []
    for c in range(n):
        L = 100 + c
        rows += [("k%d" % c, 2, 8, "a%d" % c, "L"), ("k%d" % c, L - 8, L - 2, "a%d" % c, "R")]
        body.append("r%d\t0\tk%d\t%d\t60\t20M\t*\t0\t0\t%s\t*\n" % (c, c, 3 + c % 5, "ACGT" * 5))
        body.append("q%d\t16\tk%d\t%d\t60\t20M\t*\t0\t0\t%s\t*\n" % (c, c, L - 21, "ACGT" * 5))
    p = tmp_path / "many.sam"
    p.write_text(head + "".join(reversed(body)))  # contigs first seen in an order unlike the header
    got = _check_case(str(p), rows, "many")
    assert (got >= 0).sum() == sum(1 for c in range(n) if 2 <= 2 + c % 5 < 8) + n


@needs_emu
def test_k12_synthetic_amplicon_batch():
    from kindel_b200 import synth

    amp, trows = synth.amplicon_reads(1, 6_000, 20)
    rows = []
    for k in range(len(trows) // 2):
        (c, a, b), (_, x, y) = trows[2 * k], trows[2 * k + 1]
        rows += [(c, a, b, "amp_%d" % k, "L"), (c, x, y, "amp_%d" % k, "R")]
    arr = P.amplicon_arrays(AC.scheme(rows), amp.contig_names, amp.contig_len)
    got = AC.emu_assign(amp, arr)
    assert (got >= 0).all()  # every read starts at a left primer or ends at a right one of its amplicon
    assert got.tolist() == AO.labels_of_batch(amp, rows).tolist()


# ------------------------------------------------------------------------------------------------ interface
def test_cli_amplicons_needs_primers(capsys):
    with pytest.raises(SystemExit):
        cli.main(["amplicons", "a.bam"])
    assert "--primers is required" in capsys.readouterr().err
    a = cli.build_parser().parse_args(["amplicons", "a.bam", "b.bam", "--primers", "s.bed", "--min-depth", "5",
                                       "--mask-overlaps", "--min-mapq", "3"])
    assert a.bam_path == ["a.bam", "b.bam"] and a.primers == "s.bed" and a.min_depth == 5
    assert cli._amplicon_filters(a) == dict(min_base_quality=0, min_mapq=3, exclude_flags=0, mask_overlaps=True)


def _fake_from_run(run, scheme, min_depth=20):
    """amplicons_from_run over a run that is only its name: fixed numbers per sample."""
    k = int(run[-1])
    df = pd.DataFrame({"contig": ["MN908947.3"] * 3, "amplicon": list(scheme.names), "pool": list(scheme.pool),
                       "start": scheme.start, "end": scheme.end, "insert_start": scheme.insert_start,
                       "insert_end": scheme.insert_end, "reads": [10 * k, 0, 3],
                       "mean_depth": [41.125 * k, 0.0, 19.996], "lowest_depth": [7 * k, 0, 2],
                       "covered": [0.98765, 0.0, 1.0 / 3],
                       "status": ["PASS", "dropout", "dropout"]}, columns=K.AMPLICON_COLUMNS[1:])
    df.attrs["reads"] = (20 * k, 13 * k, 5, 1, 1)
    return df


def test_cli_amplicons_tsv_and_one_block_per_sample(tmp_path, monkeypatch, capsys):
    bed = _write(tmp_path, ARTIC)
    calls = []
    monkeypatch.setattr(K, "pileup_run", lambda path, *a, **kw: (calls.append((path, a, kw)) or (str(path), None)))
    monkeypatch.setattr(K, "amplicons_from_run", _fake_from_run)
    assert cli.main(["amplicons", "--primers", str(bed), "--min-depth", "20", "x/s1", "y/s2"]) == 0
    out, err = capsys.readouterr()
    lines = out.splitlines()
    assert lines[0] == ("sample\tcontig\tamplicon\tpool\tstart\tend\tinsert_start\tinsert_end\treads\tmean_depth\t"
                        "lowest_depth\tcovered\tstatus")
    assert lines[1] == "s1\tMN908947.3\tnCoV-2019_1\t1\t30\t410\t54\t385\t10\t41.12\t7\t0.9877\tPASS"
    assert lines[2] == "s1\tMN908947.3\tnCoV-2019_2\tnCoV-2019_2\t315\t726\t342\t704\t0\t0.00\t0\t0.0000\tdropout"
    assert lines[3] == "s1\tMN908947.3\tnCoV-2019_3\t1\t642\t1028\t664\t1004\t3\t20.00\t2\t0.3333\tdropout"
    assert [ln.split("\t")[0] for ln in lines[1:]] == ["s1"] * 3 + ["s2"] * 3
    assert lines[4].split("\t")[8:10] == ["20", "82.25"]
    assert err.splitlines() == [
        "s1: 20 reads kept: 13 assigned, 5 unprimed, 1 mispaired, 1 ambiguous; 3 amplicons, 2 dropouts: "
        "nCoV-2019_2, nCoV-2019_3",
        "s2: 40 reads kept: 26 assigned, 5 unprimed, 1 mispaired, 1 ambiguous; 3 amplicons, 2 dropouts: "
        "nCoV-2019_2, nCoV-2019_3"]
    # every file piled with the scheme's rows as primers, the filters passed on
    assert [c[0] for c in calls] == ["x/s1", "y/s2"]
    assert all(isinstance(c[2]["primers"], P.PrimerSet) and c[2]["mask_overlaps"] is False for c in calls)


def test_api_names_samples_and_refuses_duplicates(tmp_path, monkeypatch):
    bed = _write(tmp_path, ARTIC)
    monkeypatch.setattr(K, "pileup_run", lambda path, *a, **kw: (str(path), None))
    monkeypatch.setattr(K, "amplicons_from_run", _fake_from_run)
    df = K.amplicons(["a/r1", "b/r2"], str(bed), samples=["one", "two"])
    assert df["sample"].tolist() == ["one"] * 3 + ["two"] * 3
    assert list(df.columns) == K.AMPLICON_COLUMNS and set(df.attrs["reads"]) == {"one", "two"}
    assert K.amplicons("a/r1", str(bed))["sample"].tolist() == ["r1"] * 3
    with pytest.raises(ValueError, match="same file name"):
        K.amplicons(["a/r1", "b/r1"], str(bed))
