"""Depth normalisation (`--normalise N`, an extension) without a GPU: K13 from its CUDA source under the kernel
emulator against the per-record oracle (oracle/py_noracle.py) on hand-made label arrays, at several SM counts (so that
groups cross the CTAs' chunk boundaries) and all three schedules, and after K12 on alignment files; the oracle's two
forms against each other; select_reads with base qualities; the API and CLI checks; the REPORT and VCF header lines."""

import numpy as np
import pytest

import amplicon_cases as AC
import emu_harness as E
from kindel_b200 import bamio, cli, vcf
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from oracle import py_noracle as NO

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
BIG = (1 << 31) - 1


def emu_normalise(labels, reverse, n_amplicons, cap, sm_count=E.SM_COUNT):
    """K13 (kdl_normalise) under the emulator: (keep uint8, total int32, dropped), each output with a poisoned element
    past its end checked."""
    lib = E.load()
    E._sm(sm_count)
    n = len(labels)
    label = np.ascontiguousarray(labels, dtype=np.int32)
    rev = np.ascontiguousarray(reverse, dtype=np.uint8)
    words = int(lib.kdl_normalise_scratch_words(n, n_amplicons))
    scratch = np.full(max(words, 1), 0x5A5A5A5A, dtype=np.int32)  # garbage: K13c must zero its rows
    keep = np.full(n + 1, 0xEE, dtype=np.uint8)
    total = np.full(2 * n_amplicons + 1, -7, dtype=np.int32)
    dropped = np.full(1, -7, dtype=np.int64)
    E._check(lib.kdl_normalise(label.ctypes.data if n else None, rev.ctypes.data if n else None, n, n_amplicons, cap,
                               scratch.ctypes.data, words, keep.ctypes.data, total.ctypes.data, dropped.ctypes.data,
                               None), "kdl_normalise")
    assert keep[n] == 0xEE and total[-1] == -7, "K13 wrote past its outputs"
    return keep[:n], total[:-1], int(dropped[0])


def _check(labels, reverse, n_amplicons, cap, sm_counts=(1, 2, 3, 7), schedules=("forward",)):
    want = NO.keep_loop(labels, reverse, cap)
    tot = NO.totals(labels, reverse, n_amplicons)
    for sm in sm_counts:
        for sched in schedules:
            E.set_schedule(sched, 7)
            try:
                keep, total, dropped = emu_normalise(labels, reverse, n_amplicons, cap, sm)
            finally:
                E.set_schedule("forward")
            assert keep.tolist() == want.tolist(), (sm, sched, cap)
            assert total.tolist() == tot.tolist(), (sm, sched)
            assert dropped == int((want == 0).sum()), (sm, sched)
    return want


# ------------------------------------------------------------------------------------------------ oracle
def test_oracle_vectorised_equals_the_loop():
    rng = np.random.default_rng(1)
    for trial in range(40):
        n = int(rng.integers(0, 3000))
        labels = rng.integers(-3, int(rng.integers(1, 30)), n)
        reverse = rng.integers(0, 2, n)
        for cap in (1, 2, 7, 100, BIG):
            assert NO.keep_vectorised(labels, reverse, cap).tolist() == NO.keep_loop(labels, reverse, cap).tolist()


# ------------------------------------------------------------------------------------------------ K13
@needs_emu
@pytest.mark.parametrize("schedule", ["forward", "reverse", "random"])
def test_k13_random_groups_every_schedule(schedule):
    rng = np.random.default_rng(3)
    n = 2600  # 11 tiles: several per CTA at every SM count below
    labels = rng.integers(-3, 9, n)
    reverse = rng.integers(0, 2, n)
    for cap in (1, 5, 40):
        _check(labels, reverse, 9, cap, schedules=(schedule,))


@needs_emu
def test_k13_caps_at_one_at_the_largest_and_at_a_groups_size():
    rng = np.random.default_rng(4)
    n = 1500
    labels = rng.integers(-1, 4, n)
    reverse = rng.integers(0, 2, n)
    size = int(((labels == 2) & (reverse == 1)).sum())
    for cap in (1, BIG, size, size - 1):
        keep = _check(labels, reverse, 4, cap)
        in_group = (labels == 2) & (reverse == 1)
        assert int(keep[in_group].sum()) == min(cap, size)
    assert _check(labels, reverse, 4, BIG).all()


@needs_emu
def test_k13_no_assigned_read_and_one_key_holding_every_read():
    n = 1800
    assert _check(np.full(n, -1), np.zeros(n), 3, 1).all()
    assert _check(np.array([-1, -2, -3] * 600), np.ones(n), 3, 1).all()
    keep = _check(np.full(n, 2), np.ones(n), 3, 700)  # the deep amplicon: every read in one group
    assert keep[:700].all() and not keep[700:].any()


@needs_emu
def test_k13_alternating_keys():
    n = 2048
    labels = np.arange(n) % 2
    reverse = (np.arange(n) // 2) % 2  # keys 0, 2, 1, 3, 0, 2, ...
    keep = _check(labels, reverse, 2, 100)
    assert int(keep.sum()) == 400 and keep[:400].all() and not keep[400:].any()


@needs_emu
def test_k13_groups_cross_every_chunk_boundary():
    # runs of one key 300 reads long (longer than a tile, offset from the tiles) over 4000 reads: at every SM count
    # each CTA's chunk starts and ends inside a group, and so do most tiles
    n = 4000
    labels = (np.arange(n) + 77) // 300 % 5
    reverse = ((np.arange(n) + 13) // 150) % 2
    for cap in (1, 100, 299, 450):
        _check(labels, reverse, 5, cap, sm_counts=(1, 2, 3, 4, 5, 8))


@needs_emu
def test_k13_more_keys_than_a_tile_and_tiny_batches():
    rng = np.random.default_rng(5)
    n = 1200
    labels = rng.integers(-3, 300, n)  # K = 600 keys, more than the 256 threads of a CTA
    reverse = rng.integers(0, 2, n)
    _check(labels, reverse, 300, 2)
    _check(labels, reverse, 300, 1)
    for n in (0, 1, 5, 31, 33):  # an empty batch, fewer reads than one warp, a warp and a bit
        _check(rng.integers(-1, 2, n), rng.integers(0, 2, n), 2, 1)
    _check(rng.integers(-3, 0, 40), rng.integers(0, 2, 40), 0, 1)  # a scheme without amplicons on these contigs


@needs_emu
def test_k13_refuses_bad_arguments():
    lib = E.load()
    lab = np.zeros(4, dtype=np.int32)
    rev = np.zeros(4, dtype=np.uint8)
    out = np.zeros(8, dtype=np.int64)
    words = int(lib.kdl_normalise_scratch_words(4, 2))
    scratch = np.zeros(words, dtype=np.int32)
    args = lambda cap, w: (lab.ctypes.data, rev.ctypes.data, 4, 2, cap, scratch.ctypes.data, w,  # noqa: E731
                           out.ctypes.data, out.ctypes.data, out.ctypes.data, None)
    assert lib.kdl_normalise(*args(0, words)) == 1  # KDL_ERR_INVALID_ARG: cap < 1
    assert lib.kdl_normalise(*args(1, words - 1)) == 1  # scratch too small
    assert lib.kdl_normalise(*args(1, words)) == 0
    assert lib.kdl_normalise_scratch_words(-1, 2) == -1


# ------------------------------------------------------------------------------------------------ K12 + K13 on files
def _file_case(tmp_path, text, rows, cap, name="n.sam", sm_counts=(1, 2, 5)):
    p = tmp_path / name
    p.write_text(text)
    b = bamio.read_alignment(p, strand=True)
    arr = P.amplicon_arrays(AC.scheme(rows), b.contig_names, b.contig_len)
    labels = AC.emu_assign(b, arr)
    want, dropped = NO.keep_by_record(str(p), b.contig_names, rows, cap)
    for sm in sm_counts:
        keep, _, n_drop = emu_normalise(labels, b.reverse, arr.n_amplicons, cap, sm)
        assert keep.tolist() == want.tolist() and n_drop == len(dropped)
    return want


@needs_emu
def test_k12_k13_many_contigs(tmp_path):
    n = 300
    head = "".join("@SQ\tSN:k%d\tLN:%d\n" % (c, 100 + c) for c in range(n))
    body, rows = [], []
    for c in range(n):
        L = 100 + c
        rows += [("k%d" % c, 2, 8, "a%d" % c, "L"), ("k%d" % c, L - 8, L - 2, "a%d" % c, "R")]
        for k in range(c % 4 + 1):
            body.append("r%d_%d\t%d\tk%d\t4\t60\t20M\t*\t0\t0\t%s\t*\n" % (c, k, 16 * (k % 2), c, "ACGT" * 5))
        body.append("q%d\t16\tk%d\t%d\t60\t20M\t*\t0\t0\t%s\t*\n" % (c, c, L - 21, "ACGT" * 5))
    text = head + "".join(reversed(body))  # contigs first seen in an order unlike the header
    want = _file_case(tmp_path, text, rows, 1)
    assert (want == 0).sum() > 0


HARD_SAM = """@SQ\tSN:c0\tLN:80
p1\t0\tc0\t60\t60\t2M30S4M\t*\t0\t0\tACGTACGTACGTACGTACGTACGTACGTACGTACGT\t*
p2\t0\tc0\t59\t60\t4M20S\t*\t0\t0\tACGTACGTACGTACGTACGTACGT\t*
p3\t0\tc0\t60\t60\t4M20S\t*\t0\t0\tACGTACGTACGTACGTACGTACGT\t*
p4\t16\tc0\t59\t60\t4M20S\t*\t0\t0\tACGTACGTACGTACGTACGTACGT\t*
u1\t0\tc0\t0\t60\t2M4S\t*\t0\t0\tACGTAC\t*
p5\t0\tc0\t61\t60\t3M10S\t*\t0\t0\tACGTACGTACGTA\t*
"""


@needs_emu
def test_k12_k13_hard_reads(tmp_path):
    rows = [("c0", 58, 62, "F", "L"), ("c0", 66, 72, "F", "R")]
    want = _file_case(tmp_path, HARD_SAM, rows, 2)
    assert want.tolist() == [1, 1, 0, 1, 1, 0]  # F forward: p1, p2 kept, p3, p5 over the cap; p4 reverse; u1 unprimed


@needs_emu
def test_k12_k13_synthetic_amplicon_batch():
    from kindel_b200 import synth

    amp, trows = synth.amplicon_reads(1, 6_000, 60)
    amp = synth.with_strands(amp, 3)
    rows = AC.tiled_rows(trows)
    arr = P.amplicon_arrays(AC.scheme(rows), amp.contig_names, amp.contig_len)
    labels = AC.emu_assign(amp, arr)
    want = NO.keep_vectorised(labels, amp.reverse, 10)
    keep, total, dropped = emu_normalise(labels, amp.reverse, arr.n_amplicons, 10, 3)
    assert keep.tolist() == want.tolist() and dropped == int((want == 0).sum()) > 0
    assert total.sum() == (labels >= 0).sum()


# ------------------------------------------------------------------------------------------------ select_reads
QUAL_SAM = """@SQ\tSN:c0\tLN:200
a\t0\tc0\t5\t60\t10M\t*\t0\t0\tACGTACGTAC\tABCDEFGHIJ
b\t16\tc0\t9\t60\t3S9M2I4M\t*\t0\t0\tGGGACGTACGTACCCGTA\t!!#$%&'()*+,-./012
c\t0\tc0\t20\t60\t12M\t*\t0\t0\tACGTACGTACGT\tKKKKKKKKKKKK
d\t0\tc0\t30\t60\t5M3D5M\t*\t0\t0\tACGTAACGTA\t0123456789
e\t16\tc0\t40\t60\t17M\t*\t0\t0\tACGTACGTACGTACGTA\tabcdefghijklmnopq
"""


def test_select_reads_carries_base_qualities(tmp_path):
    p = tmp_path / "q.sam"
    p.write_text(QUAL_SAM)
    full = bamio.read_alignment(p, qual=True, strand=True, min_base_quality=12)
    for keep in ([0, 2, 4], [1, 3], [4], [0, 1, 2, 3, 4], []):
        sub = bamio.select_reads(full, keep)
        lines = QUAL_SAM.splitlines(keepends=True)
        q = tmp_path / "sub.sam"
        q.write_text(lines[0] + "".join(lines[1 + k] for k in keep))
        want = bamio.read_alignment(q, qual=True, strand=True, min_base_quality=12)
        assert sub.qual8 is not None and np.array_equal(sub.qual8, want.qual8), keep
        for f in ("ref_start", "seq_off", "l_seq", "seq4", "reverse", "mask_read", "mask_off", "mask_qpos"):
            a, b = getattr(sub, f), getattr(want, f)
            assert (a is None and b is None) or np.array_equal(a, b), (keep, f)
    assert bamio.select_reads(bamio.read_alignment(p), [1, 2]).qual8 is None


# ------------------------------------------------------------------------------------------------ interface
def _bed(tmp_path, named=True):
    p = tmp_path / ("s.bed" if named else "plain.bed")
    p.write_text("c\t0\t5\tx_LEFT\t1\nc\t20\t25\tx_RIGHT\t1\n" if named else "c\t0\t5\nc\t20\t25\n")
    return str(p)


@pytest.mark.parametrize("value", [0, -3, 1.5, 2.0, True, "4", None])
def test_check_normalise(value):
    if value is None:
        assert K.check_normalise(None) is None
        return
    with pytest.raises(ValueError, match="normalise must be an integer >= 1"):
        K.check_normalise(value)


def test_check_normalise_takes_integers():
    assert K.check_normalise(1) == 1 and K.check_normalise(np.int64(200)) == 200 and K.check_normalise(BIG) == BIG


def test_api_normalise_needs_a_named_scheme(tmp_path):
    # refused before the file is read or a device is asked for
    with pytest.raises(ValueError, match="normalise needs a named primer scheme: pass primers="):
        K.pileup_run("missing.bam", normalise=5)
    with pytest.raises(ValueError, match="not a PrimerSet"):
        K.pileup_run("missing.bam", primers=P.load_primers(_bed(tmp_path)), normalise=5)
    with pytest.raises(ValueError, match="column 4"):
        K.pileup_run("missing.bam", primers=_bed(tmp_path, named=False), normalise=5)
    with pytest.raises(ValueError, match="normalise must be"):
        K.bam_to_consensus("missing.bam", primers=_bed(tmp_path), normalise=0)


@pytest.mark.parametrize("cmd", [["consensus", "a.bam"], ["weights", "a.bam"], ["features", "a.bam"],
                                 ["variants", "a.bam", "--vcf"], ["amplicons", "a.bam"]])
def test_cli_normalise_errors(tmp_path, capsys, cmd):
    if cmd[0] != "amplicons":  # (amplicons without --primers has its own message)
        with pytest.raises(SystemExit):
            cli.main(cmd + ["--normalise", "5"])
        assert "--normalise needs --primers" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        cli.main(cmd + ["--normalise", "5", "--primers", _bed(tmp_path, named=False)])
    assert "--normalise needs a named primer scheme" in capsys.readouterr().err
    for bad in ("0", "-1", "x", "2.5"):
        with pytest.raises(SystemExit):
            cli.main(cmd + ["--normalise", bad, "--primers", _bed(tmp_path)])
        assert "argument --normalise: invalid _normalise value" in capsys.readouterr().err


def test_cli_passes_normalise_on(tmp_path, monkeypatch, capsys):
    bed = _bed(tmp_path)
    seen = []

    class _Res:
        refs_reports, consensuses = {}, []

    monkeypatch.setattr(K, "bam_to_consensus", lambda *a, **kw: seen.append(("consensus", kw)) or _Res())
    monkeypatch.setattr(K, "variants_vcf", lambda *a, **kw: seen.append(("vcf", kw)) or "")
    cli.main(["consensus", "a.bam", "--primers", bed, "--normalise", "200"])
    cli.main(["variants", "a.bam", "b.bam", "--vcf", "--primers", bed, "--normalise", "7"])
    cli.main(["consensus", "a.bam", "--primers", bed])
    assert seen[0][1]["normalise"] == 200 and seen[1][1]["normalise"] == 7 and "normalise" not in seen[2][1]


def test_cli_amplicons_summary_names_the_dropped_reads(tmp_path, monkeypatch, capsys):
    import pandas as pd

    bed = _bed(tmp_path)

    def fake(paths, primers, min_depth, **kw):
        df = pd.DataFrame({"sample": ["s"], "contig": ["c"], "amplicon": ["x"], "pool": ["1"], "start": [0],
                           "end": [25], "insert_start": [5], "insert_end": [20], "reads": [9], "mean_depth": [9.0],
                           "lowest_depth": [9], "covered": [0.0], "status": ["dropout"]}, columns=K.AMPLICON_COLUMNS)
        df.attrs["reads"] = {"s": (12, 9, 3, 0, 0)}
        if kw.get("normalise") is not None:
            df.attrs["dropped"] = {"s": 41}
        return df

    monkeypatch.setattr(K, "amplicons", fake)
    cli.main(["amplicons", "s", "--primers", bed, "--normalise", "9"])
    assert capsys.readouterr().err.strip() == ("s: 12 reads kept: 9 assigned, 3 unprimed, 0 mispaired, 0 ambiguous; "
                                               "1 amplicons, 1 dropouts: x; 41 reads over the normalise cap dropped")
    cli.main(["amplicons", "s", "--primers", bed])
    assert "normalise" not in capsys.readouterr().err


def test_report_line_follows_the_primer_line():
    args = ("ref", K.DepthRange(0, 9), [None] * 3, None, "a.bam", False, 1, 9, 0.1, False, False)
    plain = K.build_report(*args, primers="s.bed").splitlines()
    on = K.build_report(*args, primers="s.bed", normalised=(200, 35, 965)).splitlines()
    k = plain.index("- primers: s.bed")
    assert on[:k + 1] == plain[:k + 1] and on[k + 2:] == plain[k + 1:]
    assert on[k + 1] == "- normalise: 200 per amplicon and strand, 35 of 1000 reads dropped"


def test_vcf_header_line_follows_the_primer_line(tmp_path):
    ps = P.load_primers(_bed(tmp_path))
    plain = vcf.header(["c"], [30], 1, 0.01, None, ps)
    on = vcf.header(["c"], [30], 1, 0.01, None, ps, normalise=200)
    k = plain.index("##kindelPrimers=s.bed")
    assert on == plain[:k + 1] + ["##kindelNormalise=200"] + plain[k + 1:]
    assert vcf.header(["c"], [30], 1, 0.01, None, ps, normalise=None) == plain
