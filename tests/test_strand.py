"""`variants --vcf --strand` (extension) without a GPU: the strand byte at decode and through the batch helpers, K8
from its CUDA source under the host emulator (tests/emu/emu_select.cpp) against bamio.select_reads, the oracle
(oracle/py_soracle.py) against a truth set with alleles planted on one strand, the SOR rule and the CLI."""
import os

import numpy as np
import pytest

import combo_cases as CC
import emu_select_harness as ES
import helpers as H
import limit_cases as LC
import strand_cases as S
from fuzz_cases import random_case
from kindel_b200 import bamio, cli, synth
from kindel_b200 import kindel as K
from oracle import py_soracle as SO
from oracle import samdecode

needs_emu = pytest.mark.skipif(not ES.available(), reason="needs g++ and the CUDA headers")
INPUTS = os.path.join(H.ROOT, "tests", "golden", "inputs")
FIXTURES = sorted(f for f in os.listdir(INPUTS) if f.endswith((".bam", ".sam")))


# ------------------------------------------------------------------------------------------------ decode
def _want_reverse(path, names, exclude_flags=0):
    header, records = samdecode.read_alignment_file(path)
    groups = {}
    for r in records:
        groups.setdefault(r.rname, []).append(r)
    return [1 if r.flag & 0x10 else 0 for nm in names for r in groups.get(nm, [])
            if r.mapped and len(r.seq) > 1 and not r.flag & exclude_flags]


@pytest.mark.parametrize("name", FIXTURES)
def test_reverse_is_flag_0x10_of_the_kept_records(name):
    path = os.path.join(INPUTS, name)
    readers = [("C++", lambda **kw: bamio.read_alignment(path, **kw))]
    if name.endswith(".sam"):
        readers.append(("python", lambda **kw: bamio.read_sam(path, **kw)))
    for what, read in readers:
        b = read(strand=True)
        assert b.reverse.dtype == np.uint8 and b.reverse.tolist() == _want_reverse(path, b.contig_names), what
        assert 0 < int(b.reverse.sum()) < b.n_reads, what  # the fixtures hold both strands
        assert read().reverse is None  # off by default
        x = read(strand=True, exclude_flags=0x10)
        assert x.reverse.shape == (x.n_reads,) and not x.reverse.any()
        m = read(strand=True, min_mapq=20)
        assert m.reverse.shape == (m.n_reads,)
    if name == "mm2_multi.bam":
        b = bamio.read_alignment(path, strand=True)
        assert (b.n_reads, int(b.reverse.sum())) == (915, 492)


def test_reverse_through_select_merge_save_load(tmp_path):
    b = bamio.read_alignment(os.path.join(INPUTS, "mm2_multi.bam"), strand=True, min_base_quality=20)
    idx = np.flatnonzero(np.arange(b.n_reads) % 3 != 1)
    sub = bamio.select_reads(b, idx)
    assert np.array_equal(sub.reverse, b.reverse[idx])
    parts = [bamio.select_reads(b, np.arange(0, b.n_reads, 2)), bamio.select_reads(b, np.arange(1, b.n_reads, 2))]
    merged = bamio.merge_batches(parts)
    assert merged.reverse is not None and int(merged.reverse.sum()) == int(b.reverse.sum())
    # merge sorts by start inside a contig; the strand of every read goes with it
    assert sorted(zip(merged.ref_start.tolist(), merged.seq_len.tolist(), merged.reverse.tolist())) == \
        sorted(zip(b.ref_start.tolist(), b.seq_len.tolist(), b.reverse.tolist()))
    assert bamio.merge_batches([parts[0], bamio.select_reads(bamio.read_alignment(os.path.join(INPUTS, "mm2_multi.bam")),
                                                            np.arange(1, b.n_reads, 2))]).reverse is None
    d = tmp_path / "b"
    bamio.save_batch(str(d), b)
    assert np.array_equal(bamio.load_batch(str(d)).reverse, b.reverse)
    plain = bamio.read_alignment(os.path.join(INPUTS, "mm2_multi.bam"))
    bamio.save_batch(str(d), plain)  # a batch without strands removes the old file
    assert not (d / "reverse.npy").exists() and bamio.load_batch(str(d)).reverse is None


def test_synthetic_strands(tmp_path):
    b = synth.with_strands(synth.simple_reads(4, [20_000], 20), 3)
    assert 0.45 < b.reverse.mean() < 0.55
    assert np.array_equal(synth.strands(3, b.n_reads), b.reverse)
    s = synth.strands(1, 100, forward=[0, 1, 2], reverse=[3, 4])
    assert s[:3].tolist() == [0, 0, 0] and s[3:5].tolist() == [1, 1]
    path = tmp_path / "s.bam"
    synth.write_simple_bam(str(path), b)
    assert np.array_equal(bamio.read_alignment(str(path), strand=True).reverse, b.reverse)


# ------------------------------------------------------------------------------------------------ K8
def _corpus(tmp_path):
    """(name, batch) of the fuzz, limit and combo corpora (limit and combo cases masked as well)."""
    out = []
    for seed in range(60):
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            out.append(("fuzz%d" % seed, bamio.read_alignment(p, strand=True)))
        except (ValueError, KeyError):
            pass
    for name in LC.GROUPS:
        p = tmp_path / ("limit_%s.sam" % name)
        p.write_text(LC.sam_text(name))
        out.append(("limit_" + name, bamio.read_alignment(p, strand=True, min_base_quality=20)))
    for seed in range(3):
        contigs, recs = CC.combo_case(seed)
        p = CC.write_bam(tmp_path / ("combo%d.bam" % seed), contigs, recs)
        out.append(("combo%d" % seed, bamio.read_alignment(p, strand=True, min_base_quality=20)))
    return out


def _unsorted(batch):
    """The batch with the first two reads of its first contig swapped (unsorted when their starts differ), and a keep
    that drops one of them (its subset is sorted)."""
    idx = np.arange(batch.n_reads)
    idx[0], idx[1] = 1, 0
    parent = bamio.select_reads(batch, idx)
    keep = np.ones(batch.n_reads, np.uint8)
    keep[0] = 0
    return parent, keep


@needs_emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 3)])
def test_emulated_k8_equals_select_reads(schedule, seed, tmp_path):
    ES.set_schedule(schedule, seed)
    n = hard = masked = cx = 0
    for name, b in _corpus(tmp_path):
        rng = np.random.default_rng(seed + len(name))
        keeps = [b.reverse, rng.integers(0, 2, b.n_reads).astype(np.uint8), np.zeros(b.n_reads, np.uint8),
                 np.ones(b.n_reads, np.uint8)]
        if b.n_contigs > 1:
            k = np.ones(b.n_reads, np.uint8)
            k[int(b.contig_read_off[1]):int(b.contig_read_off[2])] = 0  # a contig with no kept read
            keeps.append(k)
        for j, keep in enumerate(keeps):
            want = bamio.select_reads(b, np.flatnonzero(keep))
            ES.assert_equal(ES.select(b, keep), ES.fields(want), (name, j))
            n += 1
        hard += b.n_hard > 0
        cx += b.n_complex > b.n_hard
        masked += b.n_masked > 0
    assert n > 250 and hard > 10 and cx > 10 and masked > 10


@needs_emu
def test_emulated_k8_sorts_a_subset_of_an_unsorted_batch():
    b = synth.mixed_reads(2, [4_000, 900], 8, 0.2)
    assert b.reads_sorted and b.ref_start[0] != b.ref_start[1]
    parent, keep = _unsorted(b)
    assert not parent.reads_sorted
    got = ES.select(parent, keep)
    want = bamio.select_reads(parent, np.flatnonzero(keep))
    assert want.reads_sorted and got["reads_sorted"]
    ES.assert_equal(got, ES.fields(want), "unsorted parent")
    # and a subset that keeps the swapped pair stays unsorted
    keep2 = np.ones(b.n_reads, np.uint8)
    keep2[5] = 0
    got2 = ES.select(parent, keep2)
    assert not got2["reads_sorted"]
    ES.assert_equal(got2, ES.fields(bamio.select_reads(parent, np.flatnonzero(keep2))), "unsorted subset")


# ------------------------------------------------------------------------------------------------ oracle, SOR
def test_oracle_truth_set():
    ref, reads = S.truth_set()
    recs = S.oracle_records(reads)
    for lines in (SO.vcf_lines([("t", S.L, recs)], 1, 0.01, 3.0),
                  SO.vcf_lines([("t", ref, recs)], 1, 0.01, 3.0, reference=True)):
        got = S.parse(lines)
        one = {k[0] for k, v in got.items() if v[0] == "sor"}
        bal = [v for k, v in got.items() if k[0] == S.SNV_BAL + 1]
        assert bal[0][0] == "PASS" and bal[0][1]["SOR"] == "%.3f" % np.log(2)
        assert S.SNV_ONE + 1 in one and all(float(v[1]["SOR"]) > 4 for v in got.values() if v[0] == "sor")
    got = S.parse(SO.vcf_lines([("t", ref, recs)], 1, 0.01, 3.0, reference=True))
    assert one == {S.SNV_ONE + 1, S.INS_AT, S.DEL_AT}  # the insertion and the deletion against the reference
    ins = got[(S.INS_AT, ref[S.INS_AT - 1], ref[S.INS_AT - 1] + "GT")][1]
    dele = got[(S.DEL_AT, ref[S.DEL_AT - 1:S.DEL_AT + 2], ref[S.DEL_AT - 1])][1]
    assert (ins["ADF"].split(",")[1], ins["ADR"].split(",")[1], ins["AO"]) == ("0", "8", "8")
    assert (dele["ADF"].split(",")[1], dele["ADR"].split(",")[1], dele["AO"]) == ("8", "0", "8")
    # without a filter everything passes
    assert all(v[0] == "PASS" for v in S.parse(SO.vcf_lines([("t", ref, recs)], 1, 0.01, None, reference=True)).values())


def test_sor_rule_equals_the_oracle():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        adf = [int(x) for x in rng.integers(0, 60, 3)]
        adr = [int(x) for x in rng.integers(0, 60, 3)]
        for max_sor in (None, 0.5, 2.0):
            assert K._strand_fields(adf, adr, max_sor) == SO.strand_tail(adf, adr, max_sor)
        assert K.strand_odds_ratio(adf[0], adr[0], adf[1], adr[1]) > 0
    assert K.strand_odds_ratio(5, 5, 5, 5) == np.log(2)
    assert K._strand_fields([10, 10], [10, 0], 0.0)[0] == "sor"


def test_max_sor_and_missing_strands_raise():
    with pytest.raises(ValueError):
        K.check_max_sor(float("nan"))
    assert K.check_max_sor(None) is None and K.check_max_sor("3") == 3.0
    b = bamio.read_alignment(os.path.join(INPUTS, "mm2_gp120.bam"))
    run = K.PileupRun.from_host_tables(b, np.zeros((19, b.n_slots), np.int32), np.zeros((5, b.n_slots), np.int32),
                                       np.zeros((0, 4), np.int32))
    with pytest.raises(ValueError):
        K.variants_vcf_from_run(run, strand=True)
    with pytest.raises(ValueError):
        K.variants_vcf_from_run(run, max_sor=float("nan"))


# ------------------------------------------------------------------------------------------------ CLI
@pytest.mark.parametrize("args", [["--strand"], ["--max-sor", "3"], ["--vcf", "--max-sor", "nan"],
                                  ["--strand", "--max-sor", "2"]])
def test_cli_strand_options_need_vcf(args, capsys):
    with pytest.raises(SystemExit) as e:
        cli.main(["variants"] + args + ["x.bam"])
    assert e.value.code == 2
    assert "--vcf" in capsys.readouterr().err or "nan" in " ".join(args)


def test_cli_passes_strand(monkeypatch, capsys):
    seen = []

    def fake_vcf(path, a, r, devices=None, **kw):
        seen.append(kw)
        return "x\n"

    monkeypatch.setattr(K, "variants_vcf", fake_vcf)
    cli.main(["variants", "--vcf", "x.bam"])
    cli.main(["variants", "--vcf", "--strand", "x.bam"])
    cli.main(["variants", "--vcf", "--max-sor", "2.5", "--reference", "r.fa", "x.bam"])
    assert "strand" not in seen[0] and "max_sor" not in seen[0]
    assert seen[1]["strand"] is True and seen[1]["max_sor"] is None
    assert seen[2]["strand"] is True and seen[2]["max_sor"] == 2.5 and seen[2]["reference"] == "r.fa"
