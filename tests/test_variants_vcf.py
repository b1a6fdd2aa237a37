"""The variant sites of `variants --only-variants` and the sites-only VCF (`variants --vcf`; extensions), without a GPU.

oracle/py_voracle.py restates the rule as a per-position loop over plain ints and floats.  The product's numpy helper
(kindel.variant_alleles, through kindel.variant_sites on host tables) and K6 -- run from its CUDA source under the
host emulator (tests/emu/emu_api.cpp) -- must both reproduce it, over a threshold grid that includes negative,
NaN, non-integer and out-of-range thresholds, on the fuzz, combo and limit corpora and on adversarial tables with counts
planted in the slot behind each contig and in the padding.  The VCF writer is checked line by line and against a VCF
built from the restatement's sites."""
import math
import types

import numpy as np
import pandas as pd
import pytest

import combo_cases as CC
import emu_harness as E
import limit_cases as LC
from conftest import golden_input
from fuzz_cases import random_case
from kindel_b200 import __version__, bamio, cli, engine
from kindel_b200 import _ffi
from kindel_b200 import kindel as K
from oracle import coracle, py_voracle as V

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
NAN = float("nan")
ABS = (-5, -1, 0, 1, 2, 2 ** 31, 10 ** 12, 1.5)
REL = (-0.5, 0.0, 0.01, 0.25, 0.5, 1.0, NAN)
GRID = [(a, r) for a in ABS for r in REL]


# ---------------------------------------------------------------------------------------------- inputs
class _Batch(types.SimpleNamespace):
    """The layout fields of a ReadBatch that the variant paths read."""


def host_run(table, contig_slot, contig_len, names=None):
    """A PileupRun over a host table with the given contig layout (no reads needed)."""
    run = K.PileupRun.__new__(K.PileupRun)
    names = names or ["c%d" % c for c in range(len(contig_len))]
    run.batch = _Batch(contig_names=list(names), contig_slot=np.asarray(contig_slot, dtype=np.int64),
                       contig_len=np.asarray(contig_len, dtype=np.int32), n_contigs=len(contig_len))
    run.dbatch, run.counts, run.events, run.calls_device = None, None, None, None
    run._host_counts = np.ascontiguousarray(table, dtype=np.int32)
    run._host_derived = run._ins = None
    return run


def _oracle_run(batch):
    counts, events = coracle.pileup(batch)
    return K.PileupRun.from_host_tables(batch, counts, coracle.derive(counts), events)


def _fuzz_runs(tmp_path, seeds=range(400)):
    for seed in seeds:
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            yield "fuzz%d" % seed, _oracle_run(bamio.read_alignment(p))
        except (ValueError, KeyError, IndexError):
            continue


def combo_run(contigs, recs, path, filters, work):
    """The oracle's tables of the combo corpus under the filters (combo_cases.Piled: the record filters as unmapped
    records, the base filter by oracle/qoracle) over the product's batch layout."""
    mbq, mq, ex = filters
    piled = CC.Piled(contigs, recs, work, mbq, mq, ex)
    batch = bamio.read_alignment(path, min_mapq=mq, exclude_flags=ex, min_base_quality=mbq)
    return K.PileupRun.from_host_tables(batch, piled.counts, coracle.derive(piled.counts), piled.events)


def _combo_runs(tmp_path, seeds=(0, 1, 2)):
    for seed in seeds:
        contigs, recs = CC.combo_case(seed)
        path = CC.write_bam(tmp_path / ("combo%d.bam" % seed), contigs, recs)
        for flt in ((0, 0, 0), (20, 10, 0x400)):
            run = combo_run(contigs, recs, path, flt, tmp_path / ("combo%d_piled.bam" % seed))
            yield "combo%d/%d" % (seed, flt[0]), run, path, flt


def _limit_runs(tmp_path):
    for name in LC.GROUPS:
        p = tmp_path / ("limit_%s.sam" % name)
        p.write_text(LC.sam_text(name))
        try:
            yield "limit_" + name, _oracle_run(bamio.read_alignment(p))
        except (ValueError, KeyError, IndexError):
            continue


def adversarial(seed):
    """(table, contig_slot, contig_len) tables the corpora do not reach: ties between the top and a second allele, N
    or a deletion on top, zero-depth positions, counts near 2^31, and non-zero counts planted in the slot behind each
    contig and in the padding (which must never be sites).  Three contigs; the slot space is not a multiple of the
    1024-slot CTA span."""
    rng = np.random.default_rng(seed)
    lens = [1500, 7, 900]
    slots, s = [], 0
    for L in lens:
        slots.append(s)
        s = (s + L + 1 + 3) // 4 * 4 + 4 * int(rng.integers(0, 3))  # the slot behind the contig, padding
    n = (s + 3) // 4 * 4
    t = np.zeros((19, n), dtype=np.int64)
    t[0:6] = rng.integers(0, 5, size=(6, n))                          # ties and near-ties everywhere
    t[0:6, rng.random(n) < 0.1] = 0                                   # zero depth
    big = rng.random(n) < 0.1
    t[0:6, big] = rng.integers((1 << 31) - 4, 1 << 31, size=(6, int(big.sum())))  # near 2^31
    top_n = rng.random(n) < 0.05
    t[4, top_n] = 9                                                   # N on top
    top_d = rng.random(n) < 0.05
    t[5, top_d] = 9                                                   # deletion on top
    t[0, 5:8], t[1, 5:8] = 6, 6                                       # A and C tied on top
    t[0:6, 10] = (3, 3, 3, 3, 3, 3)                                   # all tied
    t[4, 11], t[0, 11] = 5, 2                                         # N the only variant besides REF
    t[0:6, 12] = (0, 0, 0, 0, 7, 2)                                   # N top, deletion variant
    # slot L and the padding: counts that every threshold of the grid below 2^31 would select
    is_pos = np.zeros(n, dtype=bool)
    for s0, L in zip(slots, lens):
        is_pos[s0:s0 + L] = True
    t[0:6, ~is_pos] = np.array([[100], [50], [40], [30], [20], [10]])
    t[7:, :] = rng.integers(0, 3, size=(12, n))                       # columns K6 must not read
    return t.astype(np.int32), np.array(slots), np.array(lens)


def _sites_equal(got, want, what):
    for g, w, name in zip(got, want, ("slot", "counts", "mask")):
        assert g.dtype == w.dtype, (what, name, g.dtype, w.dtype)
        np.testing.assert_array_equal(g, w, err_msg="%s: %s" % (what, name))


def _tables(tmp_path):
    """(name, table, contig_slot, contig_len) of the corpora and the adversarial tables."""
    for name, run in list(_fuzz_runs(tmp_path)) + list(_limit_runs(tmp_path)):
        yield name, run.host_counts, run.batch.contig_slot, run.batch.contig_len
    for name, run, _, _ in _combo_runs(tmp_path):
        yield name, run.host_counts, run.batch.contig_slot, run.batch.contig_len
    for seed in (1, 2, 3):
        yield ("adversarial%d" % seed,) + adversarial(seed)


# ------------------------------------------------------------------------------------ numpy helper vs loop
def test_abs_floor_clamp():
    f = engine.variant_abs_floor
    assert [f(x) for x in (-5, -1, 0, 1, 1.5, -0.5, -1.5, 2 ** 31, 10 ** 12, NAN, math.inf, -math.inf, np.int64(3))] == \
        [-1, -1, 0, 1, 1, -1, -1, 2 ** 31, 2 ** 31, 2 ** 31, 2 ** 31, -1, 3]
    # the clamp selects what the unclamped threshold selects, for every int32 count
    t = np.array([0, 1, 2, 3, (1 << 31) - 1])
    for x in (-5, -0.5, 0.5, 1.5, 2 ** 31, 10 ** 12, 3e9, NAN):
        assert np.array_equal(t > x, t > f(x)), x


def test_numpy_helper_equals_restatement(tmp_path):
    """kindel.variant_sites on host tables (the numpy helper) == the per-position loop, at every point of the threshold
    grid, on the fuzz, limit and combo corpora and the adversarial tables."""
    n_sites = n_checks = 0
    for name, table, cs, cl in _tables(tmp_path):
        run = host_run(table, cs, cl)
        for a, r in GRID:
            want = V.sites(table, cs, cl, a, r)
            _sites_equal(K.variant_sites(run, a, r), want, (name, a, r))
            n_sites += len(want[0])
            n_checks += 1
    assert n_checks > 2000 and n_sites > 100_000


def test_threshold_edges():
    table, cs, cl = adversarial(7)
    n_pos = int(cl.sum())
    run = host_run(table, cs, cl)
    for a, r in ((NAN, 0.0), (0, NAN), (2 ** 31, -1.0), (10 ** 12, -1.0)):
        assert len(K.variant_sites(run, a, r)[0]) == 0, (a, r)
    # negative thresholds: every position qualifies, zero-depth ones included (five alleles besides the top)
    slot, counts, mask = K.variant_sites(run, -1, -0.5)
    assert len(slot) == n_pos
    zero = counts.sum(axis=0) == 0
    assert zero.any() and (mask[zero] == 0b111110).all()


def test_planted_slots_are_never_sites():
    for seed in (1, 2, 3):
        table, cs, cl = adversarial(seed)
        for a, r in ((-1, -0.5), (0, 0.0), (1, 0.01)):
            slot = K.variant_sites(host_run(table, cs, cl), a, r)[0]
            c = np.searchsorted(cs, slot, side="right") - 1
            assert (slot < cs[c] + cl[c]).all() and (slot >= cs[c]).all()


# ----------------------------------------------------------------------------------------------- K6
def _emulated(table, cs, cl, a, r):
    return E.variant_sites(table, cs, cl, engine.variant_abs_floor(a), r)


@needs_emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 3)])
def test_emulated_k6_equals_restatement(schedule, seed, tmp_path):
    """K6 from its source under three thread orders == the loop: adversarial tables (not a multiple of the CTA span),
    planted slot-L / padding counts, a table with no site, and fuzz, limit and combo tables."""
    E.set_schedule(schedule, seed)
    try:
        tables = [("adversarial%d" % s,) + adversarial(s + seed) for s in (1, 2)]
        tables.append(("empty", np.zeros((19, 2052), dtype=np.int32), np.array([0, 1030]), np.array([1000, 1020])))
        fuzz = [(n, r.host_counts, r.batch.contig_slot, r.batch.contig_len)
                for n, r in _fuzz_runs(tmp_path, range(seed, 400, 40))]
        other = [t for t in _tables_small(tmp_path)]
        n_sites = 0
        for j, (name, table, cs, cl) in enumerate(tables + fuzz + other):
            grid = GRID[::5] if name.startswith("adversarial") else [GRID[(7 * j + i) % len(GRID)] for i in range(2)]
            for a, r in grid + [(1, 0.01)]:
                want = V.sites(table, cs, cl, a, r)
                _sites_equal(_emulated(table, cs, cl, a, r), want, (schedule, name, a, r))
                n_sites += len(want[0])
        assert n_sites > 5000
        assert len(_emulated(*tables[2][1:], -1, -0.5)[0]) == 2020  # the empty table: every position at < 0
        assert len(_emulated(*tables[2][1:], 0, 0.0)[0]) == 0
    finally:
        E.set_schedule("forward")


def _tables_small(tmp_path):
    for name, run in _limit_runs(tmp_path):
        if name in ("limit_contigs", "limit_edges", "limit_mixed"):
            yield name, run.host_counts, run.batch.contig_slot, run.batch.contig_len
    for name, run, _, _ in _combo_runs(tmp_path, seeds=(0,)):
        yield name, run.host_counts, run.batch.contig_slot, run.batch.contig_len


# -------------------------------------------------------------------------------------- variants frame
def test_only_variants_frame_from_sites(manifest, tmp_path):
    """variants_from_run(only_variants=True), now built from the sites, == the per-position frame filtered to its
    variant rows: columns, dtypes, RangeIndex, the empty result, with and without absolute."""
    runs = [_oracle_run(bamio.read_alignment(golden_input(e))) for e in list(manifest["files"].values())[:4]]
    runs += [run for _, run, _, _ in _combo_runs(tmp_path, seeds=(0,))]
    runs += [host_run(*adversarial(4))]
    for run in runs:
        for a, r in ((1, 0.01), (0, 0.25), (-1, -0.5), (2 ** 31, 0.0), (1.5, NAN)):
            for absolute in (False, True):
                full = K.variants_from_run(run, a, r, False, absolute)
                got = K.variants_from_run(run, a, r, True, absolute)
                t = run.host_counts
                keep = np.concatenate([K.variant_alleles(t[0:6, s:e - 1].astype(np.int64), a, r)[3].any(axis=0)
                                       for s, e in map(run.contig_slice, range(run.batch.n_contigs))])
                want = full[keep].reset_index(drop=True)
                pd.testing.assert_frame_equal(got, want)
                assert isinstance(got.index, pd.RangeIndex)
                assert got.dtypes["A"] == (np.int64 if absolute else np.float64)


# ------------------------------------------------------------------------------------------------- VCF
def _two_contig_run():
    """Contig x (L 6) and y (L 3), slot L and padding planted."""
    cols = np.array([
        # x: 0 plain A; 1 A/C; 2 N only besides REF; 3 del top, T variant; 4 N top, A + del variants; 5 depth 0
        [20, 10, 10, 0, 3, 0, 99, 0,
         # y: 0 G/T/A/del; 1 plain; 2 tie A=C (first max A)
         1, 9, 5, 99],
        [0, 8, 0, 0, 0, 0, 99, 0, 0, 0, 5, 99],
        [0, 0, 0, 0, 0, 0, 99, 0, 10, 0, 0, 99],
        [0, 0, 0, 4, 0, 0, 99, 0, 6, 0, 0, 99],
        [0, 0, 6, 0, 8, 0, 99, 0, 0, 0, 0, 99],
        [0, 0, 0, 9, 4, 0, 99, 0, 3, 0, 0, 99],
    ])
    t = np.zeros((19, 12), dtype=np.int32)
    t[0:6] = cols
    return host_run(t, [0, 8], [6, 3], ["x", "y"])


HEADER = [
    "##fileformat=VCFv4.2",
    "##source=kindel " + __version__,
    "##kindelVariants=abs_threshold=1;rel_threshold=0.01;min_base_quality=0;min_mapq=0;exclude_flags=0x0",
    "##contig=<ID=x,length=6>",
    "##contig=<ID=y,length=3>",
    '##INFO=<ID=DP,Number=1,Type=Integer,Description="Depth: A + C + G + T + N + deletions">',
    '##INFO=<ID=AD,Number=R,Type=Integer,Description="Count of REF (the most frequent allele) and of each ALT allele">',
    '##INFO=<ID=AF,Number=A,Type=Float,Description="Share of the depth of each ALT allele, rounded to 4 decimals">',
    "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO",
]


def test_vcf_pinned():
    text = K.variants_vcf_from_run(_two_contig_run(), 1, 0.01)
    assert text.endswith("\n")
    lines = text.splitlines()
    assert lines[:len(HEADER)] == HEADER
    assert lines[len(HEADER):] == [
        "x\t2\t.\tA\tC\t.\tPASS\tDP=18;AD=10,8;AF=0.4444",
        # x:3 has N as its only variant: no line
        "x\t4\t.\tN\tT\t.\tPASS\tDP=13;AD=9,4;AF=0.3077",
        "x\t5\t.\tN\tA,*\t.\tPASS\tDP=15;AD=8,3,4;AF=0.2,0.2667",
        "y\t1\t.\tG\tT,*\t.\tPASS\tDP=20;AD=10,6,3;AF=0.3,0.15",
        "y\t3\t.\tA\tC\t.\tPASS\tDP=10;AD=5,5;AF=0.5",
    ]
    # header only when nothing passes; the filters appear in the header
    text = K.variants_vcf_from_run(_two_contig_run(), 100, 0.5, filters=(20, 30, 0x904))
    assert text.splitlines()[2] == ("##kindelVariants=abs_threshold=100;rel_threshold=0.5;min_base_quality=20;"
                                    "min_mapq=30;exclude_flags=0x904")
    assert text.splitlines()[3:] == HEADER[3:] and text.endswith("\n")
    # zero depth at negative thresholds: REF N, AD 0, every ALT at AF 0.0
    zero = [ln for ln in K.variants_vcf_from_run(_two_contig_run(), -1, -0.5).splitlines() if ln.startswith("x\t6\t")]
    assert zero == ["x\t6\t.\tN\tC,G,T,*\t.\tPASS\tDP=0;AD=0,0,0,0,0;AF=0.0,0.0,0.0,0.0"]


def _check_shape(text, run, abs_threshold, rel_threshold):
    """bcftools-style shape and the AF = `variants` relative value, AD / DP from the table."""
    lines = text.splitlines()
    body = [ln for ln in lines if not ln.startswith("#")]
    assert lines[-len(body) - 1 if body else -1] == HEADER[-1]
    tsv = K.variants_from_run(run, abs_threshold, rel_threshold, only_variants=True)
    rows = {(c, p): i for i, (c, p) in enumerate(zip(tsv["chrom"], tsv["pos"]))}
    order = {name: c for c, name in enumerate(run.batch.contig_names)}
    last = (-1, 0)
    col = {"A": "A", "C": "C", "G": "G", "T": "T", "*": "deletions"}
    for ln in body:
        f = ln.split("\t")
        assert len(f) == 8 and f[2] == "." and f[5] == "." and f[6] == "PASS"
        key = (order[f[0]], int(f[1]))
        assert key > last  # table order: contigs first-seen, positions ascending
        last = key
        alts = f[4].split(",")
        assert len(set(alts)) == len(alts) and "N" not in alts and f[3] in "ACGTN" and f[3] not in alts
        info = dict(kv.split("=") for kv in f[7].split(";"))
        ad, af = info["AD"].split(","), info["AF"].split(",")
        assert len(ad) == len(alts) + 1 and len(af) == len(alts)  # Number=R, Number=A
        row = tsv.iloc[rows[(f[0], int(f[1]))]]
        assert int(info["DP"]) == row["depth"] >= sum(map(int, ad))
        for a, v in zip(alts, af):
            assert float(v) == row[col[a]]
        s = int(run.batch.contig_slot[order[f[0]]]) + int(f[1]) - 1
        t = run.host_counts[0:6, s]
        assert int(ad[0]) == t.max() and [int(x) for x in ad[1:]] == [t["ACGT*".index(a) + (a == "*")] for a in alts]


def test_vcf_shape_and_af_equal_variants(manifest, tmp_path):
    runs = [_oracle_run(bamio.read_alignment(golden_input(e))) for e in manifest["files"].values()]
    runs += [run for _, run, _, _ in _combo_runs(tmp_path, seeds=(0,))]
    runs += [_two_contig_run(), host_run(*adversarial(5))]
    n = 0
    for run in runs:
        for a, r in ((1, 0.01), (0, 0.2), (-1, -0.5)):
            text = K.variants_vcf_from_run(run, a, r)
            _check_shape(text, run, a, r)
            n += text.count("\n")
    assert n > 1000


def test_vcf_equals_restatement(manifest, tmp_path):
    """variants_vcf_from_run on oracle host tables == the header + the lines built from the restatement's sites."""
    items = [(_oracle_run(bamio.read_alignment(golden_input(e))), None) for e in manifest["files"].values()]
    items += [(run, flt) for _, run, _, flt in _combo_runs(tmp_path)]
    for run, flt in items:
        b = run.batch
        mbq, mq, ex = flt or (0, 0, 0)
        contigs = ["##contig=<ID=%s,length=%d>" % (n, L) for n, L in zip(b.contig_names, b.contig_len.tolist())]
        for a, r in ((1, 0.01), (2, 0.25), (0, 0.0)):
            sites = V.sites(run.host_counts, b.contig_slot, b.contig_len, a, r)
            header = HEADER[:2] + ["##kindelVariants=abs_threshold=%s;rel_threshold=%s;min_base_quality=%d;min_mapq=%d;"
                                   "exclude_flags=%s" % (a, r, mbq, mq, hex(ex))] + contigs + HEADER[5:]
            want = "\n".join(header + V.vcf_records(b.contig_names, b.contig_slot, *sites, a, r)) + "\n"
            assert K.variants_vcf_from_run(run, a, r, flt) == want


# ------------------------------------------------------------------------------------------------- CLI
def test_cli_parses_vcf_and_gpus():
    p = cli.build_parser()
    a = p.parse_args(["variants", "x.bam"])
    assert a.vcf is False and a.gpus is None
    a = p.parse_args(["variants", "--vcf", "--gpus", "2", "-a", "3", "-r", "0.2", "x.bam"])
    assert a.vcf is True and a.gpus == 2 and a.abs_threshold == 3 and a.rel_threshold == 0.2


@pytest.mark.parametrize("flag", ["--absolute", "--only-variants", "-o"])
def test_cli_rejects_vcf_with_table_options(flag, capsys):
    with pytest.raises(SystemExit) as e:
        cli.main(["variants", "--vcf", flag, "x.bam"])
    assert e.value.code == 2
    assert "--vcf" in capsys.readouterr().err


def test_cli_routes_vcf_and_gpus(monkeypatch, capsys):
    seen = {}

    def fake_vcf(path, a, r, devices=None, **filters):
        seen["vcf"] = (path, a, r, devices, filters)
        return "##fileformat=VCFv4.2\n"

    def fake_variants(path, a, r, only, absolute, devices=None, **filters):
        seen["tsv"] = (path, a, r, only, absolute, devices, filters)
        return pd.DataFrame({"chrom": ["x"], "pos": [1]})

    monkeypatch.setattr(K, "variants_vcf", fake_vcf)
    monkeypatch.setattr(K, "variants", fake_variants)
    assert cli.main(["variants", "--vcf", "--gpus", "2", "--min-mapq", "5", "x.bam"]) == 0
    assert capsys.readouterr().out == "##fileformat=VCFv4.2\n"
    assert seen["vcf"] == ("x.bam", 1, 0.01, 2, dict(min_base_quality=0, min_mapq=5, exclude_flags=0))
    assert cli.main(["variants", "-o", "--gpus", "3", "x.bam"]) == 0
    assert capsys.readouterr().out == "chrom\tpos\nx\t1\n"
    assert seen["tsv"] == ("x.bam", 1, 0.01, True, False, 3, dict(min_base_quality=0, min_mapq=0, exclude_flags=0))


# ------------------------------------------------------------------------------------------------- ABI
def test_abi_entry_points_refuse_bad_sizes():
    lib = _ffi.load()
    for name in ("kdl_variant_scratch_words", "kdl_variant_count", "kdl_variant_scatter"):
        assert name in _ffi.EXPORTED_SYMBOLS and getattr(lib, name)
    assert lib.kdl_variant_scratch_words(1024) == 2 and lib.kdl_variant_scratch_words(1028) == 3
    buf = np.zeros(19 * 8, dtype=np.int32)
    cs, cl = np.zeros(1, dtype=np.int64), np.full(1, 4, dtype=np.int32)
    sums = np.zeros(4, dtype=np.uint32)
    out = np.zeros(64, dtype=np.int64)

    def count(n_slots, abs_floor=1, counts=buf.ctypes.data, n_contigs=1):
        return lib.kdl_variant_count(counts, n_slots, cs.ctypes.data, cl.ctypes.data, n_contigs, abs_floor, 0.01,
                                     sums.ctypes.data, None)

    def scatter(n_slots, n_sites):
        return lib.kdl_variant_scatter(buf.ctypes.data, n_slots, cs.ctypes.data, cl.ctypes.data, 1, 1, 0.01,
                                       sums.ctypes.data, n_sites, out.ctypes.data, out.ctypes.data, out.ctypes.data,
                                       None)

    for rc in (count(6), count(0), count(-4), count(8, abs_floor=-2), count(8, abs_floor=(1 << 31) + 1),
               count(8, counts=None), count(8, n_contigs=-1), scatter(6, 0), scatter(8, -1), scatter(8, 9)):
        assert rc == 1
