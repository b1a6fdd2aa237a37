"""Several samples in one VCF (`kindel variants --vcf a.bam b.bam ...`), without a GPU.

- K6m (kdl_variant_multi_count / _scatter) under the kernel emulator gives the multi-sample oracle's sites
  (oracle/py_msoracle.py) in both modes, for S = 1, 2, 3 and 7, with counts planted behind each contig and in the
  padding, a sample lacking a contig and pooled counts above 2^31; at S = 1 its bits are K6's and K6r's.
- The product's variants_vcf over a list of paths, every kdl_* call emulated, equals the oracle's text byte for byte
  over a pairwise-covering matrix of reference x filters x primers x mask_overlaps, on BAM and SAM inputs and from
  2-rank host tables.
- A truth set of planted multi-sample cases; the list-of-one invariant; the errors."""
import os
import types

import numpy as np
import pytest

import cohort_cases as CO
import emu_harness as E
import helpers as H
import test_variants_vcf as TV
from test_vcf_combined import on_the_emulator
from kindel_b200 import __version__, bamio, cli, cohort, distributed, engine
from kindel_b200 import kindel as K
from oracle import py_msoracle as MS

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
SOURCE = "kindel {}".format(__version__)
INPUTS = os.path.join(H.ROOT, "tests", "golden", "inputs")


def emulated_k6m(T, cs, cl, ref, a, r):
    """K6m over a host stack T [S, 7, n_slots] on the emulator: (slot int64[n], mask uint8[n])."""
    lib = E.load()
    T = np.ascontiguousarray(T, dtype=np.int32)
    S, _, n_slots = T.shape
    c_slot = np.ascontiguousarray(cs, dtype=np.int64)
    c_len = np.ascontiguousarray(cl, dtype=np.int32)
    refp = None if ref is None else np.ascontiguousarray(ref, dtype=np.uint8)
    sums = np.full(int(lib.kdl_variant_scratch_words(n_slots)), 0xDEADBEEF, dtype=np.uint32)
    args = (T.ctypes.data, S, n_slots, c_slot.ctypes.data, c_len.ctypes.data, len(c_len),
            None if refp is None else refp.ctypes.data, engine.variant_abs_floor(a), float(r))
    E._check(lib.kdl_variant_multi_count(*args, sums.ctypes.data, None), "kdl_variant_multi_count")
    n = int(sums[-1])
    slot = np.full(n + 1, -7, dtype=np.int64)
    mask = np.full(n + 1, 0xEE, dtype=np.uint8)
    E._check(lib.kdl_variant_multi_scatter(*args, sums.ctypes.data, n, slot.ctypes.data, mask.ctypes.data, None),
             "kdl_variant_multi_scatter")
    assert slot[n] == -7 and mask[n] == 0xEE, "K6m wrote past the announced sites"
    return slot[:n], mask[:n]


def as_named(slot, mask, cs, cl):
    c = np.searchsorted(cs, slot, side="right") - 1
    return [("c%d" % int(k), int(s - cs[k]), int(m)) for k, s, m in zip(c.tolist(), slot.tolist(), mask.tolist())]


def k6m_cases():
    for S in (1, 2, 3, 7):
        T, cs, cl, ref, lacking = CO.stacked(10 + S, S)
        names, samples = CO.oracle_samples(T, cs, cl, lacking)
        yield S, T, cs, cl, ref, samples


@needs_emu
def test_k6m_equals_the_oracle_sites():
    n_sites = 0
    for S, T, cs, cl, ref, samples in k6m_cases():
        texts = CO.ref_texts(ref, cs, cl)
        for a, r in TV.GRID[S % 3::9]:
            for mode in ("pooled", "reference"):
                got = as_named(*emulated_k6m(T, cs, cl, ref if mode == "reference" else None, a, r), cs, cl)
                want = MS.site_bits(samples, a, r, texts if mode == "reference" else None)
                assert got == want, (S, a, r, mode)
                n_sites += len(want)
    assert n_sites > 5000


def test_stacked_tables_reach_the_cases():
    T, cs, cl, ref, lacking = CO.stacked(17, 7)
    pooled = T[:, 0:6].astype(np.int64).sum(axis=0)
    assert pooled.max() > 1 << 31 and lacking == {6: 3}
    assert (T[:, 0:6, cs[0] + cl[0]] > 0).all()  # planted in slot L


@needs_emu
def test_k6m_at_one_sample_equals_k6_and_k6r(tmp_path):
    n = 0
    tables = list(TV._tables(tmp_path))
    for j, (name, table, cs, cl) in enumerate(tables[::7] + tables[-3:]):
        table = np.ascontiguousarray(table, dtype=np.int32)
        rng = np.random.default_rng(j)
        ref = rng.integers(0, 5, size=table.shape[1]).astype(np.uint8)
        for a, r in (TV.GRID[(5 * j) % len(TV.GRID)], (1, 0.01)):
            slot, mask = emulated_k6m(table[None, 0:7], cs, cl, None, a, r)
            want = E.variant_sites(table, cs, cl, engine.variant_abs_floor(a), r)
            np.testing.assert_array_equal(slot, want[0], err_msg=name)
            np.testing.assert_array_equal(mask, want[2], err_msg=name)
            slot, mask = emulated_k6m(table[None, 0:7], cs, cl, ref, a, r)
            want = E.variant_sites_ref(table, cs, cl, ref, engine.variant_abs_floor(a), r)
            np.testing.assert_array_equal(slot, want[0], err_msg=name)
            np.testing.assert_array_equal(mask, want[3], err_msg=name)
            n += len(slot)
    assert n > 1000


def test_k6m_abi_rejects_bad_arguments():
    if not E.available():
        pytest.skip("needs g++ and the CUDA headers")
    lib = E.load()
    T = np.zeros((2, 7, 8), dtype=np.int32)
    cs, cl = np.zeros(1, dtype=np.int64), np.full(1, 4, dtype=np.int32)
    sums = np.zeros(4, dtype=np.uint32)
    ok = (T.ctypes.data, 2, 8, cs.ctypes.data, cl.ctypes.data, 1, None, 1, 0.01, sums.ctypes.data, None)
    assert lib.kdl_variant_multi_count(*ok) == 0
    assert lib.kdl_variant_multi_count(T.ctypes.data, 0, *ok[2:]) != 0            # no sample
    assert lib.kdl_variant_multi_count(T.ctypes.data, 2, 6, *ok[3:]) != 0         # n_slots % 4
    ref = np.zeros(16, dtype=np.uint8)
    assert lib.kdl_variant_multi_count(*ok[:6], ref.ctypes.data + 1, *ok[7:]) != 0  # misaligned reference


# ------------------------------------------------------------------------------------------- the product path
@pytest.fixture(scope="module")
def split(tmp_path_factory):
    d = tmp_path_factory.mktemp("cohort")
    paths, fa, bed, rows, refs = CO.split_corpus(d)
    sam_paths = CO.split_corpus(d / ".." / d.name, sam=True)[0]
    return dict(paths=paths, sam_paths=sam_paths, fa=fa, bed=bed, rows=rows, refs=refs, oracle={})


def oracle_text(split, row, names, a=1, r=0.01, paths=None):
    bq, mq, ex, pr, ref, mates = row
    samples = []
    for p in paths or split["paths"]:
        key = (p, bq, mq, ex, pr, mates)
        if key not in split["oracle"]:
            split["oracle"][key] = MS.Sample.from_path(p, bq, mq, ex, split["rows"] if pr else None, mates)
        samples.append(split["oracle"][key])
    return MS.vcf(samples, names, SOURCE, a, r, (bq, mq, ex), os.path.basename(split["bed"]) if pr else None,
                  (os.path.basename(split["fa"]), split["refs"]) if ref else None, mates)


def matrix():
    """(min_base_quality, min_mapq, exclude_flags, primers, reference, mask_overlaps) rows covering every pair."""
    values = ((0, 20), (0, 30), (0, 0x500), (False, True), (False, True), (False, True))
    return [tuple(values[k][b] for k, b in enumerate(row)) for row in CO.covering_rows(6)]


def kwargs(split, row):
    bq, mq, ex, pr, ref, mates = row
    return dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, primers=split["bed"] if pr else None,
                reference=split["fa"] if ref else None, mask_overlaps=mates)


def test_matrix_covers_every_pair():
    rows = matrix()
    for i in range(6):
        for j in range(i + 1, 6):
            assert len({(row[i], row[j]) for row in rows}) == 4


@needs_emu
def test_variants_vcf_of_samples_equals_the_oracle(split, monkeypatch):
    on_the_emulator(monkeypatch)
    names = ["s0", "s1", "s2"]
    for k, row in enumerate(matrix()):
        paths = split["sam_paths"] if k % 2 else split["paths"]
        a, r = ((1, 0.01), (0, 0.0), (2, 0.2))[k % 3]
        got = K.variants_vcf(paths, a, r, samples=names, **kwargs(split, row))
        assert got == oracle_text(split, row, names, a, r), row


@needs_emu
def test_variants_vcf_of_samples_from_host_tables(split, monkeypatch):
    """Each sample's run as a multi-GPU job leaves it: host tables summed over 2 ranks' shards, re-uploaded by
    device_tables -- the same text."""
    on_the_emulator(monkeypatch)
    from kindel_b200.kindel import PileupRun

    def two_ranks(path, devices=None, min_depth=1, min_base_quality=0, min_mapq=0, exclude_flags=0, **kw):
        assert devices == 2
        batch = bamio.read_alignment(path, min_base_quality=min_base_quality, min_mapq=min_mapq,
                                     exclude_flags=exclude_flags)
        total, evs, idx_all = None, [], []
        for rank in range(2):
            idx = distributed.shard_indices(batch, rank, 2, "reads")
            counts, events = engine.pileup(engine.upload(bamio.select_reads(batch, idx)))
            total = counts.numpy().astype(np.int64) if total is None else total + counts.numpy()
            evs.append(events.numpy())
            idx_all.append(idx)
        total = total.astype(np.int32)
        return PileupRun.from_host_tables(batch, total, E.derive(total), distributed.merge_events(evs, idx_all)), None

    monkeypatch.setattr(K, "pileup_run", two_ranks)
    for row in ((0, 0, 0, False, True, False), (20, 30, 0x500, False, False, False)):
        got = K.variants_vcf(split["paths"], 1, 0.01, devices=2, **kwargs(split, row))
        assert got == oracle_text(split, row, ["s0.bam", "s1.bam", "s2.bam"]), row


def _data(text, cols=None):
    return [ln if cols is None else "\t".join(ln.split("\t")[:cols]) for ln in text.splitlines()
            if not ln.startswith("#")]


@needs_emu
def test_a_list_of_one_gives_the_single_sample_lines(split, monkeypatch):
    on_the_emulator(monkeypatch)
    cases = [(os.path.join(INPUTS, "mm2_gp120.bam"), os.path.join(INPUTS, "hxb2-gp120-mutated.fa"), {}),
             (split["paths"][2], split["fa"], {}),
             (split["paths"][2], split["fa"], dict(min_base_quality=20, primers=split["bed"], mask_overlaps=True))]
    n = 0
    for path, fa, kw in cases:
        for ref in (None, fa):
            for a, r in ((1, 0.01), (0, 0.0)):
                one = K.variants_vcf(path, a, r, reference=ref, **kw)
                listed = K.variants_vcf([path], a, r, reference=ref, **kw)
                assert _data(listed, 8) == _data(one), (path, ref, a, r)
                head = [ln for ln in one.splitlines() if ln.startswith("##")]
                assert [ln for ln in listed.splitlines() if ln.startswith("##")][:len(head)] == head
                n += len(_data(one))
    assert n > 300


# ------------------------------------------------------------------------------------------- truth set
@needs_emu
def test_planted_truth_set(tmp_path, monkeypatch):
    on_the_emulator(monkeypatch)
    paths, fa = CO.truth_set(tmp_path)
    names = ["x", "y", "z"]
    samples = [MS.Sample.from_path(p) for p in paths]
    refs = {"a": CO.REF, "b": CO.REF}
    pooled = K.variants_vcf(paths, 1, 0.05, samples=names)
    assert pooled == MS.vcf(samples, names, SOURCE, 1, 0.05)
    by_pos = {(ln.split("\t")[0], int(ln.split("\t")[1])): ln.split("\t") for ln in _data(pooled)}
    fixed = by_pos[("a", CO.FIXED + 1)]  # A all T, B all C: C is the pooled top (first of a tie), T the ALT
    assert fixed[3:5] == ["C", "T"] and fixed[9:] == ["20:0,20:1.0", "20:20,0:0.0", "0:0,0:0.0"]
    with_ref = K.variants_vcf(paths, 1, 0.05, reference=fa, samples=names)
    assert with_ref == MS.vcf(samples, names, SOURCE, 1, 0.05, reference=("truth.fa", refs))
    lines = {(f[0], int(f[1]), f[3], f[4]): f for f in (ln.split("\t") for ln in _data(with_ref))}
    minor = next(f for k, f in lines.items() if k[1] == CO.MINOR + 1)
    assert minor[9:] == ["20:18,2:0.1", "20:20,0:0.0", "0:0,0:0.0"]
    dele = next(f for k, f in lines.items() if k[1] == CO.DEL and len(k[2]) == 3)
    assert dele[7].startswith("INDEL;DP=40;AO=4;") and dele[10].split(":")[1] == "19,1"
    ins = next(f for k, f in lines.items() if k[1] == CO.INS and k[3].endswith("GG"))
    assert ins[9].split(":")[1] == "17,3" and ins[10].split(":")[1] == "19,1"
    assert all(f[11].startswith("0:0,0") and set(f[11].split(":")[2]) <= set("0.,") for k, f in lines.items()
               if k[0] == "a")  # z has no reads on a
    assert "##contig=<ID=a,length=60>" in with_ref and "##kindelSamples=3" in with_ref


# ------------------------------------------------------------------------------------------- errors
def test_sample_names():
    assert cohort.sample_names(["/x/a.bam", "y/b.bam"]) == ["a.bam", "b.bam"]
    with pytest.raises(ValueError, match=r"/x/a.bam and /y/a.bam.*samples="):
        cohort.sample_names(["/x/a.bam", "/y/a.bam"])
    for bad in (["a", "a"], ["a", ""], ["a b", "c"], ["a"], ["a", None], ["a\tb", "c"]):
        with pytest.raises(ValueError):
            cohort.sample_names(["p", "q"], bad)
    assert cohort.sample_names(["p", "p"], ["one", "two"]) == ["one", "two"]


def test_api_errors(tmp_path):
    paths, _ = CO.truth_set(tmp_path)
    with pytest.raises(ValueError, match="strand"):
        K.variants_vcf(paths, strand=True)
    with pytest.raises(ValueError, match="strand"):
        K.variants_vcf(paths, max_sor=2.0)
    with pytest.raises(ValueError, match="samples="):
        K.variants_vcf(paths[0], samples=["x"])
    with pytest.raises(ValueError):
        K.variants_vcf([])


@needs_emu
def test_contig_length_mismatch(tmp_path, monkeypatch):
    on_the_emulator(monkeypatch)
    read = CO._read(0, 0, [(10, "M")], "ACGTACGTAC", "r")
    p1, p2 = tmp_path / "one.bam", tmp_path / "two.bam"
    bamio.write_bam(str(p1), [("a", 60)], [read])
    bamio.write_bam(str(p2), [("a", 61)], [read])
    with pytest.raises(ValueError, match=r"contig 'a' has length 60 in .*one.bam but 61 in .*two.bam"):
        K.variants_vcf([str(p1), str(p2)])


def test_layout_is_the_union_in_first_seen_order():
    lay = cohort.Layout()
    b1 = types.SimpleNamespace(contig_names=["b", "a"], contig_len=np.array([5, 9]), n_contigs=2)
    b2 = types.SimpleNamespace(contig_names=["c", "a"], contig_len=np.array([3, 9]), n_contigs=2)
    assert lay.add(b1, "p1").tolist() == [0, 1]
    slot_a = int(lay.contig_slot[1])
    assert lay.add(b2, "p2").tolist() == [2, 1]
    assert lay.contig_names == ["b", "a", "c"] and int(lay.contig_slot[1]) == slot_a  # appended, nothing moves
    assert lay.n_slots % 4 == 0 and lay.n_slots >= 5 + 9 + 3 + 3


def test_cli_parser_errors(capsys):
    parser = cli.build_parser()
    for argv, needle in ((["variants", "a.bam", "b.bam"], "need --vcf"),
                         (["variants", "--vcf", "--strand", "a.bam", "b.bam"], "--strand"),
                         (["variants", "--vcf", "--max-sor", "2", "a.bam", "b.bam"], "--max-sor")):
        with pytest.raises(SystemExit):
            cli._check_variants_args(parser, parser.parse_args(argv))
        assert needle in capsys.readouterr().err
    args = parser.parse_args(["variants", "--vcf", "a.bam", "b.bam"])
    cli._check_variants_args(parser, args)
    assert args.bam_path == ["a.bam", "b.bam"]


@needs_emu
def test_cli_writes_the_multi_sample_vcf(tmp_path, monkeypatch, capsys):
    on_the_emulator(monkeypatch)
    paths, fa = CO.truth_set(tmp_path)
    assert cli.main(["variants", "--vcf", "--reference", fa, "-r", "0.05", *paths]) == 0
    assert capsys.readouterr().out == K.variants_vcf(paths, 1, 0.05, reference=fa)
    assert cli.main(["variants", "--vcf", paths[0]]) == 0
    assert capsys.readouterr().out == K.variants_vcf(paths[0])
