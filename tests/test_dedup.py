"""Duplicate removal (`--dedup`, an extension) without a GPU: the oracle's two forms against each other and the truth
set (tests/dedup_cases.py); the C++ decoder's and the Python text reader's duplicate scores; K10p + K14k + K14s from
their CUDA source under the kernel emulator against the oracle, on the truth set, random batches, one key holding
every read, runs across every CTA boundary and tiny batches; the argument checks; the CLI, REPORT and VCF header
lines."""

import ctypes as C

import numpy as np
import pytest

import dedup_cases as D
import emu_harness as E
from kindel_b200 import _ffi, bamio, cli, synth, vcf
from kindel_b200 import kindel as K
from oracle import py_doracle as DO

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
SM_COUNTS = (1, 2, 3, 7)


def _truth_file(tmp_path, name="t.sam"):
    p = tmp_path / name
    p.write_text(D.sam_text())
    return p


# ------------------------------------------------------------------------------------------------ oracle
def _random_reads(rng, n, n_contigs, span):
    contig = np.sort(rng.integers(0, n_contigs, n))
    u = rng.integers(-3, span, n)
    strand = rng.integers(0, 2, n)
    alone = rng.random(n) < 0.1
    score = rng.integers(0, 4, n) * 100  # few values: many ties
    mate = np.full(n, -1)
    perm = rng.permutation(n)
    for k in range(0, int(0.7 * n) - 1, 2):  # disjoint pairs on one contig
        a, b = perm[k], perm[k + 1]
        if contig[a] == contig[b]:
            mate[b] = a
    return contig, u, strand, alone, score, mate


def _loop_of(contig, u, strand, alone, score, mate):
    ends = [None if a else (int(x), int(s)) for x, s, a in zip(u, strand, alone)]
    pairs = {int(r2): int(m) for r2, m in enumerate(mate) if m >= 0}
    return DO.keep_loop(contig.tolist(), ends, score.tolist(), pairs)


def test_oracle_vectorised_equals_the_loop():
    rng = np.random.default_rng(1)
    for trial in range(60):
        n = int(rng.integers(0, 400))
        args = _random_reads(rng, n, int(rng.integers(1, 4)), int(rng.integers(1, 40)))
        want, wt = _loop_of(*args)
        got, gt = DO.keep_vectorised(*args)
        assert got.tolist() == want.tolist() and gt == wt, trial


def test_oracle_matches_the_truth_set(tmp_path):
    keep, totals, removed = DO.keep_by_record(str(_truth_file(tmp_path)), D.CONTIGS)
    assert keep.tolist() == D.engine_order(D.KEEP)
    assert totals == D.TOTALS
    assert removed == {k for k, v in enumerate(D.KEEP) if not v}


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("filters", [{}, dict(min_mapq=30, exclude_flags=0x100, min_base_quality=20)])
def test_decoders_give_the_same_scores(tmp_path, filters):
    sam = _truth_file(tmp_path)
    from oracle import py_moracle

    lengths, recs = py_moracle.kept(str(sam), D.CONTIGS, filters.get("min_mapq", 0), filters.get("exclude_flags", 0))
    want = [DO.score_of(r) for _, r, *_ in recs]
    bam = tmp_path / "t.bam"
    contigs = [("c0", 2000), ("c1", 2000)]
    recs_bam = [(D.CONTIGS.index(rn), pos - 1, f, bamio.parse_cigar_text(cig), D.SEQ, q, 60,
                 None if qual == "*" else bytes(ord(c) - 33 for c in qual),
                 D.CONTIGS.index(rn) if nx == "=" else (-1 if nx == "*" else D.CONTIGS.index(nx)), pn - 1)
                for q, f, rn, pos, cig, nx, pn, qual, _ in D.ROWS]
    bamio.write_bam(str(bam), contigs, recs_bam)
    for path in (sam, bam):
        for b in (bamio.read_alignment(path, dup=True, **filters), bamio.read_sam(sam, dup=True, **filters)):
            assert b.dup_score is not None and b.dup_score.dtype == np.int32
            assert b.dup_score.tolist() == want, path
    assert bamio.read_alignment(sam, **filters).dup_score is None
    assert bamio.read_bam(bam, **filters).dup_score is None


def test_scores_saturate_and_survive_select_and_save(tmp_path):
    assert bamio.dup_score(0, "~" * 40, "A" * 40) == 93 * 40
    assert bamio.dup_score(0x100, "~~", "AC") == -1 and bamio.dup_score(0x800, "*", "AC") == -1
    assert bamio.dup_score(0, "*", "AC") == 0
    b = bamio.read_alignment(_truth_file(tmp_path), dup=True, strand=True, mates=True)
    sub = bamio.select_reads(b, [3, 1, 40])
    assert sub.dup_score.tolist() == b.dup_score[[3, 1, 40]].tolist()  # (the given order inside a contig)
    bamio.save_batch(str(tmp_path / "w"), sub)
    assert bamio.load_batch(str(tmp_path / "w")).dup_score.tolist() == sub.dup_score.tolist()
    masked = bamio.with_mask(b, np.zeros(b.n_reads, dtype=np.int64), np.zeros(0, dtype=np.uint32))
    assert masked.dup_score.tolist() == b.dup_score.tolist()
    bamio.save_batch(str(tmp_path / "w"), bamio.read_alignment(_truth_file(tmp_path)))
    assert bamio.load_batch(str(tmp_path / "w")).dup_score is None


# ------------------------------------------------------------------------------------------------ K14 under the emulator
def emu_pairs(batch):
    """K10p (kdl_mates_pair) under the emulator: mate int32 [n]."""
    lib = E.load()
    st, keep = E._host_batch(batch)
    n = batch.n_reads
    idx = np.flatnonzero(batch.pair_role)
    order = idx[np.argsort(batch.name_hash[idx], kind="stable")].astype(np.int32)
    mate = np.full(max(n, 1), -1, dtype=np.int32)
    E._check(lib.kdl_mates_pair(C.byref(st), batch.name_hash.ctypes.data, batch.mate_start.ctypes.data,
                                batch.pair_role.ctypes.data, order.ctypes.data if order.size else None, order.size,
                                mate.ctypes.data, None), "kdl_mates_pair")
    return mate[:n]


_LISTS = (("pair_contig", np.int32, 0), ("pair_e1", np.int64, 0), ("pair_e2", np.int64, 0), ("pair_rank", np.uint64, 0),
          ("pair_r1", np.int32, 0), ("pair_r2", np.int32, 0), ("single_contig", np.int32, 1),
          ("single_key", np.int64, 1), ("single_rank", np.uint64, 1), ("single_read", np.int32, 1),
          ("end", np.int64, 1), ("paired", np.uint8, 1))


def emu_dedup(batch, mate=None, sm_count=E.SM_COUNT, shuffle=None):
    """K14k + the sort + K14s under the emulator, as engine.dedup runs them: (keep uint8 [n], totals).  Every buffer
    carries a poisoned element past its end, checked.  shuffle: a seed to permute each list before the sort (the
    device compacts them in any order)."""
    lib = E.load()
    E._sm(sm_count)
    st, keepalive = E._host_batch(batch)
    n = batch.n_reads
    t = {f: np.full(max(n if full else n // 2, 1) + 1, 0x5A, dtype=dt) for f, dt, full in _LISTS}
    lists = _ffi.KdlDedupLists(*(t[f].ctypes.data for f, _, _ in _LISTS))
    keep = np.full(n + 1, 0xEE, dtype=np.uint8)
    totals = np.full(_ffi.KDL_DEDUP_TOTALS + 1, -7, dtype=np.int64)
    rev = np.ascontiguousarray(batch.reverse, dtype=np.uint8)
    score = np.ascontiguousarray(batch.dup_score, dtype=np.int32)
    mate = None if mate is None else np.ascontiguousarray(mate, dtype=np.int32)
    E._check(lib.kdl_dedup_entries(C.byref(st), rev.ctypes.data, score.ctypes.data,
                                   mate.ctypes.data if mate is not None and n else None, C.byref(lists),
                                   keep.ctypes.data, totals.ctypes.data, None), "kdl_dedup_entries")
    n_pair, n_single = int(totals[0]), int(totals[1])
    assert n_pair <= n // 2 and n_single <= n
    for f, _, full in _LISTS:
        assert t[f][-1] == 0x5A, "K14k wrote past " + f
    if shuffle is not None:  # the same entries in another order
        rng = np.random.default_rng(shuffle)
        for fields, m in ((_LISTS[:6], n_pair), (_LISTS[6:10], n_single)):
            p = rng.permutation(m)
            for f, _, _ in fields:
                t[f][:m] = t[f][:m][p]
    p_order = np.lexsort((t["pair_e2"][:n_pair], t["pair_e1"][:n_pair], t["pair_contig"][:n_pair])).astype(np.int64)
    s_order = np.lexsort((t["single_key"][:n_single], t["single_contig"][:n_single])).astype(np.int64)
    words = int(lib.kdl_dedup_scratch_words(max(n_pair, n_single)))
    scratch = np.full(max(words, 2) + 1, 0x5A5A5A5A, dtype=np.int32)
    E._check(lib.kdl_dedup_select(C.byref(lists), p_order.ctypes.data if n_pair else None, n_pair,
                                  s_order.ctypes.data if n_single else None, n_single, scratch.ctypes.data, words,
                                  keep.ctypes.data, totals.ctypes.data, None), "kdl_dedup_select")
    assert keep[n] == 0xEE and totals[-1] == -7 and scratch[-1] == 0x5A5A5A5A, "K14 wrote past its outputs"
    return keep[:n], tuple(int(x) for x in totals[2:5])


def _oracle_of_batch(batch, mate):
    """keep_vectorised over a batch's reads (ends from its CIGARs, the batch's own strands and scores)."""
    u, alone = _batch_ends(batch)
    contig = np.repeat(np.arange(batch.n_contigs), np.diff(batch.contig_read_off))
    return DO.keep_vectorised(contig, u, batch.reverse, alone | (batch.dup_score < 0), batch.dup_score, mate)


def _batch_ends(batch):
    """(u, no reference-consuming op) of every read of a batch, from its host CIGARs."""
    n = batch.n_reads
    u = np.zeros(n, dtype=np.int64)
    alone = np.zeros(n, dtype=bool)
    co = batch.cig_off.astype(np.int64)
    for r in range(n):
        ops = [(int(w >> 4), "MIDNSHP=X"[w & 15] if (w & 15) < 9 else "?") for w in batch.cigar[co[r]:co[r + 1]]]
        rec = type("R", (), dict(flag=16 if batch.reverse[r] else 0, pos=int(batch.ref_start[r]) + 1, cigars=ops))
        e = DO.end_of(rec)
        alone[r] = e is None
        u[r] = 0 if e is None else e[0]
    return u, alone


def _check_batch(batch, mate=None, sm_counts=SM_COUNTS):
    want, wt = _oracle_of_batch(batch, np.full(batch.n_reads, -1) if mate is None else mate)
    for sm in sm_counts:
        keep, totals = emu_dedup(batch, mate, sm, shuffle=sm)
        assert keep.tolist() == want.tolist(), sm
        assert totals == wt, sm
    return want, wt


@needs_emu
def test_k14_truth_set(tmp_path):
    b = bamio.read_alignment(_truth_file(tmp_path), strand=True, mates=True, dup=True)
    mate = emu_pairs(b)
    for sm in SM_COUNTS:
        keep, totals = emu_dedup(b, mate, sm)
        assert keep.tolist() == D.engine_order(D.KEEP), sm
        assert totals == D.TOTALS


@needs_emu
def test_k14_synthetic_pairs_against_the_oracle():
    b = synth.dup_pairs(2, 3000, 30, dup_frac=0.3)[0]
    mate = emu_pairs(b)
    want, wt = _check_batch(b, mate)
    assert wt[0] > 0
    # a fifth of the records gone: their mates are singles, some on a pair's end
    sub = bamio.select_reads(b, np.flatnonzero(np.random.default_rng(3).random(b.n_reads) < 0.8))
    want, wt = _check_batch(sub, emu_pairs(sub))
    assert wt[0] > 0 and wt[1] > 0 and wt[2] > 0


@needs_emu
def test_k14_random_singles_many_contigs_and_ties():
    rng = np.random.default_rng(3)
    b = synth.mixed_reads(4, [700, 500, 900], 40, 0.3)
    b.reverse = rng.integers(0, 2, b.n_reads).astype(np.uint8)
    b.dup_score = (rng.integers(-1, 3, b.n_reads) * 50).astype(np.int32)
    _check_batch(b)


@needs_emu
def test_k14_one_key_holding_every_read_and_runs_across_every_cta():
    n = 3000  # 12 CTAs of 256 entries
    b = synth.simple_reads(5, [2000], 1, read_len=40)
    starts = np.full(n, 100)
    one = bamio.finalize(b.contig_names, b.contig_len, [0, n], starts, np.arange(n) * 5, np.full(n, 40),
                         np.arange(n + 1), np.full(n, 40 << 4), np.tile(b.seq4[:5], n), n_records=n,
                         reverse=np.zeros(n, dtype=np.uint8),
                         dup_score=np.random.default_rng(6).integers(0, 1000, n).astype(np.int32))
    keep, _ = _check_batch(one)
    assert int(keep.sum()) == 1
    # runs of 300 entries, offset from the CTAs' 256
    runs = bamio.finalize(b.contig_names, b.contig_len, [0, n], (np.arange(n) + 77) // 300, np.arange(n) * 5,
                          np.full(n, 40), np.arange(n + 1), np.full(n, 40 << 4), np.tile(b.seq4[:5], n), n_records=n,
                          reverse=np.zeros(n, dtype=np.uint8), dup_score=np.full(n, 7, dtype=np.int32))
    keep, _ = _check_batch(runs)
    assert int(keep.sum()) == 11


@needs_emu
def test_k14_tiny_and_empty_batches():
    rng = np.random.default_rng(7)
    for n_reads in (0, 1, 2, 5, 31, 33):
        b = synth.simple_reads(8, [300], 1, read_len=20)
        idx = rng.integers(0, b.n_reads, n_reads) if b.n_reads else np.zeros(0, dtype=np.int64)
        sub = bamio.select_reads(b, np.sort(idx))
        sub.reverse = rng.integers(0, 2, sub.n_reads).astype(np.uint8)
        sub.dup_score = rng.integers(-1, 2, sub.n_reads).astype(np.int32)
        _check_batch(sub, sm_counts=(1, 3))


@needs_emu
def test_k14_refuses_bad_arguments():
    lib = E.load()
    b = synth.simple_reads(9, [300], 2, read_len=20)
    st, keepalive = E._host_batch(b)
    n = b.n_reads
    t = {f: np.zeros(max(n, 1), dtype=dt) for f, dt, _ in _LISTS}
    lists = _ffi.KdlDedupLists(*(t[f].ctypes.data for f, _, _ in _LISTS))
    rev = np.zeros(n, dtype=np.uint8)
    score = np.zeros(n, dtype=np.int32)
    keep = np.zeros(n, dtype=np.uint8)
    totals = np.zeros(8, dtype=np.int64)
    ok = (C.byref(st), rev.ctypes.data, score.ctypes.data, None, C.byref(lists), keep.ctypes.data, totals.ctypes.data,
          None)
    assert lib.kdl_dedup_entries(*ok) == 0
    assert lib.kdl_dedup_entries(ok[0], None, *ok[2:]) == 1  # no strands
    assert lib.kdl_dedup_entries(*ok[:4], None, *ok[5:]) == 1  # no lists
    assert lib.kdl_dedup_entries(*ok[:6], None, None) == 1  # no totals
    bad = _ffi.KdlDedupLists(*(t[f].ctypes.data for f, _, _ in _LISTS[:-1]), None)
    assert lib.kdl_dedup_entries(*ok[:4], C.byref(bad), *ok[5:]) == 1
    order = np.zeros(4, dtype=np.int64)
    words = int(lib.kdl_dedup_scratch_words(4))
    scratch = np.zeros(words, dtype=np.int32)
    sel = lambda o, m, w: (C.byref(lists), o, m, None, 0, scratch.ctypes.data, w, keep.ctypes.data,  # noqa: E731
                           totals.ctypes.data, None)
    assert lib.kdl_dedup_select(*sel(order.ctypes.data, 4, words)) == 0
    assert lib.kdl_dedup_select(*sel(order.ctypes.data, 4, words - 1)) == 1  # scratch too small
    assert lib.kdl_dedup_select(*sel(None, 4, words)) == 1  # no order
    assert lib.kdl_dedup_select(*sel(order.ctypes.data, -1, words)) == 1
    assert lib.kdl_dedup_select(*sel(None, 0, 0)) == 0  # nothing to select
    assert lib.kdl_dedup_scratch_words(-1) == -1 and lib.kdl_dedup_scratch_words(1 << 31) == -1


# ------------------------------------------------------------------------------------------------ interface
def test_dedup_off_decodes_nothing_new(tmp_path, monkeypatch):
    seen = []
    real = bamio.read_alignment
    monkeypatch.setattr(bamio, "read_alignment", lambda *a, **kw: seen.append(kw) or real(*a, **kw))
    monkeypatch.setattr(K, "PileupRun", lambda *a, **kw: (_ for _ in ()).throw(StopIteration()))
    with pytest.raises(StopIteration):
        K.pileup_run(str(_truth_file(tmp_path)))
    assert "dup" not in seen[0] and "mates" not in seen[0]
    with pytest.raises(ValueError, match="dedup must be True or False"):
        K.pileup_run("missing.bam", dedup="yes")


@pytest.mark.parametrize("cmd", [["consensus", "a.bam"], ["weights", "a.bam"], ["features", "a.bam"],
                                 ["variants", "a.bam", "--vcf"], ["variants", "a.bam", "b.bam", "--vcf"]])
def test_cli_passes_dedup_on(monkeypatch, cmd):
    seen = []

    class _Res:
        refs_reports, consensuses = {}, []

    import pandas as pd

    monkeypatch.setattr(K, "bam_to_consensus", lambda *a, **kw: seen.append(kw) or _Res())
    monkeypatch.setattr(K, "variants_vcf", lambda *a, **kw: seen.append(kw) or "")
    monkeypatch.setattr(K, "weights", lambda *a, **kw: seen.append(kw) or pd.DataFrame())
    monkeypatch.setattr(K, "features", lambda *a, **kw: seen.append(kw) or pd.DataFrame())
    cli.main(cmd + ["--dedup"])
    cli.main(cmd)
    assert seen[0]["dedup"] is True and "dedup" not in seen[1]


def test_cli_amplicons_summary_names_the_removed_duplicates(tmp_path, monkeypatch, capsys):
    import pandas as pd

    bed = tmp_path / "s.bed"
    bed.write_text("c\t0\t5\tx_LEFT\t1\nc\t20\t25\tx_RIGHT\t1\n")

    def fake(paths, primers, min_depth, **kw):
        df = pd.DataFrame({"sample": ["s"], "contig": ["c"], "amplicon": ["x"], "pool": ["1"], "start": [0],
                           "end": [25], "insert_start": [5], "insert_end": [20], "reads": [9], "mean_depth": [9.0],
                           "lowest_depth": [9], "covered": [1.0], "status": ["ok"]}, columns=K.AMPLICON_COLUMNS)
        df.attrs["reads"] = {"s": (12, 9, 3, 0, 0)}
        if kw.get("dedup"):
            df.attrs["duplicates"] = {"s": 17}
        return df

    monkeypatch.setattr(K, "amplicons", fake)
    cli.main(["amplicons", "s", "--primers", str(bed), "--dedup"])
    assert capsys.readouterr().err.strip() == ("s: 12 reads kept: 9 assigned, 3 unprimed, 0 mispaired, 0 ambiguous; "
                                               "1 amplicons, 0 dropouts; 17 duplicate reads removed")
    cli.main(["amplicons", "s", "--primers", str(bed)])
    assert "duplicate" not in capsys.readouterr().err


def test_report_line_sits_between_the_primer_and_normalise_lines():
    args = ("ref", K.DepthRange(0, 9), [None] * 3, None, "a.bam", False, 1, 9, 0.1, False, False)
    plain = K.build_report(*args, primers="s.bed", normalised=(200, 35, 965)).splitlines()
    on = K.build_report(*args, primers="s.bed", normalised=(200, 35, 965), deduplicated=(4, 3, 89, 100)).splitlines()
    k = plain.index("- primers: s.bed")
    assert on[:k + 1] == plain[:k + 1] and on[k + 2:] == plain[k + 1:]
    assert on[k + 1] == "- duplicates: 4 pairs and 3 single reads removed, 89 of 100 reads kept"
    assert on[k + 2].startswith("- normalise:")
    alone = K.build_report(*args, deduplicated=(0, 0, 5, 5)).splitlines()
    assert "- duplicates: 0 pairs and 0 single reads removed, 5 of 5 reads kept" in alone


def test_vcf_header_line_sits_between_the_primer_and_normalise_lines(tmp_path):
    from kindel_b200 import primers as P

    bed = tmp_path / "s.bed"
    bed.write_text("c\t0\t5\tx_LEFT\t1\nc\t20\t25\tx_RIGHT\t1\n")
    ps = P.load_primers(str(bed))
    plain = vcf.header(["c"], [30], 1, 0.01, None, ps, normalise=200)
    on = vcf.header(["c"], [30], 1, 0.01, None, ps, normalise=200, dedup=True)
    k = plain.index("##kindelPrimers=s.bed")
    assert on == plain[:k + 1] + ["##kindelDedup=fragment ends, base-quality score"] + plain[k + 1:]
    assert vcf.header(["c"], [30], 1, 0.01, None, ps, dedup=False) == vcf.header(["c"], [30], 1, 0.01, None, ps)
    no_primers = vcf.header(["c"], [30], 1, 0.01, None, dedup=True)
    assert "##kindelDedup=fragment ends, base-quality score" in no_primers
