"""The read selection at the engine's limits without a GPU (tests/select_limit_cases.py): K10p + K14 from their CUDA
source under the kernel emulator on every limit group with planted duplicates, at several SM counts with the lists
shuffled before the sort, against oracle/py_doracle.py; K12 + K13 under the emulator on the same files against
oracle/py_aoracle.py + oracle/py_noracle.py; the composed oracle (oracle/py_seloracle.py) against the single-stage
oracles run one after another on every corpus; the C++ decoder's and the SAM reader's duplicate scores."""
import numpy as np
import pytest

import amplicon_cases as AC
import emu_harness as E
import limit_cases as LC
import select_limit_cases as SL
import test_dedup as TD
import test_normalise as TN
from kindel_b200 import bamio
from kindel_b200 import primers as P
from oracle import py_aoracle as AO
from oracle import py_doracle as DO
from oracle import py_moracle as MO
from oracle import py_noracle as NO
from oracle import py_seloracle as SO

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
GROUPS = sorted(LC.GROUPS)
FILTERS = dict(min_mapq=20, exclude_flags=0x400)
BIG = (1 << 31) - 1


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """{name: (contigs, records, BAM path, SAM path or None)} of every input, written once."""
    d = tmp_path_factory.mktemp("select_limits")
    out = {}
    for g in GROUPS:
        contigs, recs = SL.planted(g)
        out[g] = (contigs, recs) + SL.write(d, g, contigs, recs)
    for name, (contigs, recs) in (("many300_header", SL.many(300, False)), ("many300_shuffled", SL.many(300, True)),
                                  ("twin", SL.twin()), ("interleaved", SL.interleaved())):
        out[name] = (contigs, recs) + SL.write(d, name, contigs, recs, sam=name == "interleaved")
    return out


# ------------------------------------------------------------------------------------------------ the inputs
def test_planted_groups_reach_their_shapes(corpus):
    for g in GROUPS:
        contigs, recs, bam, _ = corpus[g]
        sel = SO.select(bam, dedup=True)
        p, s, shadowed = sel.dedup_totals
        assert p > 0 and s > 0 and shadowed > 0, g
        b = bamio.read_alignment(bam, strand=True, dup=True)
        assert (b.dup_score == -1).any() and (b.dup_score == 0).any(), g
    ends = [DO.end_of(r) for _, r, *_ in MO.kept(corpus["edges"][2], SO.contig_order(corpus["edges"][2]))[1]]
    L = corpus["edges"][0][0][1]
    assert any(e and e[0] < 0 for e in ends) and any(e and e[0] >= L for e in ends)


# ------------------------------------------------------------------------------------------------ K14
@needs_emu
@pytest.mark.parametrize("group", GROUPS)
def test_k14_planted_group_against_the_oracle(corpus, group):
    _, _, bam, _ = corpus[group]
    for filters, sms in (({}, TD.SM_COUNTS), (FILTERS, (3,))):
        b = bamio.read_alignment(bam, strand=True, mates=True, dup=True, **filters)
        want, totals, _ = DO.keep_by_record(bam, b.contig_names, **filters)
        mate = TD.emu_pairs(b)
        for sm in sms:
            keep, got = TD.emu_dedup(b, mate, sm, shuffle=sm)
            assert keep.tolist() == want.tolist(), (group, filters, sm)
            assert got == totals, (group, filters, sm)


@needs_emu
@pytest.mark.parametrize("name", ["many300_header", "many300_shuffled", "twin", "interleaved"])
def test_k14_contigs_against_the_oracle(corpus, name):
    contigs, _, bam, _ = corpus[name]
    b = bamio.read_alignment(bam, strand=True, mates=True, dup=True)
    want, totals, _ = DO.keep_by_record(bam, b.contig_names)
    mate = TD.emu_pairs(b)
    for sm in (1, 7):
        keep, got = TD.emu_dedup(b, mate, sm, shuffle=sm)
        assert keep.tolist() == want.tolist() and got == totals, (name, sm)
    if name != "interleaved":  # the same ends on every contig: each contig keeps the same records
        per = np.diff(b.contig_read_off)
        assert (per == per[0]).all()
        assert (want.reshape(len(per), -1) == want[:per[0]]).all()


# ------------------------------------------------------------------------------------------------ K12 + K13
@needs_emu
@pytest.mark.parametrize("group", GROUPS)
def test_k12_k13_planted_group_against_the_oracles(corpus, group):
    contigs, _, bam, _ = corpus[group]
    rows = SL.scheme_rows(contigs)
    b = bamio.read_alignment(bam, strand=True)
    arr = P.amplicon_arrays(AC.scheme(rows), b.contig_names, b.contig_len)
    labels = AC.emu_assign(b, arr)
    assert labels.tolist() == AO.labels_by_read(bam, b.contig_names, rows).tolist()
    assert (labels >= 0).sum() > 0
    key = np.where(labels >= 0, 2 * labels + b.reverse, -1)
    size = int(np.bincount(key[key >= 0]).max()) if (key >= 0).any() else 1
    for cap in sorted({1, 2, size, BIG}):
        keep = TN._check(labels, b.reverse, arr.n_amplicons, cap)
        if cap == 1 and size > 1:
            assert (keep == 0).any()


# ------------------------------------------------------------------------------------------------ composed oracle
def _stages(tmp_path, contigs, recs, bam, rows, cap, filters):
    """(dedup removed, its totals, cap dropped, contig order of the file between the stages): py_doracle on the file,
    then py_noracle on the file of its kept records, each removed record left in as an unmapped placeholder."""
    names = bamio.read_alignment(bam, **filters).contig_names
    _, totals, gone = DO.keep_by_record(bam, names, **filters)
    mid = tmp_path / "mid.bam"
    bamio.write_bam(str(mid), contigs, SL.placeholders(recs, gone))
    _, dropped = NO.keep_by_record(str(mid), names, rows, cap, **filters)
    return names, gone, totals, dropped, SO.contig_order(str(mid))


@pytest.mark.parametrize("name", GROUPS + ["many300_header", "many300_shuffled", "twin", "interleaved"])
def test_composed_oracle_equals_the_stages_one_after_another(corpus, tmp_path, name):
    contigs, recs, bam, _ = corpus[name]
    rows = SL.scheme_rows(contigs)
    for filters in ({}, FILTERS):
        for cap in (1, 2):
            sel = SO.select(bam, dedup=True, rows=rows, normalise=cap, **filters)
            names, gone, totals, dropped, mid_order = _stages(tmp_path, contigs, recs, bam, rows, cap, filters)
            assert sel.contigs == list(names) == mid_order, (name, filters)
            assert sel.dedup_removed == gone and sel.dedup_totals == totals, (name, filters)
            assert sel.cap_dropped == dropped, (name, filters, cap)
            assert sel.kept == len(bamio.read_alignment(bam, **filters).ref_start) - len(gone) - len(dropped)
        assert SO.select(bam, **filters).removed == set()
        assert SO.select(bam, dedup=True, **filters).dedup_removed == sel.dedup_removed
    if name == "interleaved":
        assert sel.contigs == ["x2", "x0", "x1"] and 0 in sel.dedup_removed
        # the file of the survivors alone would see x0 first: the removed record still counts for the order
        bare = tmp_path / "bare.bam"
        bamio.write_bam(str(bare), contigs, [r for k, r in enumerate(recs) if k not in sel.removed])
        assert SO.contig_order(str(bare)) == ["x0", "x2", "x1"]
        assert bamio.read_alignment(str(bare)).contig_names == ["x0", "x2", "x1"]
        first = {}
        for k, r in enumerate(recs):
            first.setdefault(r[0], k)
        assert not set(first.values()) & sel.cap_dropped  # (the cap keeps the first read of every group)


# ------------------------------------------------------------------------------------------------ decoders
@pytest.mark.parametrize("filters", [{}, dict(FILTERS, min_base_quality=20)])
def test_decoders_give_the_same_scores_on_every_planted_group(corpus, filters):
    for g in GROUPS + ["interleaved"]:
        _, _, bam, sam = corpus[g]
        mf = {k: v for k, v in filters.items() if k != "min_base_quality"}
        names = bamio.read_alignment(bam, **filters).contig_names
        want = [DO.score_of(r) for _, r, *_ in MO.kept(bam, names, **mf)[1]]
        got_bam = bamio.read_bam(bam, dup=True, **filters).dup_score
        got_sam = bamio.read_sam(sam, dup=True, **filters).dup_score
        assert got_bam.tolist() == want and got_sam.tolist() == want, g


# ------------------------------------------------------------------------------------------------ K14s-c's chunk carry
@needs_emu
@pytest.mark.parametrize("mode", ["before", "after", "long"])
@pytest.mark.parametrize("scores", ["random", "tied"])
def test_k14_runs_across_the_carry_chunk(mode, scores):
    # one chunk of K14s-c (256 CTAs of 256 entries) and 300 entries more: the runs that cross into the second chunk
    # take their head from the chunk carry
    m = SL.CHUNK + 300
    rng = np.random.default_rng(len(mode))
    run, _ = SL.carry_runs(m, rng, mode)
    perm = rng.permutation(m)
    score = rng.integers(0, 5, m) * 100 if scores == "random" else np.full(m, 77)
    b = SL.hand_batch(run[perm], np.zeros(m), score, int(run[-1]) + 100)
    keep, _ = TD._check_batch(b, sm_counts=(1,))
    assert int(keep.sum()) == int(run[-1]) + 1
