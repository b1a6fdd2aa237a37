"""The read selection at the engine's limits on the GPU (tests/select_limit_cases.py): K10p + K14 and K12 + K13
through the real library against the oracles on every limit group with planted duplicates (BAM and SAM), on 2 500
contigs in header order and shuffled and on two identical contigs, each twice (the lists are compacted in any
order); K14 on hand-made batches whose sorted lists cross the chunks of its carry scan (65 536 entries), with runs
on CTA and chunk boundaries, all scores tied and both mates at the score cap; K13 at the device's own grid, the
clamped grid and one CTA; and the whole chain -- filters, `--dedup`, `--normalise N`, `--primers`,
`--mask-overlaps` -- against the same commands on a file of the composed oracle's kept records
(oracle/py_seloracle.py), every removed record left in it as an unmapped placeholder so that the contigs keep their
first-seen order."""
import random

import numpy as np
import pytest

import amplicon_cases as AC
import limit_cases as LC
import select_limit_cases as SL
from kindel_b200 import _ffi, bamio, engine, synth
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from oracle import py_aoracle as AO
from oracle import py_doracle as DO
from oracle import py_noracle as NO
from oracle import py_seloracle as SO

pytestmark = pytest.mark.gpu

GROUPS = sorted(LC.GROUPS)
FILTERS = dict(min_mapq=20, exclude_flags=0x400)
CAP = (1 << 31) - 1
MARKS = ("- bam_path:", "- duplicates:", "- normalise:", "##kindelDedup", "##kindelNormalise")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """{name: (contigs, records, BAM, SAM or None, scheme rows, BED)} of every input, written once."""
    d = tmp_path_factory.mktemp("gpu_select_limits")
    out = {}
    cases = [(g, SL.planted(g), True) for g in GROUPS]
    cases += [("many_header", SL.many(SL.N_MANY, False), False), ("many_shuffled", SL.many(SL.N_MANY, True), False),
              ("twin", SL.twin(), False), ("interleaved", SL.interleaved(), True)]
    for name, (contigs, recs), sam in cases:
        bam, sam_path = SL.write(d, name, contigs, recs, sam=sam)
        rows = SL.scheme_rows(contigs)
        bed = d / (name + ".bed")
        bed.write_text(AC.bed_text(rows))
        out[name] = (contigs, recs, bam, sam_path, rows, str(bed))
    return out


def _device_selection(path, rows, cap, filters):
    """(batch, [(dedup keep, stats, labels, normalise keep, total, dropped)] of two uploads) through the library."""
    import torch

    b = bamio.read_alignment(path, strand=True, mates=True, dup=True, **filters)
    arr = P.amplicon_arrays(AC.scheme(rows), b.contig_names, b.contig_len)
    runs = []
    for _ in range(2):
        db = engine.upload(b)
        keep, stats = engine.dedup(db)
        label = engine.assign_amplicons(db, arr)
        nk, total, dropped = engine.normalise(label, torch.from_numpy(b.reverse).to(db.device), arr.n_amplicons, cap)
        runs.append((keep.cpu().numpy(), stats, label.cpu().numpy(), nk.cpu().numpy(), total.cpu().numpy(),
                     int(dropped.item())))
    return b, runs


def _check_selection(path, rows, many, filters):
    for cap in (1, 2):
        b, runs = _device_selection(path, rows, cap, filters)
        want, totals, _ = DO.keep_by_record(path, b.contig_names, **filters)
        labels = AO.labels_of_batch(b, rows) if many else AO.labels_by_read(path, b.contig_names, rows, **filters)
        nwant = NO.keep_loop(labels, b.reverse, cap)
        for keep, stats, label, nk, total, dropped in runs:
            assert keep.tolist() == want.tolist() and stats == totals, (path, filters)
            assert label.tolist() == labels.tolist(), (path, filters)
            assert nk.tolist() == nwant.tolist() and dropped == int((nwant == 0).sum()), (path, filters, cap)
            assert total.tolist() == NO.totals(labels, b.reverse, total.shape[0] // 2).tolist()
    return b, want


@pytest.mark.parametrize("group", GROUPS)
def test_keep_bytes_on_planted_groups(files, group):
    _, _, bam, sam, rows, _ = files[group]
    for path in (bam, sam):
        for filters in ({}, FILTERS):
            _check_selection(path, rows, False, filters)


@pytest.mark.parametrize("name", ["many_header", "many_shuffled", "twin"])
def test_keep_bytes_on_many_contigs(files, name):
    contigs, _, bam, _, rows, _ = files[name]
    b, want = _check_selection(bam, rows, True, {})
    assert b.n_contigs == len(contigs)
    per = np.diff(b.contig_read_off)
    assert (per == per[0]).all() and (want.reshape(len(per), -1) == want[:per[0]]).all()  # nothing across contigs
    assert (list(b.contig_names) == sorted(b.contig_names)) == (name != "many_shuffled")


# ------------------------------------------------------------------------------------------------ K14 at GPU sizes
def _check_dedup(b, mate=None):
    keep, stats = engine.dedup(engine.upload(b), None if mate is None else engine_mate(mate))
    u = np.where(b.reverse == 1, b.ref_start.astype(np.int64) + 39, b.ref_start)
    m = np.full(b.n_reads, -1) if mate is None else mate
    want, totals = DO.keep_vectorised(np.zeros(b.n_reads), u, b.reverse, b.dup_score < 0, b.dup_score, m)
    assert keep.cpu().numpy().tolist() == want.tolist() and stats == totals
    return want, totals


def engine_mate(mate):
    import torch

    return torch.from_numpy(np.asarray(mate, dtype=np.int32)).cuda()


@pytest.mark.parametrize("m", [SL.CHUNK - 1, SL.CHUNK, SL.CHUNK + 1, 300_007])
@pytest.mark.parametrize("scores", ["random", "tied"])
@pytest.mark.parametrize("mode", SL.MODES)
def test_k14_single_list_across_the_carry_chunks(m, scores, mode):
    rng = np.random.default_rng(m)
    run, _ = SL.carry_runs(m, rng, mode)
    perm = rng.permutation(m)  # batch order unlike the sorted order: the indices decide the ties
    starts = run[perm]
    score = rng.integers(0, 5, m) * 100 if scores == "random" else np.full(m, 77)
    b = SL.hand_batch(starts, np.zeros(m), score, int(run[-1]) + 100)
    want, totals = _check_dedup(b)
    assert totals[1] == m - int(run[-1]) - 1
    if scores == "tied":  # the smallest index of every run stays
        first = np.full(int(run[-1]) + 1, m)
        np.minimum.at(first, starts, np.arange(m))
        assert np.flatnonzero(want).tolist() == sorted(first.tolist())


@pytest.mark.parametrize("n_pairs", [SL.CHUNK - 1, SL.CHUNK, SL.CHUNK + 1, 300_007])
@pytest.mark.parametrize("mode", SL.MODES)
def test_k14_pair_list_across_the_carry_chunks(n_pairs, mode):
    rng = np.random.default_rng(n_pairs)
    run, _ = SL.carry_runs(n_pairs, rng, mode)
    n_runs = int(run[-1]) + 1
    # R1 forward at the run's start, R2 reverse ending 400 further: one key (contig, E1, E2) per run
    r1_start, r2_start = run, run + 400 - 39
    starts = np.concatenate((r1_start, r2_start))
    reverse = np.concatenate((np.zeros(n_pairs), np.ones(n_pairs)))
    score = np.concatenate((rng.integers(0, 3, n_pairs), rng.integers(0, 3, n_pairs))) * 1000
    cap_runs = run % 3 == 0  # both mates at the score cap: the pair sum 2^32 - 2 fills the rank's score field
    score[:n_pairs][cap_runs] = CAP
    score[n_pairs:][cap_runs] = CAP
    perm = rng.permutation(2 * n_pairs)
    inv = np.empty_like(perm)
    inv[perm] = np.arange(2 * n_pairs)
    mate = np.full(2 * n_pairs, -1)
    mate[inv[n_pairs:]] = inv[:n_pairs]  # R2 -> R1, in batch order
    b = SL.hand_batch(starts[perm], reverse[perm], score[perm], n_runs + 500)
    want, totals = _check_dedup(b, mate)
    assert totals[0] == n_pairs - n_runs and totals[1] == 0


def test_k14_one_key_holding_every_entry():
    m = 300_007
    for score in (np.full(m, 9), np.random.default_rng(2).integers(0, 1 << 20, m)):
        want, _ = _check_dedup(SL.hand_batch(np.full(m, 50), np.zeros(m), score, 200))
        assert int(want.sum()) == 1


# ------------------------------------------------------------------------------------------------ K13 at the device grid
def _grid(n, n_amplicons):
    lib = _ffi.load()
    return int(lib.kdl_normalise_scratch_words(n, n_amplicons)) // (2 * n_amplicons)


def _labels(n, n_amplicons, per, rng):
    """Runs of one label 300 reads long, offset from the tiles, a run over every CTA boundary (every per tiles), and
    labels -1, -2, -3 interleaved."""
    lab = ((np.arange(n) + 77) // 300 * 7919) % n_amplicons
    for j, b in enumerate(range(per * 256, n, per * 256)):
        lab[max(b - 150, 0):b + 150] = (j * 31) % n_amplicons
    lab[rng.random(n) < 0.1] = -1
    lab[np.arange(n) % 7 == 3] = -2
    lab[np.arange(n) % 11 == 5] = -3
    return lab


def _check_normalise(n, n_amplicons, caps, rng):
    import torch

    g = _grid(n, n_amplicons)
    tiles = max((n + 255) // 256, 1)
    per = -(-tiles // g)
    lab = _labels(n, n_amplicons, per, rng)
    rev = rng.integers(0, 2, n)
    for cap in caps:
        keep, total, dropped = engine.normalise(torch.from_numpy(lab.astype(np.int32)).cuda(),
                                                torch.from_numpy(rev.astype(np.uint8)).cuda(), n_amplicons, cap)
        want = NO.keep_vectorised(lab, rev, cap)
        assert keep.cpu().numpy().tolist() == want.tolist(), (n, n_amplicons, cap)
        assert int(dropped.item()) == int((want == 0).sum())
        assert np.array_equal(total.cpu().numpy(), NO.totals(lab, rev, n_amplicons))
    return g


def _expected_grid(n, n_amplicons, sms):
    """normalise_grid's G: 2 per SM, at most the tiles, H within 2^24 words; then ceil(tiles / per) CTAs of per tiles."""
    tiles = max((n + 255) // 256, 1)
    g = max(min(2 * sms, tiles, (1 << 24) // (2 * n_amplicons)), 1)
    per = -(-tiles // g)
    return -(-tiles // per)


def test_k13_at_the_device_grid_the_clamped_grid_and_one_cta(capsys):
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(13)
    n = 2 * sms * 256 * 3 - 100  # three tiles per CTA, the last one short
    full = _check_normalise(n, 1000, (1, 5, 300), rng)
    assert full == 2 * sms == _expected_grid(n, 1000, sms)
    clamped = _check_normalise(n, 40_000, (1, 300), rng)
    assert 1 < clamped < 2 * sms and clamped == _expected_grid(n, 40_000, sms)
    one = _check_normalise(300_000, (1 << 23) + 1, (1, 300), rng)
    assert one == 1
    for k in (0, 1, 31, 33):
        for n_amp in (3, 40_000):
            _check_normalise(k, n_amp, (1, 2), rng)
    with capsys.disabled():
        print("\nK13 grids on %d SMs: %d, %d (clamped), %d (K > 2^24)" % (sms, full, clamped, one))


# ------------------------------------------------------------------------------------------------ the chain
def _outcome(fn):
    try:
        return ("ok", fn())
    except Exception as e:  # noqa: BLE001  (both sides must fail alike: features on several contigs, say)
        return ("error", type(e).__name__, str(e))


def _text(res):
    return [(r.name, r.sequence, r.qualities) for r in res.consensuses], res.refs_changes, \
        {k: [ln for ln in v.splitlines() if not any(m in ln for m in MARKS)] for k, v in res.refs_reports.items()}


def _frame(df):
    return df.to_csv()


def _reference(tmp_path, contigs):
    rng = random.Random(5)
    fa = tmp_path / "ref.fa"
    fa.write_text("".join(">%s\n%s\n" % (nm, "".join(rng.choice("ACGT") for _ in range(L))) for nm, L in contigs))
    return str(fa)


PLAIN = (dict(), dict(qualities=True), dict(iupac_threshold=0.6), dict(realign=True))
QUALITY = (dict(quality_vote=True, qualities=True),)


def _chain(d, contigs, recs, bam, rows, bed, cap, quality):
    """The chain on one file against the same commands on the file of the composed oracle's kept records.  quality:
    only the outputs that need every read's qualities (`--quality-vote`, VCF `--qual`), on a file that has no record
    without them; else every other output, a two-sample cohort among them."""
    d.mkdir()
    opts = dict(primers=bed, mask_overlaps=True, min_base_quality=20, **FILTERS)
    sel = SO.select(bam, dedup=True, rows=rows, normalise=cap, **FILTERS)
    sub = d / "kept.bam"
    bamio.write_bam(str(sub), contigs, SL.placeholders(recs, sel.removed))
    sub, on = str(sub), dict(dedup=True, normalise=cap)
    run, _ = K.pileup_run(bam, **opts, **on)
    assert list(run.batch.contig_names) == sel.contigs == list(K.pileup_run(sub, **opts)[0].batch.contig_names)
    assert run.deduplicated == sel.dedup_totals[:2] + (sel.after_dedup, sel.before)
    assert run.normalised == (cap, len(sel.cap_dropped), sel.kept)
    for kw in QUALITY if quality else PLAIN:
        a = _outcome(lambda: _text(K.bam_to_consensus(bam, **opts, **on, **kw)))
        assert a == _outcome(lambda: _text(K.bam_to_consensus(sub, **opts, **kw))), kw
        assert a[0] == "ok" or not quality, a
        if a[0] == "ok" and not kw:
            report = K.bam_to_consensus(bam, **opts, **on).refs_reports
            for text in report.values():
                assert "- duplicates: %d pairs and %d single reads removed, %d of %d reads kept" % (
                    sel.dedup_totals[0], sel.dedup_totals[1], sel.after_dedup, sel.before) in text.splitlines()
                assert "- normalise: %d per amplicon and strand, %d of %d reads dropped" % (
                    cap, len(sel.cap_dropped), sel.after_dedup) in text.splitlines()
    if not quality:
        for fn in (K.weights, K.features, K.variants):
            assert _outcome(lambda: _frame(fn(bam, **opts, **on))) == _outcome(lambda: _frame(fn(sub, **opts))), fn
    fa = _reference(d, contigs)
    vcf = dict(reference=fa, strand=True, qual=True) if quality else dict(reference=fa, strand=True)
    for kw in ((vcf,) if quality else (dict(), vcf)):
        a = _outcome(lambda: [ln for ln in K.variants_vcf(bam, **opts, **on, **kw).splitlines()
                              if not any(m in ln for m in MARKS)])
        assert a == _outcome(lambda: K.variants_vcf(sub, **opts, **kw).splitlines()), kw
        assert a[0] == "ok", a
    if not quality:  # a cohort (no strand or QUAL fields) whose second sample has no duplicates: the dedup alone
        sel_d = SO.select(bam, dedup=True, **FILTERS)
        sub_d = d / "dedup.bam"
        bamio.write_bam(str(sub_d), contigs, SL.placeholders(recs, sel_d.removed))
        both = dict(samples=["a", "b"], reference=fa, **opts)
        a = _outcome(lambda: [ln for ln in K.variants_vcf([bam, str(sub_d)], dedup=True, **both).splitlines()
                              if not any(m in ln for m in MARKS)])
        assert a == _outcome(lambda: K.variants_vcf([str(sub_d), str(sub_d)], **both).splitlines())
        assert a[0] == "ok", a
    if not quality:
        amp = {k: v for k, v in opts.items() if k != "primers"}
        a = _outcome(lambda: K.amplicons(bam, bed, 5, **amp, **on))
        b = _outcome(lambda: K.amplicons(sub, bed, 5, **amp))
        cols = [c for c in K.AMPLICON_COLUMNS if c != "sample"]
        assert a[0] == b[0] and (a[0] != "ok" or a[1][cols].equals(b[1][cols]))
    return sel


@pytest.mark.parametrize("name", GROUPS + ["many_header", "many_shuffled", "interleaved"])
def test_the_chain_equals_the_file_of_the_kept_records(files, tmp_path, name):
    contigs, recs, bam, _, rows, bed = files[name]
    sel = _chain(tmp_path / "all", contigs, recs, bam, rows, bed, 2, False)
    assert sel.dedup_removed and sel.cap_dropped
    if name == "interleaved":
        assert sel.contigs == ["x2", "x0", "x1"] and 0 in sel.dedup_removed
    # --qual and --quality-vote check every read the filters keep for qualities while the file is decoded, before
    # the dedup or the cap removes any: a record with QUAL `*` fails the run even when it is a removed duplicate
    noqual = [r for r in recs if r[7] is None]
    if noqual:
        with pytest.raises(ValueError, match="without base qualities"):
            K.pileup_run(bam, qual=True, dedup=True, normalise=2, primers=bed, **FILTERS)
    # so those outputs are compared on the same file without its QUAL `*` records
    with_qual = [r for r in recs if r[7] is not None]
    q_bam = str(tmp_path / "with_qual.bam")
    bamio.write_bam(q_bam, contigs, with_qual)
    sel = _chain(tmp_path / "qual", contigs, with_qual, q_bam, rows, bed, 2, True)
    assert sel.dedup_removed and sel.cap_dropped


def test_two_gpus_equal_one(files):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _, _, bam, _, _, bed = files["many_shuffled"]
    kw = dict(dedup=True, normalise=2, primers=bed, qualities=True)
    one = K.bam_to_consensus(bam, devices=1, **kw)
    two = K.bam_to_consensus(bam, devices=2, **kw)
    assert [(r.name, r.sequence, r.qualities) for r in one.consensuses] == \
        [(r.name, r.sequence, r.qualities) for r in two.consensuses]
    assert one.refs_reports == two.refs_reports
