"""The consensus with `--primers` and `--mask-overlaps` together, without a GPU: the paired corpus of
tests/pair_combo_cases.py against its composed oracle (`PairedPiled`).

- The oracle is pinned: with both options off its consensus is combo_cases.Piled's, and its tables are the C quality
  walk fed py_moracle.Masked's merged mask lists, all 19 columns and the insertion strings.
- The corpus really flips what it was built to flip, counted in both directions where masking can go both ways.
- The product's own `bam_to_consensus` -- decode, K9, K10p, K10, the pileup, K1q, K10u, K2 / K2q, K5 / K5q or the host
  assembly, the insertion table without K10's dropped rows, `_insertion_qualities`, the `--realign` patches and the
  REPORT -- runs with every kdl_* call on the kernel emulator and equals the oracle over a pairwise option matrix.
- `weights`, `features`, `variants` and `parse_bam` with both options on equal the host functions over the oracle's
  table, and every `insertions[pos]` is the oracle's dict in first-seen order.
- The sharded branch of `pileup_run` (the parent masks once, the ranks take back their own drops) equals the oracle.
- Both options off equal the keywords left out."""
import dataclasses
import os
import re

import numpy as np
import pytest
import torch

import emu_harness as E
import helpers as H
import pair_combo_cases as PC
from kindel_b200 import bamio, distributed, engine
from kindel_b200 import kindel as K
from oracle import coracle, py_poracle as PO
from oracle import py_moracle as MO
from test_vcf_combined import on_the_emulator

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("pair_combo")
    out = PC.write(d)
    out.update(dir=d, layout=bamio.read_alignment(out["bam"]), piled={})
    return out


def piled(corpus, bq=0, mq=0, ex=0, primers=False, mates=False):
    key = (bq, mq, ex, primers, mates)
    if key not in corpus["piled"]:
        corpus["piled"][key] = PC.PairedPiled(corpus["bam"], corpus["layout"], bq, mq, ex,
                                              corpus["rows"] if primers else None, mates,
                                              os.path.basename(corpus["bed"]) if primers else None)
    return corpus["piled"][key]


def same_as_oracle(got, want, what):
    assert [(r.name, r.sequence, r.qualities) for r in got.consensuses] == \
        [(n + "_cns", s, q) for n, s, _, q, _ in want], what
    assert [list(got.refs_changes[n]) for n, _, _, _, _ in want] == [c for _, _, c, _, _ in want], what


def same_reports(got, want, what):
    assert list(got.refs_reports) == list(want), what
    for name, text in want.items():
        assert got.refs_reports[name].splitlines() == text.splitlines(), (what, name)


# ------------------------------------------------------------------------------------------- oracle pins
def test_oracle_off_is_the_combo_oracle(corpus):
    """Mates and primers off: PairedPiled's consensus is combo_cases.Piled's (the C quality walk over the records with
    the filtered ones rewritten as unmapped) on the same records."""
    import combo_cases as CC

    n = 0
    for bq, (mq, ex), t, md, realign, trim, upper in ((0, (0, 0), None, 1, True, False, False),
                                                     (20, (30, 0x400), 0.6, 3, True, True, True),
                                                     (20, (0, 0), 0.99, 1, False, False, True)):
        want = CC.Piled(corpus["contigs"], corpus["recs"], corpus["dir"] / "combo.bam", bq, mq, ex).consensus(
            t, md, realign, trim, upper)
        got = piled(corpus, bq, mq, ex).consensus(t, md, realign, trim, upper)
        assert [x[:4] for x in got] == want, (bq, mq, ex, t)
        n += sum(len(x[1]) for x in got)
    assert n > 3000


def _merged_pre(path, names, bq, mq, ex, rows):
    """Per kept record (engine order): its quality-masked and primer-masked query offsets."""
    lengths, recs = MO.kept(path, names, mq, ex)
    out = []
    for nm, r, _, _, _ in recs:
        m = {q for q, v in enumerate(r.qual) if v < bq} if bq and r.qual is not None else set()
        if rows is not None:
            m |= set(PO.masked_qpos(r, lengths[nm], PO.contig_intervals(rows, nm)))
        out.append(sorted(m))
    return out


def test_oracle_tables_are_the_c_quality_walk(corpus):
    """ComposedMates' 19 columns and insertion dicts (first-seen order) == the C quality walk fed py_moracle.Masked's
    merged mask lists (quality, primer and overlap bases), minus the dropped D / I ops, without the dropped rows."""
    n_n = 0
    for bq, mq, ex, pr in ((0, 0, 0, False), (20, 30, 0x400, True), (20, 0, 0, False), (0, 30, 0x400, True)):
        plain = bamio.read_alignment(corpus["bam"], min_mapq=mq, exclude_flags=ex)
        o = MO.Masked(corpus["bam"], plain.contig_names, mq, ex,
                      pre_masked=_merged_pre(corpus["bam"], plain.contig_names, bq, mq, ex,
                                             corpus["rows"] if pr else None))
        counts, events = o.pileup(plain, dict(zip(plain.contig_names, plain.contig_slot.tolist())))
        p = piled(corpus, bq, mq, ex, pr, True)
        np.testing.assert_array_equal(p.counts, counts, err_msg=str((bq, mq, ex, pr)))
        masked = o.masked()
        ins = {}
        for slot, read, q0, ln in events.tolist():
            s = "".join("N" if q0 + k in masked[read] else ch
                        for k, ch in enumerate(H.event_string(plain, read, q0, ln)))
            ins.setdefault(slot, {})
            ins[slot][s] = ins[slot].get(s, 0) + 1
        assert {s: list(d.items()) for s, d in p.ins.items()} == {s: list(d.items()) for s, d in ins.items()}
        assert p.overlap_stats == o.stats()
        n_n += sum("N" in s for d in ins.values() for s in d)
    assert n_n >= 2


# ------------------------------------------------------------------------------------------- the corpus
def test_corpus_has_what_it_is_for(corpus):
    """Every planted shape changes the oracle's output when mask_overlaps is turned on, in both directions where
    masking can go both ways (it only removes counts, so a min_depth `N` and a clip-dominant patch can only appear)."""
    recs = corpus["recs"]
    assert {0x100, 0x400} <= {r[2] & 0x500 for r in recs} and any(r[7] is None for r in recs)
    assert corpus["layout"].contig_names == ["edge", "gone", "mix"]  # first-seen order, not the header's
    b = bamio.read_alignment(corpus["bam"], min_mapq=30, exclude_flags=0x400)
    g = b.contig_names.index("gone")
    assert b.contig_read_off[g + 1] == b.contig_read_off[g] and b.n_hard > 0
    off, on = piled(corpus), piled(corpus, mates=True)
    pairs, bases, dels, ins = on.overlap_stats
    assert pairs >= 50 and bases > 1000 and dels >= 2 and ins >= 8
    flips = dict.fromkeys(("code>base 0.6", "base>code 0.6", "code>base 0.99", "N", "I gone", "I new", "string",
                           "tie gone", "tie new", "D gone", "D new", "patch"), 0)
    lay = corpus["layout"]
    for t, up, down in ((0.6, "base>code 0.6", "code>base 0.6"), (0.99, None, "code>base 0.99")):
        a, c = off.calls(t), on.calls(t)
        flips[down] += int((((a & 0x80) != 0) & ((c & 0x80) == 0)).sum())
        if up:
            flips[up] += int((((a & 0x80) == 0) & ((c & 0x80) != 0)).sum())
    a, c = off.calls(None, 3), on.calls(None, 3)
    flips["N"] += int(((((a >> 4) & 3) != 2) & (((c >> 4) & 3) == 2)).sum())
    a, c = off.calls(), on.calls()
    ia, ic = ((a >> 4) & 3) == 3, ((c >> 4) & 3) == 3
    flips["I gone"], flips["I new"] = int((ia & ~ic).sum()), int((ic & ~ia).sum())
    da, dc = ((a >> 4) & 3) == 1, ((c >> 4) & 3) == 1
    flips["D gone"], flips["D new"] = int((da & ~dc).sum()), int((dc & ~da).sum())
    from oracle.py_oracle import base_call

    for s in np.flatnonzero(ia & ic).tolist():
        ka, _, ta = base_call(off.ins[s])
        kc, _, tc = base_call(on.ins[s])
        flips["string"] += ka != kc and not ta and not tc
        flips["tie gone"] += ta and not tc
        flips["tie new"] += tc and not ta
    e = lay.contig_names.index("edge")
    flips["patch"] = int(any(r.seq for r in on.patches(e)) and not off.patches(e))
    assert all(flips.values()), flips
    assert flips["N"] >= 30 and min(flips[k] for k in flips if "0." in k) >= 2, flips
    # the insertion at the last position of "mix", partly masked at Q20
    mix = int(lay.contig_slot[lay.contig_names.index("mix")])
    assert set(piled(corpus, 20).ins[mix + PC.CONTIGS[1][1] - 1]) == {"CA", "NA", "CN", "NN"}


def test_option_matrix_covers_every_pair():
    rows = PC.option_matrix()
    assert len(rows) <= 12
    for i in range(9):
        for j in range(i + 1, 9):
            assert {(r[i], r[j]) for r in rows} == {(a, b) for a in {r[i] for r in rows} for b in {r[j] for r in rows}}


# ------------------------------------------------------------------------------------------- the product
def consensus_kwargs(corpus, row):
    t, bq, md, realign, trim, upper, (mq, ex), pr, mates = row
    return dict(realign=realign, min_depth=md, trim_ends=trim, uppercase=upper, min_base_quality=bq, min_mapq=mq,
                exclude_flags=ex, iupac_threshold=t, primers=corpus["bed"] if pr else None, mask_overlaps=mates)


def check_consensus(corpus, row, got, path):
    t, bq, md, realign, trim, upper, (mq, ex), pr, mates = row
    p = piled(corpus, bq, mq, ex, pr, mates)
    same_as_oracle(got, p.consensus(t, md, realign, trim, upper), row)
    same_reports(got, p.reports(path, t, md, realign, trim, upper), row)


@needs_emu
def test_bam_to_consensus_matrix_emulated(corpus, monkeypatch):
    """bam_to_consensus with qualities on, every kdl_* call emulated, from BAM and from SAM text: sequence, qualities,
    change lists and REPORT lines equal the oracle's over the pairwise option matrix; qualities off gives the same
    sequences."""
    on_the_emulator(monkeypatch)
    n_i = n_patched = 0
    for k, row in enumerate(PC.option_matrix()):
        path = corpus["sam"] if k % 3 == 2 else corpus["bam"]
        kw = consensus_kwargs(corpus, row)
        got = K.bam_to_consensus(path, qualities=True, **kw)
        check_consensus(corpus, row, got, path)
        n_i += sum(len(c.sites["I"]) for c in got.refs_changes.values() if hasattr(c, "sites"))
        n_patched += any("- clip-dominant regions: \n" not in r for r in got.refs_reports.values())
        if k < 2:
            plain = K.bam_to_consensus(path, **kw)
            assert [r.sequence for r in plain.consensuses] == [r.sequence for r in got.consensuses]
            assert all(r.qualities is None for r in plain.consensuses)
    assert n_i > 10 and n_patched > 0


def one_contig(corpus):
    """The corpus's "mix" records alone, on a one-contig file (features raises the reference's IndexError on two)."""
    path = corpus["dir"] / "mix_only.bam"
    if not path.exists():
        recs = [(0,) + r[1:8] + (0 if r[8] >= 0 else -1, r[9]) for r in corpus["recs"] if r[0] == PC.MIX]
        bamio.write_bam(str(path), [PC.CONTIGS[PC.MIX]], recs)
    return str(path)


def _host_run(layout, p):
    return K.PileupRun.from_host_tables(layout, p.counts, coracle.derive(p.counts), np.zeros((0, 4), np.int32))


@needs_emu
def test_other_commands_emulated(corpus, monkeypatch):
    """weights (relative and confidence), features, variants and parse_bam's views with primers and mates on equal the
    host functions over the oracle's table; every insertions[pos] is the oracle's dict in first-seen order."""
    on_the_emulator(monkeypatch)
    mix_rows = [r for r in corpus["rows"] if r[0] == "mix"]
    for path, rows in ((corpus["bam"], corpus["rows"]), (one_contig(corpus), mix_rows)):
        layout = bamio.read_alignment(path)
        bed = corpus["dir"] / ("%s.bed" % os.path.basename(path))
        bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
        for bq, mq, ex in ((0, 0, 0), (20, 30, 0x400)):
            kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, primers=str(bed), mask_overlaps=True)
            p = PC.PairedPiled(path, layout, bq, mq, ex, rows, True)
            run = _host_run(layout, p)
            for rel, conf in ((False, True), (True, False)):
                assert K.weights(path, relative=rel, confidence=conf, **kw).equals(
                    K.weights_from_run(run, relative=rel, confidence=conf)), (path, bq, rel)
            assert K.variants(path, 1, 0.01, **kw).equals(K.variants_from_run(run, 1, 0.01)), path
            if len(layout.contig_names) == 1:
                assert K.features(path, **kw).equals(K.features_from_run(run))
            for c, (name, aln) in enumerate(K.parse_bam(path, **kw).items()):
                s0, L = int(layout.contig_slot[c]), int(layout.contig_len[c])
                want = run.alignment(c)
                np.testing.assert_array_equal(aln.table, want.table)
                assert aln.clip_start_depth == want.clip_start_depth and aln.clip_depth == want.clip_depth
                np.testing.assert_array_equal(aln.consensus_depth, want.consensus_depth)
                got_ins = [list(d.items()) for d in aln.insertions]
                assert got_ins == [list(p.ins.get(s0 + k, {}).items()) for k in range(L + 1)], (path, name, bq)


def _emulated_ranks(plan):
    """distributed.run_sharded, in process: every rank piles its shard on the emulated engine (its primer bases
    masked, its R2s' drop rows taken back), the tables add up, the vote runs over the sum, the events merge."""

    def run_sharded(batch, devices, min_depth=1, mode="fused", plan_=None, iupac_threshold=None, primers=None,
                    drops=None):
        total, evs, idxs = None, [], []
        for rank in range(devices):
            idx = distributed.shard_indices(batch, rank, devices, plan)
            db = engine.upload(bamio.select_reads(batch, idx))
            if primers is not None:
                db = engine.mask_primers(db, primers)
            if drops is not None:
                db = dataclasses.replace(db, drops=torch.from_numpy(distributed.shard_drops(drops, idx)))
            counts, events = engine.pileup(db)
            total = counts.clone() if total is None else total + counts
            evs.append(events.numpy()[:db.host.n_events])
            idxs.append(idx)
        calls = engine.vote(total, min_depth, iupac_threshold=iupac_threshold)
        return calls.numpy(), total.numpy(), engine.derive(total).numpy(), distributed.merge_events(evs, idxs)

    return run_sharded


@needs_emu
@pytest.mark.parametrize("plan", ["reads", "contigs"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_branch_emulated(corpus, monkeypatch, world, plan):
    """pileup_run with devices > 1: the product's _masked_for_shards, dropped_events, overlap_stats and
    consensus_from_run run for real over ranks emulated in process; with IUPAC, qualities and realign on the result
    equals the oracle."""
    on_the_emulator(monkeypatch)
    monkeypatch.setattr(distributed, "run_sharded", _emulated_ranks(plan))
    rows = [(0.6, 20, 3, True, False, False, (30, 0x400), True, True),
            (0.99, 0, 1, True, True, True, (0, 0), False, True),
            (0.6, 0, 1, True, False, True, (0, 0), True, False)]
    for k, row in enumerate(rows):
        path = corpus["sam"] if (k + world) % 3 == 0 else corpus["bam"]
        got = K.bam_to_consensus(path, devices=world, qualities=True, **consensus_kwargs(corpus, row))
        check_consensus(corpus, row, got, path)


@needs_emu
def test_off_is_unchanged(corpus, monkeypatch):
    """mask_overlaps=False and primers=None equal the keywords left out, for every output."""
    on_the_emulator(monkeypatch)
    one = one_contig(corpus)
    kw = dict(min_base_quality=20, min_mapq=30, exclude_flags=0x400)
    off = dict(mask_overlaps=False, primers=None)
    a = K.bam_to_consensus(corpus["bam"], realign=True, iupac_threshold=0.6, qualities=True, **kw)
    b = K.bam_to_consensus(corpus["bam"], realign=True, iupac_threshold=0.6, qualities=True, **kw, **off)
    assert [(r.sequence, r.qualities) for r in a.consensuses] == [(r.sequence, r.qualities) for r in b.consensuses]
    assert a.refs_reports == b.refs_reports and a.refs_changes == b.refs_changes
    assert not any(re.search("- (primers|mate overlaps):", r) for r in a.refs_reports.values())
    assert K.weights(corpus["bam"], **kw).equals(K.weights(corpus["bam"], **kw, **off))
    assert K.variants(corpus["bam"], **kw).equals(K.variants(corpus["bam"], **kw, **off))
    assert K.features(one, **kw).equals(K.features(one, **kw, **off))
    views = zip(K.parse_bam(corpus["bam"], **kw).items(), K.parse_bam(corpus["bam"], **kw, **off).items())
    for (n1, x), (n2, y) in views:
        assert n1 == n2 and np.array_equal(x.table, y.table) and list(x.insertions) == list(y.insertions)


def test_oracle_does_not_read_the_engine():
    """The composed oracle never imports the engine nor reads a product batch's mask list or masked bases."""
    src = open(os.path.join(H.ROOT, "tests", "pair_combo_cases.py")).read()
    oracle = src[src.index("composed oracle\n"):]
    for word in ("engine", "mask_read", "mask_off", "mask_qpos", "seq4", "n_masked", "read_alignment"):
        assert word not in oracle, word
    assert "import engine" not in src and "engine." not in src
