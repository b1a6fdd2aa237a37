"""The extensions together, without a GPU: base / read filters, the IUPAC vote and per-base qualities on one corpus
(tests/combo_cases.py) against one composed oracle.

- The host code (`consensus_from_run` over the oracle's masked tables, K2q from its CUDA source under the emulator)
  equals the composed oracle over a pairwise-covering option matrix.
- min_mapq / exclude_flags equal rewriting the records they drop as unmapped, with IUPAC and qualities on.
- The emulated device chain K0 + K1 + K1e / K1g, K1q, K2 (IUPAC), K2q, K5 + K5q equals the composed oracle."""
import os
import re

import numpy as np
import pytest
import torch

import combo_cases as CC
import emu_harness as E
import helpers as H
from kindel_b200 import bamio
from kindel_b200 import kindel as K
from oracle import coracle
from test_quality_filters import same_arrays

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
SEEDS = (1, 2)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("combo")
    out = {}
    for seed in SEEDS:
        contigs, recs = CC.combo_case(seed)
        out[seed] = (contigs, recs, CC.write_bam(d / ("c%d.bam" % seed), contigs, recs), d)
    return out


def _emulated_k2q(run, calls_all):
    """K2q from its CUDA source over the host tables (stands in for the device copy of _slot_qualities)."""
    return torch.from_numpy(E.consensus_qual(run.host_counts, calls_all))


def _host_result(path, piled, t, md, realign, trim, upper, filters):
    """consensus_from_run over the product's masked batch and the oracle's masked tables."""
    bq, mq, ex = filters
    masked = bamio.read_alignment(path, min_mapq=mq, exclude_flags=ex, min_base_quality=bq)
    run = K.PileupRun.from_host_tables(masked, piled.counts, coracle.derive(piled.counts), piled.events)
    return K.consensus_from_run(run, piled.calls(t, md), path, realign, md, 9, 0.1, 50, trim, upper,
                                filters=filters, iupac_threshold=t, qualities=True)


def _same_as_oracle(got, want, what):
    assert [(r.name, r.sequence, r.qualities) for r in got.consensuses] == \
        [(n + "_cns", s, q) for n, s, _, q in want], what
    assert [list(got.refs_changes[n]) for n, _, _, _ in want] == [c for _, _, c, _ in want], what


def test_corpus_has_what_it_is_for(corpus, tmp_path):
    """The shapes the corpus exists for are really there."""
    contigs, recs, path, _ = corpus[SEEDS[0]]
    text = CC.sam_text(contigs, recs)
    flags = {r[2] for r in recs}
    assert {0x100, 0x200, 0x400} <= {f & 0x700 for f in flags}
    assert any(r[7] is None for r in recs) and len({r[6] for r in recs}) >= 6
    assert "\t*\n" in text
    masked = bamio.read_alignment(path, min_mapq=10, exclude_flags=0x400, min_base_quality=20)
    assert masked.contig_names == ["edge", "gone", "mix"]  # first-seen order, not the header's
    assert masked.reads_sorted and masked.n_hard > 0 and masked.n_complex > masked.n_hard and masked.n_masked > 500
    gone = masked.contig_names.index("gone")
    assert masked.contig_read_off[gone + 1] == masked.contig_read_off[gone]
    p = CC.Piled(contigs, recs, tmp_path / "o.bam", 20, 10, 0x400)
    s0 = {n: int(masked.contig_slot[c]) for c, n in enumerate(masked.contig_names)}
    mix = s0["mix"]
    acgt = p.counts[0:4].sum(axis=0)
    assert all(acgt[mix + x] == 0 and p.counts[4, mix + x] == 0 for x in CC.FULL_MASK)  # every base masked
    assert all(0 < acgt[mix + x] < 3 for x in CC.THIN)  # masking thins them below min_depth 3
    strings = p.ins.get(mix + CC.INS_SITE)
    assert len(strings) >= 3 and any("N" in s for s in strings)
    last = p.ins.get(mix + CC.CONTIGS[1][1] - 1)
    assert set(last) == {"CA", "NA", "CN", "NN"}
    # masking flips IUPAC calls: at 0.6 both ways, at 0.99 (where one read of the minor allele makes a code) to a base
    flips = {(t, way): 0 for t in (0.6, 0.99) for way in (0, 1)}
    for seed in SEEDS:
        contigs, recs, _, _ = corpus[seed]
        masked_tab = CC.Piled(contigs, recs, tmp_path / "m.bam", 20, 10, 0x400)
        plain = CC.Piled(contigs, recs, tmp_path / "p.bam", 0, 10, 0x400)
        mix = int(plain.batch.contig_slot[plain.batch.contig_names.index("mix")])
        for t in (0.6, 0.99):
            a, b = plain.calls(t), masked_tab.calls(t)
            for x, _, _ in CC.MIX_SITES:
                flips[t, 0] += bool(a[mix + x] & 0x80 and not b[mix + x] & 0x80)
                flips[t, 1] += bool(b[mix + x] & 0x80 and not a[mix + x] & 0x80)
    assert flips[0.6, 0] and flips[0.6, 1] and flips[0.99, 0], flips
    assert any(r.seq for r in p.patches(masked.contig_names.index("edge")))


def test_option_matrix_covers_every_pair():
    rows = CC.option_matrix()
    assert len(rows) <= 24
    for i in range(7):
        for j in range(i + 1, 7):
            vi = {r[i] for r in rows}
            vj = {r[j] for r in rows}
            assert {(r[i], r[j]) for r in rows} == {(a, b) for a in vi for b in vj}, (i, j)


@needs_emu
def test_host_code_equals_composed_oracle(corpus, monkeypatch):
    monkeypatch.setattr(K, "_slot_qualities", _emulated_k2q)
    n_iupac = n_patched = 0
    for k, (t, bq, md, realign, trim, upper, (mq, ex)) in enumerate(CC.option_matrix()):
        seed = SEEDS[k % len(SEEDS)]
        contigs, recs, path, d = corpus[seed]
        piled = CC.Piled(contigs, recs, d / "oracle.bam", bq, mq, ex)
        want = piled.consensus(t, md, realign, trim, upper)
        got = _host_result(path, piled, t, md, realign, trim, upper, (bq, mq, ex))
        _same_as_oracle(got, want, (seed, t, bq, md, realign, trim, upper, mq, ex))
        n_iupac += sum(len(c.iupac) for c in got.refs_changes.values())
        n_patched += sum("!" in r.qualities and "- clip-dominant regions: \n" not in got.refs_reports[r.name[:-4]]
                         for r in got.consensuses) if realign else 0
    assert n_iupac > 20 and n_patched > 0


@needs_emu
def test_record_filters_equal_rewriting_as_unmapped(corpus, monkeypatch, tmp_path):
    """With IUPAC and qualities on: the decoders' batches, and the host results over the emulated pileup, are those of
    the file whose dropped records are rewritten as unmapped."""
    monkeypatch.setattr(K, "_slot_qualities", _emulated_k2q)
    contigs, recs, path, _ = corpus[SEEDS[1]]
    for mq, ex, bq in ((10, 0x400, 20), (30, 0x300, 0), (0, 0x400, 41)):
        b = CC.write_bam(tmp_path / "rewritten.bam", contigs, CC.as_unmapped(recs, mq, ex))
        s = tmp_path / "c.sam"
        s.write_text(CC.sam_text(contigs, recs))
        got = bamio.read_alignment(path, min_mapq=mq, exclude_flags=ex, min_base_quality=bq)
        want = bamio.read_alignment(b, min_base_quality=bq)
        same_arrays(got, want)
        same_arrays(bamio.read_alignment(str(s), min_mapq=mq, exclude_flags=ex, min_base_quality=bq), want)
        assert got.contig_names == want.contig_names
        results = []
        for p, filters in ((path, (bq, mq, ex)), (b, (bq, 0, 0))):
            batch = bamio.read_alignment(p, min_mapq=filters[1], exclude_flags=filters[2], min_base_quality=bq)
            counts, events = _emulated_pileup(batch)
            run = K.PileupRun.from_host_tables(batch, counts, E.derive(counts), events)
            results.append(K.consensus_from_run(run, E.vote_iupac(counts, 3, 0.6), p, True, 3, filters=filters,
                                                iupac_threshold=0.6, qualities=True))
        a, b_ = results
        assert [(r.sequence, r.qualities) for r in a.consensuses] == [(r.sequence, r.qualities) for r in b_.consensuses]
        assert a.refs_changes == b_.refs_changes
        strip = lambda rep: re.sub(r"- (bam_path|min_base_quality|min_mapq|exclude_flags): .*\n", "", rep)  # noqa: E731
        assert {k: strip(v) for k, v in a.refs_reports.items()} == {k: strip(v) for k, v in b_.refs_reports.items()}


def _emulated_pileup(batch):
    counts, events = E.pileup_pipeline(batch)
    return E.unmask(batch, counts), events


@needs_emu
def test_emulated_device_chain_equals_composed_oracle(corpus):
    """K0 + K1 + K1e / K1g, then K1q, then K2 (IUPAC or majority), then K2q, then K5 + K5q, all from their CUDA source,
    with the host's insertion strings and insertion qualities in between: text and qualities of every contig equal the
    composed oracle's."""
    n = 0
    for seed in SEEDS:
        contigs, recs, path, d = corpus[seed]
        for bq, (mq, ex), t, md in ((20, (10, 0x400), 0.6, 1), (41, (0, 0), 0.99, 3), (20, (0, 0x400), None, 3),
                                   (0, (10, 0), 1.0, 1)):
            masked = bamio.read_alignment(path, min_mapq=mq, exclude_flags=ex, min_base_quality=bq)
            counts, events = _emulated_pileup(masked)
            piled = CC.Piled(contigs, recs, d / "oracle.bam", bq, mq, ex)
            np.testing.assert_array_equal(counts, piled.counts)
            np.testing.assert_array_equal(events, piled.events)
            calls = E.vote(counts, md) if t is None else E.vote_iupac(counts, md, t)
            qual = E.consensus_qual(counts, calls)
            run = K.PileupRun.from_host_tables(masked, counts, E.derive(counts), events)
            slots = K._insertion_slots(masked, calls)
            iq = K._insertion_qualities(run, slots)
            strings = []
            for sl in slots.tolist():
                text, tie = run.ins_table.consensus_at(sl)
                strings.append("N" if tie else text.lower())
            texts, quals = E.assemble_qual(calls, qual, masked, slots, strings, [iq[s] for s in slots.tolist()])
            for trim, upper in ((False, False), (True, True)):
                want = piled.consensus(t, md, trim_ends=trim, uppercase=upper)
                for c, (name, seq, _, q) in enumerate(want):
                    s, qq = K._trim_n(texts[c], quals[c]) if trim else (texts[c], quals[c])
                    assert ((s.upper() if upper else s), qq) == (seq, q), (seed, bq, mq, ex, t, md, name)
                    n += len(q)
    assert n > 10_000


def test_oracle_does_not_read_the_engine():
    """The composed oracle never imports the engine nor reads the engine's mask list or masked bases."""
    src = open(os.path.join(H.ROOT, "tests", "combo_cases.py")).read()
    oracle = src[src.index("composed oracle\n"):]
    for word in ("engine", "mask_read", "mask_off", "mask_qpos", "seq4", "n_masked"):
        assert word not in oracle, word
    assert re.findall(r"read_alignment\((.*)\)", oracle) == ["self.path"]  # unmasked and unfiltered
