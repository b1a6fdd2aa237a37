"""The IUPAC vote (`iupac_threshold`, an extension: the reference has no such option), without a GPU.

There is no reference to pin it against, so two restatements written in different forms are held against each other:
oracle/kindel_oracle.c (`ioracle.vote_iupac`, the set / level form of the definition) and oracle/py_oracle.py (a loop
that takes the bases in descending order, a tie group at a time).  The kernels (K2, K2x, K5) run from their CUDA
source under the host emulator (tests/emu/) and must reproduce the C oracle; the host assembly, the report and the
option checks are exercised through the public API with oracle tables (`PileupRun.from_host_tables`)."""
import math

import numpy as np
import pytest

import emu_harness as E
import emu_iupac_harness as EI
import helpers as H
from clip_cases import clip_case
from conftest import golden_input
from fuzz_cases import random_case
from kindel_b200 import _ffi, bamio, cli, synth
from kindel_b200 import distributed as D
from kindel_b200 import kindel as K
from oracle import coracle, ioracle, py_ioracle, py_oracle

THRESHOLDS = (0.0, 0.25, 0.5, 0.55, 0.7, 0.75, 0.9, 0.99, 1.0)
MIN_DEPTHS = (0, 1, 7)
LETTERS = "=ACMGRSVTWYHKDBN"
needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")


# ---------------------------------------------------------------------------------------------- inputs
def _batches(manifest, tmp_path):
    """(name, batch) of the golden fixtures, the clip cases and the 400 fuzz cases that pile without raising."""
    for name, entry in manifest["files"].items():
        yield name, bamio.read_alignment(golden_input(entry))
    for seed in range(96):
        p = tmp_path / ("clip%d.sam" % seed)
        p.write_text(clip_case(seed))
        yield "clip%d" % seed, bamio.read_alignment(p)
    for seed in range(400):
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            yield "fuzz%d" % seed, bamio.read_alignment(p)
        except (ValueError, KeyError):
            continue


def _piled(manifest, tmp_path):
    for name, batch in _batches(manifest, tmp_path):
        try:
            counts, events = coracle.pileup(batch)
        except (IndexError, KeyError):
            continue
        yield name, batch, counts, events


def _py_pileup(counts_c, ins_c):
    """py_oracle's per-position dicts for one contig ([19, L+1] table, {position: OrderedDict} insertions)."""
    L = counts_c.shape[1] - 1
    weights = [{b: int(counts_c[k, i]) for b, k in (("A", 0), ("T", 3), ("G", 2), ("C", 1), ("N", 4))}
               for i in range(L)]
    insertions = [ins_c.get(i, {}) for i in range(L + 1)]
    return py_oracle.Pileup(weights, insertions, counts_c[5].tolist(), *([None] * 8))


def _contigs(batch, counts, events):
    ins = H.events_to_dicts(batch, events)
    for c in range(batch.n_contigs):
        s0, L = int(batch.contig_slot[c]), int(batch.contig_len[c])
        ins_c = {s - s0: d for s, d in ins.items() if s0 <= s <= s0 + L}
        yield s0, L, ins_c


# ------------------------------------------------------------------------------------- oracle vs oracle
def test_c_oracle_equals_python_loop(manifest, tmp_path):
    """ioracle.vote_iupac, assembled by the host code, gives py_oracle's text and changes on the golden fixtures, the
    clip cases and the fuzz cases, at every threshold and min_depth."""
    n_files = n_mixed = 0
    for name, batch, counts, events in _piled(manifest, tmp_path):
        n_files += 1
        for s0, L, ins_c in _contigs(batch, counts, events):
            p = _py_pileup(counts[:, s0:s0 + L + 1], ins_c)
            lookup = lambda pos, ins_c=ins_c: K.dict_consensus(ins_c.get(pos, {}))  # noqa: E731
            for md in MIN_DEPTHS:
                for t in THRESHOLDS:
                    calls = ioracle.vote_iupac(counts, md, t)[s0:s0 + L]
                    n_mixed += int(np.count_nonzero(calls & 0x80))
                    seq, changes = K.assemble_consensus(calls, lookup)
                    want_seq, want_changes = py_ioracle.vote(p, md, t)
                    assert seq == want_seq, (name, md, t)
                    assert list(changes) == want_changes, (name, md, t)
    assert n_files > 100 and n_mixed > 1000


def test_property_against_the_default_vote(manifest, tmp_path):
    """Where the reference's call has change D or N, or is an untied base b with count(b) >= t * depth, the IUPAC
    call byte equals it."""
    for name, batch, counts, events in _piled(manifest, tmp_path):
        w = counts[:4].astype(np.int64)
        depth = w.sum(axis=0)
        for md in MIN_DEPTHS:
            base = coracle.vote(counts, md)
            change = (base >> 4) & 3
            code = base & 7
            for t in THRESHOLDS:
                got = ioracle.vote_iupac(counts, md, t)
                dn = (change == 1) | (change == 2)
                assert np.array_equal(got[dn], base[dn]), (name, md, t)
                single = ~dn & (code < 4)
                cnt = np.take_along_axis(w, np.minimum(code, 3)[None, :].astype(np.int64), axis=0)[0]
                keep = single & (cnt.astype(np.float64) >= t * depth.astype(np.float64))
                assert np.array_equal(got[keep], base[keep]), (name, md, t)
                assert not (got[dn] & 0x80).any()


def _table(cols):
    """[19, n] table (n padded to a multiple of 4) with the given A, C, G, T(, N, D, I) rows."""
    cols = np.asarray(cols, dtype=np.int64)
    n = (cols.shape[1] + 3) // 4 * 4
    t = np.zeros((19, n), dtype=np.int32)
    t[: cols.shape[0], : cols.shape[1]] = cols
    return t


def _letter(byte):
    return LETTERS[byte & 15] if byte & 0x80 else "ACGTN"[min(byte & 7, 4)]


def test_worked_examples():
    """The definition's own examples, including the two rounding cases of the threshold product."""
    cases = [  # (A, C, G, T, N, t, letter)
        (55, 0, 45, 0, 0, 0.5, "A"), (55, 0, 45, 0, 0, 0.6, "R"), (50, 0, 50, 0, 0, 0.0, "R"),
        (50, 50, 0, 0, 0, 0.0, "M"), (0, 0, 0, 0, 9, 0.5, "N"), (1, 0, 0, 0, 9, 0.5, "A"),
        (30, 30, 30, 10, 0, 0.5, "V"), (30, 30, 30, 10, 0, 0.95, "N"), (1, 1, 1, 1, 0, 0.0, "N"),
        (0, 5, 0, 5, 0, 1.0, "Y"), (10, 0, 0, 3, 0, 1.0, "W"), (10, 0, 0, 3, 0, 0.99, "W"),
        (10, 0, 0, 3, 0, 0.76, "A"), (0, 0, 7, 7, 0, 0.3, "K"),
        # t = 0.55, D = 100: 0.55 * 100 = 55.00000000000001 > 55 -> A alone does not qualify
        (55, 45, 0, 0, 0, 0.55, "M"),
        # t = 0.7, D = 90: 0.7 * 90 = 62.99999999999999 <= 63 -> A alone qualifies
        (63, 0, 27, 0, 0, 0.7, "A"),
    ]
    assert 0.55 * 100 == 55.00000000000001 and 0.7 * 90 == 62.99999999999999
    for a, c, g, t_, n, thr, want in cases:
        tab = _table([[a], [c], [g], [t_], [n]])
        got = ioracle.vote_iupac(tab, 1, thr)[0]
        assert _letter(got) == want, (a, c, g, t_, n, thr)
        assert py_ioracle.iupac_call({"A": a, "C": c, "G": g, "T": t_, "N": n}, thr) == want
        if E.available():
            assert _letter(EI.vote_iupac(tab, 1, thr)[0]) == want


# ------------------------------------------------------------------------------------------ kernels
def _adversarial(seed):
    """Tables the fuzz cases do not reach: many ties and exact boundary equalities (counts 0..4), the two rounding
    examples, per-column counts near 2^29 (the depth overflows int32), random deletion / insertion columns."""
    rng = np.random.default_rng(seed)
    n = 4096
    small = rng.integers(0, 5, size=(7, n))
    small[4] = rng.integers(0, 3, size=n)
    small[5] = np.where(rng.random(n) < 0.15, rng.integers(0, 6, size=n), 0)
    small[6] = np.where(rng.random(n) < 0.15, rng.integers(0, 6, size=n), 0)
    big = rng.integers(0, 4, size=(7, n)) + (1 << 29) - 2
    big[:4] *= rng.random((4, n)) < 0.8
    big[4:] = 0
    big[5] = np.where(rng.random(n) < 0.05, (1 << 30), 0)
    big[6] = np.where(rng.random(n) < 0.05, (1 << 30) + 1, 0)
    rounding = np.array([[55, 63], [45, 0], [0, 27], [0, 0], [0, 0], [0, 0], [0, 0]])
    return [_table(small), _table(big), _table(rounding)]


@needs_emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 1)])
def test_emulated_k2_iupac_equals_oracle(schedule, seed, tmp_path):
    EI.set_schedule(schedule, seed)
    try:
        tables = _adversarial(seed + 11)
        for s in range(0, 400, 8):
            p = tmp_path / ("fuzz%d.sam" % s)
            p.write_text(random_case(s))
            try:
                tables.append(coracle.pileup(bamio.read_alignment(p))[0])
            except (ValueError, KeyError, IndexError):
                continue
        for tab in tables:
            for md in MIN_DEPTHS:
                for t in THRESHOLDS:
                    np.testing.assert_array_equal(EI.vote_iupac(tab, md, t), ioracle.vote_iupac(tab, md, t),
                                                  err_msg="%s md=%d t=%s" % (schedule, md, t))
    finally:
        EI.set_schedule("forward")


@needs_emu
@pytest.mark.parametrize("world", [2, 3])
def test_emulated_exchange_iupac_equals_one_table(world):
    """K2x with the IUPAC vote over `world` ranks' footprint-clipped tables (then K2g) gives every rank the call
    bytes of the one summed table."""
    flags = {k: [np.zeros(16, dtype=np.int32) for _ in range(world)] for k in ("ready", "done")}
    flags["counter"] = [np.zeros(1, dtype=np.int32) for _ in range(world)]
    bufs = None
    for epoch, (seed, t) in enumerate(((74, 0.6), (75, 0.99), (76, 0.0)), start=1):
        batch = synth.mixed_reads(seed, [9000], 30, 0.3)
        shards = [D.shard_batch(batch, r, world) for r in range(world)]
        full, _ = coracle.pileup(batch)
        tables = [coracle.pileup(s)[0] for s in shards]
        feet = [D.footprint(s) for s in shards]
        n_slots = full.shape[1]
        slices = D.footprint_slices(feet, n_slots)
        if bufs is None:
            bufs = [[np.full(n_slots, 0xEE, dtype=np.uint8) for _ in range(world)] for _ in range(2)]
        calls = bufs[epoch & 1]
        EI.exchange_epoch(tables, feet, slices, calls, flags, epoch, t, min_depth=2)
        want = ioracle.vote_iupac(full, 2, t)
        assert (want & 0x80).any()
        for r in range(world):
            np.testing.assert_array_equal(calls[r], want, err_msg="epoch %d rank %d" % (epoch, r))


def _insertion_strings(run, calls):
    slots = np.flatnonzero(((calls >> 4) & 3) == 3)
    c = np.searchsorted(run.batch.contig_slot, slots, side="right") - 1
    slots = slots[slots < run.batch.contig_slot[c] + run.batch.contig_len[c].astype(np.int64)]
    strings = []
    for sl in slots.tolist():
        text, tie = run.ins_table.consensus_at(sl)
        strings.append("N" if tie else text.lower())
    return slots, strings


@needs_emu
def test_emulated_k5_on_iupac_calls_equals_host_assembly(manifest, tmp_path):
    """K5 from its source writes the same text for bit-7 calls as the host assembly (_emit_range)."""
    n_mixed = 0
    for k, (name, batch, counts, events) in enumerate(_piled(manifest, tmp_path)):
        if k % 5:
            continue
        run = K.PileupRun.from_host_tables(batch, counts, coracle.derive(counts), events)
        for t in (0.0, 0.7, 1.0):
            calls = ioracle.vote_iupac(counts, 1, t)
            n_mixed += int(np.count_nonzero(calls & 0x80))
            got = EI.assemble(calls, batch, *_insertion_strings(run, calls))
            for c in range(batch.n_contigs):
                s, e = run.contig_slice(c)
                want, _ = K.assemble_consensus(calls[s:e - 1], lambda p, s=s: run.ins_table.consensus_at(s + p))
                assert got[c] == want, (name, t, c)
    assert n_mixed > 100


# --------------------------------------------------------------------------------------- public API
def _host_run(path):
    batch = bamio.read_alignment(path)
    counts, events = coracle.pileup(batch)
    return K.PileupRun.from_host_tables(batch, counts, coracle.derive(counts), events), counts, events


def _two_haplotypes(path, seed=5, L=600, frac=0.35):
    """A mixed sample: a share `frac` of the reads comes from a haplotype with a substitution every ~15 bases."""
    rng = np.random.default_rng(seed)
    ref = "".join(rng.choice(list("ACGT"), size=L))
    alt = list(ref)
    for i in range(7, L, 15):
        alt[i] = "ACGT"[("ACGT".index(ref[i]) + 1 + i % 3) % 4]
    alt = "".join(alt)
    records = []
    for _ in range(900):
        start = int(rng.integers(0, L - 80))
        src = alt if rng.random() < frac else ref
        records.append((0, start, 0, [80 << 4], src[start:start + 80]))
    records.sort(key=lambda r: r[1])
    bamio.write_bam(path, [("hap", L)], records)
    return ref, alt


def test_consensus_from_run_plain_and_realign(manifest, tmp_path):
    """The host half of bam_to_consensus with oracle IUPAC calls: plain, the text is py_oracle's; with --realign the
    changes are the default run's and the text differs from it only where the vote can differ."""
    paths = [golden_input(e) for e in manifest["files"].values()]
    for seed in range(0, 96, 6):
        p = tmp_path / ("clip%d.sam" % seed)
        p.write_text(clip_case(seed))
        paths.append(str(p))
    n_mixed = 0
    for path in paths:
        run, counts, events = _host_run(path)
        contigs = list(_contigs(run.batch, counts, events))
        for t in (0.0, 0.6, 0.99):
            calls = ioracle.vote_iupac(counts, 1, t)
            res = K.consensus_from_run(run, calls, path, iupac_threshold=t)
            base = K.consensus_from_run(run, coracle.vote(counts, 1), path)
            for c, name in enumerate(run.batch.contig_names):
                s, e = run.contig_slice(c)
                want_seq, want_changes = py_ioracle.vote(_py_pileup(counts[:, s:e], contigs[c][2]), 1, t)
                assert res.consensuses[c].sequence == want_seq
                assert list(res.refs_changes[name]) == want_changes
                sites = [str(k + 1) for k in np.flatnonzero(calls[s:e - 1] & 0x80)]
                n_mixed += len(sites)
                lines = res.refs_reports[name].splitlines()
                assert lines[lines.index("- uppercase: False") + 1] == "- iupac_threshold: %s" % t
                at = next(i for i, ln in enumerate(lines) if ln.startswith("- ambiguous sites:"))
                assert lines[at + 1] == "- iupac sites: " + ", ".join(sites)
                assert [ln for ln in lines if "iupac" not in ln] == base.refs_reports[name].splitlines()
            real = K.consensus_from_run(run, calls, path, realign=True, min_overlap=7, iupac_threshold=t)
            real0 = K.consensus_from_run(run, coracle.vote(counts, 1), path, realign=True, min_overlap=7)
            for c, name in enumerate(run.batch.contig_names):
                a, b = real.consensuses[c].sequence, real0.consensuses[c].sequence
                assert len(a) == len(b) and list(real.refs_changes[name]) == list(real0.refs_changes[name])
                for x, y in zip(a, b):
                    assert x == y or (y in "ACGTN" and x in "ACGTMRWSYKVHDBN"), (path, t)
                lines = real.refs_reports[name].splitlines()
                assert [ln for ln in lines if "iupac" not in ln] == real0.refs_reports[name].splitlines()
                assert sum(1 for ln in lines if ln.startswith("- iupac")) == 2
    assert n_mixed > 50


def test_two_haplotype_sample(tmp_path):
    """A 65/35 mixture: the default consensus is the major haplotype; at t = 0.7 the mixed sites become IUPAC
    codes of the two alleles, everywhere the minor allele is frequent enough."""
    path = str(tmp_path / "mix.bam")
    ref, alt = _two_haplotypes(path)
    run, counts, _ = _host_run(path)
    res = K.consensus_from_run(run, ioracle.vote_iupac(counts, 1, 0.7), path, iupac_threshold=0.7)
    seq = res.consensuses[0].sequence
    codes = {frozenset(k): v for k, v in (("AC", "M"), ("AG", "R"), ("AT", "W"), ("CG", "S"), ("CT", "Y"), ("GT", "K"))}
    w = counts[:4, :len(ref)].astype(np.int64)
    n_code = 0
    for i, (r, a) in enumerate(zip(ref, alt)):
        d = int(w[:, i].sum())
        if r != a and d and w["ACGT".index(r), i] < 0.7 * d and w["ACGT".index(a), i] > 0:
            assert seq[i] == codes[frozenset(r + a)], i
            n_code += 1
        elif r == a and d:
            assert seq[i] == r
    assert n_code > 20
    assert res.refs_reports["hap"].count("- iupac sites: ") == 1


def test_report_unchanged_when_off():
    args = ("ref", K.DepthRange(1, 5), [None, "N"], None, "x.bam", False, 1, 7, 0.1, False, False)
    plain = K.build_report(*args)
    assert K.build_report(*args, iupac_threshold=None) == plain
    assert K.build_report(*args, filters=(0, 0, 0), iupac_threshold=None) == plain
    changes = K._changes_list(np.array([0x00, 0x25, 0x85, 0xB3, 0x02], dtype=np.uint8))
    assert changes.iupac == ["3", "4"] and list(changes) == [None, "N", None, "I", None]
    lines = K.build_report(*args[:2], changes, *args[3:], filters=(20, 0, 0), iupac_threshold=0.25).splitlines()
    at = lines.index("- exclude_flags: 0x0")
    assert lines[at + 1] == "- iupac_threshold: 0.25"
    assert lines[lines.index("- ambiguous sites: 2") + 1] == "- iupac sites: 3, 4"


def test_host_letters_of_every_call_byte():
    """_emit_range's letters: bits 0-2 as before, bit 7 the IUPAC code of the nibble."""
    for mask in range(1, 16):
        for change in (0, 3):
            byte = 0x80 | change << 4 | mask
            out, changes = [], K._Changes([None])
            changes.iupac = []
            K._emit_range(np.array([byte], dtype=np.uint8), 0, 1, lambda p: ("ac", False), out, changes)
            assert "".join(out) == ("ac" if change == 3 else "") + LETTERS[mask]
            assert changes.iupac == ["1"]


# ------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("bad", ["-0.1", "1.5", "nan", "x"])
def test_cli_rejects(bad, capsys):
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["consensus", "x.bam", "--iupac-threshold", bad])


def test_cli_accepts():
    p = cli.build_parser()
    assert p.parse_args(["consensus", "x.bam"]).iupac_threshold is None
    assert p.parse_args(["consensus", "x.bam", "--iupac-threshold", "0.6"]).iupac_threshold == 0.6
    assert p.parse_args(["consensus", "x.bam", "--iupac-threshold", "1"]).iupac_threshold == 1.0


@pytest.mark.parametrize("bad", [-0.1, 1.5, float("nan"), float("inf")])
def test_api_and_abi_reject(bad, tmp_path):
    """ValueError before any device work; the C entry points refuse the threshold before they launch anything."""
    with pytest.raises(ValueError):
        K.bam_to_consensus(str(tmp_path / "never_read.bam"), iupac_threshold=bad)
    with pytest.raises(ValueError):
        K.consensus_sequence([{"A": 1, "C": 0, "G": 0, "T": 0, "N": 0}], [{}, {}], [0, 0], None, False, 1, False,
                             iupac_threshold=bad)
    batch = synth.simple_reads(1, [2000], 4)
    with pytest.raises(ValueError):
        D.run_sharded(batch, 2, 1, iupac_threshold=bad)
    lib = _ffi.load()
    buf = np.zeros(7 * 8, dtype=np.int32)
    calls = np.zeros(8, dtype=np.uint8)
    assert lib.kdl_vote_iupac(buf.ctypes.data, 8, 1, bad, calls.ctypes.data, None) == 1
    assert lib.kdl_exchange_vote_iupac(None, 8, 1, bad, 1, None) == 1
    assert math.isnan(bad) or not 0 <= bad <= 1


def test_peer_mode_has_no_iupac_vote():
    batch = synth.simple_reads(1, [2000], 4)
    with pytest.raises(ValueError, match="peer"):
        D.run_sharded(batch, 2, 1, mode="peer", iupac_threshold=0.5)


def test_new_symbols_are_exported():
    lib = _ffi.load()
    for name in ("kdl_vote_iupac", "kdl_exchange_vote_iupac"):
        assert name in _ffi.EXPORTED_SYMBOLS and getattr(lib, name)
