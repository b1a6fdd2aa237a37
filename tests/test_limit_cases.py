"""The engine at its own limits (tests/limit_cases.py), on the CPU.

Every read of the corpus lands in the class it was built for (simple, tile-eligible or KDL_HARD) with the right
l_seq word, whichever decoder reads it; the C oracle matches what the unmodified reference computed for the same
files (tests/golden/reference_digests.json); K0 + K1 (both instantiations, every flush mode, the depth split), K1e,
K1g and the whole pipeline, run from their CUDA source in the emulator, equal the oracle under three thread
orders; K1q equals the masking oracle on the corpus's quality lattice; and every shard's table lies inside its
footprint.  The corpus's mirror of the capacities is read back out of the sources, so it cannot drift."""
import json
import os
import re

import numpy as np
import pytest

import emu_harness as E
import limit_cases as LC
from conftest import GOLDEN, ROOT
from kindel_b200 import _ffi, bamio
from kindel_b200 import distributed as D
from oracle import coracle, qoracle
from oracle import make_reference_digests as R
from test_quality_filters import sam_quals, sam_to_bam, same_arrays

GROUPS = list(LC.GROUPS)
emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("limits")
    out = {}
    for name in GROUPS:
        text = LC.sam_text(name)
        sam, bam = str(d / (name + ".sam")), str(d / (name + ".bam"))
        with open(sam, "w") as fh:
            fh.write(text)
        sam_to_bam(text, bam)
        out[name] = (text, sam, bam)
    return out


_batches = {}


def batch_of(files, name, **kw):
    key = (name, tuple(sorted(kw.items())))
    if key not in _batches:
        _batches[key] = bamio.read_bam(files[name][2], **kw)
    return _batches[key]


def _source(*parts):
    with open(os.path.join(ROOT, *parts)) as fh:
        return fh.read()


def test_capacities_match_the_sources():
    h = _source("include", "kindel_b200.h")
    for k in ("KDL_FAST_MAXLEN", "KDL_TILE_MAXOPS", "KDL_TILE_MAXREACH", "KDL_LEN_MASK", "KDL_TILE"):
        m = re.search(r"#define %s\s+(0x[0-9a-fA-F]+u?|\d+)" % k, h)
        assert m, k
        assert int(m.group(1).rstrip("u"), 0) == getattr(LC, k), k
        if hasattr(_ffi, k):
            assert getattr(_ffi, k) == getattr(LC, k), k
    tc = _source("kindel_b200", "csrc", "tile_common.cuh")
    assert int(re.search(r"constexpr int F_FLUSH_BLOCKS = (\d+);", tc).group(1)) == LC.F_FLUSH_BLOCKS
    assert int(re.search(r"constexpr int F_WIN = (\d+);", tc).group(1)) == LC.F_WIN
    pt = _source("kindel_b200", "csrc", "pileup_tile.cu")
    two = pt.split("#if KDL_W_STAGES == 2", 1)[1].split("#elif", 1)[0]
    for cx in (False, True):
        body = two.split("struct TileCfg<%s>" % ("true" if cx else "false"), 1)[1].split("};", 1)[0]
        cfg = {k: int(v) for k, v in re.findall(r"(k\w+) = (\d+);", body)}
        assert cfg["kRmax"] == LC.RMAX[cx] and cfg["kCapW"] == LC.CAPW[cx], cx
        if cx:
            assert cfg["kPcap"] == LC.PCAP
    assert int(re.search(r"constexpr int W_PRODUCERS = (\d+);", pt).group(1)) * 32 == LC.W_PT
    # the corpus's shapes need these relations to mean what they say
    assert 10 * LC.KDL_TILE_MAXOPS <= LC.PCAP < 11 * LC.KDL_TILE_MAXOPS
    assert LC.RMAX[False] * 19 == LC.CAPW[False] and LC.RMAX[True] * 20 == LC.CAPW[True]


def _classes(batch):
    w = batch.l_seq.view(np.uint32).astype(np.int64)
    return ["h" if x & _ffi.KDL_HARD else "t" if x & _ffi.KDL_COMPLEX else "s" for x in w.tolist()]


def _n_match(batch):
    ops = batch.cigar & 15
    is_m = ((ops == 0) | (ops == 7) | (ops == 8)).astype(np.int64)
    c = np.concatenate(([0], np.cumsum(is_m)))
    co = batch.cig_off.astype(np.int64)
    return c[co[1:]] - c[co[:-1]]


@pytest.mark.parametrize("name", GROUPS)
def test_classes_and_decoders_agree(files, name):
    """Each read's class and l_seq word, the same from the C++ BAM decoder, the C++ SAM converter and
    bamio.finalize (the Python SAM reader), with and without the base-quality mask."""
    text, sam, bam = files[name]
    want = LC.expected_classes(name)
    for thr in (0, LC.MASK_QUAL):
        py = bamio.read_sam(sam, min_base_quality=thr)
        same_arrays(bamio.read_bam(sam, min_base_quality=thr), py)
        same_arrays(bamio.read_bam(bam, min_base_quality=thr), py)
        assert _classes(py) == want
        lseq = py.seq_len.astype(np.int64)
        word = np.where(np.array(want) == "s", lseq,
                        np.where(np.array(want) == "t", lseq | (_n_match(py) << _ffi.KDL_NM_SHIFT) | _ffi.KDL_COMPLEX,
                                 lseq | _ffi.KDL_COMPLEX | _ffi.KDL_HARD))
        assert np.array_equal(py.l_seq.view(np.uint32).astype(np.int64), word)
        assert py.reads_sorted and py.n_reads == len(want)
        if thr:
            assert py.n_masked > 0


def test_every_limit_is_reached_from_both_sides(files):
    """The corpus is not vacuous: the exact values on and past each limit occur, in the class they must have."""
    seen = {}
    for name in GROUPS:
        b = batch_of(files, name)
        cls = _classes(b)
        co = b.cig_off.astype(np.int64)
        for r in range(b.n_reads):
            ops = [(int(x) >> 4, int(x) & 15) for x in b.cigar[co[r]:co[r + 1]]]
            n_ops = len(ops)
            lead = ops[0][0] if ops and ops[0][1] == 4 else 0
            span = sum(n for k, (n, op) in enumerate(ops) if op in (0, 2, 7, 8) or (op == 4 and k > 0))
            start = int(b.ref_start[r])
            L = int(b.contig_len[np.searchsorted(b.contig_read_off, r, side="right") - 1])
            lseq = int(b.seq_len[r])
            if cls[r] == "s":
                seen.setdefault(("simple_len", lseq), set()).add("s")
                if start + lseq == L:
                    seen.setdefault(("simple_end", lseq >= 8192), set()).add("s")
                continue
            # each limit, with every OTHER condition of tile eligibility met
            value = {"ops": n_ops, "cx_len": lseq, "slot0": start - lead - 1, "last": start + span - (L - 1),
                     "span": span, "lead": lead}
            ok = {"ops": n_ops <= 64, "cx_len": lseq <= 8192, "slot0": start - lead - 1 >= 0,
                  "last": start + span <= L - 1, "span": span <= 1023, "lead": lead <= 1023}
            for k in value:
                if all(v for o, v in ok.items() if o != k):
                    seen.setdefault((k, value[k]), set()).add(cls[r])
    want = {("simple_len", 8191): {"s"}, ("simple_len", 8192): {"s"}, ("simple_end", True): {"s"},
            ("ops", 64): {"t"}, ("ops", 65): {"h"}, ("span", 1023): {"t"}, ("span", 1024): {"h"},
            ("lead", 1023): {"t"}, ("lead", 1024): {"h"}, ("slot0", 0): {"t"}, ("slot0", -1): {"h"},
            ("last", 0): {"t"}, ("last", 1): {"h"}, ("cx_len", 8192): {"t"}, ("cx_len", 8193): {"h"}}
    for k, v in want.items():
        assert seen.get(k) == v, (k, seen.get(k))
    # simple reads past KDL_FAST_MAXLEN are hard
    b = batch_of(files, "simple_len")
    assert [c for c, n in zip(_classes(b), b.seq_len.tolist()) if n == 8193] == ["h", "h"]


def _k0_items(batch, tile):
    """(reads, staged words) of the first item K1 makes of `tile` (K0's read range, kRmax / kCapW cuts)."""
    g0 = tile * LC.KDL_TILE
    start = batch.contig_slot[0] + batch.ref_start.astype(np.int64)
    lo = int(np.searchsorted(start, g0 - batch.reach_right + 1))
    hi = int(np.searchsorted(start, g0 + LC.KDL_TILE + batch.reach_left))
    wa = int(batch.seq_off[lo]) & ~3
    wend = int(batch.seq_off[hi]) if hi < batch.n_reads else int(batch.seq4.shape[0])
    return hi - lo, wend - wa


def test_items_sit_on_the_capacities(files):
    b = batch_of(files, "items")
    assert b.n_contigs == 1
    shapes = [_k0_items(b, t) for t in range(6)]
    assert shapes[0] == (LC.RMAX[False], LC.CAPW[False])          # exactly full, both ways
    assert shapes[1] == (LC.RMAX[False], LC.CAPW[False] + 1)      # one word over
    assert shapes[2][0] == LC.RMAX[False] + 1
    assert shapes[3] == (LC.RMAX[True], LC.CAPW[True])
    assert shapes[4] == (LC.RMAX[True], LC.CAPW[True] + 1)
    assert shapes[5][0] == LC.RMAX[True] + 1
    p = batch_of(files, "pieces")
    n_m = _n_match(p)
    per_tile = [int(n_m[(p.ref_start // LC.KDL_TILE) == t].sum()) for t in range(4)]
    assert per_tile[:3] == [LC.PCAP, LC.PCAP + 1, 11 * LC.KDL_TILE_MAXOPS]


@pytest.mark.parametrize("name", GROUPS)
def test_oracle_matches_the_reference(files, name):
    """The C oracle's tables, insertion dicts, changes and FASTA equal what the unmodified reference computed for the
    same file (oracle/make_reference_digests.py)."""
    import helpers as H
    from kindel_b200 import kindel as K

    with open(os.path.join(GOLDEN, "reference_digests.json")) as fh:
        ref = json.load(fh)["limit_cases"][name]
    b = bamio.read_alignment(files[name][1])
    counts, events = coracle.pileup(b)
    calls = coracle.vote(counts, 1)
    ins = H.events_to_dicts(b, events)
    assert b.contig_names == ref["contigs"]
    got = []
    for c in range(b.n_contigs):
        t = H.contig_view(b, counts, c)
        s = int(b.contig_slot[c])
        L = int(b.contig_len[c])
        dicts = [ins.get(s + i, {}) for i in range(L + 1)]
        changes = H.calls_to_changes(calls[s:s + L])
        got.append(R.table_digest(t, dicts, changes))
    assert got == ref["digests"]
    run = K.PileupRun.from_host_tables(b, counts, coracle.derive(counts), events)
    res = K.consensus_from_run(run, calls, files[name][1])
    assert R.fasta_digest([(r.name, r.sequence) for r in res.consensuses]) == ref["fasta"]


# ---- the kernels from their CUDA source -------------------------------------------------------------------------
def _hard_table(batch):
    return coracle.pileup(D.select_reads(batch, batch.hard_idx))[0] if batch.n_hard else 0


@emu
@pytest.mark.parametrize("cx", [False, True], ids=["lean", "cx"])
@pytest.mark.parametrize("name", GROUPS)
def test_limit_tile_kernel(files, name, cx, monkeypatch):
    """K0 + K1 (+ K1e<8> behind the lean instantiation, K1e<1> behind kCx, + K1g) as kdl_pileup_range launches them, in
    F_STORE over garbage, F_ADD, and F_ATOMIC with 2 and 5 CTAs per tile: the whole table and every event, exactly.  A
    group without tile-eligible complex reads runs kCx by a direct launch (no entry point picks it there): everything
    but the hard reads."""
    b = batch_of(files, name)
    assert E.tileable(b)
    want_c, want_e = coracle.pileup(b)
    direct = cx and b.n_complex == b.n_hard
    monkeypatch.setenv("KDL_CX", "pieces" if cx else "atomics")
    for fresh, split in ((True, 1), (False, 1), (False, 2), (False, 5)):
        what = "%s fresh=%s split=%d" % (name, fresh, split)
        if direct:
            got = E.tile_cx_pileup(b, fresh, split, zero_rest=fresh)
            np.testing.assert_array_equal(got, want_c - _hard_table(b), err_msg=what)
            continue
        monkeypatch.setenv("KDL_SPLIT", str(split))
        got, ev = E.run_pileup(b, fresh, want_events=True, zero_rest=fresh)
        np.testing.assert_array_equal(got, want_c, err_msg=what)
        np.testing.assert_array_equal(ev, want_e, err_msg=what)


@emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 3)])
def test_limit_pipeline(files, schedule, seed, monkeypatch):
    """The whole pileup pipeline (K0 + K1 + K1e + K1g, as kdl_pileup launches them) under three thread orders."""
    E.set_schedule(schedule, seed)
    try:
        for name in GROUPS:
            b = batch_of(files, name)
            want_c, want_e = coracle.pileup(b)
            for split in ((1, 2) if schedule == "forward" else (1,)):
                monkeypatch.setenv("KDL_SPLIT", str(split))
                got_c, got_e = E.pileup_pipeline(b)
                np.testing.assert_array_equal(got_c, want_c, err_msg="%s %s split=%d" % (name, schedule, split))
                np.testing.assert_array_equal(got_e, want_e, err_msg=name)
    finally:
        E.set_schedule("forward")


@emu
@pytest.mark.parametrize("schedule", ["forward", "random"])
def test_limit_k1q_mask_lattice(files, schedule, monkeypatch):
    """K1q after the pipeline on the corpus's quality lattice equals the masking oracle."""
    E.set_schedule(schedule, 7)
    try:
        for name in GROUPS:
            text, sam, bam = files[name]
            plain = batch_of(files, name)
            masked = batch_of(files, name, min_base_quality=LC.MASK_QUAL)
            qual = sam_quals(text)
            assert masked.n_masked == int((qual < LC.MASK_QUAL).sum()) > 0
            want_c, want_e = qoracle.pileup(plain, qual, LC.MASK_QUAL)
            for split in (1, 3):
                monkeypatch.setenv("KDL_SPLIT", str(split))
                got_c, got_e = E.pileup_pipeline(masked)
                np.testing.assert_array_equal(E.unmask(masked, got_c), want_c, err_msg=name)
                np.testing.assert_array_equal(got_e, want_e, err_msg=name)
    finally:
        E.set_schedule("forward")


# ---- footprints ---------------------------------------------------------------------------------------------------
def _check_footprints(batch, label):
    for world in (2, 3, 4):
        for rank in range(world):
            shard = D.shard_batch(batch, rank, world)
            try:
                t, _ = coracle.pileup(shard)
            except (IndexError, KeyError):
                continue
            lo, hi = D.footprint(shard)
            assert not t[:, :lo].any() and not t[:, hi:].any(), (label, world, rank, (lo, hi))


def test_footprints_hold_on_the_fuzz_cases(tmp_path):
    from fuzz_cases import random_case

    checked = 0
    for seed in range(400):
        p = tmp_path / ("f%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            b = bamio.read_alignment(p)
        except (ValueError, KeyError):
            continue
        _check_footprints(b, seed)
        checked += 1
    assert checked > 300


def test_footprints_hold_on_the_limit_cases(files):
    for name in GROUPS:
        _check_footprints(batch_of(files, name), name)
