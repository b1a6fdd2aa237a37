"""The dirty-sector map of a reused count table (kdl_pileup_range_map): a pileup zeroes only the 32-byte sectors of
columns 5..18 that the map marks, and every kernel that writes those columns marks what it writes -- or, for complex
reads as dense as 1 in 16 and more, the zeroing kernel leaves the whole range marked.

Sequences of batches go through ONE reused table -- complex batch A, complex batch B (other seed, so other dirty
sectors; both 4 % complex, so their writers mark), a simple batch, A again, a config-3 batch with its edge tail (hard
reads; dense: the range is left marked), and for the order-independent kernels an unsorted batch -- and after every
pileup the table and the events equal the C oracle's and every non-zero (column 5..18, sector) has its bit set.  A map
with every bit set gives the same results.  The emulator half runs the kernel sources on the CPU (tests/emu/); the
`gpu` half runs the same through engine.pileup (masked reads, slot-range shards) and the host-buffer context.

The emulator also runs the sharded step's table sequence: every rank's two parity tables, each bounded by the rank's
footprint, piled into epoch after epoch with the fused exchange in between (tests/test_gpu_sharded_epochs.py runs
distributed.ShardedConsensus itself the same way on one GPU)."""
import numpy as np
import pytest

import emu_harness as E
from kindel_b200 import distributed as D
from kindel_b200 import synth
from oracle import coracle, qoracle

L = 6000


def _sequence(contig_len=L, depth=30, unsorted=False):
    a = synth.mixed_reads(11, [contig_len], depth, 0.04)
    seq = [("complex A", a),
           ("complex B", synth.mixed_reads(12, [contig_len], depth, 0.04)),
           ("simple", synth.simple_reads(13, [contig_len], depth)),
           ("complex A again", a),
           ("cfg3 with edge tail", synth.complex_reads(14, contig_len, depth))]
    if unsorted:  # the order-independent kernels: zeroing pass + K1s + K1g over every complex read
        seq.append(("unsorted tail", synth.complex_reads(15, contig_len, depth, unsorted_tail=True)))
    assert len({b.n_slots for _, b in seq}) == 1
    return seq


def dirty_sectors(counts: np.ndarray) -> np.ndarray:
    """bool [windows, 14, 8]: which (window, column 5 + b, sector) of the table holds a non-zero count."""
    n_slots = counts.shape[1]
    w = (n_slots + 63) // 64
    rest = np.zeros((14, w * 64), dtype=bool)
    rest[:, :n_slots] = counts[5:] != 0
    return rest.reshape(14, w, 8, 8).any(axis=3).transpose(1, 0, 2)


def map_bits(dirty_map: np.ndarray) -> np.ndarray:
    """bool [windows, 14, 8] of a map (uint32 / int32 words, 16 bytes per window; byte b = column 5 + b)."""
    rec = np.ascontiguousarray(dirty_map).view(np.uint8).reshape(-1, 16)[:, :14]
    return ((rec[:, :, None] >> np.arange(8, dtype=np.uint8)) & 1).astype(bool)


def assert_map_covers(counts, dirty_map, what):
    missing = dirty_sectors(counts) & ~map_bits(dirty_map)
    assert not missing.any(), "%s: %d non-zero sectors without their bit" % (what, int(missing.sum()))


# ---------------------------------------------------------------------------------------------- emulator
emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")


@emu
@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("cx", [False, True], ids=["atomics", "pieces"])
def test_reused_table_sequence_emulated(cx, split, monkeypatch):
    monkeypatch.setenv("KDL_CX", "pieces" if cx else "atomics")
    monkeypatch.setenv("KDL_SPLIT", str(split))
    seq = _sequence(unsorted=True)
    n_slots = seq[0][1].n_slots
    table = np.zeros((19, n_slots), dtype=np.int32)   # what CountTable allocates: zeros, map zero
    dmap = np.zeros(E.dirty_map_words(n_slots), dtype=np.uint32)
    ones = np.full((19, n_slots), 0x3B3B3B3B, dtype=np.int32)  # garbage, map all ones: everything is zeroed
    omap = np.full_like(dmap, 0xFFFFFFFF)
    prev_complex = False
    marked = []
    for name, b in seq:
        want, want_ev = coracle.pileup(b)
        what = "%s (cx=%s, split=%d)" % (name, cx, split)
        ev = E.fresh_pileup(b, table, dmap, zero_rest=prev_complex)
        np.testing.assert_array_equal(table, want, err_msg=what)
        np.testing.assert_array_equal(ev, want_ev, err_msg=what)
        assert_map_covers(table, dmap, what)
        if b.n_complex == 0 and prev_complex:
            assert not dmap.any(), what + ": the zeroing must clear the records of what it zeroed"
        if b.n_complex * 16 >= b.n_reads:
            assert (dmap == 0xFFFFFFFF).all(), what + ": dense complex reads leave the range marked"
        marked.append(map_bits(dmap).mean())
        ev = E.fresh_pileup(b, ones, omap, zero_rest=True)
        np.testing.assert_array_equal(ones, want, err_msg=what + " (map of ones)")
        np.testing.assert_array_equal(ev, want_ev, err_msg=what + " (map of ones)")
        assert_map_covers(ones, omap, what + " (map of ones)")
        omap[:] = 0xFFFFFFFF
        prev_complex = b.n_complex > 0
    assert 0 < marked[0] < 0.5 and 0 < marked[1] < 0.5, marked  # marked op by op: far from every sector


@emu
def test_null_map_zeroes_everything_emulated():
    """Without a map (kdl_pileup_range) the zeroing is the full one: a table of garbage comes out right."""
    for _, b in _sequence()[:3]:
        t = np.full((19, b.n_slots), 0x3B3B3B3B, dtype=np.int32)
        ev = E.fresh_pileup(b, t, None, zero_rest=True)
        want, want_ev = coracle.pileup(b)
        np.testing.assert_array_equal(t, want)
        np.testing.assert_array_equal(ev, want_ev)


def test_map_helpers_agree():
    """The test's own reading of the layout: a sector set in the table shows in dirty_sectors, a bit in map_bits."""
    counts = np.zeros((19, 200), dtype=np.int32)
    counts[5 + 9, 64 + 8 * 3 + 5] = 1      # column 14, window 1, sector 3
    got = dirty_sectors(counts)
    assert got.shape == (4, 14, 8) and got.sum() == 1 and got[1, 9, 3]
    dmap = np.zeros(16, dtype=np.uint32)
    dmap[4 + 2] = 1 << (8 * 1 + 3)          # window 1, word 2, byte 1 = record byte 9
    assert map_bits(dmap)[1, 9, 3] and map_bits(dmap).sum() == 1


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["atomics", "pieces"])
def test_engine_table_sequence(monkeypatch, mode):
    import torch

    from kindel_b200 import engine

    monkeypatch.setenv("KDL_CX", mode)
    dev = engine.require_cuda()
    for split in ("1", "4"):
        monkeypatch.setenv("KDL_SPLIT", split)
        seq = _sequence(200_000, 60, unsorted=True)
        table = engine.CountTable(seq[0][1].n_slots, dev)
        for name, b in seq:
            counts, events = engine.pileup(engine.upload(b, dev), table=table)
            torch.cuda.synchronize()
            want, want_ev = coracle.pileup(b)
            what = "%s (%s, split %s)" % (name, mode, split)
            got = counts.cpu().numpy()
            np.testing.assert_array_equal(got, want, err_msg=what)
            np.testing.assert_array_equal(events.cpu().numpy(), want_ev, err_msg=what)
            assert_map_covers(got, table.dirty_map.cpu().numpy(), what)


@pytest.mark.gpu
def test_engine_masked_reads_and_shards():
    """Masked bases (K1q takes back counts the pileup marked) and slot-range shards, into one reused table."""
    import torch

    from kindel_b200 import engine

    dev = engine.require_cuda()
    plain = synth.mixed_reads(21, [300_000], 50, 0.03)  # sparse: K1e marks, K1q takes back
    masked, qual = synth.with_qualities(plain, 22)
    simple = synth.simple_reads(23, [300_000], 50)
    table = engine.CountTable(plain.n_slots, dev)
    for k in range(4):
        b, (want, want_ev) = ((masked, qoracle.pileup(plain, qual, 20)) if k % 2 == 0 else
                              (simple, coracle.pileup(simple)))
        counts, events = engine.pileup(engine.upload(b, dev), table=table)
        torch.cuda.synchronize()
        got = counts.cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg="step %d" % k)
        np.testing.assert_array_equal(events.cpu().numpy(), want_ev, err_msg="step %d" % k)
        assert_map_covers(got, table.dirty_map.cpu().numpy(), "step %d" % k)
    # shards of a complex batch, each bounded by its footprint, in one table
    full = synth.mixed_reads(24, [300_000], 50, 0.3)
    table = engine.CountTable(full.n_slots, dev)
    for rank in (0, 1, 2, 1, 0):
        shard = D.shard_batch(full, rank, 3)
        counts, events = engine.pileup(engine.upload(shard, dev), table=table, slot_range=D.footprint(shard))
        torch.cuda.synchronize()
        got = counts.cpu().numpy()
        want, want_ev = coracle.pileup(shard)
        np.testing.assert_array_equal(got, want, err_msg="shard %d" % rank)
        np.testing.assert_array_equal(events.cpu().numpy(), want_ev, err_msg="shard %d" % rank)
        assert_map_covers(got, table.dirty_map.cpu().numpy(), "shard %d" % rank)


@pytest.mark.gpu
def test_adopted_and_declared_dirty_tables_zero_everything():
    """A table adopted from a tensor, or declared dirty from outside, has every sector marked: garbage goes."""
    import torch

    from kindel_b200 import engine

    dev = engine.require_cuda()
    b = synth.mixed_reads(31, [200_000], 40, 0.1)
    want, want_ev = coracle.pileup(b)
    t = torch.full((19, b.n_slots), 7, dtype=torch.int32, device=dev)
    adopted = engine.CountTable(b.n_slots, dev, tensor=t)
    assert bool((adopted.dirty_map == -1).all())
    adopted.dirty, adopted._dirty_rest = (0, b.n_slots), True
    declared = engine.CountTable(b.n_slots, dev)
    assert not bool(declared.dirty_map.any())
    declared.t.fill_(7)
    declared.dirty, declared.dirty_rest = (0, b.n_slots), True
    assert bool((declared.dirty_map == -1).all())
    for table in (adopted, declared):
        counts, events = engine.pileup(engine.upload(b, dev), table=table)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(counts.cpu().numpy(), want)
        np.testing.assert_array_equal(events.cpu().numpy(), want_ev)


@pytest.mark.gpu
def test_host_context_alternating_batches():
    """kdl_ctx_consensus called again and again on one layout: its own map decides what is zeroed."""
    from kindel_b200 import engine

    seq = _sequence(200_000, 60)
    seq = seq + seq[::-1]
    ctx = engine.HostContext(0)
    try:
        for k, (name, b) in enumerate(seq):
            want, want_ev = coracle.pileup(b)
            counts = np.full((19, b.n_slots), -1, dtype=np.int32)
            events = np.full((max(b.n_events, 1), 4), -1, dtype=np.int32)
            calls = ctx.consensus(b, 1, counts_out=counts, events_out=events)
            what = "call %d (%s)" % (k, name)
            np.testing.assert_array_equal(counts, want, err_msg=what)
            np.testing.assert_array_equal(events[:b.n_events], want_ev, err_msg=what)
            np.testing.assert_array_equal(calls, coracle.vote(want, 1), err_msg=what)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------- sharded epochs, emulated
class _EmuRankTable:
    """One parity table of a rank as distributed.ShardedConsensus holds it, on the host: adopted from a zero-filled
    block (CountTable(tensor=...): every map bit set, nothing dirty yet), with engine.pileup's bookkeeping around
    each pileup -- the range is the footprint joined with what earlier pileups dirtied, tile-aligned, and columns
    5..18 are zeroed (where the map says) once a complex batch has been piled into the table."""

    def __init__(self, n_slots):
        self.t = np.zeros((19, n_slots), dtype=np.int32)
        self.map = np.full(E.dirty_map_words(n_slots), 0xFFFFFFFF, dtype=np.uint32)
        self.dirty, self.dirty_rest = None, False

    def pileup(self, batch, slot_range):
        n_slots = self.t.shape[1]
        lo, hi = slot_range
        if self.dirty is not None:
            lo, hi = min(lo, self.dirty[0]), max(hi, self.dirty[1])
        lo, hi = max(0, lo // 512 * 512), min(n_slots, (hi + 511) // 512 * 512)
        ev = E.fresh_pileup(batch, self.t, self.map, self.dirty_rest, slot_range=(lo, hi))
        self.dirty, self.dirty_rest = (lo, hi), batch.n_complex > 0
        return ev


def _sharded_case(kind):
    if kind == "contigs":  # 3 ranks over 2 contigs: the middle rank gets no reads and a zero-width slice
        return synth.mixed_reads(16, [3000, 2500], 30, 0.04), "contigs"
    if kind == "dense":    # 1 in 16 and more complex, hard reads of the edge tail: ranges are left marked
        return synth.complex_reads(17, L, 30), "reads"
    return synth.mixed_reads(18, [L], 30, 0.04), "reads"  # sparse: the kernels mark sector by sector


@emu
@pytest.mark.parametrize("world,kind", [(2, "sparse"), (3, "sparse"), (2, "dense"), (3, "contigs")])
def test_sharded_epochs_emulated(world, kind):
    """The fused sharded step of every rank on the emulated kernels: each rank keeps its shard and its two parity
    tables, piles into the epoch's table over its footprint with a live map (every table reused), then K2x + K2g run
    over that epoch's tables.  After every epoch each rank's calls equal the oracle's vote of the whole batch, each
    table equals its shard's oracle table (zero outside the footprint) with its map covering it, the tables add up to
    the whole batch's and the shards' events merge into its events."""
    full, plan = _sharded_case(kind)
    n_slots = full.n_slots
    want, want_ev = coracle.pileup(full)
    want_calls = coracle.vote(want, 2)
    idx = [D.shard_indices(full, r, world, plan) for r in range(world)]
    shards = [D.select_reads(full, i) for i in idx]
    shard_want = [coracle.pileup(s)[0] for s in shards]
    feet = [D.footprint(s) for s in shards]
    slices = D.footprint_slices(feet, n_slots)
    if kind == "contigs":
        assert [s.n_reads == 0 for s in shards] == [False, True, False] and slices[1][0] == slices[1][1]
    tables = [[_EmuRankTable(n_slots) for _ in range(2)] for _ in range(world)]
    calls = [[np.full(n_slots, 0xEE, dtype=np.uint8) for _ in range(world)] for _ in range(2)]
    flags = {k: [np.zeros(16, dtype=np.int32) for _ in range(world)] for k in ("ready", "done")}
    flags["counter"] = [np.zeros(1, dtype=np.int32) for _ in range(world)]
    for epoch in range(1, 5):
        par = epoch & 1
        evs = [tables[r][par].pileup(shards[r], feet[r]) for r in range(world)]
        E.exchange_epoch([tables[r][par].t for r in range(world)], feet, slices, calls[par], flags, epoch, min_depth=2)
        for r in range(world):
            what = "%s world %d epoch %d rank %d" % (kind, world, epoch, r)
            np.testing.assert_array_equal(calls[par][r], want_calls, err_msg=what)
            tab = tables[r][par]
            np.testing.assert_array_equal(tab.t, shard_want[r], err_msg=what)
            lo, hi = feet[r]
            assert not tab.t[:, :lo].any() and not tab.t[:, hi:].any(), what
            for k in range(2):
                assert_map_covers(tables[r][k].t, tables[r][k].map, what + " parity %d" % k)
        np.testing.assert_array_equal(sum(tables[r][par].t.astype(np.int64) for r in range(world)), want)
        np.testing.assert_array_equal(D.merge_events(evs, idx), want_ev)
