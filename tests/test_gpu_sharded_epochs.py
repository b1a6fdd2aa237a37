"""distributed.ShardedConsensus for 2 and 3 ranks in ONE process on one GPU, epoch after epoch, against the oracle.

The ranks are the product's own ShardedConsensus objects.  Only what needs a second process is stood in for:
  * the process group: rank and world, the footprint all_gather (filled from the precomputed shards, in rank order),
    a barrier that does nothing, and in allreduce mode an all_reduce whose first call of an epoch sums columns 0..6 of
    every rank's table into all of them (every rank's pileup is already in the stream);
  * the CUDA IPC mappings of PeerTables: every rank's block is allocated once on this device, with PeerTables' layout,
    and the peers' pointers are those blocks.  exchange_struct, counts, calls and close are the product's own.

Every kernel goes into ONE stream, in an order in which nothing waits for a kernel behind it: every rank's pileup
(`pile`), every rank's ready signal, every rank's vote (K2x, `exchange`), then every rank's pull of the peers' call
slices (K2g, which waits for the peers' K2x: the driver issues it after all of them).  `step()` is never called rank
after rank here: its K2g would wait for the next rank's K2x, behind it in the stream.

Each rank keeps its shard for every epoch, as the product and bench.py do, so each of its two parity tables is piled
into again and again with a live dirty-sector map.  After every epoch: every rank's calls equal the oracle's vote of
the whole batch; each rank's own table equals its shard's oracle table (fused: zero outside the footprint; allreduce:
columns 0..6 summed over all ranks); every table's map covers its non-zero sectors; the ranks' tables reduce to the
whole batch's table; their events merge into its events; and K2p over the epoch's parity tables agrees."""
import ctypes as C
import math

import numpy as np
import pytest

from kindel_b200 import _ffi, bamio, synth
from kindel_b200 import distributed as D
from oracle import coracle, ioracle, qoracle
from test_sparse_zero import assert_map_covers

pytestmark = pytest.mark.gpu

EPOCHS = 6  # each parity table piled into three times
MIN_DEPTH = 2


class _World:
    """What the ranks of the stand-in group share."""

    def __init__(self, n, feet):
        self.n, self.feet = n, feet
        self.blocks = None  # device pointer of every rank's block
        self.ranks = []     # the ShardedConsensus objects, in rank order
        self.reduced_epoch = 0


class _Group:
    def __init__(self, world: _World, rank: int):
        self.world, self.rank = world, rank


def _all_gather_object(out, obj, group=None):
    assert obj == group.world.feet[group.rank]  # (ShardedConsensus gathers its footprint)
    out[:] = list(group.world.feet)


def _all_reduce(tensor, op=None, group=None):
    import torch

    w = group.world
    me = w.ranks[group.rank]
    assert tensor.data_ptr() == me.last_counts.data_ptr() and tensor.shape[0] == _ffi.KDL_NVOTE_COL
    if w.reduced_epoch == me.epoch:
        return
    w.reduced_epoch = me.epoch
    cols = [sc.last_counts[: _ffi.KDL_NVOTE_COL] for sc in w.ranks]
    total = torch.stack(cols).sum(0, dtype=torch.int32)
    for c in cols:
        c.copy_(total)


class _OneProcessPeerTables(D.PeerTables):
    """PeerTables without IPC: the first rank allocates every rank's block (kdl_table_alloc: zero-filled), with the
    layout of PeerTables -- [table 0][table 1][calls 0][calls 1][flags] -- and the peers' pointers are the blocks."""

    def __init__(self, n_slots: int, device, group=None):
        import torch

        w = group.world
        self.lib = _ffi.load()
        self.n_slots, self.device, self.group = n_slots, device, group
        self.world, self.rank = w.n, group.rank
        self.table_bytes = _ffi.KDL_NCOL * n_slots * 4
        self.calls_off = 2 * self.table_bytes
        self.flags_off = self.calls_off + 2 * n_slots
        if w.blocks is None:
            w.blocks = []
            with torch.cuda.device(device):
                for _ in range(w.n):
                    p = C.c_void_p()
                    _ffi.check(self.lib.kdl_table_alloc(self.flags_off + 256, C.byref(p)), "kdl_table_alloc")
                    w.blocks.append(p.value)
        self.ptr = w.blocks[self.rank]
        self.peer_ptrs = list(w.blocks)
        self._opened = []
        self.counts = [D._wrap_device_memory(self.ptr + k * self.table_bytes, (_ffi.KDL_NCOL, n_slots), device)
                       for k in range(2)]
        self.calls = [D._wrap_device_memory(self.ptr + self.calls_off + k * n_slots, (n_slots,), device, "|u1")
                      for k in range(2)]


class _DeferredWait:
    """The library as a rank's `exchange` sees it, except that K2g (kdl_exchange_wait) is only recorded: the driver
    issues it once every rank's K2x is in the stream."""

    def __init__(self, lib, pending):
        self._lib, self._pending = lib, pending

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def kdl_exchange_wait(self, x, epoch, stream):
        self._pending.append((x, epoch, stream))
        return _ffi.KDL_OK


class _Lockstep:
    """`world` ranks of one sharded job, driven epoch by epoch in one process on one device."""

    def __init__(self, monkeypatch, full, world, mode, plan="reads", qual=None, masked=None):
        import torch
        import torch.distributed as dist

        self.full, self.world, self.mode = full, world, mode
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.lib = _ffi.load()
        self.idx = [D.shard_indices(full, r, world, plan) for r in range(world)]
        src = full if masked is None else masked
        self.shards = [D.select_reads(src, i) for i in self.idx]
        if qual is None:
            self.want, self.want_ev = coracle.pileup(full)
            self.shard_want = [coracle.pileup(D.select_reads(full, i))[0] for i in self.idx]
        else:  # masked bases: the oracle reads them as N and does not count them
            self.want, self.want_ev = qoracle.pileup(full, qual, 20)
            lens = full.seq_len.astype(np.int64)
            starts = np.cumsum(lens) - lens
            self.shard_want = [qoracle.pileup(D.select_reads(full, i), bamio._ragged_gather(qual, starts[i], lens[i]),
                                              20)[0] for i in self.idx]
            assert all(s.n_masked for s in self.shards)
        self.feet = [D.footprint(s) for s in self.shards]
        self.w = _World(world, self.feet)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: group.world.n)
        monkeypatch.setattr(dist, "get_rank", lambda group=None: group.rank)
        monkeypatch.setattr(dist, "all_gather_object", _all_gather_object)
        monkeypatch.setattr(dist, "barrier", lambda group=None: None)
        monkeypatch.setattr(dist, "all_reduce", _all_reduce)
        monkeypatch.setattr(D, "PeerTables", _OneProcessPeerTables)
        try:
            for r in range(world):
                self.w.ranks.append(D.ShardedConsensus(self.shards[r], self.dev, mode=mode, group=_Group(self.w, r)))
        except BaseException:
            self.close()
            raise

    def close(self):
        owned = set()
        for sc in self.w.ranks:
            if sc.tables is not None:
                owned.add(sc.tables.ptr)
            sc.close()
        for p in self.w.blocks or []:  # blocks of ranks that were never built
            if p not in owned:
                self.lib.kdl_table_free(p)
        self.w.ranks, self.w.blocks = [], None

    def epoch(self, iupac_threshold=None):
        """One step of every rank.  Returns the call bytes of every rank (host)."""
        import torch

        ranks = self.w.ranks
        for sc in ranks:
            sc.pile()
        if self.mode == "allreduce":  # before the all_reduce puts every rank's sums into columns 5, 6
            for r, sc in enumerate(ranks):
                what = "allreduce world %d epoch %d rank %d, after the pileup" % (self.world, sc.epoch, r)
                got = sc.last_counts.cpu().numpy()
                np.testing.assert_array_equal(got, self.shard_want[r], err_msg=what)
                assert_map_covers(got, sc.table[sc.epoch & 1].dirty_map.cpu().numpy(), what)
        if self.mode == "fused":
            st = int(torch.cuda.current_stream(self.dev).cuda_stream)
            for sc in ranks:
                _ffi.check(self.lib.kdl_exchange_signal(C.byref(sc.xstruct[sc.epoch & 1]), sc.epoch, st), "signal")
            pending = []
            for sc in ranks:
                sc.lib = _DeferredWait(self.lib, pending)
            try:
                calls = [sc.exchange(MIN_DEPTH, iupac_threshold) for sc in ranks]
            finally:
                for sc in ranks:
                    sc.lib = self.lib
            assert len(pending) == self.world
            for x, ep, s in pending:
                _ffi.check(self.lib.kdl_exchange_wait(x, ep, s), "kdl_exchange_wait")
        else:
            calls = [sc.exchange(MIN_DEPTH, iupac_threshold) for sc in ranks]
        torch.cuda.synchronize()
        return [c.cpu().numpy() for c in calls]

    def check(self, calls, iupac_threshold=None):
        """Everything the module docstring lists, for the epoch that just ran."""
        ranks = self.w.ranks
        epoch = ranks[0].epoch
        par = epoch & 1
        want_calls = (coracle.vote(self.want, MIN_DEPTH) if iupac_threshold is None
                      else ioracle.vote_iupac(self.want, MIN_DEPTH, iupac_threshold))
        nv = _ffi.KDL_NVOTE_COL
        own = []
        for r, sc in enumerate(ranks):
            what = "%s world %d epoch %d rank %d" % (self.mode, self.world, epoch, r)
            np.testing.assert_array_equal(calls[r], want_calls, err_msg=what)
            tabs = [sc.table[k].t.cpu().numpy() for k in range(2)]
            got = tabs[par]
            np.testing.assert_array_equal(sc.last_counts.cpu().numpy(), got, err_msg=what)
            if self.mode == "fused":
                np.testing.assert_array_equal(got, self.shard_want[r], err_msg=what)
                lo, hi = self.feet[r]
                assert not got[:, :lo].any() and not got[:, hi:].any(), what + ": counts outside the footprint"
                if epoch > 1:  # last epoch's table, untouched since
                    np.testing.assert_array_equal(tabs[par ^ 1], self.shard_want[r], err_msg=what + " (other parity)")
                for k in range(2):
                    assert_map_covers(tabs[k], sc.table[k].dirty_map.cpu().numpy(), what + " parity %d" % k)
            else:
                np.testing.assert_array_equal(got[:nv], self.want[:nv], err_msg=what + " (reduced columns)")
                np.testing.assert_array_equal(got[nv:], self.shard_want[r][nv:], err_msg=what + " (own columns)")
            own.append(got)
        # what reduce_table sums on its destination rank
        if self.mode == "fused":
            reduced = sum(t.astype(np.int64) for t in own)
        else:
            reduced = np.concatenate([own[0][:nv], sum(t[nv:].astype(np.int64) for t in own)])
        np.testing.assert_array_equal(reduced, self.want, err_msg="reduced table, epoch %d" % epoch)
        evs = [sc.dbatch.tensors["_events"][: s.n_events].cpu().numpy() if s.n_events else np.zeros((0, 4), np.int32)
               for sc, s in zip(ranks, self.shards)]
        np.testing.assert_array_equal(D.merge_events(evs, self.idx), self.want_ev, err_msg="events, epoch %d" % epoch)
        if self.mode == "fused" and iupac_threshold is None:
            self.check_peer_vote(want_calls)

    def check_peer_vote(self, want_calls):
        """K2p (kdl_vote_peers_sparse) over this epoch's parity tables, every rank on its own slice."""
        import torch

        st = int(torch.cuda.current_stream(self.dev).cuda_stream)
        n_slots = self.full.n_slots
        for r, sc in enumerate(self.w.ranks):
            lo, hi = sc.slices[r]
            calls = torch.full((n_slots,), 0xEE, dtype=torch.uint8, device=self.dev)
            reduced = torch.zeros((_ffi.KDL_NVOTE_COL, n_slots), dtype=torch.int32, device=self.dev)
            rc = self.lib.kdl_vote_peers_sparse(sc.ptr_arr[sc.epoch & 1], sc.foot_lo, sc.foot_hi, self.world, n_slots,
                                                lo, hi, int(math.ceil(MIN_DEPTH)), calls.data_ptr(), reduced.data_ptr(), st)
            _ffi.check(rc, "kdl_vote_peers_sparse")
            what = "K2p epoch %d rank %d" % (sc.epoch, r)
            np.testing.assert_array_equal(calls[lo:hi].cpu().numpy(), want_calls[lo:hi], err_msg=what)
            np.testing.assert_array_equal(reduced[:, lo:hi].cpu().numpy(), self.want[: _ffi.KDL_NVOTE_COL, lo:hi],
                                          err_msg=what)

    def run(self, thresholds=None):
        """EPOCHS epochs; thresholds(epoch) -> the IUPAC threshold of that epoch, or None for the majority vote."""
        try:
            for epoch in range(1, EPOCHS + 1):
                t = thresholds(epoch) if thresholds else None
                self.check(self.epoch(t), t)
        finally:
            self.close()


def _iupac_on_odd_epochs(epoch):
    return (0.0, 0.6, 1.0)[(epoch - 1) // 2 % 3] if epoch & 1 else None


L = 150_000


@pytest.mark.parametrize("frac", [0.01, 0.04])
@pytest.mark.parametrize("world", [2, 3])
def test_fused_sparse_complex(monkeypatch, world, frac):
    """1 % and 4 % complex reads in sorted simple ones: K1e / K1g mark the map op by op."""
    full = synth.mixed_reads(101, [L], 40, frac)
    assert 0 < full.n_complex * 16 < full.n_reads
    _Lockstep(monkeypatch, full, world, "fused").run()


@pytest.mark.parametrize("kind", ["30pct", "edge_tail"])
@pytest.mark.parametrize("world", [2, 3])
def test_fused_dense_complex(monkeypatch, world, kind):
    """Complex reads dense enough (>= 1 in 16) that the range is left marked; the config-3 batch has hard reads."""
    full = synth.mixed_reads(102, [L], 40, 0.3) if kind == "30pct" else synth.complex_reads(103, 40_000, 60)
    assert full.n_complex * 16 >= full.n_reads and (kind == "30pct" or full.n_hard > 0)
    _Lockstep(monkeypatch, full, world, "fused").run()


@pytest.mark.parametrize("world", [2, 3])
def test_fused_iupac_and_majority(monkeypatch, world):
    """The IUPAC vote (t = 0, 0.6, 1) on odd epochs, the majority vote on even ones, through K2x."""
    full = synth.mixed_reads(104, [L], 40, 0.04)
    _Lockstep(monkeypatch, full, world, "fused").run(_iupac_on_odd_epochs)


@pytest.mark.parametrize("world", [2, 3])
def test_fused_masked_shards(monkeypatch, world):
    """Bases below Q20 masked: K1q takes back counts in a reused rank table after every pileup."""
    plain = synth.mixed_reads(105, [L], 40, 0.03)
    masked, qual = synth.with_qualities(plain, 106)
    _Lockstep(monkeypatch, plain, world, "fused", qual=qual, masked=masked).run()


@pytest.mark.parametrize("world,lens", [(2, [60_000, 45_000, 30_000, 50_000]), (3, [60_000, 45_000])],
                         ids=["2_ranks_4_contigs", "3_ranks_2_contigs"])
def test_fused_contig_plan(monkeypatch, world, lens):
    """Whole contigs per rank (no slot shared); three ranks over two contigs leave one rank without reads, with a
    zero-width slice that still takes part in the flag protocol."""
    full = synth.mixed_reads(107, lens, 40, 0.04)
    drv = _Lockstep(monkeypatch, full, world, "fused", plan="contigs")
    if world == 3:
        assert [s.n_reads == 0 for s in drv.shards] == [False, True, False]
        lo, hi = drv.w.ranks[1].slices[1]
        assert lo == hi
    drv.run()


@pytest.mark.parametrize("frac", [0.04, 0.3])
@pytest.mark.parametrize("world", [2, 3])
def test_allreduce_majority_and_iupac(monkeypatch, world, frac):
    """allreduce mode: columns 5, 6 of every table hold the sums of all ranks after a step, so the next pileup must
    zero all of the table's columns 5..18 -- with 4 % complex reads the map alone would leave other ranks' sums."""
    full = synth.mixed_reads(108, [L], 40, frac)
    _Lockstep(monkeypatch, full, world, "allreduce").run(_iupac_on_odd_epochs)
