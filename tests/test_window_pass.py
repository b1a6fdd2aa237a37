"""K1w, the complex-read window pass (kindel_b200/csrc/pileup_general.cu), at its window edges, on the CPU under the
kernel emulator: every update of a tile-eligible complex read is counted by the CTA whose window of CW_SLOTS slots
holds it, so a read that straddles an edge, reaches three windows or shares a window with other contigs must come out
exactly as the C oracle piles it -- with one CTA per window and with windows shared by `split` CTAs, over the whole
table and over a slot range, and into a reused table whose dirty-sector map an earlier pileup left.  K1w runs behind
K1's lean instantiation (KDL_CX=atomics); the same cases behind the piece instantiation (K1e) are the control."""
from __future__ import annotations

import numpy as np
import pytest

import emu_harness as E
from limit_cases import _Group
from oracle import coracle

from kindel_b200 import bamio

pytestmark = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")

W = 1024  # CW_SLOTS


def _edges_group():
    g = _Group("windows")
    c = g.contig(6000)
    g.background(c, 6000, step=97)
    for e in (W, 2 * W, 4 * W):                      # the reads below sit on window edges e
        g.read(c, e - 20, "10M10D30M", "t")          # deletion up to the slot before the edge, bases across it
        g.read(c, e - 10, "5M20D25M", "t")           # deletion across the edge
        g.read(c, e - 24, "24M2I30M", "t")           # insertion on the edge's first slot
        g.read(c, e - 25, "24M2I30M", "t")           # ... and on the slot before it
        g.read(c, e + 10, "40S60M", "t")             # leading clip reaching back across the edge
        g.read(c, e, "1S60M", "t")                   # leading clip on the slot before the edge
        g.read(c, e - 40, "40M30S", "t")             # trailing clip starting on the edge
        g.read(c, e - 41, "40M30S", "t")             # clip_starts on the slot before the edge
    g.read(c, W + 40, "1000S10M1003D10M", "t")       # reach 1024 to the right from a start in window 1, clip bases
    #                                                  from window 0: three windows
    g.read(c, 2 * W - 1, "2S10M3I1003D7M", "t")
    for L in (300, 200, 400, 90):                    # four contigs inside one window, complex reads on each
        d = g.contig(L)
        g.read(d, 5, "3S20M2D20M4S", "t")
        g.read(d, L - 60, "10M1I20M5D10M2S", "t")
    return g


def _batch(g, tmp_path):
    p = tmp_path / ("%s.sam" % g.name)
    p.write_text(g.sam())
    b = bamio.read_sam(str(p))
    assert b.reads_sorted and (b.n_complex > b.n_hard or g.name == "simple")
    return b


@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("cx", ["atomics", "pieces"])
def test_window_edges(cx, split, tmp_path, monkeypatch):
    """Reads on and across window edges, a read reaching three windows, several contigs in one window, windows
    without complex reads; added to a table and into a fresh one."""
    monkeypatch.setenv("KDL_CX", cx)
    monkeypatch.setenv("KDL_SPLIT", str(split))
    b = _batch(_edges_group(), tmp_path)
    want_c, want_e = coracle.pileup(b)
    for fresh in (False, True):
        got, ev = E.run_pileup(b, fresh, want_events=True, zero_rest=fresh)
        np.testing.assert_array_equal(got, want_c)
        np.testing.assert_array_equal(ev, want_e)


@pytest.mark.parametrize("cx", ["atomics", "pieces"])
def test_slot_range(cx, tmp_path, monkeypatch):
    """A batch whose reads lie in [2 * 512, 11 * 512): the range call's windows start at slot 512, not 0."""
    monkeypatch.setenv("KDL_CX", cx)
    monkeypatch.setenv("KDL_SPLIT", "1")
    g = _Group("ranged")
    c = g.contig(8000)
    g.background(c, 5500, step=41, lo=1600)
    for p in (1530, 1600, 2040, 2550, 3060, 4090, 5100):
        g.read(c, p, "30S50M4D20M3I20M", "t")
    b = _batch(g, tmp_path)
    want_c, want_e = coracle.pileup(b)
    assert not want_c[:, :512].any() and not want_c[:, 11 * 512:].any()
    got, ev = E.run_pileup(b, True, slot_range=(512, 11 * 512), want_events=True)
    np.testing.assert_array_equal(got[:, 512: 11 * 512], want_c[:, 512: 11 * 512])
    np.testing.assert_array_equal(ev, want_e)


@pytest.mark.parametrize("cx", ["atomics", "pieces"])
def test_reused_table_after_dense(cx, tmp_path, monkeypatch):
    """A dense-complex pileup leaves the map saturated; the sparse one after it zeroes what the map marks, and K1w's
    flush marks the sectors of columns 5 and 6 it changed (and the clip updates theirs), so a third pileup of a batch
    without complex reads clears everything again."""
    monkeypatch.setenv("KDL_CX", cx)
    monkeypatch.setenv("KDL_SPLIT", "1")
    dense = _Group("dense")
    c = dense.contig(6000)
    for p in range(40, 5800, 37):
        dense.read(c, p, "5S40M2D40M1I30M", "t")
    sparse = _edges_group()
    simple = _Group("simple")
    for L in (6000, 300, 200, 400, 90):
        simple.contig(L, "windows_%d" % len(simple.contigs))
    dense.contigs = list(sparse.contigs)  # one layout for the three batches: reads on every contig
    dense.reads = [("windows_0",) + r[1:] for r in dense.reads]
    for name, L in simple.contigs:
        simple.background(name, L, step=53, read_len=50)
        dense.read(name, 10, "2S30M1D10M", "t")
    batches = [_batch(g, tmp_path) for g in (dense, sparse, simple)]
    n_slots = int(batches[0].n_slots)
    assert all(int(x.n_slots) == n_slots for x in batches)
    table = np.zeros((19, n_slots), dtype=np.int32)
    dmap = np.zeros(E.dirty_map_words(n_slots), dtype=np.uint32)
    prev = False
    for b in batches:
        want_c, want_e = coracle.pileup(b)
        ev = E.fresh_pileup(b, table, dmap, zero_rest=prev)
        np.testing.assert_array_equal(table, want_c)
        np.testing.assert_array_equal(ev, want_e)
        bits = np.unpackbits(dmap.view(np.uint8).reshape(-1, 16)[:, :14], axis=1, bitorder="little")
        bits = bits.reshape(-1, 14, 8).transpose(1, 0, 2).reshape(14, -1)  # [column 5.., sector]
        sect = table[5:, : bits.shape[1] * 8].reshape(14, -1, 8).any(axis=2)
        assert not (sect & ~bits[:, : sect.shape[1]].astype(bool)).any(), "a changed sector without its bit"
        prev = b.n_complex > 0
    assert not dmap.any()
