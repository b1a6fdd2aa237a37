"""Per-amplicon reads and depth (`kindel amplicons`, an extension) -- test infrastructure: named schemes, K12 and K12d
under the kernel emulator."""
from __future__ import annotations

import ctypes as C

import numpy as np

import emu_harness as E
from kindel_b200 import engine
from kindel_b200 import primers as P


def bed_text(rows, pools=True):
    """A named BED of rows (chrom, start, end, amplicon, side): primer names `<amplicon>_LEFT` / `_RIGHT` (an `_altN`
    suffix on repeats), column 5 the pool when `pools`."""
    seen, lines = {}, []
    for c, a, b, amp, side in rows:
        key = (c, amp, side)
        k = seen.get(key, -1) + 1
        seen[key] = k
        name = "%s_%s%s" % (amp, "LEFT" if side == "L" else "RIGHT", "_alt%d" % k if k else "")
        lines.append("%s\t%d\t%d\t%s" % (c, a, b, name) + ("\t%s\t%s" % (amp, "+-"[side == "R"]) if pools else ""))
    return "\n".join(lines) + "\n"


def scheme(rows, name="scheme.bed"):
    return P.read_scheme(bed_text(rows).encode(), name)


def random_scheme_rows(rng, contigs, n_max=6):
    """Random amplicons on contigs [(name, L)]: 1-2 left and 1-2 right primers each, overlapping other amplicons'
    primers now and then (ambiguous segments), at the contig's start and end included; plus an amplicon of a contig
    the alignment does not have."""
    rows = []
    for name, L in contigs:
        if L < 12:
            continue
        for k in range(int(rng.integers(0, n_max + 1))):
            a = int(rng.integers(0, L - 10))
            b = int(rng.integers(a + 10, min(L, a + 400) + 1))
            amp = "%s_a%d" % (name, k)
            for _ in range(int(rng.integers(1, 3))):
                x = int(rng.integers(a, a + 3))
                rows.append((name, x, x + int(rng.integers(1, 5)), amp, "L"))
            for _ in range(int(rng.integers(1, 3))):
                y = int(rng.integers(b - 2, b + 1))
                rows.append((name, y - int(rng.integers(1, 5)), y, amp, "R"))
    rows.append(("elsewhere", 0, 5, "far", "L"))
    rows.append(("elsewhere", 10, 15, "far", "R"))
    # keep amplicons with an insert only
    ok = []
    for amp in sorted({r[3] for r in rows}):
        mine = [r for r in rows if r[3] == amp]
        if max(r[2] for r in mine if r[4] == "L") < min(r[1] for r in mine if r[4] == "R"):
            ok += mine
    return ok


def emu_assign(batch, arrays):
    """K12 (kdl_amplicons_assign) under the emulator: int32 labels, with a poisoned element past the end checked."""
    lib = E.load()
    struct, hold = engine.host_struct(batch)
    keep = {f: np.ascontiguousarray(getattr(arrays, f)) for f in engine._AMPLICON_FIELDS}
    a = engine.amplicons_struct(arrays, {f: (x.ctypes.data if x.size else None) for f, x in keep.items()})
    out = np.full(batch.n_reads + 1, 0x7777, dtype=np.int32)
    E._check(lib.kdl_amplicons_assign(C.byref(struct), C.byref(a), out.ctypes.data, None), "kdl_amplicons_assign")
    assert out[-1] == 0x7777, "K12 wrote past the labels"
    del hold, keep
    return out[:-1]


def emu_depth(counts, batch, arrays, min_depth):
    """K12d (kdl_amplicons_depth) under the emulator over a host table: int64 [n_amplicons, 3]."""
    lib = E.load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    keep = {f: np.ascontiguousarray(getattr(arrays, f)) for f in engine._AMPLICON_FIELDS}
    a = engine.amplicons_struct(arrays, {f: (x.ctypes.data if x.size else None) for f, x in keep.items()})
    slot = np.ascontiguousarray(batch.contig_slot, dtype=np.int64)
    length = np.ascontiguousarray(batch.contig_len, dtype=np.int32)
    out = np.full(3 * arrays.n_amplicons + 1, -7, dtype=np.int64)
    E._check(lib.kdl_amplicons_depth(counts.ctypes.data, counts.shape[1], slot.ctypes.data, length.ctypes.data,
                                     len(length), C.byref(a), int(min_depth), out.ctypes.data, None),
             "kdl_amplicons_depth")
    assert out[-1] == -7, "K12d wrote past the stats"
    del keep
    return out[:-1].reshape(-1, 3)


def tiled_rows(rows):
    """synth.tiled_scheme's rows as (chrom, start, end, amplicon, side), named as synth.named_scheme_bed names them."""
    out, k_of = [], {}
    for i in range(0, len(rows), 2):
        (c, a, b), (_, x, y) = rows[i], rows[i + 1]
        k = k_of.get(c, 0)
        k_of[c] = k + 1
        out += [(c, a, b, "amp_%d" % k, "L"), (c, x, y, "amp_%d" % k, "R")]
    return out
