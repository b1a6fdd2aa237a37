"""Builds and drives the kernel emulator (tests/emu/): test infrastructure.

`tests/emu/emu_api.cpp` compiles kindel_b200/csrc/api.cu -- the C ABI with its launch code, and every kernel -- for the
host on top of `tests/emu/cuda_emu.h`, a functional model of the CUDA execution model (fibres per thread, warp
collectives, shared memory, mbarrier / bulk copy / cp.async with late completion).  The helpers below call the
emulated kdl_* entry points with the product's own prototypes (kindel_b200._ffi), host buffers and no stream, so the
kernels run with exactly the grids, order and choices the product launches; the environment knobs KDL_CX and
KDL_SPLIT pin the pileup's choices as they do on the device.  Output buffers sit between guard zones or carry a
poisoned tail, which is checked."""
from __future__ import annotations

import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "emu")
OUT_DIR = os.path.join(EMU_DIR, "_build")
# KDL_EMU_DEFS="-DKDL_W_STAGES=2" builds (and loads) a variant of the emulated kernels next to the default one
EXTRA_DEFS = os.environ.get("KDL_EMU_DEFS", "").split()
LIB = os.path.join(OUT_DIR, "libkdl_emu%s.so" % "".join(c if c.isalnum() else "_" for c in "".join(EXTRA_DEFS)))
CUDA_INCLUDE = os.environ.get("CUDA_INCLUDE", "/usr/local/cuda/include")
# what the emulated sm_count() returns unless a call asks for another: small, so that grid-stride loops stride
SM_COUNT = 2

_lib = None


def available() -> bool:
    return shutil.which("g++") is not None and os.path.exists(os.path.join(CUDA_INCLUDE, "cuda_runtime.h"))


def _sources():
    dirs = [os.path.join(ROOT, "kindel_b200", "csrc"), os.path.join(ROOT, "include"), EMU_DIR]
    return [os.path.join(d, f) for d in dirs for f in os.listdir(d) if os.path.isfile(os.path.join(d, f))]


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in _sources())):
        os.makedirs(OUT_DIR, exist_ok=True)
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-I", CUDA_INCLUDE, "-I", os.path.join(ROOT, "include"),
               *EXTRA_DEFS, os.path.join(EMU_DIR, "emu_api.cpp"), "-o", LIB]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the kernel emulator failed:\n" + res.stdout + res.stderr)
    from kindel_b200 import _ffi

    lib = C.CDLL(LIB)
    for name, (restype, argtypes) in _ffi._PROTOTYPES.items():
        fn = getattr(lib, name, None)  # the entry points that need a real device are not built for the emulator
        if fn is not None:
            fn.restype, fn.argtypes = restype, argtypes
    lib.emu_last_error.restype = C.c_char_p
    lib.emu_set_schedule.argtypes = [C.c_int, C.c_ulonglong]
    lib.emu_set_schedule.restype = None
    lib.emu_set_sm_count.argtypes = [C.c_int]
    lib.emu_set_sm_count.restype = None
    lib.emu_pileup_tile_cx.argtypes = [C.POINTER(_ffi.KdlBatch), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int]
    _lib = lib
    return lib


def _check(rc, what):
    if rc:
        why = _lib.emu_last_error() if rc == 2 else _lib.kdl_status_string(rc)  # 2: KDL_ERR_CUDA, a failed launch
        raise RuntimeError("%s: %s (status %d)" % (what, why.decode(), rc))


def set_schedule(mode: str = "forward", seed: int = 1):
    """Order in which the emulator runs the threads of a block within a scheduler round: "forward", "reverse" or
    "random" (a fresh pseudo-random order every round) -- different interleavings of producers and consumers."""
    load().emu_set_schedule({"forward": 0, "reverse": 1, "random": 2}[mode], seed)


def _sm(n):
    load().emu_set_sm_count(int(n))


def tileable(batch) -> bool:
    """kdl_pileup_range's test for the tile-owner path."""
    from kindel_b200 import _ffi

    return (batch.n_reads > batch.n_hard and int(batch.n_slots) % 512 == 0 and bool(batch.reads_sorted)
            and 0 < int(batch.reach_right) <= _ffi.KDL_FAST_MAXLEN + _ffi.KDL_TILE_MAXREACH)


def _host_batch(batch):
    """(kdl_batch over host arrays with a tile-index scratch, keepalive)."""
    from kindel_b200 import engine

    st, keep = engine.host_struct(batch)
    index = np.zeros(8 * (int(batch.n_slots) // 512) + 8, dtype=np.uint32)
    st.tile_index = index.ctypes.data
    return st, (keep, index)


def _guarded_table(n_slots):
    """(arena, table [19, n_slots] inside it): the table sits between two canary zones."""
    guard = 4096
    arena = np.full(19 * n_slots + 2 * guard, 0x7A7A7A7A, dtype=np.int32)
    return arena, arena[guard:guard + 19 * n_slots].reshape(19, n_slots)


def _assert_guards(arena):
    assert (arena[:4096] == 0x7A7A7A7A).all() and (arena[-4096:] == 0x7A7A7A7A).all(), "write outside the count table"


def run_pileup(batch, fresh: bool = True, slot_range=None, counts: np.ndarray = None, want_events: bool = False,
               zero_rest: bool = False, sm_count: int = SM_COUNT):
    """kdl_pileup_range over `slot_range` = (lo, hi) (multiples of 512; default: the whole table) of `batch` (a
    bamio.ReadBatch) into a table that sits between canary zones.

    fresh: KDL_PILEUP_FRESH_WEIGHTS -- the weight columns of the range hold garbage on entry (and with zero_rest,
    KDL_PILEUP_ZERO_REST, so do columns 5..18); else the kernels add to `counts` (zeros by default).  KDL_CX and
    KDL_SPLIT pick the instantiation and the depth split.  Returns int32 [19, n_slots] (and the event rows)."""
    from kindel_b200 import _ffi

    lib = load()
    _sm(sm_count)
    st, keep = _host_batch(batch)
    n_slots = int(batch.n_slots)
    lo, hi = (0, n_slots) if slot_range is None else (int(slot_range[0]), int(slot_range[1]))
    arena, table = _guarded_table(n_slots)
    if counts is None:
        table[:] = 0
        if fresh:
            table[0:5, lo:hi] = 0x5A5A5A5A
            if zero_rest:
                table[5:, lo:hi] = 0x3B3B3B3B
    else:
        table[:] = counts
    events = np.full((max(int(batch.n_events), 1), 4), -1, dtype=np.int32)
    flag = np.zeros(4, dtype=np.int32)
    flags = (_ffi.KDL_PILEUP_FRESH_WEIGHTS if fresh else 0) | (_ffi.KDL_PILEUP_ZERO_REST if zero_rest else 0)
    _check(lib.kdl_pileup_range(C.byref(st), table.ctypes.data, n_slots, lo, hi, flags, events.ctypes.data,
                                flag.ctypes.data, None), "kdl_pileup_range")
    del keep
    _assert_guards(arena)
    assert not flag[0], "a read raised"
    return (table.copy(), events[: int(batch.n_events)]) if want_events else table.copy()


def tile_cx_pileup(batch, fresh: bool = True, split: int = 1, zero_rest: bool = False, sm_count: int = SM_COUNT):
    """K0 + K1's piece (kCx) instantiation over a batch without tile-eligible complex reads, which no kdl_* entry point
    launches (emu_pileup_tile_cx); the table is prepared as run_pileup prepares it.  Returns int32 [19, n_slots]."""
    lib = load()
    _sm(sm_count)
    assert batch.n_complex == batch.n_hard and tileable(batch)
    st, keep = _host_batch(batch)
    n_slots = int(batch.n_slots)
    arena, table = _guarded_table(n_slots)
    table[:] = 0
    if fresh and split == 1:
        table[0:5] = 0x5A5A5A5A
        if zero_rest:
            table[5:] = 0x3B3B3B3B
    _check(lib.emu_pileup_tile_cx(C.byref(st), table.ctypes.data, n_slots, int(fresh), int(split), int(zero_rest)),
           "emu_pileup_tile_cx")
    del keep
    _assert_guards(arena)
    return table.copy()


def pileup_pipeline(batch, sm_count: int = SM_COUNT):
    """kdl_pileup into a zeroed table, and on a raised error flag kdl_diagnose, as engine.pileup does.  Returns
    (counts [19, n_slots], events [n_events, 4]) or raises IndexError / KeyError(base) exactly like
    kindel_b200.engine.pileup."""
    from kindel_b200 import _ffi, engine

    lib = load()
    _sm(sm_count)
    st, keep = _host_batch(batch)
    n_slots = int(batch.n_slots)
    arena, counts = _guarded_table(n_slots)
    counts[:] = 0
    events = np.zeros((max(int(batch.n_events), 1), 4), dtype=np.int32)
    flag = np.zeros(4, dtype=np.int32)
    _check(lib.kdl_pileup(C.byref(st), counts.ctypes.data, n_slots, events.ctypes.data, flag.ctypes.data, None),
           "kdl_pileup")
    _assert_guards(arena)
    if flag[0]:
        diag = _ffi.KdlDiag()
        _check(lib.kdl_diagnose(C.byref(st), C.addressof(diag), None), "kdl_diagnose")
        assert diag.status, "error flag raised but no offending read found"
        engine.raise_like_reference(diag.status, diag.read, diag.nibble, diag.op_index)
    del keep
    return counts.copy(), events[: int(batch.n_events)]


def dirty_map_words(n_slots: int) -> int:
    """uint32 words of a table's dirty-sector map: one 16-byte record per 64-slot window."""
    return 4 * ((int(n_slots) + 63) // 64)


def fresh_pileup(batch, counts: np.ndarray, dirty_map, zero_rest: bool, slot_range=None, sm_count: int = SM_COUNT):
    """kdl_pileup_range_map with KDL_PILEUP_FRESH_WEIGHTS (| KDL_PILEUP_ZERO_REST when zero_rest) over the slot range
    `slot_range` = (lo, hi) (multiples of 4, of 512 for the tile kernel; default: the whole table): `counts` (int32
    [19, n_slots]) is a reused table -- weight columns stale, columns 5..18 as the previous pileup left them -- and
    `dirty_map` (uint32 [dirty_map_words], or None = zero all of columns 5..18) its map; both are updated in place.
    Returns the event rows; raises if a read raised."""
    from kindel_b200 import _ffi

    lib = load()
    _sm(sm_count)
    st, keep = _host_batch(batch)
    n_slots = int(batch.n_slots)
    assert counts.dtype == np.int32 and counts.shape == (19, n_slots) and counts.flags.c_contiguous
    assert dirty_map is None or (dirty_map.dtype == np.uint32 and dirty_map.size == dirty_map_words(n_slots))
    events = np.full((max(int(batch.n_events), 1), 4), -1, dtype=np.int32)
    flag = np.zeros(4, dtype=np.int32)
    lo, hi = (0, n_slots) if slot_range is None else (int(slot_range[0]), int(slot_range[1]))
    flags = _ffi.KDL_PILEUP_FRESH_WEIGHTS | (_ffi.KDL_PILEUP_ZERO_REST if zero_rest else 0)
    _check(lib.kdl_pileup_range_map(C.byref(st), counts.ctypes.data, n_slots, lo, hi, flags,
                                    None if dirty_map is None else dirty_map.ctypes.data, events.ctypes.data,
                                    flag.ctypes.data, None), "kdl_pileup_range_map")
    del keep
    assert not flag[0], "a read raised"
    return events[: int(batch.n_events)]


def unmask(batch, counts):
    """K1q (kdl_unmask) over a host count table (in place): takes back the counts of the batch's masked bases."""
    from kindel_b200 import engine

    lib = load()
    st, keep = engine.host_struct(batch)
    qm, qkeep = engine.host_qmask(batch)
    if qm is not None:
        _check(lib.kdl_unmask(C.byref(st), C.byref(qm), counts.ctypes.data, int(batch.n_slots), None), "kdl_unmask")
    del keep, qkeep
    return counts


def vote(counts: np.ndarray, min_depth=1) -> np.ndarray:
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    calls = np.zeros(counts.shape[1], dtype=np.uint8)
    _check(lib.kdl_vote(counts.ctypes.data, counts.shape[1], int(math.ceil(min_depth)), calls.ctypes.data, None),
           "kdl_vote")
    return calls


def vote_iupac(counts: np.ndarray, min_depth, threshold) -> np.ndarray:
    """K2 with the IUPAC vote (kdl_vote_iupac) over a host table."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    calls = np.zeros(counts.shape[1], dtype=np.uint8)
    _check(lib.kdl_vote_iupac(counts.ctypes.data, counts.shape[1], int(math.ceil(min_depth)), float(threshold),
                              calls.ctypes.data, None), "kdl_vote_iupac")
    return calls


def derive(counts: np.ndarray) -> np.ndarray:
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    out = np.zeros((5, counts.shape[1]), dtype=np.int32)
    _check(lib.kdl_derive(counts.ctypes.data, counts.shape[1], out.ctypes.data, None), "kdl_derive")
    return out


def vote_peers(tables, feet, slot_lo, slot_hi, min_depth=1, want_reduced=False):
    """K2p (kdl_vote_peers_sparse) over host tables: vote of the SUM of `tables` on [slot_lo, slot_hi); feet =
    [(lo, hi)] or None."""
    lib = load()
    n = len(tables)
    n_slots = tables[0].shape[1]
    ptrs = (C.c_void_p * n)(*[t.ctypes.data for t in tables])
    lo = (C.c_int64 * n)(*[f[0] for f in feet]) if feet else None
    hi = (C.c_int64 * n)(*[f[1] for f in feet]) if feet else None
    calls = np.zeros(n_slots, dtype=np.uint8)
    reduced = np.zeros((7, n_slots), dtype=np.int32) if want_reduced else None
    _check(lib.kdl_vote_peers_sparse(ptrs, lo, hi, n, n_slots, slot_lo, slot_hi, int(math.ceil(min_depth)),
                                     calls.ctypes.data, reduced.ctypes.data if want_reduced else None, None),
           "kdl_vote_peers_sparse")
    return (calls, reduced) if want_reduced else calls


def _exchange(tables, feet, slices, calls, flags, epoch, vote_one, sm_count):
    """One epoch of the fused multi-GPU exchange with the ranks' buffers in host memory: kdl_exchange_signal of every
    rank, then vote_one(exchange, rank) (K2x) of every rank, then kdl_exchange_wait (K2g) of every rank.  A kernel
    runs to completion here, so every ready flag has to be up before the first K2x waits for them."""
    from kindel_b200 import _ffi

    lib = load()
    _sm(sm_count)
    n = len(tables)
    xs = (_ffi.KdlExchange * n)()
    for r in range(n):
        x = xs[r]
        x.n_ranks, x.rank = n, r
        for p in range(n):
            x.tables[p] = tables[p].ctypes.data
            x.calls[p] = calls[p].ctypes.data
            x.ready[p] = flags["ready"][p].ctypes.data
            x.done[p] = flags["done"][p].ctypes.data
            x.foot_lo[p], x.foot_hi[p] = feet[p]
            x.slice_lo[p], x.slice_hi[p] = slices[p]
        x.counter = flags["counter"][r].ctypes.data
    for r in range(n):
        _check(lib.kdl_exchange_signal(C.byref(xs[r]), epoch, None), "kdl_exchange_signal")
    for r in range(n):
        _check(vote_one(C.byref(xs[r])), "K2x")
    for r in range(n):
        _check(lib.kdl_exchange_wait(C.byref(xs[r]), epoch, None), "kdl_exchange_wait")


def exchange_epoch(tables, feet, slices, calls, flags, epoch, min_depth=1, sm_count: int = SM_COUNT):
    """One epoch of the fused exchange (kdl_exchange_vote).  tables[r]: int32 [19, n_slots]; calls[r]: uint8 [n_slots];
    flags: dict of per-rank int32 arrays 'ready', 'done' (16 each) and 'counter' (1), persistent across epochs."""
    lib = load()
    n_slots, md = tables[0].shape[1], int(math.ceil(min_depth))
    _exchange(tables, feet, slices, calls, flags, epoch,
              lambda x: lib.kdl_exchange_vote(x, n_slots, md, epoch, None), sm_count)


def exchange_epoch_iupac(tables, feet, slices, calls, flags, epoch, threshold, min_depth=1, sm_count: int = SM_COUNT):
    """One epoch of the fused exchange with the IUPAC vote (kdl_exchange_vote_iupac); arguments as exchange_epoch."""
    lib = load()
    n_slots, md = tables[0].shape[1], int(math.ceil(min_depth))
    _exchange(tables, feet, slices, calls, flags, epoch,
              lambda x: lib.kdl_exchange_vote_iupac(x, n_slots, md, float(threshold), epoch, None), sm_count)


def cdr_flags(counts: np.ndarray, slot_lo: int, slot_hi: int, decay: float):
    """K4 (kdl_cdr_flags) over a host table: (flags, bases) uint8 of slots [slot_lo, slot_hi), like engine.cdr_flags.
    Slots outside the range keep the canary 0xEE, which is checked."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    n = counts.shape[1]
    flags = np.full(n, 0xEE, dtype=np.uint8)
    bases = np.full(n, 0xEE, dtype=np.uint8)
    _check(lib.kdl_cdr_flags(counts.ctypes.data, n, int(slot_lo), int(slot_hi), float(decay), flags.ctypes.data,
                             bases.ctypes.data, None), "kdl_cdr_flags")
    assert (flags[:slot_lo] == 0xEE).all() and (flags[slot_hi:] == 0xEE).all(), "K4 wrote outside its slot range"
    assert (bases[:slot_lo] == 0xEE).all() and (bases[slot_hi:] == 0xEE).all(), "K4 wrote outside its slot range"
    return flags[slot_lo:slot_hi].copy(), bases[slot_lo:slot_hi].copy()


def _assemble(calls, batch, ins_slots, ins_strings):
    """kdl_assemble over host buffers: (offsets, text buffer, keepalive)."""
    lib = load()
    calls = np.ascontiguousarray(calls, dtype=np.uint8)
    n_slots = calls.shape[0]
    enc = [x.encode("ascii") for x in ins_strings]
    ins_off = np.zeros(len(enc) + 1, dtype=np.uint32)
    if enc:
        ins_off[1:] = np.cumsum([len(x) for x in enc])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8).copy()
    slots = np.ascontiguousarray(ins_slots if len(enc) else np.zeros(1), dtype=np.int64)
    c_slot = np.ascontiguousarray(batch.contig_slot, dtype=np.int64)
    c_len = np.ascontiguousarray(batch.contig_len, dtype=np.int32)
    sums = np.zeros(int(lib.kdl_assemble_scratch_words(n_slots)), dtype=np.uint32)
    offsets = np.zeros(n_slots + 1, dtype=np.uint32)
    out = np.zeros(n_slots + int(ins_off[-1]) + 16, dtype=np.uint8)
    _check(lib.kdl_assemble(calls.ctypes.data, n_slots, c_slot.ctypes.data, c_len.ctypes.data, len(c_len),
                            slots.ctypes.data, ins_off.ctypes.data, blob.ctypes.data, len(enc), sums.ctypes.data,
                            offsets.ctypes.data, out.ctypes.data, None), "kdl_assemble")
    spans = [(int(offsets[s]), int(offsets[s + L])) for s, L in zip(c_slot.tolist(), c_len.tolist())]
    return offsets, out, spans, (slots, len(enc))


def assemble(calls: np.ndarray, batch, ins_slots, ins_strings):
    """K5 (kdl_assemble) over host call bytes: the consensus text of every contig, like engine.assemble."""
    offsets, out, spans, _ = _assemble(calls, batch, ins_slots, ins_strings)
    text = out[: int(offsets[-1])].tobytes()
    return [text[a:b].decode("ascii") for a, b in spans]


def consensus_qual(counts: np.ndarray, calls: np.ndarray) -> np.ndarray:
    """K2q (kdl_consensus_qual) over a host table and its call bytes."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    calls = np.ascontiguousarray(calls, dtype=np.uint8)
    qual = np.full(counts.shape[1], 0xEE, dtype=np.uint8)
    _check(lib.kdl_consensus_qual(counts.ctypes.data, calls.ctypes.data, counts.shape[1], qual.ctypes.data, None),
           "kdl_consensus_qual")
    return qual


def assemble_qual(calls, qual, batch, ins_slots, ins_strings, ins_qual):
    """K5 + K5q (kdl_assemble, then kdl_assemble_qual on its offsets) over host buffers: (texts, quality texts), one
    per contig, like engine.assemble(..., qual=...)."""
    lib = load()
    offsets, out, spans, (slots, n_ins) = _assemble(calls, batch, ins_slots, ins_strings)
    qual = np.ascontiguousarray(qual, dtype=np.uint8)
    iq = np.ascontiguousarray(ins_qual if n_ins else np.zeros(1), dtype=np.uint8)
    qout = np.full(out.size, 0xEE, dtype=np.uint8)
    _check(lib.kdl_assemble_qual(offsets.ctypes.data, qual.ctypes.data, qual.shape[0], slots.ctypes.data,
                                 iq.ctypes.data, n_ins, qout.ctypes.data, None), "kdl_assemble_qual")
    total = int(offsets[-1])
    assert (qout[total:] == 0xEE).all(), "K5q wrote past the text"
    text, qtext = out[:total].tobytes(), qout[:total].tobytes()
    return [text[a:b].decode("ascii") for a, b in spans], [qtext[a:b].decode("latin-1") for a, b in spans]


def variant_sites(counts, contig_slot, contig_len, abs_floor, rel_threshold):
    """K6 (kdl_variant_count, a read of the total, kdl_variant_scatter) over a host table: (slot int64[n], counts
    int32[6, n], mask uint8[n]) like engine.variant_sites.  abs_floor is the clamped integer threshold
    (engine.variant_abs_floor)."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    n_slots = counts.shape[1]
    c_slot = np.ascontiguousarray(contig_slot, dtype=np.int64)
    c_len = np.ascontiguousarray(contig_len, dtype=np.int32)
    sums = np.full(int(lib.kdl_variant_scratch_words(n_slots)), 0xDEADBEEF, dtype=np.uint32)
    args = (counts.ctypes.data, n_slots, c_slot.ctypes.data, c_len.ctypes.data, len(c_len), int(abs_floor),
            float(rel_threshold))
    _check(lib.kdl_variant_count(*args, sums.ctypes.data, None), "kdl_variant_count")
    n = int(sums[-1])
    # one record more than announced, poisoned: the scatter must write exactly n and leave the rest alone
    slot = np.full(n + 1, -7, dtype=np.int64)
    mask = np.full(n + 1, 0xEE, dtype=np.uint8)
    flat = np.full(6 * n + 1, -7, dtype=np.int32)
    _check(lib.kdl_variant_scatter(*args, sums.ctypes.data, n, slot.ctypes.data, flat.ctypes.data, mask.ctypes.data,
                                   None), "kdl_variant_scatter")
    assert slot[n] == -7 and mask[n] == 0xEE and flat[6 * n] == -7, "K6 wrote past the announced sites"
    return slot[:n], flat[:6 * n].reshape(6, n).copy(), mask[:n]


def variant_sites_ref(counts, contig_slot, contig_len, ref_codes, abs_floor, rel_threshold):
    """K6r (kdl_variant_ref_count, a read of the total, kdl_variant_ref_scatter) over a host table: (slot int64[n],
    counts int32[7, n], dpa int64[n], mask uint8[n]) like engine.variant_sites_ref.  abs_floor is the clamped integer
    threshold (engine.variant_abs_floor)."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    n_slots = counts.shape[1]
    c_slot = np.ascontiguousarray(contig_slot, dtype=np.int64)
    c_len = np.ascontiguousarray(contig_len, dtype=np.int32)
    ref = np.ascontiguousarray(ref_codes, dtype=np.uint8)
    assert ref.shape == (n_slots,)
    sums = np.full(int(lib.kdl_variant_scratch_words(n_slots)), 0xDEADBEEF, dtype=np.uint32)
    args = (counts.ctypes.data, n_slots, c_slot.ctypes.data, c_len.ctypes.data, len(c_len), ref.ctypes.data,
            int(abs_floor), float(rel_threshold))
    _check(lib.kdl_variant_ref_count(*args, sums.ctypes.data, None), "kdl_variant_ref_count")
    n = int(sums[-1])
    # one record more than announced, poisoned: the scatter must write exactly n and leave the rest alone
    slot = np.full(n + 1, -7, dtype=np.int64)
    dpa = np.full(n + 1, -7, dtype=np.int64)
    mask = np.full(n + 1, 0xEE, dtype=np.uint8)
    flat = np.full(7 * n + 1, -7, dtype=np.int32)
    _check(lib.kdl_variant_ref_scatter(*args, sums.ctypes.data, n, slot.ctypes.data, flat.ctypes.data, dpa.ctypes.data,
                                       mask.ctypes.data, None), "kdl_variant_ref_scatter")
    assert slot[n] == -7 and dpa[n] == -7 and mask[n] == 0xEE and flat[7 * n] == -7, "K6r wrote past the sites"
    return slot[:n], flat[:7 * n].reshape(7, n).copy(), dpa[:n], mask[:n]


def deletion_events(batch):
    """K7 (kdl_deletion_count, a read of the total, kdl_deletion_scatter) over a host ReadBatch: (slot int64[m],
    length int32[m]) in read order, then op order."""
    from kindel_b200 import engine

    lib = load()
    struct, keep = engine.host_struct(batch)
    sums = np.full(int(lib.kdl_deletion_scratch_words(batch.n_reads)), 0xDEADBEEF, dtype=np.uint32)
    _check(lib.kdl_deletion_count(C.byref(struct), sums.ctypes.data, None), "kdl_deletion_count")
    m = int(sums[-1])
    slot = np.full(m + 1, -7, dtype=np.int64)
    length = np.full(m + 1, -7, dtype=np.int32)
    _check(lib.kdl_deletion_scatter(C.byref(struct), sums.ctypes.data, m, slot.ctypes.data, length.ctypes.data, None),
           "kdl_deletion_scatter")
    assert slot[m] == -7 and length[m] == -7, "K7 wrote past the events"
    del keep
    return slot[:m], length[:m]


def select(batch, keep):
    """K8 (kdl_select_count, one read of the totals record, kdl_select_scatter) over a host ReadBatch and keep bytes
    -> the fields of the sub-batch (see strand_cases.fields)."""
    from kindel_b200 import _ffi, engine

    lib = load()
    keep = np.ascontiguousarray(keep, dtype=np.uint8)
    struct, hold = engine.host_struct(batch)
    qmask, qhold = engine.host_qmask(batch)
    qp = C.byref(qmask) if qmask is not None else None
    scratch = np.full(int(lib.kdl_select_scratch_words(batch.n_reads)), 0xDEADBEEF, dtype=np.uint32)
    _check(lib.kdl_select_count(C.byref(struct), qp, keep.ctypes.data, scratch.ctypes.data, None), "kdl_select_count")
    tot = scratch[-16:].astype(np.int64)
    n, n_words, n_cx, n_hard, n_evt, n_mr, n_mb = (int(x) for x in tot[:7])
    # one element more than announced, poisoned: the scatter must write exactly the announced ones
    out = dict(ref_start=np.full(n + 1, -7, np.int32), seq_off=np.full(n + 1, 7, np.uint32),
               l_seq=np.full(n + 1, -7, np.int32), seq4=np.full(n_words + 1, 7, np.uint32),
               contig_read_off=np.full(batch.n_contigs + 2, -7, np.int64), complex_idx=np.full(n_cx + 1, 7, np.uint32),
               hard_idx=np.full(n_hard + 1, 7, np.uint32), mask_read=np.full(n_mr + 1, 7, np.uint32),
               mask_off=np.full(n_mr + 2, 7, np.uint32), mask_qpos=np.full(n_mb + 1, 7, np.uint32))
    o = _ffi.KdlBatch()
    o.n_reads, o.seq4_words, o.n_contigs = n, n_words, batch.n_contigs
    o.reads_sorted, o.max_simple_len, o.reach_right, o.reach_left = (int(x) for x in tot[7:11])
    o.n_complex, o.n_hard = n_cx, n_hard
    for f in ("ref_start", "seq_off", "l_seq", "seq4", "contig_read_off", "complex_idx", "hard_idx"):
        setattr(o, f, out[f].ctypes.data)
    o.contig_len, o.contig_slot = struct.contig_len, struct.contig_slot
    om = None
    if n_mr:
        om = _ffi.KdlQmask()
        om.n_reads, om.n_bases = n_mr, n_mb
        om.read_idx, om.off, om.qpos = out["mask_read"].ctypes.data, out["mask_off"].ctypes.data, out["mask_qpos"].ctypes.data
    _check(lib.kdl_select_scatter(C.byref(struct), qp, keep.ctypes.data, scratch.ctypes.data, C.byref(o),
                                  C.byref(om) if om is not None else None, None), "kdl_select_scatter")
    sizes = dict(ref_start=n, seq_off=n, l_seq=n, seq4=n_words, contig_read_off=batch.n_contigs + 1, complex_idx=n_cx,
                 hard_idx=n_hard, mask_read=n_mr, mask_off=n_mr + 1 if n_mr else 0, mask_qpos=n_mb)
    for f, k in sizes.items():
        a = out[f]
        assert np.all(a[k:] == a[-1]) and a[-1] in (7, -7), "K8 wrote past %s" % f
    del hold, qhold
    got = {f: out[f][:k] for f, k in sizes.items()}
    got.update(n_events=n_evt, reads_sorted=bool(tot[7]), max_simple_len=int(tot[8]), reach_right=int(tot[9]),
               reach_left=int(tot[10]))
    if not n_mr:
        got.update(mask_read=None, mask_off=None, mask_qpos=None)
    return got
