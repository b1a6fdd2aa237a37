"""Builds and drives the emulated pileup with a dirty-sector map (tests/emu/emu_map.cpp): test infrastructure.

The kernel sources are compiled for the host on top of tests/emu/cuda_emu.h, as tests/emu_harness.py does for the
pileup without a map, into a library of its own.  `fresh_pileup` runs what kdl_pileup_range_map launches for a reused
table: the table and its map are updated in place."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from emu_harness import CUDA_INCLUDE, EMU_DIR, OUT_DIR, ROOT, available  # noqa: F401  (available: re-exported)

LIB = os.path.join(OUT_DIR, "libkdl_emu_map.so")

_lib = None


def _sources():
    csrc = os.path.join(ROOT, "kindel_b200", "csrc")
    return [os.path.join(EMU_DIR, "cuda_emu.h"), os.path.join(EMU_DIR, "emu_map.cpp"),
            os.path.join(csrc, "kdl_common.cuh"), os.path.join(csrc, "tile_common.cuh"), os.path.join(csrc, "pileup_tile.cu"),
            os.path.join(csrc, "pileup_general.cu"), os.path.join(csrc, "pileup_simple.cu"),
            os.path.join(ROOT, "include", "kindel_b200.h")]


def load():
    global _lib
    if _lib is not None:
        return _lib
    src = _sources()
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in src)):
        os.makedirs(OUT_DIR, exist_ok=True)
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-I", CUDA_INCLUDE, "-I", os.path.join(ROOT, "include"),
               os.path.join(EMU_DIR, "emu_map.cpp"), "-o", LIB]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the dirty-map emulator failed:\n" + res.stdout + res.stderr)
    from kindel_b200 import _ffi

    lib = C.CDLL(LIB)
    lib.emu_map_last_error.restype = C.c_char_p
    lib.emu_map_pileup.restype = C.c_int
    vp = C.c_void_p
    ll = C.c_longlong
    lib.emu_map_pileup.argtypes = [C.POINTER(_ffi.KdlBatch), vp, ll, ll, ll, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp,
                                   C.c_int]
    _lib = lib
    return lib


def dirty_map_words(n_slots: int) -> int:
    """uint32 words of a table's dirty-sector map: one 16-byte record per 64-slot window."""
    return 4 * ((int(n_slots) + 63) // 64)


def fresh_pileup(batch, counts: np.ndarray, dirty_map, zero_rest: bool, split: int = 1, cx: bool = None,
                 grid: int = 3, slot_range=None):
    """What kdl_pileup_range_map does with KDL_PILEUP_FRESH_WEIGHTS (| KDL_PILEUP_ZERO_REST when zero_rest) over the
    slot range `slot_range` = (lo, hi) (multiples of 4, of 512 for the tile kernel; default: the whole table):
    `counts` (int32 [19, n_slots]) is a reused table -- weight columns stale, columns 5..18 as the previous pileup
    left them -- and `dirty_map` (uint32 [dirty_map_words], or None = zero all of columns 5..18) its
    map; both are updated in place.  split > 1: the depth split.  cx: which K1 instantiation (default: the piece one
    when the batch has tile-eligible complex reads).  Returns the event rows; raises if a read raised."""
    from kindel_b200 import engine

    lib = load()
    st, keep = engine.host_struct(batch)
    n_slots = int(batch.n_slots)
    assert counts.dtype == np.int32 and counts.shape == (19, n_slots) and counts.flags.c_contiguous
    assert dirty_map is None or (dirty_map.dtype == np.uint32 and dirty_map.size == dirty_map_words(n_slots))
    if cx is None:
        cx = batch.n_complex > batch.n_hard
    index = np.zeros(8 * (n_slots // 512) + 8, dtype=np.uint32)
    events = np.full((max(int(batch.n_events), 1), 4), -1, dtype=np.int32)
    flag = np.zeros(4, dtype=np.int32)
    lo, hi = (0, n_slots) if slot_range is None else (int(slot_range[0]), int(slot_range[1]))
    rc = lib.emu_map_pileup(C.byref(st), counts.ctypes.data, n_slots, lo, hi, index.ctypes.data,
                            None if dirty_map is None else dirty_map.ctypes.data, 1 if zero_rest else 0, split,
                            1 if cx else 0, events.ctypes.data, flag.ctypes.data, grid)
    del keep
    if rc:
        raise RuntimeError(lib.emu_map_last_error().decode())
    assert not flag[0], "a read raised"
    return events[: int(batch.n_events)]
