"""Builds and drives the emulated IUPAC vote and K5 (tests/emu/emu_iupac.cpp): test infrastructure.

The sources of kindel_b200/csrc/vote.cu and assemble.cu are compiled for the host on top of tests/emu/cuda_emu.h, as
tests/emu_harness.py does for the other kernels, into a library of its own.  `vote_iupac` is K2 with the IUPAC vote,
`exchange_epoch` one epoch of K2x (IUPAC) + K2g for every rank, `assemble` the consensus text K5 writes, `cdr_flags` the --realign predicates of K4."""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np

from emu_harness import CUDA_INCLUDE, EMU_DIR, OUT_DIR, ROOT, available  # noqa: F401  (available: re-exported)

LIB = os.path.join(OUT_DIR, "libkdl_emu_iupac.so")

_lib = None


def _sources():
    csrc = os.path.join(ROOT, "kindel_b200", "csrc")
    return [os.path.join(EMU_DIR, "cuda_emu.h"), os.path.join(EMU_DIR, "emu_iupac.cpp"),
            os.path.join(csrc, "kdl_common.cuh"), os.path.join(csrc, "vote.cu"), os.path.join(csrc, "assemble.cu"),
            os.path.join(ROOT, "include", "kindel_b200.h")]


def load():
    global _lib
    if _lib is not None:
        return _lib
    src = _sources()
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in src)):
        os.makedirs(OUT_DIR, exist_ok=True)
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-I", CUDA_INCLUDE, "-I", os.path.join(ROOT, "include"),
               os.path.join(EMU_DIR, "emu_iupac.cpp"), "-o", LIB]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the IUPAC-vote emulator failed:\n" + res.stdout + res.stderr)
    from kindel_b200 import _ffi

    lib = C.CDLL(LIB)
    vp = C.c_void_p
    lib.emu_iupac_last_error.restype = C.c_char_p
    lib.emu_iupac_set_schedule.argtypes = [C.c_int, C.c_ulonglong]
    lib.emu_iupac_set_schedule.restype = None
    lib.emu_vote_iupac.argtypes = [vp, C.c_longlong, C.c_longlong, C.c_double, vp]
    lib.emu_exchange_epoch_iupac.argtypes = [C.POINTER(_ffi.KdlExchange), C.c_int, C.c_longlong, C.c_longlong,
                                             C.c_double, C.c_int, C.c_int]
    lib.emu_assemble.argtypes = [vp, C.c_longlong, vp, vp, C.c_int, vp, vp, vp, C.c_longlong, vp, vp, vp]
    lib.emu_cdr_flags.argtypes = [vp, C.c_longlong, C.c_longlong, C.c_longlong, C.c_double, vp, vp]
    _lib = lib
    return lib


def _check(rc):
    if rc:
        raise RuntimeError(_lib.emu_iupac_last_error().decode())


def vote_iupac(counts: np.ndarray, min_depth, threshold) -> np.ndarray:
    """K2 with the IUPAC vote (kdl_vote_iupac) over a host table."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    calls = np.zeros(counts.shape[1], dtype=np.uint8)
    _check(lib.emu_vote_iupac(counts.ctypes.data, counts.shape[1], int(math.ceil(min_depth)), float(threshold),
                              calls.ctypes.data))
    return calls


def exchange_epoch(tables, feet, slices, calls, flags, epoch, threshold, min_depth=1, grid=3):
    """One epoch of the fused multi-GPU exchange with the IUPAC vote (kdl_exchange_vote_iupac, then K2g) with the
    ranks' buffers in host memory; arguments as emu_harness.exchange_epoch."""
    from kindel_b200 import _ffi

    lib = load()
    n = len(tables)
    n_slots = tables[0].shape[1]
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
    _check(lib.emu_exchange_epoch_iupac(xs, n, n_slots, int(math.ceil(min_depth)), float(threshold), epoch, grid))


def assemble(calls: np.ndarray, batch, ins_slots, ins_strings):
    """K5 (kdl_assemble) over host call bytes: the consensus text of every contig, like engine.assemble."""
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
    n_blocks = (n_slots + 1 + 1023) // 1024
    sums = np.zeros(n_blocks + 1, dtype=np.uint32)
    offsets = np.zeros(n_slots + 1, dtype=np.uint32)
    out = np.zeros(n_slots + int(ins_off[-1]) + 16, dtype=np.uint8)
    _check(lib.emu_assemble(calls.ctypes.data, n_slots, c_slot.ctypes.data, c_len.ctypes.data, len(c_len),
                            slots.ctypes.data, ins_off.ctypes.data, blob.ctypes.data, len(enc), sums.ctypes.data,
                            offsets.ctypes.data, out.ctypes.data))
    text = out[: int(offsets[n_slots])].tobytes()
    return [text[int(offsets[s]):int(offsets[s + L])].decode("ascii") for s, L in zip(c_slot.tolist(), c_len.tolist())]


def cdr_flags(counts: np.ndarray, slot_lo: int, slot_hi: int, decay: float):
    """K4 (kdl_cdr_flags) over a host table: (flags, bases) uint8 of slots [slot_lo, slot_hi), like engine.cdr_flags.
    Slots outside the range keep the canary 0xEE, which is checked."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    n = counts.shape[1]
    flags = np.full(n, 0xEE, dtype=np.uint8)
    bases = np.full(n, 0xEE, dtype=np.uint8)
    _check(lib.emu_cdr_flags(counts.ctypes.data, n, int(slot_lo), int(slot_hi), float(decay), flags.ctypes.data,
                             bases.ctypes.data))
    assert (flags[:slot_lo] == 0xEE).all() and (flags[slot_hi:] == 0xEE).all(), "K4 wrote outside its slot range"
    assert (bases[:slot_lo] == 0xEE).all() and (bases[slot_hi:] == 0xEE).all(), "K4 wrote outside its slot range"
    return flags[slot_lo:slot_hi].copy(), bases[slot_lo:slot_hi].copy()


def set_schedule(mode: str = "forward", seed: int = 1):
    """Thread order of the emulated blocks: "forward", "reverse" or "random" (see emu_harness.set_schedule)."""
    load().emu_iupac_set_schedule({"forward": 0, "reverse": 1, "random": 2}[mode], seed)
