"""Builds and drives the emulated consensus-quality kernels (tests/emu/emu_qual.cpp): test infrastructure.

The source of kindel_b200/csrc/assemble.cu is compiled for the host on top of tests/emu/cuda_emu.h, as
tests/emu_iupac_harness.py does for the vote, into a library of its own.  `consensus_qual` is K2q, `assemble_qual`
K5 followed by K5q over K5's offsets."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from emu_harness import CUDA_INCLUDE, EMU_DIR, OUT_DIR, ROOT, available  # noqa: F401  (available: re-exported)

LIB = os.path.join(OUT_DIR, "libkdl_emu_qual.so")

_lib = None


def _sources():
    csrc = os.path.join(ROOT, "kindel_b200", "csrc")
    return [os.path.join(EMU_DIR, "cuda_emu.h"), os.path.join(EMU_DIR, "emu_qual.cpp"),
            os.path.join(csrc, "kdl_common.cuh"), os.path.join(csrc, "assemble.cu"),
            os.path.join(ROOT, "include", "kindel_b200.h")]


def load():
    global _lib
    if _lib is not None:
        return _lib
    src = _sources()
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in src)):
        os.makedirs(OUT_DIR, exist_ok=True)
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-I", CUDA_INCLUDE, "-I", os.path.join(ROOT, "include"),
               os.path.join(EMU_DIR, "emu_qual.cpp"), "-o", LIB]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the consensus-quality emulator failed:\n" + res.stdout + res.stderr)
    lib = C.CDLL(LIB)
    vp = C.c_void_p
    lib.emu_qual_last_error.restype = C.c_char_p
    lib.emu_qual_set_schedule.argtypes = [C.c_int, C.c_ulonglong]
    lib.emu_qual_set_schedule.restype = None
    lib.emu_consensus_qual.argtypes = [vp, vp, C.c_longlong, vp]
    lib.emu_assemble_qual.argtypes = [vp, vp, C.c_longlong, vp, vp, C.c_int, vp, vp, vp, vp, C.c_longlong, vp, vp, vp,
                                      vp]
    _lib = lib
    return lib


def _check(rc):
    if rc:
        raise RuntimeError(_lib.emu_qual_last_error().decode())


def consensus_qual(counts: np.ndarray, calls: np.ndarray) -> np.ndarray:
    """K2q (kdl_consensus_qual) over a host table and its call bytes."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    calls = np.ascontiguousarray(calls, dtype=np.uint8)
    qual = np.full(counts.shape[1], 0xEE, dtype=np.uint8)
    _check(lib.emu_consensus_qual(counts.ctypes.data, calls.ctypes.data, counts.shape[1], qual.ctypes.data))
    return qual


def assemble_qual(calls, qual, batch, ins_slots, ins_strings, ins_qual):
    """K5 + K5q over host buffers: (texts, quality texts), one per contig, like engine.assemble(..., qual=...)."""
    lib = load()
    calls = np.ascontiguousarray(calls, dtype=np.uint8)
    qual = np.ascontiguousarray(qual, dtype=np.uint8)
    n_slots = calls.shape[0]
    enc = [x.encode("ascii") for x in ins_strings]
    ins_off = np.zeros(len(enc) + 1, dtype=np.uint32)
    if enc:
        ins_off[1:] = np.cumsum([len(x) for x in enc])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8).copy()
    slots = np.ascontiguousarray(ins_slots if len(enc) else np.zeros(1), dtype=np.int64)
    iq = np.ascontiguousarray(ins_qual if len(enc) else np.zeros(1), dtype=np.uint8)
    c_slot = np.ascontiguousarray(batch.contig_slot, dtype=np.int64)
    c_len = np.ascontiguousarray(batch.contig_len, dtype=np.int32)
    n_blocks = (n_slots + 1 + 1023) // 1024
    sums = np.zeros(n_blocks + 1, dtype=np.uint32)
    offsets = np.zeros(n_slots + 1, dtype=np.uint32)
    size = n_slots + int(ins_off[-1]) + 16
    out = np.zeros(size, dtype=np.uint8)
    qout = np.full(size, 0xEE, dtype=np.uint8)
    _check(lib.emu_assemble_qual(calls.ctypes.data, qual.ctypes.data, n_slots, c_slot.ctypes.data, c_len.ctypes.data,
                                 len(c_len), slots.ctypes.data, ins_off.ctypes.data, blob.ctypes.data, iq.ctypes.data,
                                 len(enc), sums.ctypes.data, offsets.ctypes.data, out.ctypes.data, qout.ctypes.data))
    total = int(offsets[n_slots])
    assert (qout[total:] == 0xEE).all(), "K5q wrote past the text"
    text, qtext = out[:total].tobytes(), qout[:total].tobytes()
    spans = [(int(offsets[s]), int(offsets[s + L])) for s, L in zip(c_slot.tolist(), c_len.tolist())]
    return [text[a:b].decode("ascii") for a, b in spans], [qtext[a:b].decode("latin-1") for a, b in spans]


def set_schedule(mode: str = "forward", seed: int = 1):
    """Thread order of the emulated blocks: "forward", "reverse" or "random" (see emu_harness.set_schedule)."""
    load().emu_qual_set_schedule({"forward": 0, "reverse": 1, "random": 2}[mode], seed)
