"""Builds and drives the emulated K6r / K7 kernels (tests/emu/emu_variants_ref.cpp): test infrastructure.

The source of kindel_b200/csrc/variants.cu (and of assemble.cu, whose scan kernel it uses) is compiled for the host on
top of tests/emu/cuda_emu.h into a library of its own.  `variant_sites_ref` runs K6r as engine.variant_sites_ref does
(the count, a read of the total, the scatter); `deletion_events` runs K7 as engine.deletion_events does, over a
kdl_batch of host pointers."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from emu_harness import CUDA_INCLUDE, EMU_DIR, OUT_DIR, ROOT, available  # noqa: F401  (available: re-exported)

LIB = os.path.join(OUT_DIR, "libkdl_emu_variants_ref.so")

_lib = None


def _sources():
    csrc = os.path.join(ROOT, "kindel_b200", "csrc")
    return [os.path.join(EMU_DIR, "cuda_emu.h"), os.path.join(EMU_DIR, "emu_variants_ref.cpp"),
            os.path.join(csrc, "kdl_common.cuh"), os.path.join(csrc, "assemble.cu"), os.path.join(csrc, "variants.cu"),
            os.path.join(ROOT, "include", "kindel_b200.h")]


def load():
    global _lib
    if _lib is not None:
        return _lib
    src = _sources()
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in src)):
        os.makedirs(OUT_DIR, exist_ok=True)
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-I", CUDA_INCLUDE, "-I", os.path.join(ROOT, "include"),
               os.path.join(EMU_DIR, "emu_variants_ref.cpp"), "-o", LIB]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the reference-variant emulator failed:\n" + res.stdout + res.stderr)
    lib = C.CDLL(LIB)
    vp, ll = C.c_void_p, C.c_longlong
    lib.emu_variants_ref_last_error.restype = C.c_char_p
    lib.emu_variants_ref_set_schedule.argtypes = [C.c_int, C.c_ulonglong]
    lib.emu_variants_ref_set_schedule.restype = None
    lib.emu_variant_ref_count.argtypes = [vp, ll, vp, vp, C.c_int, vp, ll, C.c_double, vp]
    lib.emu_variant_ref_scatter.argtypes = [vp, ll, vp, vp, C.c_int, vp, ll, C.c_double, vp, ll, vp, vp, vp, vp]
    lib.emu_deletion_count.argtypes = [vp, vp]
    lib.emu_deletion_scatter.argtypes = [vp, vp, ll, vp, vp]
    _lib = lib
    return lib


def _check(rc):
    if rc:
        raise RuntimeError(_lib.emu_variants_ref_last_error().decode())


def variant_sites_ref(counts, contig_slot, contig_len, ref_codes, abs_floor, rel_threshold):
    """K6r over a host table: (slot int64[n], counts int32[7, n], dpa int64[n], mask uint8[n]) like
    engine.variant_sites_ref.  abs_floor is the clamped integer threshold (engine.variant_abs_floor)."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    n_slots = counts.shape[1]
    c_slot = np.ascontiguousarray(contig_slot, dtype=np.int64)
    c_len = np.ascontiguousarray(contig_len, dtype=np.int32)
    ref = np.ascontiguousarray(ref_codes, dtype=np.uint8)
    assert ref.shape == (n_slots,) and ref.ctypes.data % 4 == 0
    n_blocks = (n_slots + 1023) // 1024
    sums = np.full(n_blocks + 1, 0xDEADBEEF, dtype=np.uint32)
    args = (counts.ctypes.data, n_slots, c_slot.ctypes.data, c_len.ctypes.data, len(c_len), ref.ctypes.data,
            int(abs_floor), float(rel_threshold))
    _check(lib.emu_variant_ref_count(*args, sums.ctypes.data))
    n = int(sums[n_blocks])
    # one record more than announced, poisoned: the scatter must write exactly n and leave the rest alone
    slot = np.full(n + 1, -7, dtype=np.int64)
    dpa = np.full(n + 1, -7, dtype=np.int64)
    mask = np.full(n + 1, 0xEE, dtype=np.uint8)
    flat = np.full(7 * n + 1, -7, dtype=np.int32)
    _check(lib.emu_variant_ref_scatter(*args, sums.ctypes.data, n, slot.ctypes.data, flat.ctypes.data, dpa.ctypes.data,
                                       mask.ctypes.data))
    assert slot[n] == -7 and dpa[n] == -7 and mask[n] == 0xEE and flat[7 * n] == -7, "K6r wrote past the sites"
    return slot[:n], flat[:7 * n].reshape(7, n).copy(), dpa[:n], mask[:n]


def deletion_events(batch):
    """K7 over a host ReadBatch: (slot int64[m], length int32[m]) in read order, then op order."""
    from kindel_b200 import engine

    lib = load()
    struct, keep = engine.host_struct(batch)
    n_blocks = (batch.n_reads + 255) // 256
    sums = np.full(n_blocks + 1, 0xDEADBEEF, dtype=np.uint32)
    _check(lib.emu_deletion_count(C.addressof(struct), sums.ctypes.data))
    m = int(sums[n_blocks])
    slot = np.full(m + 1, -7, dtype=np.int64)
    length = np.full(m + 1, -7, dtype=np.int32)
    _check(lib.emu_deletion_scatter(C.addressof(struct), sums.ctypes.data, m, slot.ctypes.data, length.ctypes.data))
    assert slot[m] == -7 and length[m] == -7, "K7 wrote past the events"
    del keep
    return slot[:m], length[:m]


def set_schedule(mode: str = "forward", seed: int = 1):
    """Thread order of the emulated blocks: "forward", "reverse" or "random" (see emu_harness.set_schedule)."""
    load().emu_variants_ref_set_schedule({"forward": 0, "reverse": 1, "random": 2}[mode], seed)
