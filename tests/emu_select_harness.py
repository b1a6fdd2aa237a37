"""Builds and drives the emulated K8 read selection (tests/emu/emu_select.cpp): test infrastructure.

kindel_b200/csrc/select.cu is compiled for the host on top of tests/emu/cuda_emu.h into a library of its own.
`select` runs K8 as engine.select_reads does (the count, one read of the totals record, the scatter) over a kdl_batch
of host pointers; `fields` / `assert_equal` compare such a result with bamio.select_reads field for field."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from emu_harness import CUDA_INCLUDE, EMU_DIR, OUT_DIR, ROOT, available  # noqa: F401  (available: re-exported)

LIB = os.path.join(OUT_DIR, "libkdl_emu_select.so")

_lib = None


def _sources():
    csrc = os.path.join(ROOT, "kindel_b200", "csrc")
    return [os.path.join(EMU_DIR, "cuda_emu.h"), os.path.join(EMU_DIR, "emu_select.cpp"),
            os.path.join(csrc, "kdl_common.cuh"), os.path.join(csrc, "select.cu"),
            os.path.join(ROOT, "include", "kindel_b200.h")]


def load():
    global _lib
    if _lib is not None:
        return _lib
    src = _sources()
    if not (os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in src)):
        os.makedirs(OUT_DIR, exist_ok=True)
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-I", CUDA_INCLUDE, "-I", os.path.join(ROOT, "include"),
               os.path.join(EMU_DIR, "emu_select.cpp"), "-o", LIB]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("building the read-selection emulator failed:\n" + res.stdout + res.stderr)
    lib = C.CDLL(LIB)
    vp = C.c_void_p
    lib.emu_select_last_error.restype = C.c_char_p
    lib.emu_select_set_schedule.argtypes = [C.c_int, C.c_ulonglong]
    lib.emu_select_set_schedule.restype = None
    lib.emu_select_scratch_words.argtypes = [C.c_longlong]
    lib.emu_select_scratch_words.restype = C.c_longlong
    lib.emu_select_count.argtypes = [vp, vp, vp, vp]
    lib.emu_select_scatter.argtypes = [vp, vp, vp, vp, vp, vp]
    _lib = lib
    return lib


def _check(rc):
    if rc:
        raise RuntimeError(_lib.emu_select_last_error().decode())


def set_schedule(mode: str = "forward", seed: int = 1):
    """Thread order of the emulated blocks: "forward", "reverse" or "random" (see emu_harness.set_schedule)."""
    load().emu_select_set_schedule({"forward": 0, "reverse": 1, "random": 2}[mode], seed)


def select(batch, keep):
    """K8 over a host ReadBatch and keep bytes -> the fields of the sub-batch (see `fields`)."""
    from kindel_b200 import _ffi, engine

    lib = load()
    keep = np.ascontiguousarray(keep, dtype=np.uint8)
    struct, hold = engine.host_struct(batch)
    qmask, qhold = engine.host_qmask(batch)
    qp = C.addressof(qmask) if qmask is not None else None
    words = int(lib.emu_select_scratch_words(batch.n_reads))
    scratch = np.full(words, 0xDEADBEEF, dtype=np.uint32)
    _check(lib.emu_select_count(C.addressof(struct), qp, keep.ctypes.data, scratch.ctypes.data))
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
    _check(lib.emu_select_scatter(C.addressof(struct), qp, keep.ctypes.data, scratch.ctypes.data, C.addressof(o),
                                  C.addressof(om) if om is not None else None))
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


_ARRAYS = ("ref_start", "seq_off", "l_seq", "seq4", "contig_read_off", "complex_idx", "hard_idx")
_SCALARS = ("n_events", "reads_sorted", "max_simple_len", "reach_right", "reach_left")
_MASK = ("mask_read", "mask_off", "mask_qpos")


def fields(batch) -> dict:
    """The fields K8 produces, of a host ReadBatch (what select_reads gives)."""
    out = {f: np.asarray(getattr(batch, f)) for f in _ARRAYS}
    out.update({f: getattr(batch, f) for f in _SCALARS})
    out.update({f: (np.asarray(getattr(batch, f)) if batch.n_masked else None) for f in _MASK})
    return out


def assert_equal(got: dict, want: dict, what=""):
    for f in _ARRAYS:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        assert g.shape == w.shape and np.array_equal(g.view(np.uint8) if g.size else g,
                                                     w.astype(g.dtype).view(np.uint8) if w.size else w.astype(g.dtype)), (what, f)
    for f in _SCALARS:
        assert int(got[f]) == int(want[f]), (what, f, got[f], want[f])
    for f in _MASK:
        if want[f] is None:
            assert got[f] is None, (what, f)
        else:
            assert got[f] is not None and np.array_equal(np.asarray(got[f], dtype=np.int64),
                                                         np.asarray(want[f], dtype=np.int64)), (what, f)
