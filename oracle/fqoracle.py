"""TEST INFRASTRUCTURE ONLY -- ctypes front-end of oracle/kindel_fqoracle.c, the CPU checker of the per-base consensus
qualities (an extension).

    qual(counts, calls) -> uint8[n_slots]                  Q of the base every slot emits (linear search over q)
    fastq(counts, calls, s0, L, ins, patches, trim_ends, uppercase) -> (text, qualities)
                                                           one contig walked position by position

`ins` maps a contig position to its insertion dict (string -> count, first-seen order); `patches` are the merged CDR
Regions (start, end, seq) as the host code applies them.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .py_oracle import base_call

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kindel_fqoracle.c")
_LIB = os.path.join(_HERE, "_build", "libkindel_fqoracle.so")
_NO_PATCH = -(1 << 63)

_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(_LIB), exist_ok=True)
        subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-Wall", _SRC, "-o", _LIB], check=True)
    return _LIB


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        vp, i64 = C.c_void_p, C.c_int64
        lib.fqoracle_phred.restype = C.c_int
        lib.fqoracle_phred.argtypes = [i64, i64]
        lib.fqoracle_qual.restype = None
        lib.fqoracle_qual.argtypes = [vp, vp, i64, vp]
        lib.fqoracle_fastq.restype = i64
        lib.fqoracle_fastq.argtypes = [vp, i64, i64, i64, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp]
        _lib = lib
    return _lib


def phred(depth: int, support: int) -> int:
    return _load().fqoracle_phred(int(depth), int(support))


def qual(counts, calls) -> np.ndarray:
    lib = _load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    calls = np.ascontiguousarray(calls, dtype=np.uint8)
    out = np.zeros(counts.shape[1], dtype=np.uint8)
    lib.fqoracle_qual(counts.ctypes.data, calls.ctypes.data, counts.shape[1], out.ctypes.data)
    return out


def fastq(counts, calls, s0, L, ins, patches=None, trim_ends=False, uppercase=False):
    lib = _load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    calls = np.ascontiguousarray(calls, dtype=np.uint8)
    ins_k = np.zeros(L, dtype=np.int64)
    ins_off = np.zeros(L + 1, dtype=np.int64)
    blob = []
    for p in range(L):
        text = ""
        if p in ins:
            key, cnt, tie = base_call(ins[p])
            ins_k[p] = -1 if tie else cnt
            text = key
        blob.append(text.encode("ascii"))
        ins_off[p + 1] = ins_off[p] + len(blob[-1])
    skip = np.full(L, _NO_PATCH, dtype=np.int64)
    p_off = np.zeros(L + 1, dtype=np.int64)
    p_text = [b""] * L
    for r in patches or []:
        if r.seq and 0 <= r.start < L and skip[r.start] == _NO_PATCH:
            first = next(x for x in patches if x.start == r.start)  # the first Region starting there
            skip[r.start] = first.end - first.start - 1
            p_text[r.start] = first.seq.encode("ascii")
    for p in range(L):
        p_off[p + 1] = p_off[p] + len(p_text[p])
    ib = np.frombuffer(b"".join(blob) + b"\0", dtype=np.uint8).copy()
    pb = np.frombuffer(b"".join(p_text) + b"\0", dtype=np.uint8).copy()
    cap = L + int(ins_off[-1]) + int(p_off[-1]) + 1
    text = np.zeros(cap, dtype=np.uint8)
    q = np.zeros(cap, dtype=np.uint8)
    n = lib.fqoracle_fastq(counts.ctypes.data, counts.shape[1], int(s0), int(L), calls.ctypes.data, ins_k.ctypes.data,
                           ins_off.ctypes.data, ib.ctypes.data, skip.ctypes.data, p_off.ctypes.data, pb.ctypes.data,
                           int(bool(trim_ends)), int(bool(uppercase)), text.ctypes.data, q.ctypes.data)
    return text[:n].tobytes().decode("ascii"), q[:n].tobytes().decode("ascii")
