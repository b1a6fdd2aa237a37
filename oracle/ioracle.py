"""TEST INFRASTRUCTURE ONLY -- ctypes front-end of oracle/kindel_ioracle.c, the CPU checker of the IUPAC vote (an
extension).

    vote_iupac(counts, min_depth, t) -> calls uint8[n_slots]    (counts int32[>= 7, n_slots], as oracle.coracle.vote)

Multi-base calls carry bit 7 and their base set as a BAM nibble in bits 0-3; every other byte is encoded like
oracle.coracle.vote's.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kindel_ioracle.c")
_LIB = os.path.join(_HERE, "_build", "libkindel_ioracle.so")

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
        lib.ioracle_vote.restype = None
        lib.ioracle_vote.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_double, C.c_void_p]
        _lib = lib
    return _lib


def vote_iupac(counts, min_depth, t):
    lib = _load()
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    n_slots = counts.shape[1]
    calls = np.zeros(n_slots, dtype=np.uint8)
    lib.ioracle_vote(counts.ctypes.data, n_slots, int(math.ceil(min_depth)), float(t), calls.ctypes.data)
    return calls
