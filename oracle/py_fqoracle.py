"""TEST INFRASTRUCTURE ONLY -- the per-base consensus qualities (an extension) restated in numpy, as an independent
check of oracle/kindel_fqoracle.c: every slot tests all 61 q at once, and Q is the number of q in 1..60 that pass
(the test is monotone in q and always passes at q = 0).

    TEN                          this module's copy of the 61 hex-float constants
    qual(counts, calls)          uint8[n_slots], the Q of the base each slot emits
    insertion_qual(d, dn, k)     Q of inserted strings (k < 0: a tie), vectorised
"""
from __future__ import annotations

import numpy as np

TEN = np.array([float.fromhex(h) for h in (
    "0x1.0000000000000p+0", "0x1.4248ef8fc2604p+0", "0x1.95bb8f6d46052p+0", "0x1.fec982d5bb8afp+0",
    "0x1.41857e9d4cc5fp+1", "0x1.94c583ada5b53p+1", "0x1.fd93c1f526de0p+1", "0x1.40c28430012e7p+2",
    "0x1.93d00d2348996p+2", "0x1.fc5ebcec13541p+2", "0x1.4000000000000p+3", "0x1.92db2b73b2f85p+3",
    "0x1.fb2a734897867p+3", "0x1.3f3df1c59536ep+4", "0x1.91e6de449ff77p+4", "0x1.f9f6e4990f227p+4",
    "0x1.3e7c5939384acp+5", "0x1.90f3253c017a1p+5", "0x1.f8c4106c1abfbp+5", "0x1.3dbb36138c149p+6",
    "0x1.9000000000000p+6", "0x1.f791f6509fb66p+6", "0x1.3cfa880d5eb40p+7", "0x1.8f0d6e36fa849p+7",
    "0x1.f66095d5c7f54p+7", "0x1.3c3a4edfa9759p+8", "0x1.8e1b6f87865d7p+8", "0x1.f52fee8b01d89p+8",
    "0x1.3b7a8a4390b7dp+9", "0x1.8d2a03986f19bp+9", "0x1.f400000000000p+9", "0x1.3abb39f263d20p+10",
    "0x1.8c392a10b6611p+10", "0x1.f2d0c9c4b925bp+10", "0x1.39fc5da59cf95p+11", "0x1.8b48e29793d2fp+11",
    "0x1.f1a24b6967f4cp+11", "0x1.393df516e1276p+12", "0x1.8a592cd474e5cp+12", "0x1.f074847e8ae02p+12",
    "0x1.3880000000000p+13", "0x1.896a086efcc67p+13", "0x1.ef477494e3f95p+13", "0x1.37c27e1af3b79p+14",
    "0x1.887b750f0437ap+14", "0x1.ee1b1b3d78c7ap+14", "0x1.37056f21e0f90p+15", "0x1.878d725c99713p+15",
    "0x1.ecef7809921f4p+15", "0x1.3648d2cf16cc1p+16", "0x1.86a0000000000p+16", "0x1.ebc48a8abbf81p+16",
    "0x1.358ca8dd0e7bdp+17", "0x1.85b31da1b0a57p+17", "0x1.ea9a5252c5458p+17", "0x1.34d0f1066b7ccp+18",
    "0x1.84c6caea59374p+18", "0x1.e970cef3bfcd8p+18", "0x1.3415ab05fb538p+19", "0x1.83db0782dc7f1p+19",
    "0x1.e848000000000p+19",
)], dtype=np.float64)


def _q(depth, support):
    depth = np.asarray(depth, dtype=np.int64)
    support = np.asarray(support, dtype=np.int64)
    e = (depth - support + 1).astype(np.float64)[..., None]
    lim = (depth + 2).astype(np.float64)[..., None]
    ok = (e * TEN[1:]) <= lim  # [n, 60]: one correctly rounded multiply per q
    return np.where(support > 0, ok.sum(axis=-1), 0).astype(np.uint8)


def qual(counts, calls):
    w = np.asarray(counts[:4], dtype=np.int64)
    calls = np.asarray(calls, dtype=np.uint8)
    depth = w.sum(axis=0)
    multi = (calls & 0x80) != 0
    mask = (calls & 15).astype(np.int64)
    bits = (mask[None, :] >> np.arange(4)[:, None]) & 1
    k_multi = np.where(mask == 15, 0, (w * bits).sum(axis=0))
    code = (calls & 7).astype(np.int64)
    k_one = np.where(code < 4, np.take_along_axis(w, np.minimum(code, 3)[None, :], axis=0)[0], 0)
    return _q(depth, np.where(multi, k_multi, k_one))


def insertion_qual(depth, depth_next, k):
    k = np.asarray(k, dtype=np.int64)
    d = np.maximum(np.minimum(np.asarray(depth, dtype=np.int64), np.asarray(depth_next, dtype=np.int64)), k)
    return np.where(k < 0, 0, _q(d, np.maximum(k, 0))).astype(np.uint8)
