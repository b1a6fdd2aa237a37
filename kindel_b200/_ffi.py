"""ctypes binding of libkindel_b200.so (the C ABI in include/kindel_b200.h).

There is no fallback: if the shared library is missing it is built in-tree with nvcc
(`kindel_b200.build`); if that fails, importing the engine raises.  Nothing in this package computes
a pileup or a vote on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

c_i32p = C.POINTER(C.c_int32)
c_u32p = C.POINTER(C.c_uint32)
c_i64p = C.POINTER(C.c_int64)
c_u8p = C.POINTER(C.c_uint8)

KDL_NCOL = 19
KDL_NVOTE_COL = 7
KDL_COMPLEX = 0x80000000
KDL_HARD = 0x40000000
KDL_LEN_MASK = 0xFFFF
KDL_NM_SHIFT = 16
KDL_NM_MASK = 0x7F
KDL_TILE_MAXOPS = 64
KDL_TILE_MAXREACH = 1024
KDL_TILE = 512
KDL_PILEUP_FRESH_WEIGHTS = 1
KDL_PILEUP_ZERO_REST = 2
KDL_FAST_MAXLEN = 8192
KDL_OK = 0
KDL_ERR_INDEX = 10
KDL_ERR_KEY = 11
KDL_DEDUP_TOTALS = 8


class KdlBatch(C.Structure):
    _fields_ = [
        ("n_reads", C.c_int64),
        ("seq4_words", C.c_int64),
        ("ref_start", C.c_void_p),
        ("seq_off", C.c_void_p),
        ("l_seq", C.c_void_p),
        ("seq4", C.c_void_p),
        ("n_contigs", C.c_int32),
        ("reads_sorted", C.c_int32),
        ("max_simple_len", C.c_int32),
        ("reach_right", C.c_int32),
        ("reach_left", C.c_int32),
        ("reserved0", C.c_int32),
        ("contig_read_off", C.c_void_p),
        ("contig_len", C.c_void_p),
        ("contig_slot", C.c_void_p),
        ("n_complex", C.c_int64),
        ("n_hard", C.c_int64),
        ("complex_idx", C.c_void_p),
        ("hard_idx", C.c_void_p),
        ("tile_index", C.c_void_p),
    ]


class KdlQmask(C.Structure):
    _fields_ = [
        ("n_reads", C.c_int64),
        ("n_bases", C.c_int64),
        ("read_idx", C.c_void_p),
        ("off", C.c_void_p),
        ("qpos", C.c_void_p),
    ]


class KdlPrimers(C.Structure):
    _fields_ = [
        ("n_contigs", C.c_int32),
        ("reserved", C.c_int32),
        ("n_intervals", C.c_int64),
        ("contig_off", C.c_void_p),
        ("start_sorted", C.c_void_p),
        ("end_max", C.c_void_p),
        ("end_sorted", C.c_void_p),
        ("start_min", C.c_void_p),
    ]


class KdlAmplicons(C.Structure):
    _fields_ = [
        ("n_contigs", C.c_int32),
        ("n_amplicons", C.c_int32),
        ("left_off", C.c_void_p),
        ("left_at", C.c_void_p),
        ("left_label", C.c_void_p),
        ("right_off", C.c_void_p),
        ("right_at", C.c_void_p),
        ("right_label", C.c_void_p),
        ("amp_contig", C.c_void_p),
        ("insert_start", C.c_void_p),
        ("insert_end", C.c_void_p),
    ]


class KdlDedupLists(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in ("pair_contig", "pair_e1", "pair_e2", "pair_rank", "pair_r1", "pair_r2",
                                          "single_contig", "single_key", "single_rank", "single_read", "end",
                                          "paired")]


class KdlExchange(C.Structure):
    _fields_ = [
        ("n_ranks", C.c_int32),
        ("rank", C.c_int32),
        ("tables", C.c_void_p * 16),
        ("calls", C.c_void_p * 16),
        ("ready", C.c_void_p * 16),
        ("done", C.c_void_p * 16),
        ("foot_lo", C.c_int64 * 16),
        ("foot_hi", C.c_int64 * 16),
        ("slice_lo", C.c_int64 * 16),
        ("slice_hi", C.c_int64 * 16),
        ("counter", C.c_void_p),
    ]


class KdlDiag(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("reserved", C.c_int32),
        ("read", C.c_int64),
        ("nibble", C.c_int32),
        ("op_index", C.c_int32),
    ]


# every symbol include/kindel_b200.h declares, with its prototype
_PROTOTYPES = {
    "kdl_abi_version": (C.c_int, []),
    "kdl_status_string": (C.c_char_p, [C.c_int]),
    "kdl_launch_count": (C.c_int64, []),
    "kdl_pileup": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_pileup_range": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_pileup_range_map": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_diagnose": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_void_p]),
    "kdl_unmask": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.c_void_p, C.c_int64, C.c_void_p]),
    "kdl_vote": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "kdl_vote_iupac": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_void_p]),
    "kdl_derive": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "kdl_cdr_flags": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_assemble_scratch_words": (C.c_int64, [C.c_int64]),
    "kdl_assemble": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_consensus_qual": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "kdl_assemble_qual": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                    C.c_void_p]),
    "kdl_variant_scratch_words": (C.c_int64, [C.c_int64]),
    "kdl_variant_count": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_double,
                                    C.c_void_p, C.c_void_p]),
    "kdl_variant_scatter": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_double,
                                      C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_variant_ref_count": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_int64, C.c_double, C.c_void_p, C.c_void_p]),
    "kdl_variant_ref_scatter": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                          C.c_int64, C.c_double, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_variant_multi_count": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32,
                                          C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_void_p]),
    "kdl_variant_multi_scatter": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32,
                                            C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_int64, C.c_void_p,
                                            C.c_void_p, C.c_void_p]),
    "kdl_deletion_scratch_words": (C.c_int64, [C.c_int64]),
    "kdl_deletion_count": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_void_p]),
    "kdl_deletion_scatter": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "kdl_left_align_deletions": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                           C.c_void_p]),
    "kdl_left_align_insertions": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_select_scratch_words": (C.c_int64, [C.c_int64]),
    "kdl_select_count": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_select_scatter": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.c_void_p, C.c_void_p,
                                     C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.c_void_p]),
    "kdl_primers_scratch_words": (C.c_int64, [C.c_int64]),
    "kdl_primers_count": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.POINTER(KdlPrimers), C.c_void_p,
                                    C.c_void_p]),
    "kdl_primers_apply": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.POINTER(KdlPrimers), C.c_void_p,
                                    C.c_void_p, C.POINTER(KdlQmask), C.c_void_p]),
    "kdl_mates_pair": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                 C.c_void_p, C.c_void_p]),
    "kdl_overlap_scratch_words": (C.c_int64, [C.c_int64]),
    "kdl_overlap_count": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_overlap_apply": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.POINTER(KdlQmask), C.c_void_p, C.c_int64, C.c_void_p]),
    "kdl_overlap_untake": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "kdl_quality_pileup": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "kdl_quality_weights": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "kdl_vote_quality": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_amplicons_assign": (C.c_int, [C.POINTER(KdlBatch), C.POINTER(KdlAmplicons), C.c_void_p, C.c_void_p]),
    "kdl_amplicons_depth": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32,
                                      C.POINTER(KdlAmplicons), C.c_int64, C.c_void_p, C.c_void_p]),
    "kdl_normalise_scratch_words": (C.c_int64, [C.c_int64, C.c_int32]),
    "kdl_normalise": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_int64,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_dedup_entries": (C.c_int, [C.POINTER(KdlBatch), C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.POINTER(KdlDedupLists), C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_dedup_scratch_words": (C.c_int64, [C.c_int64]),
    "kdl_dedup_select": (C.c_int, [C.POINTER(KdlDedupLists), C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                   C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_vote_peers":(C.c_int, [C.POINTER(C.c_void_p), C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_vote_peers_sparse": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int32,
                                        C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_exchange_signal": (C.c_int, [C.POINTER(KdlExchange), C.c_int32, C.c_void_p]),
    "kdl_exchange_vote": (C.c_int, [C.POINTER(KdlExchange), C.c_int64, C.c_int64, C.c_int32, C.c_void_p]),
    "kdl_exchange_vote_iupac": (C.c_int, [C.POINTER(KdlExchange), C.c_int64, C.c_int64, C.c_double, C.c_int32,
                                          C.c_void_p]),
    "kdl_exchange_wait": (C.c_int, [C.POINTER(KdlExchange), C.c_int32, C.c_void_p]),
    "kdl_table_alloc": (C.c_int, [C.c_int64, C.POINTER(C.c_void_p)]),
    "kdl_table_free": (C.c_int, [C.c_void_p]),
    "kdl_ipc_export": (C.c_int, [C.c_void_p, C.c_char_p]),
    "kdl_ipc_open": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "kdl_ipc_close": (C.c_int, [C.c_void_p]),
    "kdl_ctx_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "kdl_ctx_destroy": (None, [C.c_void_p]),
    "kdl_ctx_consensus": (C.c_int, [C.c_void_p, C.POINTER(KdlBatch), C.c_int64, C.c_int64, C.c_int64,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(KdlDiag)]),
    "kdl_ctx_consensus_masked": (C.c_int, [C.c_void_p, C.POINTER(KdlBatch), C.POINTER(KdlQmask), C.c_int64, C.c_int64,
                                           C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(KdlDiag)]),
    "kdl_ctx_last_timing": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "kdl_bam_open": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]),
    "kdl_bam_close": (None, [C.c_void_p]),
    "kdl_bam_header_text": (C.c_void_p, [C.c_void_p, C.POINTER(C.c_int64)]),
    "kdl_bam_n_ref": (C.c_int32, [C.c_void_p]),
    "kdl_bam_ref_name": (C.c_char_p, [C.c_void_p, C.c_int32]),
    "kdl_bam_ref_len": (C.c_int32, [C.c_void_p, C.c_int32]),
    "kdl_bam_prepare": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "kdl_bam_contigs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_bam_fill": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_bam_set_filter": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "kdl_bam_fill_mask": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_bam_fill_strand": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "kdl_bam_fill_mates": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "kdl_bam_fill_qual": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "kdl_bam_fill_dup": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_PROTOTYPES)

_lib = None


def lib_path() -> str:
    return _build.LIB_PATH


def load():
    """Load (building first if needed) the engine library.  Raises if it cannot be had."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if not os.path.exists(path):
        path = _build.build_engine()
    lib = C.CDLL(path)
    for name, (res, args) in _PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.kdl_abi_version() != 2:
        raise RuntimeError("libkindel_b200.so ABI version mismatch")
    _lib = lib
    return lib


def status_string(code: int) -> str:
    return load().kdl_status_string(code).decode()


def check(code: int, what: str = "") -> None:
    if code != KDL_OK:
        raise RuntimeError("kindel_b200 %s failed: %s (status %d)" % (what, status_string(code), code))
