"""Device side of the pileup/consensus engine: torch tensors as buffers, kernels through the C ABI.

PyTorch is used for device memory, streams and (in `distributed.py`) the NCCL process group only;
every count and every vote is computed by the hand-written sm_90a kernels in
`kindel_b200/csrc/` reached through `libkindel_b200.so` (include/kindel_b200.h).  There is no CPU
implementation behind these functions: without a CUDA device they raise.

    upload(batch)              ReadBatch (host numpy) -> DeviceBatch (device tensors + kdl_batch [+ kdl_qmask])
    pileup(dbatch)             K1 (+ K1q for masked bases): count table [19, n_slots] int32 + insertion events
    vote(counts, min_depth)    K2: call byte per slot (iupac_threshold=t: the IUPAC vote)
    derive(counts)             derived depth columns [5, n_slots]
    consensus_qual(counts, calls)  K2q: Phred quality of the base each slot emits (extension)
    assemble(calls, ...)       K5 (+ K5q): consensus text (and its quality text) of every contig
    variant_sites(counts, ...) K6: the variant sites of `variants --only-variants` and the VCF (extension)
    variant_sites_ref(...)     K6r: the SNV and insertion-candidate sites against a reference (extension)
    deletion_alleles(dbatch, counts, ...)  K7 + grouping: the deletion alleles against a reference (extension)
    deletion_union(groups, table, ...)  the same rule over S samples' K7 groups: the keys that pass in some sample
    select_reads(dbatch, keep) K8: the sub-batch of the kept reads, built on the device (extension)
    mask_primers(dbatch, arrays)  K9: the batch with its amplicon primer bases masked (extension)
    mask_overlaps(dbatch)      K10p + K10: the batch with its read pairs' second mates masked where the first covers
                               (extension); pileup then runs K10u
    quality_sums(dbatch, qual8)  K0 + K11 + K11g: the counted bases' qualities summed per slot (extension)
    quality_weights(dbatch, qual8)  K0 + K11w + K11g-w: their quality weights summed per slot and base (extension)
    vote_quality(counts, wsum)  K2w: the vote with the base by summed quality weights, and its Q (extension)
    assign_amplicons(dbatch, arrays)  K12: each read's amplicon label (extension: `kindel amplicons`)
    amplicon_depth(counts, arrays, min_depth, ...)  K12d: per amplicon the sum, minimum and covered positions of the
                               depth of its insert (extension)
    normalise(label, reverse, n_amplicons, cap)  K13: the reads each (amplicon, strand) cap keeps, in batch order
                               (extension: `--normalise N`)
    dedup(dbatch, mate)        K10p + K14k + sort + K14s: the reads and read pairs duplicate removal keeps (extension:
                               `--dedup`)
    left_align_deletions(key, cnt, ref, ...)  K15d + regrouping: deletion groups moved to their leftmost place against
                               the reference (extension: `--left-align`)
    left_align_insertions(dbatch, events, ref)  K15i: each insertion row's leftmost slot and string rotation, and the
                               per-slot count of the moved rows (extension: `--left-align`)
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _ffi
from .bamio import NIBBLES, ReadBatch


def require_cuda(device=None) -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError(
            "kindel_b200 needs a CUDA device (H100, sm_90a): the pileup and the vote exist only as "
            "CUDA kernels and there is no CPU fallback")
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return torch.device(device)


def _stream_ptr(device) -> int:
    return int(torch.cuda.current_stream(device).cuda_stream)


@dataclass
class DeviceBatch:
    host: ReadBatch
    device: torch.device
    tensors: dict
    struct: _ffi.KdlBatch
    qmask: _ffi.KdlQmask = None  # the batch's masked bases (min_base_quality); None when there are none
    primer_masked: tuple = (0, 0)  # (reads, bases) K9 masked in it (mask_primers)
    # K10 (mask_overlaps): the dropped R2 ops, int32 [m, 4] = (slot, len, read, event row or -1 for a D), whose counts
    # pileup takes back (K10u); None when off
    drops: torch.Tensor = None
    overlap_masked: tuple = None  # (pairs, bases, deletions, insertions) K10 masked in it; None when off

    @property
    def n_slots(self) -> int:
        return self.host.n_slots


def make_struct(host: ReadBatch, ptr: dict) -> _ffi.KdlBatch:
    s = _ffi.KdlBatch()
    s.n_reads = host.n_reads
    s.seq4_words = int(host.seq4.shape[0])
    s.ref_start = ptr["ref_start"]
    s.seq_off = ptr["seq_off"]
    s.l_seq = ptr["l_seq"]
    s.seq4 = ptr["seq4"]
    s.n_contigs = host.n_contigs
    s.reads_sorted = 1 if host.reads_sorted else 0
    s.max_simple_len = int(host.max_simple_len)
    s.reach_right = int(host.reach_right)
    s.reach_left = int(host.reach_left)
    s.contig_read_off = ptr["contig_read_off"]
    s.contig_len = ptr["contig_len"]
    s.contig_slot = ptr["contig_slot"]
    s.n_complex = host.n_complex
    s.n_hard = host.n_hard
    s.complex_idx = ptr["complex_idx"] if host.n_complex else None
    s.hard_idx = ptr["hard_idx"] if host.n_hard else None
    s.tile_index = ptr.get("tile_index")
    return s


@dataclass
class BatchShape:
    """The scalars of a batch that lives only on the device (a K8 result): what DeviceBatch and the pileup read of
    their host batch, without the read data."""

    n_reads: int
    n_words: int
    n_contigs: int
    n_slots: int
    n_complex: int
    n_hard: int
    n_events: int
    n_masked: int
    n_mask_reads: int
    reads_sorted: bool
    max_simple_len: int
    reach_right: int
    reach_left: int


_FIELDS = ("ref_start", "seq_off", "l_seq", "seq4", "contig_read_off", "contig_len", "contig_slot", "complex_idx",
           "hard_idx")


_MASK_FIELDS = ("mask_read", "mask_off", "mask_qpos")


def host_struct(host: ReadBatch):
    """kdl_batch over HOST pointers (for the kdl_ctx_* entry points).  Returns (struct, keepalive)."""
    keep = {f: np.ascontiguousarray(getattr(host, f)) for f in _FIELDS}
    ptr = {f: (a.ctypes.data if a.size else None) for f, a in keep.items()}
    return make_struct(host, ptr), keep


def make_qmask(host: ReadBatch, ptr: dict) -> _ffi.KdlQmask:
    q = _ffi.KdlQmask()
    q.n_reads = host.n_mask_reads
    q.n_bases = host.n_masked
    q.read_idx, q.off, q.qpos = ptr["mask_read"], ptr["mask_off"], ptr["mask_qpos"]
    return q


def host_qmask(host: ReadBatch):
    """kdl_qmask over HOST pointers, or (None, None) when the batch has no masked base."""
    if not host.n_masked:
        return None, None
    keep = {f: np.ascontiguousarray(getattr(host, f), dtype=np.uint32) for f in _MASK_FIELDS}
    return make_qmask(host, {f: a.ctypes.data for f, a in keep.items()}), keep


def upload(host: ReadBatch, device=None, non_blocking: bool = False) -> DeviceBatch:
    device = require_cuda(device)
    tensors = {}
    for f in _FIELDS:
        a = np.ascontiguousarray(getattr(host, f))
        if a.dtype == np.uint32:  # torch has no first-class uint32 arithmetic; the bits are what matter
            a = a.view(np.int32)
        t = torch.from_numpy(a) if a.size else torch.zeros(4, dtype=torch.from_numpy(a).dtype)
        tensors[f] = t.to(device, non_blocking=non_blocking)
    qmask = None
    if host.n_masked:
        for f in _MASK_FIELDS:
            tensors[f] = torch.from_numpy(np.ascontiguousarray(getattr(host, f), dtype=np.uint32).view(np.int32)).to(
                device, non_blocking=non_blocking)
    # scratch for the tile index kdl_pileup builds on the device (K0)
    tensors["tile_index"] = torch.empty(8 * (host.n_slots // _ffi.KDL_TILE), dtype=torch.int32, device=device)
    ptr = {f: int(t.data_ptr()) for f, t in tensors.items()}
    if host.n_masked:
        qmask = make_qmask(host, ptr)
    return DeviceBatch(host=host, device=device, tensors=tensors, struct=make_struct(host, ptr), qmask=qmask)


def raise_like_reference(status: int, read: int, nibble: int, op_index: int):
    if status == _ffi.KDL_ERR_KEY:
        exc = KeyError(NIBBLES[nibble])  # e.g. KeyError('R'): kindel.py:52,72,79
    else:
        exc = IndexError("list index out of range (read %d, CIGAR op %d walks off its contig or its SEQ)"
                         % (read, op_index))
    exc.kdl_read = int(read)  # which read of the batch raised (the sharded driver orders errors by it)
    raise exc


class CountTable:
    """A count table [19, n_slots] that is REUSED across pileups without being memset.

    It remembers which slot range earlier pileups may have dirtied and whether the non-weight
    columns (5..18: indels, clips -- only complex reads write them) are dirty, and asks the kernels
    to overwrite / zero exactly that (KDL_PILEUP_FRESH_WEIGHTS / KDL_PILEUP_ZERO_REST) instead of
    clearing 76 bytes per slot every time.  Inside columns 5..18 its dirty-sector map (`dirty_map`,
    kdl_pileup_range_map) narrows the zeroing to the 32-byte sectors complex reads wrote.

    A table adopted from a caller's tensor starts with every sector marked dirty.  Setting `dirty_rest = True`
    from outside says columns 5..18 were written by other means: every sector is marked dirty again."""

    def __init__(self, n_slots: int, device, tensor: torch.Tensor = None):
        self.n_slots = n_slots
        self.device = device
        self.t = tensor if tensor is not None else torch.zeros((_ffi.KDL_NCOL, n_slots), dtype=torch.int32,
                                                                device=device)
        # uint32 per word (held as int32): 16 bytes per 64-slot window, byte b = column 5 + b, bit s = sector s
        self.dirty_map = torch.full((4 * ((n_slots + 63) // 64),), 0 if tensor is None else -1, dtype=torch.int32,
                                    device=device)
        self.dirty = None         # (lo, hi) slot range holding counts of an earlier pileup
        self._dirty_rest = False  # columns 5..18 non-zero somewhere inside `dirty` (where: dirty_map)

    @property
    def dirty_rest(self) -> bool:
        return self._dirty_rest

    @dirty_rest.setter
    def dirty_rest(self, value: bool):
        if value:
            self.dirty_map.fill_(-1)
        self._dirty_rest = bool(value)


def _tile_align(lo: int, hi: int, n_slots: int):
    t = _ffi.KDL_TILE
    return max(0, lo // t * t), min(n_slots, (hi + t - 1) // t * t)


def pileup(dbatch: DeviceBatch, counts: torch.Tensor = None, check: bool = True, table: CountTable = None,
           slot_range=None):
    """K1 (+ K1q when the batch has masked bases, + K10u when it has dropped mate ops).  Returns (counts int32[19, n_slots], events int32[n_events, 4]) on
    the device.

    counts=<tensor>  accumulate into a table the caller zeroed (several batches / shards may add up).
    table=<CountTable>  fresh result in a reused table: nothing is memset, the kernels overwrite the
                     weight columns and zero the others only if an earlier pileup dirtied them.
                     slot_range = (lo, hi) bounds what the batch can touch (default: everything).
    With check=True the error flag is read back (one 16-byte D2H) and, if set, the exact first
    offending read is located on the device and the reference's exception is raised."""
    lib = _ffi.load()
    dev = dbatch.device
    n_slots = dbatch.n_slots
    with torch.cuda.device(dev):
        # scratch that lives with the batch: the insertion-event rows and the 16-byte error flag
        events = dbatch.tensors.get("_events")
        if events is None:
            events = dbatch.tensors["_events"] = torch.empty((max(dbatch.host.n_events, 1), 4), dtype=torch.int32,
                                                             device=dev)
            dbatch.tensors["_flag"] = torch.zeros(4, dtype=torch.int32, device=dev)
        flag = dbatch.tensors["_flag"]
        if check:
            flag.zero_()  # unchecked calls (hot loops) never read it
        if table is not None:
            counts = table.t
            lo, hi = slot_range if slot_range is not None else (0, n_slots)
            if table.dirty is not None:
                lo, hi = min(lo, table.dirty[0]), max(hi, table.dirty[1])
            lo, hi = _tile_align(lo, hi, n_slots)
            flags = _ffi.KDL_PILEUP_FRESH_WEIGHTS | (_ffi.KDL_PILEUP_ZERO_REST if table.dirty_rest else 0)
            rc = lib.kdl_pileup_range_map(C.byref(dbatch.struct), counts.data_ptr(), n_slots, lo, hi, flags,
                                          table.dirty_map.data_ptr(), events.data_ptr(), flag.data_ptr(),
                                          _stream_ptr(dev))
            table.dirty = (lo, hi)
            table._dirty_rest = dbatch.host.n_complex > 0  # (the kernels marked where in the map)
        else:
            if counts is None:
                counts = torch.zeros((_ffi.KDL_NCOL, n_slots), dtype=torch.int32, device=dev)
            rc = lib.kdl_pileup(C.byref(dbatch.struct), counts.data_ptr(), n_slots, events.data_ptr(),
                                flag.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_pileup")
        if dbatch.qmask is not None:
            # K1q only touches columns 5..18 (clip bases) for complex reads, which already mark them dirty
            assert table is None or table.dirty_rest or dbatch.host.n_complex == 0
            rc = lib.kdl_unmask(C.byref(dbatch.struct), C.byref(dbatch.qmask), counts.data_ptr(), n_slots,
                                _stream_ptr(dev))
            _ffi.check(rc, "kdl_unmask")
        if dbatch.drops is not None and dbatch.drops.shape[0]:
            # K10u: only columns 5 and 6 of complex reads, whose sectors the pileup already marked dirty
            rc = lib.kdl_overlap_untake(dbatch.drops.data_ptr(), int(dbatch.drops.shape[0]), counts.data_ptr(), n_slots,
                                        _stream_ptr(dev))
            _ffi.check(rc, "kdl_overlap_untake")
        if check and int(flag[0].item()) != 0:
            diagnose_and_raise(dbatch)
    return counts, events[: dbatch.host.n_events]


def diagnose_and_raise(dbatch: DeviceBatch):
    lib = _ffi.load()
    dev = dbatch.device
    diag = torch.zeros(6, dtype=torch.int32, device=dev)  # sizeof(kdl_diag) == 24
    rc = lib.kdl_diagnose(C.byref(dbatch.struct), diag.data_ptr(), _stream_ptr(dev))
    _ffi.check(rc, "kdl_diagnose")
    raw = diag.cpu().numpy().tobytes()
    d = _ffi.KdlDiag.from_buffer_copy(raw)
    if d.status:
        raise_like_reference(d.status, d.read, d.nibble, d.op_index)
    raise RuntimeError("pileup raised its error flag but no offending read was found")


def check_iupac_threshold(t):
    """None (off) or a float in [0, 1]; anything else (NaN included) raises ValueError."""
    if t is None:
        return None
    t = float(t)
    if not 0.0 <= t <= 1.0:
        raise ValueError("iupac_threshold must lie in [0, 1], got %r" % t)
    return t


def vote(counts: torch.Tensor, min_depth=1, out: torch.Tensor = None, iupac_threshold=None) -> torch.Tensor:
    """K2.  counts int32[>=7, n_slots] (contiguous) -> calls uint8[n_slots] (`out` reuses a buffer).
    iupac_threshold (extension, default None = off): the IUPAC vote of kdl_vote_iupac, multi-base calls as IUPAC
    codes (bit 7 of the call byte)."""
    t = check_iupac_threshold(iupac_threshold)
    lib = _ffi.load()
    dev = counts.device
    n_slots = counts.shape[1]
    with torch.cuda.device(dev):
        calls = out if out is not None else torch.empty(n_slots, dtype=torch.uint8, device=dev)
        if t is None:
            rc = lib.kdl_vote(counts.data_ptr(), n_slots, int(math.ceil(min_depth)), calls.data_ptr(),
                              _stream_ptr(dev))
            _ffi.check(rc, "kdl_vote")
        else:
            rc = lib.kdl_vote_iupac(counts.data_ptr(), n_slots, int(math.ceil(min_depth)), t, calls.data_ptr(),
                                    _stream_ptr(dev))
            _ffi.check(rc, "kdl_vote_iupac")
    return calls


def derive(counts: torch.Tensor) -> torch.Tensor:
    """Derived columns [5, n_slots]: consensus_depth, clip_start_depth, clip_end_depth, clip_depth,
    acgt_depth (kindel.py:83-96, :450)."""
    lib = _ffi.load()
    dev = counts.device
    n_slots = counts.shape[1]
    with torch.cuda.device(dev):
        out = torch.empty((5, n_slots), dtype=torch.int32, device=dev)
        rc = lib.kdl_derive(counts.data_ptr(), n_slots, out.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_derive")
    return out


def cdr_flags(counts: torch.Tensor, slot_lo: int, slot_hi: int, clip_decay_threshold: float):
    """K4: (flags uint8[slot_hi - slot_lo], bases uint8[...]) on the host for slots [slot_lo, slot_hi): the
    --realign predicates (kindel.py:182-185,202,243-246,256), 2 bytes per slot instead of the 76-byte table row."""
    lib = _ffi.load()
    dev = counts.device
    n_slots = counts.shape[1]
    with torch.cuda.device(dev):
        flags = torch.empty(n_slots, dtype=torch.uint8, device=dev)
        bases = torch.empty(n_slots, dtype=torch.uint8, device=dev)
        rc = lib.kdl_cdr_flags(counts.data_ptr(), n_slots, int(slot_lo), int(slot_hi), float(clip_decay_threshold),
                               flags.data_ptr(), bases.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_cdr_flags")
    return flags[slot_lo:slot_hi].cpu().numpy(), bases[slot_lo:slot_hi].cpu().numpy()


def consensus_qual(counts: torch.Tensor, calls: torch.Tensor) -> torch.Tensor:
    """K2q (extension): the Phred quality 0..60 of the base every slot emits, uint8[n_slots] on the device, from the
    call bytes of any vote over `counts` (int32[>= 4, n_slots], contiguous; n_slots % 4 == 0).  The rule:
    kindel_b200/quality.py."""
    lib = _ffi.load()
    dev = counts.device
    n_slots = counts.shape[1]
    with torch.cuda.device(dev):
        qual = torch.empty(n_slots, dtype=torch.uint8, device=dev)
        rc = lib.kdl_consensus_qual(counts.data_ptr(), calls.data_ptr(), n_slots, qual.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_consensus_qual")
    return qual


def assemble(calls: torch.Tensor, host: ReadBatch, ins_slots: np.ndarray, ins_strings, qual: torch.Tensor = None,
             ins_qual=None):
    """K5: consensus text of every contig from the device call bytes.  ins_slots (ascending) / ins_strings: the
    chosen insertion string of every slot whose call carries change 'I'.  Returns a list of str, one per contig.
    qual (extension): K2q's per-slot qualities on the device, ins_qual the Q of each inserted string (host ints, one
    per ins_slots entry); K5q then writes the Phred+33 quality text beside the consensus text and the call returns
    (texts, quality texts)."""
    lib = _ffi.load()
    dev = calls.device
    n_slots = int(calls.shape[0])
    enc = [x.encode("ascii") for x in ins_strings]
    ins_off = np.zeros(len(enc) + 1, dtype=np.uint32)
    if enc:
        ins_off[1:] = np.cumsum([len(x) for x in enc])
    blob = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    with torch.cuda.device(dev):
        def put(a):
            a = np.ascontiguousarray(a)
            return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).to(dev)

        t_slot = put(np.asarray(host.contig_slot, dtype=np.int64))
        t_len = put(np.asarray(host.contig_len, dtype=np.int32))
        t_is = put(np.asarray(ins_slots, dtype=np.int64) if len(enc) else np.zeros(1, dtype=np.int64))
        t_io = put(ins_off)
        t_ib = put(blob.copy())
        sums = torch.empty(int(lib.kdl_assemble_scratch_words(n_slots)), dtype=torch.int32, device=dev)
        offsets = torch.empty(n_slots + 1, dtype=torch.int32, device=dev)
        out = torch.empty(n_slots + int(ins_off[-1]) + 16, dtype=torch.uint8, device=dev)
        rc = lib.kdl_assemble(calls.data_ptr(), n_slots, t_slot.data_ptr(), t_len.data_ptr(), host.n_contigs,
                              t_is.data_ptr(), t_io.data_ptr(), t_ib.data_ptr(), len(enc), sums.data_ptr(),
                              offsets.data_ptr(), out.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_assemble")
        if qual is not None:
            t_iq = put(np.asarray(ins_qual, dtype=np.uint8) if len(enc) else np.zeros(1, dtype=np.uint8))
            qout = torch.empty_like(out)
            rc = lib.kdl_assemble_qual(offsets.data_ptr(), qual.data_ptr(), n_slots, t_is.data_ptr(), t_iq.data_ptr(),
                                       len(enc), qout.data_ptr(), _stream_ptr(dev))
            _ffi.check(rc, "kdl_assemble_qual")
        starts = torch.from_numpy(np.asarray(host.contig_slot, dtype=np.int64)).to(dev)
        ends = starts + torch.from_numpy(np.asarray(host.contig_len, dtype=np.int64)).to(dev)
        lo = offsets[starts].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        hi = offsets[ends].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        total = int(offsets[n_slots].item()) & 0xFFFFFFFF
        text = out[:total].cpu().numpy().tobytes()
        texts = [text[a:b].decode("ascii") for a, b in zip(lo.tolist(), hi.tolist())]
        if qual is None:
            return texts
        qtext = qout[:total].cpu().numpy().tobytes()
    return texts, [qtext[a:b].decode("ascii") for a, b in zip(lo.tolist(), hi.tolist())]


def variant_abs_floor(abs_threshold) -> int:
    """The absolute threshold as K6 takes it: for an integer count t, t > x is t > floor(x), and with counts in
    [0, 2^31) floor(x) clamped to [-1, 2^31] selects the same counts; NaN selects nothing (2^31)."""
    if isinstance(abs_threshold, (int, np.integer)):
        x = int(abs_threshold)
    else:
        x = float(abs_threshold)
        if math.isnan(x):
            return 1 << 31
        if math.isinf(x):
            return 1 << 31 if x > 0 else -1
        x = math.floor(x)
    return max(-1, min(1 << 31, x))


def variant_sites(counts: torch.Tensor, contig_slot, contig_len, abs_threshold, rel_threshold):
    """K6 (extension): the variant sites of a device table (int32[>= 6, n_slots], contiguous, n_slots % 4 == 0) --
    the positions where an allele other than the first most frequent one passes both thresholds (kindel.variant_alleles
    is the rule).  Returns (slot int64[n], counts int32[6, n], mask uint8[n]) on the host, in ascending slot order;
    bit k of mask: allele k (A, C, G, T, N, deletions) is a variant.  One 4-byte read-back sizes the result."""
    lib = _ffi.load()
    dev = counts.device
    n_slots = int(counts.shape[1])
    a, r = variant_abs_floor(abs_threshold), float(rel_threshold)
    n_contigs = len(contig_len)
    with torch.cuda.device(dev):
        t_slot = torch.from_numpy(np.ascontiguousarray(contig_slot, dtype=np.int64) if n_contigs
                                  else np.zeros(1, dtype=np.int64)).to(dev)
        t_len = torch.from_numpy(np.ascontiguousarray(contig_len, dtype=np.int32) if n_contigs
                                 else np.zeros(1, dtype=np.int32)).to(dev)
        sums = torch.empty(int(lib.kdl_variant_scratch_words(n_slots)), dtype=torch.int32, device=dev)
        args = (counts.data_ptr(), n_slots, t_slot.data_ptr(), t_len.data_ptr(), n_contigs, a, r, sums.data_ptr())
        rc = lib.kdl_variant_count(*args, _stream_ptr(dev))
        _ffi.check(rc, "kdl_variant_count")
        n = int(sums[-1].item()) & 0xFFFFFFFF
        site_slot = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        site_counts = torch.empty((6, max(n, 1)), dtype=torch.int32, device=dev)
        site_mask = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        rc = lib.kdl_variant_scatter(*args, n, site_slot.data_ptr(), site_counts.data_ptr(), site_mask.data_ptr(),
                                     _stream_ptr(dev))
        _ffi.check(rc, "kdl_variant_scatter")
        if n == 0:
            return np.zeros(0, dtype=np.int64), np.zeros((6, 0), dtype=np.int32), np.zeros(0, dtype=np.uint8)
        return site_slot.cpu().numpy(), site_counts[:, :n].cpu().numpy(), site_mask.cpu().numpy()


def _device_layout(contig_slot, contig_len, dev):
    n_contigs = len(contig_len)
    t_slot = torch.from_numpy(np.ascontiguousarray(contig_slot, dtype=np.int64) if n_contigs
                              else np.zeros(1, dtype=np.int64)).to(dev)
    t_len = torch.from_numpy(np.ascontiguousarray(contig_len, dtype=np.int32) if n_contigs
                             else np.zeros(1, dtype=np.int32)).to(dev)
    return t_slot, t_len, n_contigs


def variant_sites_ref(counts: torch.Tensor, contig_slot, contig_len, ref, abs_threshold, rel_threshold):
    """K6r (extension): the candidate sites of `variants --vcf --reference` in a device table (int32[>= 7, n_slots],
    contiguous, n_slots % 4 == 0) against reference codes `ref` (uint8[n_slots], 0-3 = A, C, G, T, 4 = other; a device
    tensor or a host array, uploaded).  Returns (slot int64[n], counts int32[7, n], dpa int64[n], mask uint8[n]) on the
    host in ascending slot order: bits 0-3 of mask are the SNV alleles A, C, G, T, bit 6 the insertion candidate, dpa
    the depth the slot's insertions are measured against (include/kindel_b200.h has the rule)."""
    lib = _ffi.load()
    dev = counts.device
    n_slots = int(counts.shape[1])
    a, r = variant_abs_floor(abs_threshold), float(rel_threshold)
    with torch.cuda.device(dev):
        if not isinstance(ref, torch.Tensor):
            ref = torch.from_numpy(np.ascontiguousarray(ref, dtype=np.uint8))
        ref = ref.to(dev).contiguous()
        if ref.dtype != torch.uint8 or ref.numel() != n_slots:
            raise ValueError("reference codes must be uint8[%d], got %s[%d]" % (n_slots, ref.dtype, ref.numel()))
        t_slot, t_len, n_contigs = _device_layout(contig_slot, contig_len, dev)
        sums = torch.empty(int(lib.kdl_variant_scratch_words(n_slots)), dtype=torch.int32, device=dev)
        args = (counts.data_ptr(), n_slots, t_slot.data_ptr(), t_len.data_ptr(), n_contigs, ref.data_ptr(), a, r,
                sums.data_ptr())
        _ffi.check(lib.kdl_variant_ref_count(*args, _stream_ptr(dev)), "kdl_variant_ref_count")
        n = int(sums[-1].item()) & 0xFFFFFFFF
        site_slot = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        site_counts = torch.empty((7, max(n, 1)), dtype=torch.int32, device=dev)
        site_dpa = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        site_mask = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        rc = lib.kdl_variant_ref_scatter(*args, n, site_slot.data_ptr(), site_counts.data_ptr(), site_dpa.data_ptr(),
                                         site_mask.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_variant_ref_scatter")
        if n == 0:
            return (np.zeros(0, dtype=np.int64), np.zeros((7, 0), dtype=np.int32), np.zeros(0, dtype=np.int64),
                    np.zeros(0, dtype=np.uint8))
        return (site_slot.cpu().numpy(), site_counts[:, :n].cpu().numpy(), site_dpa.cpu().numpy(),
                site_mask.cpu().numpy())


def variant_sites_multi(counts: torch.Tensor, contig_slot, contig_len, ref, abs_threshold, rel_threshold):
    """K6m (extension): the sites of several samples at once in a stacked device table (int32[S, 7, n_slots],
    contiguous, n_slots % 4 == 0; sample s's columns 0-6 over one shared layout).  ref None: the pooled mode (bits
    0-5, the alleles of kindel.variant_alleles tested in each sample, the pooled top left out); else reference codes
    as for variant_sites_ref (bits 0-3 SNV alleles, bit 6 the insertion candidate, each sample tested against its own
    DPa).  Each bit is ORed over the samples (include/kindel_b200.h has the rule).  Returns (slot int64[n], mask
    uint8[n]) as device tensors in ascending slot order; the samples' rows stay in `counts`."""
    lib = _ffi.load()
    dev = counts.device
    if counts.dim() != 3 or counts.shape[1] != 7 or counts.dtype != torch.int32 or not counts.is_contiguous():
        raise ValueError("the stacked table must be a contiguous int32[S, 7, n_slots], got %s %s"
                         % (counts.dtype, tuple(counts.shape)))
    n_samples, n_slots = int(counts.shape[0]), int(counts.shape[2])
    a, r = variant_abs_floor(abs_threshold), float(rel_threshold)
    with torch.cuda.device(dev):
        ref_ptr = None
        if ref is not None:
            if not isinstance(ref, torch.Tensor):
                ref = torch.from_numpy(np.ascontiguousarray(ref, dtype=np.uint8))
            ref = ref.to(dev).contiguous()
            if ref.dtype != torch.uint8 or ref.numel() != n_slots:
                raise ValueError("reference codes must be uint8[%d], got %s[%d]" % (n_slots, ref.dtype, ref.numel()))
            ref_ptr = ref.data_ptr()
        t_slot, t_len, n_contigs = _device_layout(contig_slot, contig_len, dev)
        sums = torch.empty(int(lib.kdl_variant_scratch_words(n_slots)), dtype=torch.int32, device=dev)
        args = (counts.data_ptr(), n_samples, n_slots, t_slot.data_ptr(), t_len.data_ptr(), n_contigs, ref_ptr, a, r,
                sums.data_ptr())
        _ffi.check(lib.kdl_variant_multi_count(*args, _stream_ptr(dev)), "kdl_variant_multi_count")
        n = int(sums[-1].item()) & 0xFFFFFFFF
        site_slot = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        site_mask = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        rc = lib.kdl_variant_multi_scatter(*args, n, site_slot.data_ptr(), site_mask.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_variant_multi_scatter")
    return site_slot[:n], site_mask[:n]


_SELECT_TOTALS = 16  # words of K8's totals record (include/kindel_b200.h)


def select_reads(dbatch: DeviceBatch, keep: torch.Tensor) -> DeviceBatch:
    """K8 (extension): the sub-batch of the reads with keep[r] != 0 (uint8[n_reads], device), built on the device;
    it equals bamio.select_reads(host, np.flatnonzero(keep)) field for field.  One 64-byte read-back sizes it; its
    host side is a BatchShape (scalars only), and contig_len / contig_slot are shared with the parent."""
    lib = _ffi.load()
    dev = dbatch.device
    n = int(dbatch.struct.n_reads)
    with torch.cuda.device(dev):
        keep = keep.to(dev, torch.uint8).contiguous()
        if keep.numel() != n:
            raise ValueError("keep must hold one byte per read (%d), got %d" % (n, keep.numel()))
        qmask = C.byref(dbatch.qmask) if dbatch.qmask is not None else None
        scratch = torch.empty(int(lib.kdl_select_scratch_words(n)), dtype=torch.int32, device=dev)
        args = (C.byref(dbatch.struct), qmask, keep.data_ptr() if n else None, scratch.data_ptr())
        _ffi.check(lib.kdl_select_count(*args, _stream_ptr(dev)), "kdl_select_count")
        tot = scratch[-_SELECT_TOTALS:].cpu().numpy().view(np.uint32).astype(np.int64)
        n_out, n_words, n_cx, n_hard, n_evt, n_mr, n_mb = (int(x) for x in tot[:7])

        def empty(k, dtype=torch.int32):
            return torch.empty(max(k, 1), dtype=dtype, device=dev)

        t = dict(ref_start=empty(n_out), seq_off=empty(n_out), l_seq=empty(n_out), seq4=empty(n_words),
                 contig_read_off=empty(dbatch.struct.n_contigs + 1, torch.int64), complex_idx=empty(n_cx),
                 hard_idx=empty(n_hard), contig_len=dbatch.tensors["contig_len"],
                 contig_slot=dbatch.tensors["contig_slot"],
                 tile_index=torch.empty(8 * (dbatch.n_slots // _ffi.KDL_TILE), dtype=torch.int32, device=dev))
        if n_mr:
            t.update(mask_read=empty(n_mr), mask_off=empty(n_mr + 1), mask_qpos=empty(n_mb))
        host = BatchShape(n_reads=n_out, n_words=n_words, n_contigs=int(dbatch.struct.n_contigs), n_slots=dbatch.n_slots,
                          n_complex=n_cx, n_hard=n_hard, n_events=n_evt, n_masked=n_mb, n_mask_reads=n_mr,
                          reads_sorted=bool(tot[7]), max_simple_len=int(tot[8]), reach_right=int(tot[9]),
                          reach_left=int(tot[10]))
        ptr = {f: int(x.data_ptr()) for f, x in t.items()}
        s = _ffi.KdlBatch()
        s.n_reads, s.seq4_words, s.n_contigs = n_out, n_words, host.n_contigs
        s.reads_sorted, s.max_simple_len = int(host.reads_sorted), host.max_simple_len
        s.reach_right, s.reach_left = host.reach_right, host.reach_left
        for f in ("ref_start", "seq_off", "l_seq", "seq4", "contig_read_off", "contig_len", "contig_slot", "tile_index"):
            setattr(s, f, ptr[f])
        s.n_complex, s.n_hard = n_cx, n_hard
        s.complex_idx = ptr["complex_idx"] if n_cx else None
        s.hard_idx = ptr["hard_idx"] if n_hard else None
        q = make_qmask(host, ptr) if n_mr else None
        rc = lib.kdl_select_scatter(*args, C.byref(s), C.byref(q) if q is not None else None, _stream_ptr(dev))
        _ffi.check(rc, "kdl_select_scatter")
        drops = None
        if dbatch.drops is not None:  # the kept reads' drop rows, their read numbers those of the sub-batch
            kept = keep[dbatch.drops[:, 2].long()] != 0
            drops = dbatch.drops[kept].clone()
            drops[:, 2] = (torch.cumsum(keep.to(torch.int64), 0) - 1).index_select(0, drops[:, 2].long()).to(torch.int32)
    return DeviceBatch(host=host, device=dev, tensors=t, struct=s, qmask=q, drops=drops)


_PRIMER_TOTALS = 8  # words of K9's totals record (include/kindel_b200.h)


def primers_struct(arrays, ptr: dict) -> _ffi.KdlPrimers:
    """kdl_primers over the pointers `ptr` of a primers.PrimerArrays' fields."""
    p = _ffi.KdlPrimers()
    p.n_contigs, p.n_intervals = arrays.n_contigs, arrays.n_intervals
    for f in ("contig_off", "start_sorted", "end_max", "end_sorted", "start_min"):
        setattr(p, f, ptr[f])
    return p


def mask_primers(dbatch: DeviceBatch, arrays) -> DeviceBatch:
    """K9 (extension: `--primers`): the batch with every read's primer bases masked (include/kindel_b200.h has the
    rule), as min_base_quality masks a base: N in seq4 and listed in the mask list, whose count K1q takes back.

    `arrays`: primers.PrimerArrays over the batch's contigs.  The nibbles are written into the batch's own device seq4,
    in place -- the upload of one run, which nothing else reads -- and the result shares every tensor with `dbatch`
    except the mask list, the union of the batch's own and the primer bases.  So `dbatch` itself must not be piled
    after this call.  One 32-byte read-back sizes the list; a batch without a primer base comes back as it is.  The
    host ReadBatch is never touched.  `primer_masked` of the result = (reads, bases) masked by the primers.  A batch
    that already carries drop rows (mask_overlaps) keeps them."""
    lib = _ffi.load()
    dev = dbatch.device
    n = int(dbatch.struct.n_reads)
    if arrays.n_contigs != int(dbatch.struct.n_contigs):
        raise ValueError("primer arrays for %d contigs, the batch has %d" % (arrays.n_contigs, dbatch.struct.n_contigs))
    if arrays.n_intervals == 0 or n == 0:
        return dbatch
    with torch.cuda.device(dev):
        t = {f: torch.from_numpy(np.ascontiguousarray(getattr(arrays, f))).to(dev)
             for f in ("contig_off", "start_sorted", "end_max", "end_sorted", "start_min")}
        p = primers_struct(arrays, {f: int(x.data_ptr()) for f, x in t.items()})
        qmask = C.byref(dbatch.qmask) if dbatch.qmask is not None else None
        scratch = torch.empty(int(lib.kdl_primers_scratch_words(n)), dtype=torch.int32, device=dev)
        args = (C.byref(dbatch.struct), qmask, C.byref(p), scratch.data_ptr())
        _ffi.check(lib.kdl_primers_count(*args, _stream_ptr(dev)), "kdl_primers_count")
        tot = scratch[-_PRIMER_TOTALS:].cpu().numpy().view(np.uint32).astype(np.int64)
        n_mr, n_mb, n_pr, n_pb = (int(x) for x in tot[:4])
        if n_pb == 0:
            return dbatch
        tensors = dict(dbatch.tensors)
        tensors.update(mask_read=torch.empty(n_mr, dtype=torch.int32, device=dev),
                       mask_off=torch.empty(n_mr + 1, dtype=torch.int32, device=dev),
                       mask_qpos=torch.empty(n_mb, dtype=torch.int32, device=dev))
        q = _ffi.KdlQmask()
        q.n_reads, q.n_bases = n_mr, n_mb
        q.read_idx, q.off, q.qpos = (int(tensors[f].data_ptr()) for f in ("mask_read", "mask_off", "mask_qpos"))
        rc = lib.kdl_primers_apply(*args, int(dbatch.tensors["seq4"].data_ptr()), C.byref(q), _stream_ptr(dev))
        _ffi.check(rc, "kdl_primers_apply")
    return DeviceBatch(host=dbatch.host, device=dev, tensors=tensors, struct=dbatch.struct, qmask=q,
                       primer_masked=(n_pr, n_pb), drops=dbatch.drops, overlap_masked=dbatch.overlap_masked)


_AMPLICON_FIELDS = ("left_off", "left_at", "left_label", "right_off", "right_at", "right_label", "contig",
                    "insert_start", "insert_end")


def amplicons_struct(arrays, ptr: dict) -> _ffi.KdlAmplicons:
    """kdl_amplicons over the pointers `ptr` of a primers.AmpliconArrays' fields."""
    a = _ffi.KdlAmplicons()
    a.n_contigs, a.n_amplicons = arrays.n_contigs, arrays.n_amplicons
    for f in _AMPLICON_FIELDS:
        setattr(a, "amp_contig" if f == "contig" else f, ptr[f])
    return a


def _amplicons_on(arrays, dev):
    """(kdl_amplicons, keepalive tensors) of the arrays uploaded to `dev`."""
    t = {f: torch.from_numpy(np.ascontiguousarray(getattr(arrays, f))).to(dev) for f in _AMPLICON_FIELDS}
    return amplicons_struct(arrays, {f: (int(x.data_ptr()) if x.numel() else None) for f, x in t.items()}), t


def assign_amplicons(dbatch: DeviceBatch, arrays) -> torch.Tensor:
    """K12 (extension: `kindel amplicons`): int32 [n_reads] on the device, each read's amplicon -- an index into
    `arrays` (primers.AmpliconArrays over the batch's contigs) -- or -1 (unprimed), -2 (mispaired), -3 (ambiguous);
    include/kindel_b200.h has the rule.  Reads the batch's CIGARs and starts only, so a primer-masked batch gives the
    same labels."""
    lib = _ffi.load()
    dev = dbatch.device
    n = int(dbatch.struct.n_reads)
    if arrays.n_contigs != int(dbatch.struct.n_contigs):
        raise ValueError("amplicon arrays for %d contigs, the batch has %d" % (arrays.n_contigs, dbatch.struct.n_contigs))
    with torch.cuda.device(dev):
        label = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        a, keep = _amplicons_on(arrays, dev)
        rc = lib.kdl_amplicons_assign(C.byref(dbatch.struct), C.byref(a), label.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_amplicons_assign")
        del keep  # (the stream orders the kernel before any reuse of the freed blocks)
    return label[:n]


def amplicon_depth(counts: torch.Tensor, arrays, min_depth, contig_slot, contig_len) -> torch.Tensor:
    """K12d (extension: `kindel amplicons`): int64 [n_amplicons, 3] on the device -- per amplicon of `arrays` the sum,
    the minimum and the number of positions >= min_depth of A+C+G+T (columns 0-3 of `counts`) over its insert; the
    table's layout is contig_slot / contig_len (the batch's)."""
    lib = _ffi.load()
    dev = counts.device
    n = arrays.n_amplicons
    with torch.cuda.device(dev):
        stats = torch.zeros((max(n, 1), 3), dtype=torch.int64, device=dev)
        slot, length, n_contigs = _device_layout(contig_slot, contig_len, dev)
        a, keep = _amplicons_on(arrays, dev)
        rc = lib.kdl_amplicons_depth(counts.data_ptr(), int(counts.shape[1]), slot.data_ptr(), length.data_ptr(),
                                     n_contigs, C.byref(a), int(math.ceil(min_depth)), stats.data_ptr(),
                                     _stream_ptr(dev))
        _ffi.check(rc, "kdl_amplicons_depth")
        del keep
    return stats[:n]


def normalise(label: torch.Tensor, reverse: torch.Tensor, n_amplicons: int, cap: int):
    """K13 (extension: `--normalise N`): (keep uint8 [n], total int32 [2 * n_amplicons], dropped int64 [1]) on the
    device.  keep[r] = 0 for a read with an amplicon label (K12's, `label`) that has `cap` reads of its amplicon and
    strand (`reverse`, 1 = FLAG & 0x10) before it in the batch, else 1; total = the reads of each (amplicon, strand),
    2 * amplicon + strand; dropped = the reads with keep 0.  include/kindel_b200.h has the rule."""
    lib = _ffi.load()
    dev = label.device
    n = int(label.numel())
    if int(reverse.numel()) != n:
        raise ValueError("normalise: %d labels and %d strand bytes" % (n, int(reverse.numel())))
    with torch.cuda.device(dev):
        label = label.to(torch.int32).contiguous()
        reverse = reverse.to(torch.uint8).contiguous()
        words = int(lib.kdl_normalise_scratch_words(n, int(n_amplicons)))
        scratch = torch.empty(max(words, 1), dtype=torch.int32, device=dev)
        keep = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        total = torch.empty(max(2 * int(n_amplicons), 1), dtype=torch.int32, device=dev)
        dropped = torch.empty(1, dtype=torch.int64, device=dev)
        rc = lib.kdl_normalise(label.data_ptr(), reverse.data_ptr(), n, int(n_amplicons), int(cap), scratch.data_ptr(),
                               words, keep.data_ptr(), total.data_ptr(), dropped.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_normalise")
    return keep[:n], total[:2 * int(n_amplicons)], dropped


def _lexsort(keys):
    """int64 permutation that orders the rows by `keys` (device tensors, most significant first): one stable
    torch.sort per key, least significant first."""
    perm = None
    for k in reversed(keys):
        idx = torch.sort(k if perm is None else k.index_select(0, perm), stable=True)[1]
        perm = idx if perm is None else perm.index_select(0, idx)
    return perm.contiguous()


_DEDUP_LISTS = (("pair_contig", torch.int32, 0), ("pair_e1", torch.int64, 0), ("pair_e2", torch.int64, 0),
                ("pair_rank", torch.int64, 0), ("pair_r1", torch.int32, 0), ("pair_r2", torch.int32, 0),
                ("single_contig", torch.int32, 1), ("single_key", torch.int64, 1), ("single_rank", torch.int64, 1),
                ("single_read", torch.int32, 1), ("end", torch.int64, 1), ("paired", torch.uint8, 1))


def dedup(dbatch: DeviceBatch, mate: torch.Tensor = None):
    """K14 (extension: `--dedup`): (keep uint8 [n] on the device, (pairs removed, singles removed, singles shadowed by
    a pair end)).  keep[r] = 0 for a read that duplicate removal takes out (include/kindel_b200.h has the rule).  Needs a
    host batch decoded with strand and dup (its `reverse` and `dup_score`); mate: K10p's result, run here when the
    batch has its mates and mate is None (no mates: every read is a single).  K14k fills the two entry lists; one
    read-back of the totals record sizes them; each is sorted by key on the device (stable torch.sort passes); K14s
    selects, and a second read-back gives the totals."""
    h = dbatch.host
    if getattr(h, "dup_score", None) is None or getattr(h, "reverse", None) is None:
        raise ValueError("dedup needs the reads' strands and duplicate scores: decode with strand=True, dup=True")
    lib = _ffi.load()
    dev = dbatch.device
    n = int(dbatch.struct.n_reads)
    if mate is None and getattr(h, "mates", None) is not None:
        mate = pair_mates(dbatch)
    with torch.cuda.device(dev):
        reverse = torch.from_numpy(np.ascontiguousarray(h.reverse, dtype=np.uint8)).to(dev)
        score = torch.from_numpy(np.ascontiguousarray(h.dup_score, dtype=np.int32)).to(dev)
        if mate is not None:
            mate = mate.to(dev, torch.int32).contiguous()
        t = {f: torch.empty(max(n if full else n // 2, 1), dtype=dt, device=dev) for f, dt, full in _DEDUP_LISTS}
        lists = _ffi.KdlDedupLists(*(int(t[f].data_ptr()) for f, _, _ in _DEDUP_LISTS))
        keep = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        totals = torch.zeros(_ffi.KDL_DEDUP_TOTALS, dtype=torch.int64, device=dev)
        rc = lib.kdl_dedup_entries(C.byref(dbatch.struct), reverse.data_ptr(), score.data_ptr(),
                                   mate.data_ptr() if mate is not None and n else None, C.byref(lists),
                                   keep.data_ptr(), totals.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_dedup_entries")
        n_pair, n_single = (int(x) for x in totals[:2].cpu())
        one = int(dbatch.struct.n_contigs) <= 1  # (one contig: its key needs no pass)
        pk = [t["pair_e1"][:n_pair], t["pair_e2"][:n_pair]]
        sk = [t["single_key"][:n_single]]
        p_order = _lexsort(pk if one else [t["pair_contig"][:n_pair]] + pk) if n_pair else None
        s_order = _lexsort(sk if one else [t["single_contig"][:n_single]] + sk) if n_single else None
        words = int(lib.kdl_dedup_scratch_words(max(n_pair, n_single)))
        scratch = torch.empty(max(words, 2), dtype=torch.int32, device=dev)
        rc = lib.kdl_dedup_select(C.byref(lists), p_order.data_ptr() if n_pair else None, n_pair,
                                  s_order.data_ptr() if n_single else None, n_single, scratch.data_ptr(), words,
                                  keep.data_ptr(), totals.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_dedup_select")
        stats = tuple(int(x) for x in totals[2:5].cpu())
    return keep[:n], stats


_OVERLAP_TOTALS = 8  # words of K10's totals record (include/kindel_b200.h)


def pair_mates(dbatch: DeviceBatch, order: torch.Tensor = None) -> torch.Tensor:
    """K10p (extension: `--mask-overlaps`): int32[n_reads] on the device, the R1 of every paired R2 and -1 elsewhere
    (include/kindel_b200.h has the rule).  The reads with pair_role != 0 are compacted and sorted by name hash here
    (torch, on the device); `order` gives that sorted index list instead.  Needs a host batch decoded with mates."""
    h = dbatch.host
    if getattr(h, "mates", None) is None:
        raise ValueError("mask_overlaps needs the reads' mates: decode the batch with mates=True")
    lib = _ffi.load()
    dev = dbatch.device
    n = h.n_reads
    with torch.cuda.device(dev):
        t_hash = torch.from_numpy(np.ascontiguousarray(h.name_hash, dtype=np.uint64).view(np.int64)).to(dev)
        t_mate = torch.from_numpy(np.ascontiguousarray(h.mate_start, dtype=np.int32)).to(dev)
        t_role = torch.from_numpy(np.ascontiguousarray(h.pair_role, dtype=np.uint8)).to(dev)
        if order is None:
            idx = torch.nonzero(t_role, as_tuple=True)[0]
            order = idx.index_select(0, torch.sort(t_hash.index_select(0, idx), stable=True)[1])
        order = order.to(dev, torch.int32).contiguous()
        mate = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        rc = lib.kdl_mates_pair(C.byref(dbatch.struct), t_hash.data_ptr(), t_mate.data_ptr(), t_role.data_ptr(),
                                order.data_ptr(), int(order.numel()), mate.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_mates_pair")
    return mate[:n]


def mask_overlaps(dbatch: DeviceBatch, mate: torch.Tensor = None) -> DeviceBatch:
    """K10 (extension: `--mask-overlaps`): the batch with every read pair's second mate (R2) masked where the first
    (R1) covers it, as min_base_quality masks a base, and the drop rows of R2's deletions and insertions there, whose
    counts pileup takes back after K1q (K10u).  include/kindel_b200.h has the rule.

    mate: K10p's result (pair_mates runs when it is None).  Like mask_primers, the nibbles are written into the batch's
    own device seq4 -- run it after mask_primers, so that primer-masked R1 bases cover nothing -- and the result shares
    every tensor with `dbatch` but the mask list; `dbatch` must not be piled after this call.  One 32-byte read-back
    sizes the outputs.  `overlap_masked` of the result = (pairs, bases, deletions, insertions)."""
    lib = _ffi.load()
    dev = dbatch.device
    n = int(dbatch.struct.n_reads)
    if mate is None:
        mate = pair_mates(dbatch)
    with torch.cuda.device(dev):
        mate = mate.to(dev, torch.int32).contiguous()
        qmask = C.byref(dbatch.qmask) if dbatch.qmask is not None else None
        scratch = torch.empty(int(lib.kdl_overlap_scratch_words(n)), dtype=torch.int32, device=dev)
        args = (C.byref(dbatch.struct), qmask, mate.data_ptr() if n else None, scratch.data_ptr())
        _ffi.check(lib.kdl_overlap_count(*args, _stream_ptr(dev)), "kdl_overlap_count")
        tot = scratch[-_OVERLAP_TOTALS:].cpu().numpy().view(np.uint32).astype(np.int64)
        n_mr, n_mb, n_drops, n_pairs, n_ob, n_od, n_oi = (int(x) for x in tot[:7])
        drops = torch.empty((n_drops, 4), dtype=torch.int32, device=dev)
        stats = (n_pairs, n_ob, n_od, n_oi)
        if n_ob == 0 and n_drops == 0:
            return dataclasses.replace(dbatch, drops=drops, overlap_masked=stats)
        tensors = dict(dbatch.tensors)
        q = dbatch.qmask
        if n_ob:
            tensors.update(mask_read=torch.empty(n_mr, dtype=torch.int32, device=dev),
                           mask_off=torch.empty(n_mr + 1, dtype=torch.int32, device=dev),
                           mask_qpos=torch.empty(n_mb, dtype=torch.int32, device=dev))
            q = _ffi.KdlQmask()
            q.n_reads, q.n_bases = n_mr, n_mb
            q.read_idx, q.off, q.qpos = (int(tensors[f].data_ptr()) for f in ("mask_read", "mask_off", "mask_qpos"))
        # (no overlap base: the merged list is the batch's own, and only the drop rows are written)
        out = C.byref(q) if n_ob and n_mr else None
        rc = lib.kdl_overlap_apply(*args, int(dbatch.tensors["seq4"].data_ptr()), out,
                                   drops.data_ptr() if n_drops else None, n_drops, _stream_ptr(dev))
        _ffi.check(rc, "kdl_overlap_apply")
    return dataclasses.replace(dbatch, tensors=tensors, qmask=q, drops=drops, overlap_masked=stats)


def quality_sums(dbatch: DeviceBatch, qual8: torch.Tensor):
    """K0 + K11 (+ K11g): (qsum int32 [4, n_slots] holding uint32 bits, emass int64 [n_slots] holding uint64 bits) on
    the device -- per slot the summed Phred of the counted A / C / G / T bases and the summed EPS of all of them
    (include/kindel_b200.h kdl_quality_pileup).  qual8: uint8 [8 * words of seq4] on the batch's device.  Reads the
    batch's seq4 as it is now, so after K9 / K10 a primer or overlap base counts nowhere; the batch's tile-index
    scratch is rebuilt."""
    lib = _ffi.load()
    dev = dbatch.device
    n_slots = dbatch.n_slots
    with torch.cuda.device(dev):
        qsum = torch.empty((4, n_slots), dtype=torch.int32, device=dev)
        emass = torch.empty(n_slots, dtype=torch.int64, device=dev)
        q = qual8 if qual8.numel() else torch.zeros(8, dtype=torch.uint8, device=dev)
        rc = lib.kdl_quality_pileup(C.byref(dbatch.struct), q.data_ptr(), qsum.data_ptr(), emass.data_ptr(), n_slots,
                                    _stream_ptr(dev))
        _ffi.check(rc, "kdl_quality_pileup")
    return qsum, emass


def quality_weights(dbatch: DeviceBatch, qual8: torch.Tensor) -> torch.Tensor:
    """K0 + K11w (+ K11g-w): wsum int64 [4, n_slots] holding uint64 bits on the device -- per slot the summed
    weight W[min(q, 93)] (kindel_b200/quality.py WEIGHT) of the counted A / C / G / T bases (include/kindel_b200.h
    kdl_quality_weights).  The counted bases and qual8 are quality_sums'."""
    lib = _ffi.load()
    dev = dbatch.device
    n_slots = dbatch.n_slots
    with torch.cuda.device(dev):
        wsum = torch.empty((4, n_slots), dtype=torch.int64, device=dev)
        q = qual8 if qual8.numel() else torch.zeros(8, dtype=torch.uint8, device=dev)
        rc = lib.kdl_quality_weights(C.byref(dbatch.struct), q.data_ptr(), wsum.data_ptr(), n_slots, _stream_ptr(dev))
        _ffi.check(rc, "kdl_quality_weights")
    return wsum


def vote_quality(counts: torch.Tensor, wsum: torch.Tensor, min_depth=1, out: torch.Tensor = None):
    """K2w (extension: quality_vote): (calls uint8[n_slots], qual uint8[n_slots]) on the device.  The change bits are
    kdl_vote's; the emitted base is the one with the largest summed weight in wsum (quality_weights), N on a tie or
    when no base has weight; qual is its Q (include/kindel_b200.h kdl_vote_quality)."""
    lib = _ffi.load()
    dev = counts.device
    n_slots = counts.shape[1]
    with torch.cuda.device(dev):
        calls = out if out is not None else torch.empty(n_slots, dtype=torch.uint8, device=dev)
        qual = torch.empty(n_slots, dtype=torch.uint8, device=dev)
        rc = lib.kdl_vote_quality(counts.data_ptr(), wsum.data_ptr(), n_slots, int(math.ceil(min_depth)),
                                  calls.data_ptr(), qual.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_vote_quality")
    return calls, qual


def dropped_event_rows(dbatch: DeviceBatch) -> np.ndarray:
    """The insertion-event rows K10 dropped (int64, ascending) -- the rows no insertion string may read."""
    if dbatch.drops is None or dbatch.drops.shape[0] == 0:
        return np.zeros(0, dtype=np.int64)
    evt = dbatch.drops[:, 3].cpu().numpy().astype(np.int64)
    return np.sort(evt[evt >= 0])


def download_fields(dbatch: DeviceBatch) -> dict:
    """The device arrays and scalars of a batch, as host numpy (for checking a K8 result against the host's)."""
    h = dbatch.host
    sizes = dict(ref_start=h.n_reads, seq_off=h.n_reads, l_seq=h.n_reads, contig_read_off=h.n_contigs + 1,
                 complex_idx=h.n_complex, hard_idx=h.n_hard)
    sizes["seq4"] = h.n_words if isinstance(h, BatchShape) else int(h.seq4.shape[0])
    if h.n_masked:
        sizes.update(mask_read=h.n_mask_reads, mask_off=h.n_mask_reads + 1, mask_qpos=h.n_masked)
    out = {f: dbatch.tensors[f][:k].cpu().numpy() for f, k in sizes.items()}
    for f in ("seq_off", "seq4", "complex_idx", "hard_idx", "mask_read", "mask_off", "mask_qpos"):
        if f in out:
            out[f] = out[f].view(np.uint32)
    if not h.n_masked:
        out.update(mask_read=None, mask_off=None, mask_qpos=None)
    out.update(n_events=h.n_events, reads_sorted=bool(h.reads_sorted), max_simple_len=int(h.max_simple_len),
               reach_right=int(h.reach_right), reach_left=int(h.reach_left))
    return out


def deletion_events(dbatch: DeviceBatch):
    """K7 (extension): every deletion event (slot, length) of the batch's CIGARs, in read order and then op order, as
    device tensors (int64[m], int32[m]).  A D op is an event when it lies inside its contig (include/kindel_b200.h)."""
    lib = _ffi.load()
    dev = dbatch.device
    with torch.cuda.device(dev):
        sums = torch.empty(int(lib.kdl_deletion_scratch_words(dbatch.host.n_reads)), dtype=torch.int32, device=dev)
        _ffi.check(lib.kdl_deletion_count(C.byref(dbatch.struct), sums.data_ptr(), _stream_ptr(dev)),
                   "kdl_deletion_count")
        m = int(sums[-1].item()) & 0xFFFFFFFF
        ev_slot = torch.empty(max(m, 1), dtype=torch.int64, device=dev)
        ev_len = torch.empty(max(m, 1), dtype=torch.int32, device=dev)
        rc = lib.kdl_deletion_scatter(C.byref(dbatch.struct), sums.data_ptr(), m, ev_slot.data_ptr(), ev_len.data_ptr(),
                                      _stream_ptr(dev))
        _ffi.check(rc, "kdl_deletion_scatter")
    return ev_slot[:m], ev_len[:m]


_LEN_BITS = 28  # a CIGAR op length has 28 bits


def _deletion_groups(dbatch: DeviceBatch, ref: torch.Tensor = None):
    """K7's events grouped by (slot, length) on the device: (key = slot << 28 | length, count), keys ascending.  The
    deletions K10 dropped (mask_overlaps) are subtracted by the same key, and groups left empty are removed.  ref
    (extension: left_align): the device reference codes of the batch's slots; the groups are then left-aligned
    against them (left_align_deletions) after the drops are subtracted."""
    ev_slot, ev_len = deletion_events(dbatch)
    with torch.cuda.device(dbatch.device):
        key, cnt = torch.unique((ev_slot << _LEN_BITS) | ev_len.to(torch.int64), sorted=True, return_counts=True)
        d = dbatch.drops
        if d is not None and key.numel():
            d = d[d[:, 3] < 0]
        if d is not None and key.numel() and d.shape[0]:
            dk, dc = torch.unique((d[:, 0].to(torch.int64) << _LEN_BITS) | d[:, 1].to(torch.int64), return_counts=True)
            at = torch.searchsorted(key, dk).clamp(max=key.numel() - 1)
            cnt = cnt.clone()
            cnt.index_add_(0, at, torch.where(key[at] == dk, -dc, torch.zeros_like(dc)))  # (each is one of the events)
            live = cnt > 0
            key, cnt = key[live], cnt[live]
        if ref is None:
            return key, cnt
        return left_align_deletions(key, cnt, ref, dbatch.tensors["contig_slot"], int(dbatch.struct.n_contigs))


def left_align_deletions(key: torch.Tensor, cnt: torch.Tensor, ref: torch.Tensor, contig_slot: torch.Tensor,
                         n_contigs: int):
    """K15d (extension: left_align): deletion groups (key = slot << 28 | length, count; device tensors) moved to their
    leftmost place against the device reference codes `ref` (uint8 [n_slots]) over the layout's first slots
    (contig_slot, int64 device), and grouped again: (key, count) with the counts of keys that met summed, keys
    ascending.  include/kindel_b200.h has the rule."""
    lib = _ffi.load()
    dev = key.device
    with torch.cuda.device(dev):
        n = int(key.numel())
        if n == 0:
            return key, cnt
        key = key.contiguous()
        moved = torch.empty_like(key)
        rc = lib.kdl_left_align_deletions(key.data_ptr(), n, contig_slot.data_ptr(), int(n_contigs), ref.data_ptr(),
                                          moved.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_left_align_deletions")
        out, inv = torch.unique(moved, sorted=True, return_inverse=True)
        total = torch.zeros(out.numel(), dtype=cnt.dtype, device=dev).index_add_(0, inv, cnt)
    return out, total


def left_align_insertions(dbatch: DeviceBatch, events: torch.Tensor, ref: torch.Tensor, dead: torch.Tensor = None):
    """K15i (extension: left_align): (norm_slot int64 [n], rot int32 [n], hist int32 [n_slots]) on the device for the
    insertion event rows `events` (int32 [n, 4] on the device, the batch's pileup rows in their order): each row's
    leftmost slot against the device reference codes `ref` (uint8 [n_slots]), the right rotation of its string there,
    and per slot the number of live rows moved to it.  dead (uint8 [n] or None): rows K10 dropped, which get norm_slot
    -1 and count nowhere.  include/kindel_b200.h has the rule."""
    lib = _ffi.load()
    dev = dbatch.device
    n = int(events.shape[0])
    with torch.cuda.device(dev):
        events = events.to(dev, torch.int32).contiguous()
        norm_slot = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        rot = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        hist = torch.zeros(dbatch.n_slots, dtype=torch.int32, device=dev)
        if dead is not None:
            dead = dead.to(dev, torch.uint8).contiguous()
        rc = lib.kdl_left_align_insertions(C.byref(dbatch.struct), events.data_ptr() if n else None, n,
                                           dead.data_ptr() if dead is not None and n else None, ref.data_ptr(),
                                           norm_slot.data_ptr(), rot.data_ptr(), hist.data_ptr(), _stream_ptr(dev))
        _ffi.check(rc, "kdl_left_align_insertions")
    return norm_slot[:n], rot[:n], hist


def dead_event_rows(dbatch: DeviceBatch, n_events: int):
    """uint8 [n_events] on the device, 1 at the insertion-event rows K10 dropped (mask_overlaps); None when none."""
    d = dbatch.drops
    if d is None or d.shape[0] == 0:
        return None
    evt = d[:, 3].to(torch.int64)
    evt = evt[evt >= 0]
    if evt.numel() == 0:
        return None
    with torch.cuda.device(dbatch.device):
        return torch.zeros(n_events, dtype=torch.uint8, device=dbatch.device).index_fill_(0, evt, 1)


def _group_counts(key, cnt, q):
    """The count of each queried key q in the groups (key ascending, cnt), 0 where it has none; on the device."""
    if key.numel() == 0:
        return torch.zeros_like(q)
    at = torch.searchsorted(key, q).clamp(max=key.numel() - 1)
    return torch.where(key[at] == q, cnt[at], torch.zeros_like(cnt[at]))


def deletion_alleles(dbatch: DeviceBatch, counts: torch.Tensor, abs_threshold, rel_threshold, ref=None):
    """deletion_union of one sample: K7's events of `dbatch` grouped on the device against `counts`, a device table
    of the same batch; (slot, length, count, depth), int64 numpy arrays sorted by slot, then length.  ref (extension:
    left_align): device reference codes, the groups left-aligned against them (_deletion_groups)."""
    slot, length, cnt, depth = deletion_union([_deletion_groups(dbatch, ref)], counts[None], abs_threshold,
                                              rel_threshold)
    return slot, length, cnt[0], depth[0]


def deletion_union(groups, table: torch.Tensor, abs_threshold, rel_threshold):
    """The deletion alleles of `variants --vcf --reference` (extension) of S samples: groups holds each sample's K7
    events grouped by (slot, length) (_deletion_groups) in the slots of `table`, the samples' device tables
    (int32 [S, >= 6, n_slots]).  A group passes in its sample when its count c > abs_threshold and c / D >
    rel_threshold (0 at D = 0), D the sample's six-allele depth at the deletion's first slot.  Only the union of the
    keys that pass in some sample leaves the device: (slot int64[n], length int64[n], count int64 [S, n], depth int64
    [S, n]) as numpy arrays sorted by slot, then length, with every sample's c (0 without the event) and D."""
    a, r = variant_abs_floor(abs_threshold), float(rel_threshold)
    with torch.cuda.device(table.device):
        passing = []
        for i, (key, cnt) in enumerate(groups):
            depth = table[i, 0:6].index_select(1, key >> _LEN_BITS).to(torch.int64).sum(dim=0)
            share = torch.where(depth > 0, cnt.to(torch.float64) / depth.clamp(min=1).to(torch.float64),
                                torch.zeros((), dtype=torch.float64, device=table.device))
            passing.append(key[(cnt > a) & (share > r)])
        union = torch.unique(torch.cat(passing), sorted=True)
        slot = union >> _LEN_BITS
        counts = torch.stack([_group_counts(key, cnt, union) for key, cnt in groups])
        depths = torch.stack([table[i, 0:6].index_select(1, slot).to(torch.int64).sum(dim=0)
                              for i in range(len(groups))])
        return (slot.cpu().numpy(), (union & ((1 << _LEN_BITS) - 1)).cpu().numpy(),
                counts.cpu().numpy().astype(np.int64), depths.cpu().numpy())


def deletion_counts(dbatch: DeviceBatch, slot, length, ref=None) -> np.ndarray:
    """K7 over `dbatch` grouped on the device: how many of its deletion events are (slot[i], length[i]), for each
    queried pair (host int64 arrays); int64 numpy.  `variants --vcf --strand` asks it of the reverse-strand reads.
    ref (extension: left_align): device reference codes, the events left-aligned against them (_deletion_groups)."""
    q = (np.asarray(slot, dtype=np.int64) << _LEN_BITS) | np.asarray(length, dtype=np.int64)
    if q.size == 0:
        return np.zeros(0, dtype=np.int64)
    key, cnt = _deletion_groups(dbatch, ref)
    with torch.cuda.device(dbatch.device):
        return _group_counts(key, cnt, torch.from_numpy(q).to(key.device)).cpu().numpy().astype(np.int64)


class HostContext:
    """kdl_ctx_*: host buffers in, host buffers out (the path a non-CUDA host program binds)."""

    def __init__(self, device: int = 0):
        self._lib = _ffi.load()
        h = C.c_void_p()
        rc = self._lib.kdl_ctx_create(int(device), C.byref(h))
        _ffi.check(rc, "kdl_ctx_create")
        self._h = h

    def close(self):
        if self._h:
            self._lib.kdl_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def consensus(self, host: ReadBatch, min_depth=1, calls_out=None, counts_out=None, events_out=None,
                  struct=None, qmask=None):
        """Runs H2D + K1 (+ K1q) + K2 + D2H.  Returns calls (numpy uint8[n_slots]).  struct / qmask: prebuilt
        kdl_batch / kdl_qmask over host buffers the caller keeps alive (e.g. pinned memory)."""
        if struct is None:
            struct, keep = host_struct(host)
        if qmask is None:
            qmask, qkeep = host_qmask(host)
        if calls_out is None:
            calls_out = np.empty(host.n_slots, dtype=np.uint8)
        diag = _ffi.KdlDiag()
        outs = (int(math.ceil(min_depth)), calls_out.ctypes.data, counts_out.ctypes.data if counts_out is not None else None,
                events_out.ctypes.data if (events_out is not None and host.n_events) else None, C.byref(diag))
        if qmask is None:
            rc = self._lib.kdl_ctx_consensus(self._h, C.byref(struct), host.n_slots, host.n_events, *outs)
        else:
            rc = self._lib.kdl_ctx_consensus_masked(self._h, C.byref(struct), C.byref(qmask), host.n_slots,
                                                    host.n_events, *outs)
        if rc in (_ffi.KDL_ERR_INDEX, _ffi.KDL_ERR_KEY):
            raise_like_reference(rc, diag.read, diag.nibble, diag.op_index)
        _ffi.check(rc, "kdl_ctx_consensus")
        return calls_out

    def last_timing(self):
        a, b, c = C.c_float(), C.c_float(), C.c_float()
        self._lib.kdl_ctx_last_timing(self._h, C.byref(a), C.byref(b), C.byref(c))
        return {"h2d_ms": a.value, "kernel_ms": b.value, "d2h_ms": c.value}
