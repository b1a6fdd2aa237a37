"""kindel's Python API on top of the H100 engine (drop-in for `kindel.kindel` of bede/kindel 1.2.1).

Same names, signatures, defaults and return shapes as the reference module `kindel/kindel.py`
(SURVEY.md 8b).  What changed is where the two hot loops run:

  parse_records / parse_bam   (reference kindel/kindel.py:21-153)  -> K1 pileup kernels
  consensus_sequence          (reference kindel/kindel.py:384-430) -> K2 vote kernel + host string
                                                                      assembly

Everything the north star leaves on the host stays on the host and is restated here in numpy:
BAM/SAM decode (bamio.py), `--realign` clip-dominant-region reassembly (kindel.py:156-366),
report text (kindel.py:437-485) and the float tails of `weights` / `features` (kindel.py:558-664).
There is no CPU implementation of the pileup or the vote in this package.
"""
from __future__ import annotations

import functools
import logging
import os
from collections import OrderedDict, namedtuple

import numpy as np

from . import bamio, engine, quality, vcf
from .primers import AmpliconScheme, PrimerSet, amplicon_arrays, as_primer_set, as_scheme, primer_arrays
from .insertions import InsertionTable, dict_consensus
from .views import Alignment, BaseCounts, Insertions
from .vcf import QUAL_CAP, allele_quality, strand_odds_ratio  # noqa: F401  (kindel's VCF names)

Region = namedtuple("Region", ["start", "end", "seq", "direction"])
result = namedtuple("result", ["consensuses", "refs_changes", "refs_reports"])

_BASE_CHARS = np.frombuffer(b"ACGTN", dtype=np.uint8)
_CHANGE_LUT = (None, "D", "N", "I")
# letter of every call byte: bits 0-2 = base code (0..4 = A,C,G,T,N), or with bit 7 set (the IUPAC vote's multi-base
# calls) bits 0-3 = the base set as a BAM nibble, A=1 C=2 G=4 T=8
_CALL_LETTERS = np.array([ord("=ACMGRSVTWYHKDBN"[c & 15]) if c & 0x80 else ord("ACGTN"[min(c & 7, 4)])
                          for c in range(256)], dtype=np.uint8)

try:  # the reference wraps consensus sequences in dnaio.Sequence (kindel.py:433-434)
    from dnaio import Sequence as _Sequence
except Exception:  # dnaio not installed: same three attributes

    class _Sequence:
        __slots__ = ("name", "sequence", "qualities")

        def __init__(self, name=None, sequence=None, qualities=None):
            self.name, self.sequence, self.qualities = name, sequence, qualities

        def __repr__(self):
            return "Sequence(name=%r, sequence=%r)" % (self.name, self.sequence)


# ------------------------------------------------------------------------------------ pileup
class PileupRun:
    """One file's pileup on the device: count table, events, and lazily the host copies."""

    _device = None   # (count table, DeviceBatch) of host tables, uploaded on demand (device_tables)
    _reverse = None  # (count table, DeviceBatch) of the reverse-strand reads (reverse_table)
    _quality = None  # (qsum, emass) of the counted bases' qualities (quality_table)
    _weights = None  # wsum of the counted bases' quality weights (quality_weights)
    vote_qual = None  # K2w's Q per slot on the device after vote(quality=True), else None
    primers = None   # the PrimerSet whose primer bases the pileup masked (extension), None when off
    mask_overlaps = False  # the pileup counted each read pair once where its mates overlap (extension, K10)
    _dropped_events = None  # K10's dropped insertion-event rows of host tables
    _host_events = None  # the event rows of host tables in their order, K10's dropped rows included (left_align)
    _overlap_stats = None   # K10's (pairs, bases, deletions, insertions) of host tables
    normalised = None  # (N, dropped, kept) of the --normalise cap the batch went through (extension), None when off
    deduplicated = None  # (pairs removed, singles removed, kept, before) of --dedup (extension), None when off

    def __init__(self, batch: bamio.ReadBatch, device=None, primers=None, mask_overlaps=False):
        self.batch = batch
        self.primers = primers
        self.mask_overlaps = bool(mask_overlaps)
        self.dbatch = _upload(batch, device, primers, self.mask_overlaps)
        self.counts, self.events = engine.pileup(self.dbatch)
        self.calls_device = None
        self._host_counts = None
        self._host_derived = None
        self._ins = None

    @classmethod
    def from_host_tables(cls, batch, counts, derived, events, primers=None, mask_overlaps=False, dropped_events=None,
                         overlap_stats=None):
        """Wrap tables that already sit in host memory (results copied back by another path, e.g.
        the kdl_ctx_* host-buffer call or a multi-GPU reduction).  Does no computation.  primers: the PrimerSet the
        tables were piled with (a re-upload of the batch masks the same bases).  mask_overlaps: the tables count each
        read pair once (a re-upload masks the same mates again); dropped_events: K10's dropped insertion-event rows,
        which the insertion table leaves out; overlap_stats: K10's (pairs, bases, deletions, insertions) for the
        REPORT."""
        run = cls.__new__(cls)
        run.batch, run.dbatch, run.counts, run.events, run.calls_device = batch, None, None, None, None
        run.primers = primers
        run.mask_overlaps = bool(mask_overlaps)
        run._dropped_events = dropped_events
        run._overlap_stats = None if overlap_stats is None else tuple(int(x) for x in overlap_stats)
        run._host_counts = np.ascontiguousarray(counts, dtype=np.int32)
        run._host_derived = np.ascontiguousarray(derived, dtype=np.int32)
        run._ins = None
        run._host_events = np.ascontiguousarray(events, dtype=np.int32).reshape(-1, 4)
        run._ins = run._insertion_table(events)
        return run

    def device_tables(self):
        """(count table, DeviceBatch) on a device.  Host tables (a multi-GPU result): the reduced table and the batch
        go to this process's GPU, once (its primer bases and mate overlaps masked again, as the ranks saw them)."""
        if self.counts is not None:
            return self.counts, self.dbatch
        if self._device is None:
            import torch

            dev = engine.require_cuda()
            self._device = (torch.from_numpy(self.host_counts).to(dev),
                            _upload(self.batch, dev, self.primers, self.mask_overlaps))
        return self._device

    def reverse_table(self):
        """(count table, DeviceBatch) of the reverse-strand reads alone (extension: `variants --vcf --strand`), built
        once: K8 selects the reads whose `reverse` byte is set into a device batch, and the unchanged pileup counts
        them.  The forward table is the total minus this one.  Needs a batch decoded with strand=True.  K8 carries the
        merged mask list, and the sub-batch keeps the drop rows of its reverse R2 reads (mask_overlaps), which its
        pileup takes back."""
        if self._reverse is None:
            import torch

            if self.batch.reverse is None:
                raise ValueError("strand needs the reads' strands: decode the batch with strand=True")
            _, dbatch = self.device_tables()
            keep = torch.from_numpy(np.ascontiguousarray(self.batch.reverse, dtype=np.uint8)).to(dbatch.device)
            sub = engine.select_reads(dbatch, keep)
            self._reverse = (engine.pileup(sub)[0], sub)
        return self._reverse

    def quality_table(self):
        """(qsum int32 [4, n_slots], emass int64 [n_slots]) on a device, built once (extension: `variants --vcf
        --qual`): K11 over the run's masked device batch (device_tables(), so a multi-GPU result too) and its qual8,
        uploaded here and only here.  The bits are uint32 / uint64 (engine.quality_sums).  Needs a batch decoded with
        qual=True."""
        if self._quality is None:
            import torch

            if self.batch.qual8 is None:
                raise ValueError("qual needs the reads' qualities: decode the batch with qual=True")
            _, dbatch = self.device_tables()
            self._quality = engine.quality_sums(dbatch, torch.from_numpy(self.batch.qual8).to(dbatch.device))
        return self._quality

    def quality_weights(self):
        """wsum int64 [4, n_slots] (uint64 bits) on a device, built once (extension: quality_vote): K11w over the run's
        masked device batch (device_tables(), so a multi-GPU result too) and its qual8, uploaded here.  Needs a batch
        decoded with qual=True."""
        if self._weights is None:
            import torch

            if self.batch.qual8 is None:
                raise ValueError("quality_vote needs the reads' qualities: decode the batch with qual=True")
            _, dbatch = self.device_tables()
            self._weights = engine.quality_weights(dbatch, torch.from_numpy(self.batch.qual8).to(dbatch.device))
        return self._weights

    def vote(self, min_depth=1, iupac_threshold=None, quality=False) -> np.ndarray:
        """K2 over the whole table -> call bytes on the host (the device copy is kept for K5).  iupac_threshold:
        extension, see bam_to_consensus.  quality (extension): K2w over the table of device_tables() and
        quality_weights() instead, its Q kept in vote_qual."""
        if quality:
            counts, _ = self.device_tables()
            self.calls_device, self.vote_qual = engine.vote_quality(counts, self.quality_weights(), min_depth)
        else:
            self.calls_device = engine.vote(self.counts, min_depth, iupac_threshold=iupac_threshold)
        return self.calls_device.cpu().numpy()

    def quality_vote_sites(self, min_depth=1) -> np.ndarray:
        """The slots (int64, ascending) whose call byte of vote(quality=True) differs from kdl_vote's over the same
        table: one more K2 and a compare on the device; only those slots come back."""
        import torch

        if self.vote_qual is None:
            raise ValueError("quality_vote_sites needs the quality vote: call vote(quality=True) first")
        counts, _ = self.device_tables()
        base = engine.vote(counts, min_depth)
        return torch.nonzero(base != self.calls_device).flatten().cpu().numpy().astype(np.int64)

    @property
    def ins_table(self) -> InsertionTable:
        if self._ins is None:
            self._ins = self._insertion_table(self.events.cpu().numpy())
        return self._ins

    def _dropped_rows(self):
        """The insertion-event rows K10 dropped (mask_overlaps), or None."""
        dropped = self._dropped_events
        if dropped is None and self.dbatch is not None:
            dropped = engine.dropped_event_rows(self.dbatch)
        return dropped

    def _insertion_table(self, events) -> InsertionTable:
        """The one place the run's event rows become its insertion table: without the rows K10 dropped
        (mask_overlaps), so that no insertion string, VCF record or `alignment` view reads them."""
        dropped = self._dropped_rows()
        if dropped is not None and len(dropped):
            events = np.delete(np.asarray(events).reshape(-1, 4), np.asarray(dropped, dtype=np.int64), axis=0)
        return InsertionTable(self.batch, events)

    def left_aligned_insertions(self, ref):
        """(hist int32 [n_slots] on the device, InsertionTable) of the insertions left-aligned against the device
        reference codes `ref` (extension: left_align): K15i over the run's event rows in their order -- host tables'
        rows uploaded next to device_tables()' batch -- with the rows K10 dropped excluded first.  hist counts the live
        rows per left-aligned slot; the table holds the live rows at those slots with their strings' rotations."""
        import torch

        _, dbatch = self.device_tables()
        events = self.events if self.events is not None else torch.from_numpy(self._host_events).to(dbatch.device)
        n = int(events.shape[0])
        dead = None
        dropped = self._dropped_rows()
        if dropped is not None and len(dropped):
            dead = torch.zeros(n, dtype=torch.uint8, device=dbatch.device)
            dead[torch.from_numpy(np.asarray(dropped, dtype=np.int64)).to(dbatch.device)] = 1
        norm_slot, rot, hist = engine.left_align_insertions(dbatch, events, ref, dead)
        slots, rot, rows = norm_slot.cpu().numpy(), rot.cpu().numpy(), events.cpu().numpy()
        live = slots >= 0
        return hist, InsertionTable(self.batch, rows[live], slots[live], rot[live])

    @property
    def overlap_stats(self):
        """(pairs, bases, deletions, insertions) K10 masked (mask_overlaps), None when off."""
        if not self.mask_overlaps:
            return None
        if self._overlap_stats is not None:
            return self._overlap_stats
        return (self.dbatch if self.dbatch is not None else self.device_tables()[1]).overlap_masked

    @property
    def host_counts(self) -> np.ndarray:
        if self._host_counts is None:
            self._host_counts = self.counts.cpu().numpy()
        return self._host_counts

    @property
    def host_derived(self) -> np.ndarray:
        if self._host_derived is None:
            self._host_derived = engine.derive(self.counts).cpu().numpy()
        return self._host_derived

    def contig_slice(self, c: int):
        s = int(self.batch.contig_slot[c])
        return s, s + int(self.batch.contig_len[c]) + 1

    def alignment(self, c: int) -> Alignment:
        s, e = self.contig_slice(c)
        return Alignment(self.batch.contig_names[c], self.host_counts[:, s:e], self.host_derived[:, s:e],
                         self.ins_table, s)

    def alignments(self) -> OrderedDict:
        return OrderedDict((self.batch.contig_names[c], self.alignment(c)) for c in range(self.batch.n_contigs))


def _upload(batch, device, primers, mask_overlaps=False):
    """The batch on a device; with a PrimerSet (extension) its primer bases masked there by K9 (engine.mask_primers),
    then with mask_overlaps (extension) each pair's second mate masked where the first covers it, K10p + K10
    (engine.mask_overlaps): after K9, so that a primer-masked base of R1 covers nothing."""
    dbatch = engine.upload(batch, device)
    if primers is not None:
        dbatch = engine.mask_primers(dbatch, primer_arrays(primers, batch.contig_names, batch.contig_len))
    if mask_overlaps:
        dbatch = engine.mask_overlaps(dbatch)
    return dbatch


def _masked_for_shards(batch, primers, mask_overlaps):
    """(host batch, drop rows, K10's (pairs, bases, deletions, insertions)) of a sharded job with mask_overlaps: mates
    may land on different ranks, so K9 and K10 run once here, on this process's GPU; the merged mask list comes back
    and is applied to the host batch (the ranks pile it without primers), and each rank takes back its own R2s' drop
    rows (distributed.shard_drops)."""
    dbatch = _upload(batch, engine.require_cuda(), primers, True)
    drops = dbatch.drops.cpu().numpy().astype(np.int32).reshape(-1, 4)
    stats = dbatch.overlap_masked
    q = dbatch.qmask
    if q is None:
        return batch, drops, stats
    n_mr, n_mb = int(q.n_reads), int(q.n_bases)
    read = dbatch.tensors["mask_read"][:n_mr].cpu().numpy().view(np.uint32).astype(np.int64)
    off = dbatch.tensors["mask_off"][:n_mr + 1].cpu().numpy().view(np.uint32).astype(np.int64)
    qpos = dbatch.tensors["mask_qpos"][:n_mb].cpu().numpy().view(np.uint32)
    counts = np.zeros(batch.n_reads, dtype=np.int64)
    counts[read] = np.diff(off)
    return bamio.with_mask(batch, counts, qpos), drops, stats


def _op_word(length, op):
    code = bamio._OP_CODE.get(op, 15) if op is not None else 15
    return (int(length) << 4) | code


def flatten_records(ref_id, ref_len, records) -> bamio.ReadBatch:
    """Record objects (.pos 1-based, .mapped, .seq, .cigars) -> ReadBatch of one contig.
    The filter is the reference's (kindel.py:43-46)."""
    ref_start, l_seq, cig_off, cigar, seq_off, parts = [], [], [0], [], [], []
    words = 0
    n_rec = 0
    for rec in records:
        n_rec += 1
        if not rec.mapped or len(rec.seq) <= 1:
            continue
        ref_start.append(int(rec.pos) - 1)
        l_seq.append(len(rec.seq))
        cigar.extend(_op_word(ln, op) for ln, op in rec.cigars)
        cig_off.append(len(cigar))
        enc = bamio.encode_seq(rec.seq)
        seq_off.append(words)
        words += enc.size
        parts.append(enc)
    seq4 = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint32)
    return bamio.finalize([ref_id], np.array([ref_len], dtype=np.int64), np.array([0, len(ref_start)], dtype=np.int64),
                          np.array(ref_start, dtype=np.int64), np.array(seq_off, dtype=np.int64),
                          np.array(l_seq, dtype=np.int64), np.array(cig_off, dtype=np.int64),
                          np.array(cigar, dtype=np.int64), seq4, n_records=n_rec)


def parse_records(ref_id, ref_len, records):
    """Pileup of one contig's records -> `alignment` (reference kindel/kindel.py:21-128)."""
    return PileupRun(flatten_records(ref_id, ref_len, records)).alignment(0)


def _default_devices(devices):
    """`devices` = number of GPUs of this node to shard the pileup over (None: $KINDEL_GPUS, else 1)."""
    if devices is None:
        devices = int(os.environ.get("KINDEL_GPUS", "1") or 1)
    return max(1, int(devices))


def check_normalise(normalise):
    """The one check of the normalise option: None (off) or an integer >= 1 (ValueError otherwise)."""
    if normalise is None:
        return None
    if isinstance(normalise, (bool, np.bool_)) or not isinstance(normalise, (int, np.integer)) or normalise < 1:
        raise ValueError("normalise must be an integer >= 1, got %r" % (normalise,))
    return int(normalise)


def _normalise_scheme(primers, normalise):
    """(PrimerSet or None, AmpliconScheme or None) of pileup_run's primers: normalise needs a named scheme."""
    if normalise is None:
        return as_primer_set(primers.primers if isinstance(primers, AmpliconScheme) else primers), None
    if primers is None:
        raise ValueError("normalise needs a named primer scheme: pass primers= (a BED whose 4th column names each "
                         "primer <amplicon>_LEFT or <amplicon>_RIGHT)")
    if isinstance(primers, PrimerSet):
        raise ValueError("normalise needs a named primer scheme: pass the BED's path or an AmpliconScheme "
                         "(primers.load_scheme), not a PrimerSet")
    scheme = as_scheme(primers)
    return scheme.primers, scheme


def _normalise(batch, scheme, cap, strand):
    """(the batch of the reads the cap keeps, (cap, dropped, kept)) (extension: normalise): K12 labels every read of
    the uploaded batch with its amplicon under `scheme`, K13 keeps the first `cap` reads of each (amplicon, strand)
    group in batch order, and only when it drops a read do the keep bytes (1 B per read) come back and the host batch
    is rebuilt from the kept reads (bamio.select_reads).  The strand bytes stay only when `strand` asked for them."""
    import torch

    arrays = amplicon_arrays(scheme, batch.contig_names, batch.contig_len)
    dbatch = engine.upload(batch, engine.require_cuda())
    label = engine.assign_amplicons(dbatch, arrays)
    reverse = torch.from_numpy(np.ascontiguousarray(batch.reverse, dtype=np.uint8)).to(dbatch.device)
    keep, _, dropped = engine.normalise(label, reverse, arrays.n_amplicons, cap)
    n_dropped = int(dropped.item())
    if n_dropped:
        batch = bamio.select_reads(batch, np.flatnonzero(keep.cpu().numpy()))
    del dbatch, label, reverse, keep
    if not strand:
        batch.reverse = None
    return batch, (cap, n_dropped, int(batch.n_reads))


def check_dedup(dedup) -> bool:
    """The one check of the dedup option: True or False (ValueError otherwise)."""
    if not isinstance(dedup, (bool, np.bool_)):
        raise ValueError("dedup must be True or False, got %r" % (dedup,))
    return bool(dedup)


def _dedup(batch, strand, mates):
    """(the batch of the reads duplicate removal keeps, (pairs removed, singles removed, kept, before)) (extension:
    dedup): K10p pairs the mates of the uploaded batch, K14k / the sort / K14s find the duplicates on the device, and
    only when a read is removed do the keep bytes (1 B per read) come back and the host batch is rebuilt from the kept
    reads (bamio.select_reads).  The strand bytes and the mates stay only when `strand` / `mates` asked for them."""
    dbatch = engine.upload(batch, engine.require_cuda())
    keep, (pairs, singles, _) = engine.dedup(dbatch)
    before = int(batch.n_reads)
    if pairs or singles:
        batch = bamio.select_reads(batch, np.flatnonzero(keep.cpu().numpy()))
    del dbatch, keep
    batch.dup_score = None
    if not strand:
        batch.reverse = None
    if not mates:
        batch.name_hash = batch.mate_start = batch.pair_role = None
    return batch, (pairs, singles, int(batch.n_reads), before)


def pileup_run(bam_path, devices=None, min_depth=1, min_base_quality=0, min_mapq=0, exclude_flags=0,
               iupac_threshold=None, strand=False, primers=None, mask_overlaps=False, qual=False, normalise=None,
               dedup=False):
    """(PileupRun, calls) of an alignment file on `devices` GPUs.  devices > 1: one process per GPU, reads (or whole
    contigs) sharded, counts exchanged over NVLink in front of the vote (distributed.run_sharded); the result is
    bit-identical to one GPU.  min_base_quality / min_mapq / exclude_flags (extension, all off by default): a record
    with MAPQ < min_mapq or FLAG & exclude_flags is treated as unmapped; a base with Phred quality < min_base_quality
    is read as N and not counted (kindel_b200/bamio.py).  iupac_threshold: the vote of the sharded job (extension,
    see bam_to_consensus); calls is None for one GPU, where the caller votes.  strand (extension): the batch keeps
    the reads' strands (PileupRun.reverse_table).  primers (extension, default None = off): a BED path or a
    primers.PrimerSet; the bases of every read that copy an amplicon primer are then read as N and not counted, as
    min_base_quality does with a low-quality base (K9, kindel_b200/primers.py has the rule).  With several GPUs every
    rank masks its own shard; the result is the same.  mask_overlaps (extension, default False = off): each read pair
    is counted once where its mates overlap -- the second mate's bases, deletions and insertions there are masked or
    dropped where the first mate has information (K10p / K10 / K10u, include/kindel_b200.h has the rule); the batch is
    then decoded with its mates.  With several GPUs the pairing and the masking run once on this process's GPU, and
    every rank takes back its own second mates' drops; the result is the same.  qual (extension, default False =
    off): the batch keeps its reads' base qualities (PileupRun.quality_table); a kept read without them is a
    ValueError.  normalise (extension, default None = off): an integer N >= 1 that needs `primers` to be a named
    scheme (primers.load_scheme: a BED path or an AmpliconScheme; ValueError otherwise).  After the filters, each read
    gets its amplicon (K12's label) and strand (FLAG & 0x10); of the reads with an amplicon, only the first N of each
    (amplicon, strand) in batch order are kept (K13), and the others are removed from the batch as if they were not
    in the file: no count, clip, event or mate of theirs.  Reads without an amplicon are never capped.  Everything
    else -- primer masking, mate pairing, the pileup, several GPUs -- then runs on the kept reads; the run's
    `normalised` holds (N, dropped, kept).  dedup (extension, default False = off): after the filters and before
    normalise, duplicate reads and read pairs are removed as samtools markdup -r removes them: by fragment ends (each
    read's unclipped 5' end and strand, both mates' for a pair) and a base-quality score, the best of each duplicate set
    staying (K14, include/kindel_b200.h has the rule).  The removed reads are taken out as if they were not in the
    file, on this process's GPU before any sharding; the run's `deduplicated` holds (pairs removed, singles removed,
    kept, before).  A 0x400 flag in the file is not read: `exclude_flags=0x400` honours it.  A read that dedup or
    normalise removes still counts for the first-seen order of contigs, as a filtered record does: the run reports
    the whole file's contigs in the whole file's order."""
    iupac_threshold = check_iupac_threshold(iupac_threshold)
    normalise = check_normalise(normalise)
    dedup = check_dedup(dedup)
    primers, scheme = _normalise_scheme(primers, normalise)
    decode = dict(min_mapq=min_mapq, exclude_flags=exclude_flags, min_base_quality=min_base_quality,
                  strand=strand or normalise is not None or dedup)
    if mask_overlaps or dedup:  # (the keyword only when on: the decode stays as it was otherwise)
        decode["mates"] = True
    if qual:
        decode["qual"] = True
    if dedup:
        decode["dup"] = True
    batch = bamio.read_alignment(bam_path, **decode)
    deduplicated = normalised = None
    if dedup:
        batch, deduplicated = _dedup(batch, strand or normalise is not None, mask_overlaps)
    if normalise is not None:
        batch, normalised = _normalise(batch, scheme, normalise, strand)
    arrays = primer_arrays(primers, batch.contig_names, batch.contig_len) if primers is not None else None
    devices = _default_devices(devices)
    if devices <= 1:
        run = PileupRun(batch, primers=primers, mask_overlaps=mask_overlaps)
        run.normalised, run.deduplicated = normalised, deduplicated
        return run, None
    from . import distributed

    shards, drops, stats = batch, None, None
    if mask_overlaps:
        shards, drops, stats = _masked_for_shards(batch, primers, True)
        arrays = None  # (the primer bases are in the merged mask list already)
    calls, counts, derived, events = distributed.run_sharded(shards, devices, min_depth, iupac_threshold=iupac_threshold,
                                                             primers=arrays, drops=drops)
    dropped = None if drops is None else np.sort(drops[drops[:, 3] >= 0, 3].astype(np.int64))
    run = PileupRun.from_host_tables(batch, counts, derived, events, primers=primers, mask_overlaps=mask_overlaps,
                                     dropped_events=dropped, overlap_stats=stats)
    run.normalised, run.deduplicated = normalised, deduplicated
    return run, calls


def parse_bam(bam_path, devices=None, min_base_quality=0, min_mapq=0, exclude_flags=0, primers=None,
              mask_overlaps=False, normalise=None, dedup=False):
    """Alignment information for each reference sequence, first-seen order
    (reference kindel/kindel.py:131-153).  devices, the filters, primers, mask_overlaps, normalise and dedup:
    extensions, see pileup_run."""
    return pileup_run(bam_path, devices, 1, min_base_quality, min_mapq, exclude_flags,
                      primers=primers, mask_overlaps=mask_overlaps, normalise=normalise, dedup=dedup)[0].alignments()


# --------------------------------------------------------------------------------- consensus
def consensus(weight):
    """(base, frequency, proportion, tie) of one count dict (reference kindel/kindel.py:369-381):
    first maximum in dict order; ("N", 0) when empty/all zero; tie = another key shares it."""
    total = sum(weight.values())
    base, frequency = "N", 0
    if total:
        first = True
        for k, v in weight.items():
            if first or v > frequency:
                base, frequency, first = k, v, False
    tie = bool(frequency) and any(v == frequency for k, v in weight.items() if k != base)
    proportion = round(frequency / total, 2) if total else 0
    return (base, frequency, proportion, tie)


def _vote_columns(weights, insertions, deletions):
    """The 7 vote columns [7, L+1] from either engine views or plain lists of dicts."""
    L = len(weights)
    cols = np.zeros((7, L + 1), dtype=np.int32)
    if isinstance(weights, BaseCounts):
        cols[0:5, :L] = weights.cols
    else:
        for i, w in enumerate(weights):
            cols[0, i], cols[1, i], cols[2, i], cols[3, i], cols[4, i] = w["A"], w["C"], w["G"], w["T"], w["N"]
    dele = np.asarray(deletions[:L] if not isinstance(deletions, np.ndarray) else deletions[:L], dtype=np.int64)
    cols[5, : dele.shape[0]] = dele
    if isinstance(insertions, Insertions):
        cols[6, :L] = insertions.totals[:L]
    else:
        for i in range(L):
            d = insertions[i]
            cols[6, i] = sum(d.values()) if d else 0
    return cols


def check_iupac_threshold(t):
    """The one check of the iupac_threshold option: None (off) or a number in [0, 1], else ValueError."""
    return engine.check_iupac_threshold(t)


def _device_vote(cols: np.ndarray, min_depth, iupac_threshold=None) -> np.ndarray:
    import torch

    dev = engine.require_cuda()
    n = cols.shape[1]
    n_pad = (n + 3) // 4 * 4
    t = torch.zeros((7, n_pad), dtype=torch.int32, device=dev)
    t[:, :n] = torch.from_numpy(np.ascontiguousarray(cols)).to(dev)
    return engine.vote(t, min_depth, iupac_threshold=iupac_threshold).cpu().numpy()[:n]


def _emit_range(calls, lo, hi, ins_lookup, out, changes, qual=None, ins_qual=None, qout=None):
    """Append the consensus text of positions [lo, hi) to `out` (kindel.py:413-424).  A bit-7 call (IUPAC vote)
    emits its ambiguity code; when `changes` keeps an `iupac` list, its 1-based position is added there.
    qual (extension): per-position Q (uint8 array like calls); then the Phred+33 text of every emitted character goes
    to `qout`, an inserted string's from ins_qual(position)."""
    if hi <= lo:
        return
    seg = calls[lo:hi]
    change = (seg >> 4) & 3
    chars = _CALL_LETTERS[seg]
    qchars = (np.asarray(qual[lo:hi], dtype=np.uint8) + 33).astype(np.uint8) if qual is not None else None
    for k in np.flatnonzero(change).tolist():
        changes[lo + k] = _CHANGE_LUT[change[k]]
    iupac = getattr(changes, "iupac", None)
    if iupac is not None:
        iupac.extend(str(lo + k + 1) for k in np.flatnonzero(seg & 0x80).tolist())
    ins_pos = np.flatnonzero(change == 3)
    keep = change != 1

    def emit(a, b):
        out.append(chars[a:b][keep[a:b]].tobytes().decode("ascii"))
        if qchars is not None:
            qout.append(qchars[a:b][keep[a:b]].tobytes().decode("ascii"))

    if ins_pos.size == 0:
        emit(0, hi - lo)
        return
    prev = 0
    for k in ins_pos.tolist():
        emit(prev, k)
        s, tie = ins_lookup(lo + k)
        text = "N" if tie else s.lower()
        out.append(text)
        if qchars is not None:
            qout.append(chr(33 + ins_qual(lo + k)) * len(text))
        prev = k
    emit(prev, hi - lo)


def assemble_consensus(calls, ins_lookup, cdr_patches=None, trim_ends=False, uppercase=False, qual=None,
                       ins_qual=None):
    """Call bytes of one contig (length L) -> (consensus string, changes list).

    Restates the sequential part of consensus_sequence (kindel.py:387-401, 425-430): CDR patches
    (first Region whose start == pos, provided some Region starting there has a truthy seq) emit
    their lower-cased sequence and skip `end - start - 1` further positions without looking at them.
    qual / ins_qual (extension): per-position Q (uint8[L]) and the Q of the inserted string at a position; the call
    then returns (string, changes, quality string), a patch's characters at Q0 and trim_ends cutting both alike.
    """
    L = calls.shape[0]
    changes = _Changes([None] * L)
    changes.iupac = []  # positions of multi-base IUPAC calls that were emitted
    out = []
    qout = [] if qual is not None else None
    starts = sorted({r.start for r in cdr_patches if r.seq and 0 <= r.start < L}) if cdr_patches else []
    pos = 0
    for st in starts:
        if st < pos:
            continue  # lies inside a span that is being skipped
        _emit_range(calls, pos, st, ins_lookup, out, changes, qual, ins_qual, qout)
        patch = next(r for r in cdr_patches if r.start == st)
        out.append(patch.seq.lower())
        if qout is not None:
            qout.append("!" * len(patch.seq))  # no aligned read supports a patch: Q0
        skip = (patch.end - patch.start) - 1
        if skip < 0:  # the reference's counter goes negative and never recovers: nothing more is emitted
            pos = L
            break
        pos = st + 1 + skip
    _emit_range(calls, pos, L, ins_lookup, out, changes, qual, ins_qual, qout)
    seq = "".join(out)
    quals = "".join(qout) if qout is not None else None
    if trim_ends:
        seq, quals = _trim_n(seq, quals)
    if uppercase:
        seq = seq.upper()
    return (seq, changes) if qual is None else (seq, changes, quals)


def _trim_n(seq, quals=None):
    """seq.strip("N") (trim_ends), and the quality characters at exactly the stripped positions removed."""
    left = seq.lstrip("N")
    out = left.rstrip("N")
    if quals is None:
        return out, None
    a = len(seq) - len(left)
    return out, quals[a:a + len(out)]


def consensus_sequence(weights, insertions, deletions, cdr_patches, trim_ends, min_depth, uppercase,
                       iupac_threshold=None):
    """Per-position vote -> (consensus string, changes) (reference kindel/kindel.py:384-430).
    The vote itself runs on the GPU (K2); strings are assembled here.  iupac_threshold: extension, see
    bam_to_consensus."""
    iupac_threshold = check_iupac_threshold(iupac_threshold)
    calls = _device_vote(_vote_columns(weights, insertions, deletions), min_depth, iupac_threshold)[: len(weights)]
    return assemble_consensus(calls, lambda p: dict_consensus(insertions[p]), cdr_patches, trim_ends, uppercase)


def consensus_seqrecord(consensus, ref_id, qualities=None):
    """The record of one contig; qualities (extension): its Phred+33 quality string, None when not asked for."""
    return _Sequence(name=f"{ref_id}_cns", sequence=consensus, qualities=qualities)


# ---------------------------------------------------------------- realign (host, kindel.py:156-366)
def _first_max_base(cols: np.ndarray) -> np.ndarray:
    """consensus(w)[0] for every column of a [5, n] A,C,G,T,N block: first max in A,T,G,C,N order."""
    order = np.array([0, 3, 2, 1, 4])
    stacked = cols[order]
    idx = order[np.argmax(stacked, axis=0)]
    idx = np.where(cols.sum(axis=0) == 0, 4, idx)
    return _BASE_CHARS[idx]


def _cols_of(base_counts) -> np.ndarray:
    if isinstance(base_counts, BaseCounts):
        return np.asarray(base_counts.cols, dtype=np.int64)
    n = len(base_counts)
    cols = np.zeros((5, n), dtype=np.int64)
    for i, w in enumerate(base_counts):
        cols[:, i] = (w["A"], w["C"], w["G"], w["T"], w["N"])
    return cols


def _masked(n: int, mask_ends: int) -> np.ndarray:
    m = np.zeros(n, dtype=bool)
    r = range(n)
    m[list(r[:mask_ends])] = True
    m[list(r[-mask_ends:])] = True  # mask_ends == 0 masks everything, like positions[-0:]
    return m


def _cdr_inputs(weights, deletions, clip_weights, clip_depth, clip_decay_threshold, mask_ends):
    w = _cols_of(weights)
    n = w.shape[1]
    depth = w.sum(axis=0)  # all five keys (sum(w.values()), kindel.py:182)
    dele = np.asarray(deletions, dtype=np.int64)[:n]
    cd = np.asarray(clip_depth, dtype=np.int64)[:n]
    dominant = (cd / (depth + dele + 1) > 0.5) & ~_masked(n, mask_ends)
    extend = cd > (depth + dele) * clip_decay_threshold
    bases = _first_max_base(_cols_of(clip_weights))
    return n, dominant, extend, bases


def _start_regions(n, dominant, extend, bases):
    """-> regions from the per-position predicates (reference kindel/kindel.py:156-213)."""
    stops = np.flatnonzero(~extend)
    regions = []
    for pos in np.flatnonzero(dominant).tolist():
        if any(r.start <= pos < r.end for r in regions):
            continue
        k = np.searchsorted(stops, pos)
        if k < stops.shape[0]:
            end = int(stops[k])
            seq_end = end
        else:  # ran to the contig end without decaying
            end = n - 1
            seq_end = n
        regions.append(Region(pos, end, bases[pos:seq_end].tobytes().decode("ascii"), "\u2192"))
    return regions


def _end_regions(n, dominant, extend, bases):
    """<- regions from the per-position predicates (reference kindel/kindel.py:216-275)."""
    stops = np.flatnonzero(~extend)
    regions = []
    for pos in np.flatnonzero(dominant)[::-1].tolist():
        if any(r.start <= pos < r.end for r in regions):
            continue
        # extension walks pos-1, pos-2, ... and stops at the first position that has decayed
        k = np.searchsorted(stops, pos) - 1  # last stop < pos
        if pos == 0:
            start, seq = 0, ""
        elif k >= 0:
            start = int(stops[k])
            seq = bases[start + 1:pos + 1].tobytes().decode("ascii") if start < pos - 1 else ""
        else:
            start = 0
            seq = bases[0:pos + 1].tobytes().decode("ascii")
        regions.append(Region(start, pos + 1, seq, "\u2190"))
    return regions


def cdr_start_consensuses(weights, deletions, clip_start_weights, clip_start_depth, clip_decay_threshold,
                          mask_ends):
    """Right-clipped (->) consensuses of clip-dominant regions (reference kindel/kindel.py:156-213)."""
    return _start_regions(*_cdr_inputs(weights, deletions, clip_start_weights, clip_start_depth, clip_decay_threshold,
                                       mask_ends))


def cdr_end_consensuses(weights, deletions, clip_end_weights, clip_end_depth, clip_decay_threshold, mask_ends):
    """Left-clipped (<-) consensuses of clip-dominant regions (reference kindel/kindel.py:216-275)."""
    return _end_regions(*_cdr_inputs(weights, deletions, clip_end_weights, clip_end_depth, clip_decay_threshold,
                                     mask_ends))


def _pair_regions(fwd, rev):
    pairs = []
    for f in fwd:
        for r in rev:
            if max(f.start, r.start) < min(f.end, r.end):
                pairs.append((f, r))
                break
    return pairs


def cdrps_from_device(counts, s, e, clip_decay_threshold, mask_ends):
    """cdrp_consensuses for the contig at slots [s, e) straight from the device table: K4 evaluates the
    clip-dominance and decay predicates and the clip consensus bases per position (2 bytes per position come
    back instead of the 76-byte table row); regions, pairing and merging are the same host code."""
    n = e - s
    flags, bases = engine.cdr_flags(counts, s, e, clip_decay_threshold)
    keep = ~_masked(n, mask_ends)
    fwd = _start_regions(n, ((flags & 1) != 0) & keep, (flags & 2) != 0, _BASE_CHARS[bases & 7])
    rev = _end_regions(n, ((flags & 4) != 0) & keep, (flags & 8) != 0, _BASE_CHARS[(bases >> 4) & 7])
    return _pair_regions(fwd, rev)


def cdrp_consensuses(weights, deletions, clip_start_weights, clip_end_weights, clip_start_depth, clip_end_depth,
                     clip_decay_threshold, mask_ends):
    """Pairs of overlapping -> / <- clip consensuses (reference kindel/kindel.py:278-320)."""
    fwd = cdr_start_consensuses(weights, deletions, clip_start_weights, clip_start_depth, clip_decay_threshold,
                                mask_ends)
    rev = cdr_end_consensuses(weights, deletions, clip_end_weights, clip_end_depth, clip_decay_threshold,
                              mask_ends)
    return _pair_regions(fwd, rev)


def merge_by_lcs(s1, s2, min_overlap):
    """Superstring of s1 and s2 about their longest common substring if it is at least
    min_overlap long, else None (reference kindel/kindel.py:323-347).  Among equally long common
    substrings the one ending first in s1 wins, as in the reference's row-major scan."""
    longest, x_longest = 0, 0
    if s1 and s2:
        b = np.frombuffer(s2.encode("utf-32-le"), dtype=np.uint32)
        prev = np.zeros(b.shape[0] + 1, dtype=np.int64)
        for x, ch in enumerate(s1, start=1):
            row = np.zeros_like(prev)
            hit = b == ord(ch)
            row[1:][hit] = prev[:-1][hit] + 1
            m = int(row.max())
            if m > longest:
                longest, x_longest = m, x
            prev = row
    lcs = s1[x_longest - longest:x_longest]
    if len(lcs) < min_overlap:
        return None
    return s1.split(lcs, 1)[0] + lcs + s2.split(lcs, 1)[1]


def merge_cdrps(cdrps, min_overlap):
    """Merged clip-dominant region pairs as Regions (reference kindel/kindel.py:350-366)."""
    merged = []
    for fwd_cdr, rev_cdr in cdrps:
        seq = merge_by_lcs(fwd_cdr.seq, rev_cdr.seq, min_overlap)
        if not seq:
            logging.warning(
                f"No overlap found for clip dominant region spanning positions {fwd_cdr.start}-{rev_cdr.end} (min_overlap = {min_overlap})"
            )
        merged.append(Region(fwd_cdr.start, rev_cdr.end, seq, None))
    return merged


# -------------------------------------------------------------------------------------- report
DepthRange = namedtuple("DepthRange", ["dmin", "dmax"])  # min / max ACGT depth of a contig (kindel.py:450,477-479)


def build_report(ref_id, weights, changes, cdr_patches, bam_path, realign, min_depth, min_overlap,
                 clip_decay_threshold, trim_ends, uppercase, filters=None, iupac_threshold=None, primers=None,
                 overlaps=None, quality_vote_sites=None, normalised=None, deduplicated=None):
    """REPORT text block (reference kindel/kindel.py:437-485).  filters (extension): (min_base_quality, min_mapq,
    exclude_flags); when any is set, three option lines follow `- uppercase:`, otherwise the text is the reference's.
    iupac_threshold (extension): when set, `- iupac_threshold:` follows the option lines and `- iupac sites:` (the
    positions of multi-base calls, from the `iupac` list of a changes list this module built) follows
    `- ambiguous sites:`.  primers (extension): the primer BED's file name; when set, `- primers:` follows the filter
    lines.  overlaps (extension: mask_overlaps): K10's (pairs, bases, deletions, insertions); when set,
    `- mate overlaps:` follows the filter and primer lines.  quality_vote_sites (extension: quality_vote): the 1-based
    positions (strings) whose call differs from the reference's vote; when set, `- quality_vote: True` follows the
    option lines and `- quality-vote sites:` follows `- ambiguous sites:`.  normalised (extension: normalise): the run's
    (N, dropped, kept); when set, `- normalise:` follows the primer line.  deduplicated (extension: dedup): the run's
    (pairs removed, singles removed, kept, before); when set, `- duplicates:` follows the primer line, before
    `- normalise:`."""
    if isinstance(weights, DepthRange):  # already reduced on the device: no table copy needed
        dmin, dmax = weights.dmin, weights.dmax
    elif isinstance(weights, BaseCounts):
        acgt = weights.cols[0:4].sum(axis=0)
        dmin, dmax = (int(acgt.min()), int(acgt.max()))
    else:
        depths = [w["A"] + w["C"] + w["G"] + w["T"] for w in weights]
        dmin, dmax = min(depths), max(depths)
    sites = getattr(changes, "sites", None)  # (a list built by _changes_list knows its sites already)
    if sites is None:
        sites = {"N": [], "I": [], "D": []}
        for pos, change in enumerate(changes, start=1):
            if change in sites:
                sites[change].append(str(pos))
    patches = ["{}-{}: {}".format(r.start, r.end, r.seq) for r in cdr_patches] if cdr_patches else ""
    lines = [
        "========================= REPORT ===========================",
        "reference: {}".format(ref_id),
        "options:",
        "- bam_path: {}".format(bam_path),
        "- min_depth: {}".format(min_depth),
        "- realign: {}".format(realign),
        "    - min_overlap: {}".format(min_overlap),
        "    - clip_decay_threshold: {}".format(clip_decay_threshold),
        "- trim_ends: {}".format(trim_ends),
        "- uppercase: {}".format(uppercase),
    ]
    if filters is not None and any(filters):
        lines += ["- min_base_quality: {}".format(filters[0]), "- min_mapq: {}".format(filters[1]),
                  "- exclude_flags: {:#x}".format(filters[2])]
    if primers is not None:
        lines.append("- primers: {}".format(primers))
    if deduplicated is not None:
        lines.append("- duplicates: {} pairs and {} single reads removed, {} of {} reads kept".format(*deduplicated))
    if normalised is not None:
        cap, dropped, kept = normalised
        lines.append("- normalise: {} per amplicon and strand, {} of {} reads dropped".format(cap, dropped,
                                                                                           dropped + kept))
    if overlaps is not None:
        lines.append("- mate overlaps: {} pairs, {} bases, {} deletions, {} insertions masked".format(*overlaps))
    if iupac_threshold is not None:
        lines.append("- iupac_threshold: {}".format(iupac_threshold))
    if quality_vote_sites is not None:
        lines.append("- quality_vote: True")
    lines += [
        "observations:",
        "- min, max observed depth: {}, {}".format(dmin, dmax),
        "- ambiguous sites: {}".format(", ".join(sites["N"])),
    ]
    if iupac_threshold is not None:
        lines.append("- iupac sites: {}".format(", ".join(getattr(changes, "iupac", None) or [])))
    if quality_vote_sites is not None:
        lines.append("- quality-vote sites: {}".format(", ".join(quality_vote_sites)))
    lines += [
        "- insertion sites: {}".format(", ".join(sites["I"])),
        "- deletion sites: {}".format(", ".join(sites["D"])),
        "- clip-dominant regions: {}".format(", ".join(patches)),
    ]
    return "\n".join(lines) + "\n"


# --------------------------------------------------------------------------------- public API
def bam_to_consensus(bam_path, realign=False, min_depth=1, min_overlap=9, clip_decay_threshold=0.1,
                     mask_ends=50, trim_ends=False, uppercase=False, devices=None, min_base_quality=0, min_mapq=0,
                     exclude_flags=0, iupac_threshold=None, qualities=False, primers=None, mask_overlaps=False,
                     quality_vote=False, normalise=None, dedup=False):
    """Consensus sequence(s) of an alignment file (reference kindel/kindel.py:488-555).

    Device work per file: one pileup (K1) and one vote (K2) over all contigs at once; only the
    call bytes, the insertion events and -- for --realign and the report -- count columns come
    back to the host.  `devices` (extension; default $KINDEL_GPUS or 1) shards the pileup over that many GPUs of
    the node.  min_base_quality / min_mapq / exclude_flags / primers / mask_overlaps / normalise / dedup: extension,
    see pileup_run; with normalise the REPORT gains `- normalise:` after `- primers:`, with dedup `- duplicates:`
    between the two.

    iupac_threshold (extension; default None = off, the reference's vote): t in [0, 1].  Where a base is emitted,
    the call is the smallest set of the most frequent bases (A, C, G, T; N is not an allele) that holds at least
    t * depth of the reads, tied bases entering together, written as its IUPAC code (R = A/G, Y = C/T, ...,
    N = all four).  The D / N / I changes and the inserted strings are those of the reference's vote.

    qualities (extension; default False): every record's `.qualities` is then a Phred+33 string, one character per
    character of `.sequence` (kindel_b200/quality.py has the rule); the sequence, changes and reports are those of
    qualities=False.  Off, `.qualities` is None and nothing else runs.

    quality_vote (extension; default False = off): where a base is emitted, it is the one whose reads' base qualities
    give it the largest summed log-likelihood weight (W[q], kindel_b200/quality.py; the haploid maximum-likelihood base
    under uniform priors), N on a tie or when no base has weight; an N count no longer makes the call N.  The D / N / I
    changes and the inserted strings are those of the reference's vote.  With qualities, a base's Q is the weight gap
    to the runner-up in Phred, capped at 60.  The batch is decoded with its qualities, so a kept read without them is a
    ValueError; not together with iupac_threshold (ValueError)."""
    iupac_threshold = check_iupac_threshold(iupac_threshold)
    quality_vote = check_quality_vote(quality_vote, iupac_threshold)
    filters = (min_base_quality, min_mapq, exclude_flags)
    run, calls = pileup_run(bam_path, devices, min_depth, *filters, iupac_threshold=iupac_threshold, primers=primers,
                            mask_overlaps=mask_overlaps, qual=quality_vote, normalise=normalise, dedup=dedup)
    if calls is None or quality_vote:  # (several GPUs: the ranks' majority calls give way to the reduced table's)
        calls = run.vote(min_depth, iupac_threshold, quality=quality_vote)
    return consensus_from_run(run, calls, bam_path, realign, min_depth, min_overlap,
                              clip_decay_threshold, mask_ends, trim_ends, uppercase, filters=filters,
                              iupac_threshold=iupac_threshold, qualities=qualities, quality_vote=quality_vote)


def check_quality_vote(quality_vote, iupac_threshold=None) -> bool:
    """The one check of the quality_vote option: it cannot be combined with an IUPAC threshold (ValueError)."""
    quality_vote = bool(quality_vote)
    if quality_vote and iupac_threshold is not None:
        raise ValueError("quality_vote cannot be combined with iupac_threshold")
    return quality_vote


class _Changes(list):
    """The reference's `changes` list (None / 'D' / 'N' / 'I' per position) that also remembers where its few
    non-None entries are, so the report needs no pass over millions of Nones, and (`iupac`) the 1-based positions
    of multi-base IUPAC calls, which the list itself cannot show."""

    __slots__ = ("sites", "iupac")


def _changes_list(calls):
    """Per-position change codes (None / 'D' / 'N' / 'I') of one contig's call bytes."""
    change = (calls >> 4) & 3
    out = _Changes([None] * calls.shape[0])
    at = np.flatnonzero(change)
    out.sites = {"N": [], "I": [], "D": []}
    for k, code in zip(at.tolist(), change[at].tolist()):
        name = _CHANGE_LUT[code]
        out[k] = name
        out.sites[name].append(str(k + 1))
    out.iupac = [str(k + 1) for k in np.flatnonzero(calls & 0x80).tolist()]
    return out


def _insertion_slots(batch, calls_all):
    """Ascending slots whose call carries change 'I', positions only: the extra slot behind a contig never emits
    (kindel.py:390 loops over weights)."""
    slots = np.flatnonzero(((calls_all >> 4) & 3) == 3)
    if slots.size:
        c = np.searchsorted(batch.contig_slot, slots, side="right") - 1
        slots = slots[slots < batch.contig_slot[c] + batch.contig_len[c].astype(np.int64)]
    return slots


def _acgt_depth(run, slots):
    """A + C + G + T at the given slots, from the device table (a gather, not a copy of it) or the host one."""
    if run.counts is not None:
        import torch

        idx = torch.from_numpy(np.asarray(slots, dtype=np.int64)).to(run.counts.device)
        return run.counts[0:4].index_select(1, idx).sum(dim=0, dtype=torch.int64).cpu().numpy()
    return run.host_counts[0:4, slots].astype(np.int64).sum(axis=0)


def _insertion_qualities(run, slots):
    """{slot: Q of its inserted string} (kindel_b200/quality.py): D = max(min(depth, depth_next), count of the chosen
    string), the two depths the vote's 'I' rule compares; depth_next at a contig's last position is the empty slot
    behind it (kindel.py:405-412: 0)."""
    if len(slots) == 0:
        return {}
    slots = np.asarray(slots, dtype=np.int64)
    depth, depth_next = _acgt_depth(run, slots), _acgt_depth(run, slots + 1)
    out = {}
    for sl, d, dn in zip(slots.tolist(), depth.tolist(), depth_next.tolist()):
        _, tie, k = run.ins_table.consensus_count_at(sl)
        out[sl] = quality.insertion_phred(d, dn, k, tie)
    return out


def _slot_qualities(run, calls_all):
    """K2q over the run's table and calls: the device tensor when the table is on the device, else (host tables, e.g.
    a multi-GPU result) the four base columns and the calls go up to the current device and 1 B per slot comes back."""
    if run.vote_qual is not None:  # (the quality vote wrote its own Q)
        return run.vote_qual
    if run.counts is not None and run.calls_device is not None:
        return engine.consensus_qual(run.counts, run.calls_device)
    import torch

    dev = engine.require_cuda()
    n = calls_all.shape[0]
    n_pad = (n + 3) // 4 * 4
    cols = torch.zeros((4, n_pad), dtype=torch.int32, device=dev)
    calls = torch.zeros(n_pad, dtype=torch.uint8, device=dev)
    src = run.counts[0:4] if run.counts is not None else torch.from_numpy(np.ascontiguousarray(run.host_counts[0:4]))
    cols[:, :n] = src.to(dev)
    calls[:n] = torch.from_numpy(np.ascontiguousarray(calls_all, dtype=np.uint8)).to(dev)
    return engine.consensus_qual(cols, calls)[:n]


def _device_texts(run, calls_all, qual=None, ins_q=None):
    """K5: the consensus text of every contig assembled on the device (emitted-length scan + scatter); only the
    insertion strings of the 'I' sites are resolved on the host (from the event list) and handed over.  qual
    (extension): K2q's device qualities; K5q then adds the quality texts and the call returns (texts, quality
    texts)."""
    batch = run.batch
    slots = _insertion_slots(batch, calls_all)
    strings = []
    for sl in slots.tolist():
        text, tie = run.ins_table.consensus_at(sl)
        strings.append("N" if tie else text.lower())
    if qual is None:
        return engine.assemble(run.calls_device, batch, slots, strings)
    return engine.assemble(run.calls_device, batch, slots, strings, qual=qual,
                           ins_qual=[ins_q[sl] for sl in slots.tolist()])


def consensus_from_run(run, calls_all, bam_path, realign=False, min_depth=1, min_overlap=9,
                       clip_decay_threshold=0.1, mask_ends=50, trim_ends=False, uppercase=False, filters=None,
                       iupac_threshold=None, qualities=False, quality_vote=False):
    """Host half of bam_to_consensus: per contig, optional CDR patches, string assembly, report.  The call bytes
    already carry the vote; iupac_threshold (extension) only adds its lines to the report.  qualities (extension):
    see bam_to_consensus -- K2q (and, with the device text, K5q) on the device, the host assembly otherwise.
    quality_vote (extension): the calls are the run's vote(quality=True); the qualities are then K2w's and the report
    gains its lines."""
    qv_slots = None
    if quality_vote:
        if getattr(run, "vote_qual", None) is None:
            raise ValueError("quality_vote needs the run's quality vote: call vote(quality=True) first")
        qv_slots = run.quality_vote_sites(min_depth)
    ins_table = run.ins_table
    consensuses, refs_changes, refs_reports = [], {}, {}
    primers_name = getattr(getattr(run, "primers", None), "name", None)
    overlaps = run.overlap_stats if getattr(run, "mask_overlaps", False) else None
    on_device = run.counts is not None
    device_text = on_device and not realign and run.calls_device is not None
    qual_all = ins_q = qtexts = None
    if qualities:
        qual_all = _slot_qualities(run, calls_all)
        ins_q = _insertion_qualities(run, _insertion_slots(run.batch, calls_all))
        if not device_text:
            qual_all = qual_all.cpu().numpy()  # 1 B per slot for the host assembly
    texts = None
    if device_text:
        texts = _device_texts(run, calls_all, qual_all, ins_q) if qualities else _device_texts(run, calls_all)
        if qualities:
            texts, qtexts = texts
    for c, ref_id in enumerate(run.batch.contig_names):
        s, e = run.contig_slice(c)
        if on_device:
            # the call bytes, the insertion events and, for the report, the min / max ACGT depth are all that is
            # needed: reduced on the device instead of copying 76 B per position back
            d = run.counts[0:4, s:e - 1].sum(dim=0)
            report_weights = DepthRange(int(d.min().item()), int(d.max().item())) if e - 1 > s else DepthRange(0, 0)
        else:
            aln = run.alignment(c)  # host tables (another path produced them)
            report_weights = aln.weights
        if realign:
            if on_device:
                cdrps = cdrps_from_device(run.counts, s, e - 1, clip_decay_threshold, mask_ends)
            else:
                cdrps = cdrp_consensuses(aln.weights, aln.deletions, aln.clip_start_weights, aln.clip_end_weights,
                                         aln.clip_start_depth, aln.clip_end_depth, clip_decay_threshold, mask_ends)
            cdr_patches = merge_cdrps(cdrps, min_overlap)
        else:
            cdr_patches = None
        quals = None
        if texts is not None:
            cons, changes = texts[c], _changes_list(calls_all[s:e - 1])
            if qtexts is not None:
                quals = qtexts[c]
            if trim_ends:
                cons, quals = _trim_n(cons, quals)
            if uppercase:
                cons = cons.upper()
        elif qualities:
            cons, changes, quals = assemble_consensus(
                calls_all[s:e - 1], lambda p, s=s: ins_table.consensus_at(s + p), cdr_patches, trim_ends, uppercase,
                qual=qual_all[s:e - 1], ins_qual=lambda p, s=s: ins_q[s + p])
        else:
            cons, changes = assemble_consensus(calls_all[s:e - 1], lambda p, s=s: ins_table.consensus_at(s + p),
                                               cdr_patches, trim_ends, uppercase)
        qv_sites = None
        if qv_slots is not None:
            lo, hi = np.searchsorted(qv_slots, [s, e - 1])
            qv_sites = [str(x - s + 1) for x in qv_slots[lo:hi].tolist()]
        report = build_report(ref_id, report_weights, changes, cdr_patches, bam_path, realign, min_depth,
                              min_overlap, clip_decay_threshold, trim_ends, uppercase, filters, iupac_threshold,
                              primers=primers_name, overlaps=overlaps, quality_vote_sites=qv_sites,
                              normalised=getattr(run, "normalised", None),
                              deduplicated=getattr(run, "deduplicated", None))
        consensuses.append(consensus_seqrecord(cons, ref_id, quals))
        refs_reports[ref_id] = report
        refs_changes[ref_id] = changes
    return result(consensuses, refs_changes, refs_reports)


def weights(bam_path: "path to SAM/BAM file", relative: "output relative nucleotide frequencies" = False,
            confidence: "calculate confidence interval" = True, confidence_alpha: "confidence interval alpha" = 0.01,
            devices=None, min_base_quality=0, min_mapq=0, exclude_flags=0, primers=None, mask_overlaps=False,
            normalise=None, dedup=False):
    """DataFrame of per-site nucleotide frequencies, depth, consensus, clip starts/ends, confidence
    interval and entropy (reference kindel/kindel.py:558-630).  Integer columns come from the GPU
    table; the float tail is the reference's arithmetic, vectorised.  devices, the filters, primers,
    mask_overlaps, normalise and dedup: extensions, see pileup_run."""
    run = pileup_run(bam_path, devices, 1, min_base_quality, min_mapq, exclude_flags, primers=primers,
                     mask_overlaps=mask_overlaps, normalise=normalise, dedup=dedup)[0]
    return weights_from_run(run, relative, confidence, confidence_alpha)


def weights_from_run(run, relative=False, confidence=True, confidence_alpha=0.01):
    """Host half of `weights`: DataFrame from the count table of a finished pileup."""
    import pandas as pd
    import scipy.stats

    tab = run.host_counts
    frames = []
    for c, chrom in enumerate(run.batch.contig_names):
        s, e = run.contig_slice(c)
        L = e - s - 1
        t = tab[:, s:e].astype(np.int64)
        frames.append(pd.DataFrame({
            "chrom": [chrom] * L, "pos": np.arange(1, L + 1, dtype=np.int64),
            "A": t[0, :L], "C": t[1, :L], "G": t[2, :L], "T": t[3, :L], "N": t[4, :L],
            "insertions": t[6, 1:L + 1],  # row i reports the insertions of slot i (kindel.py:581)
            "deletions": t[5, :L], "clip_starts": t[7, :L], "clip_ends": t[8, :L],
        }))
    cols = ["chrom", "pos", "A", "C", "G", "T", "N", "insertions", "deletions", "clip_starts", "clip_ends"]
    weights_df = pd.concat(frames, ignore_index=True) if frames else pd.DataFrame(columns=cols)
    six = ["A", "C", "G", "T", "N", "deletions"]
    weights_df["depth"] = weights_df[six].sum(axis=1)
    consensus_depths = weights_df[six].max(axis=1)
    weights_df["consensus"] = consensus_depths.divide(weights_df.depth)
    rel = pd.DataFrame()
    for nt in six:
        rel[[nt]] = weights_df[[nt]].divide(weights_df.depth, axis=0)
        rel = rel.round({k: 4 for k in six})
    acgt = rel[["A", "C", "G", "T"]].values
    with np.errstate(invalid="ignore", divide="ignore"):
        weights_df["shannon"] = scipy.stats.entropy(acgt, axis=1) if len(acgt) else []
    if confidence:
        cnt = consensus_depths.to_numpy()
        nobs = weights_df["depth"].to_numpy()
        # Jeffreys interval per (count, depth) pair (kindel.py:569-574,619-624): an elementwise function of two small
        # integers, and megabases of positions share a few thousand distinct pairs -- evaluate those, gather the rest
        # (the same scipy call on the same inputs: bit-identical to the per-row result)
        base = int(nobs.max()) + 1 if len(nobs) else 1
        pair, inverse = np.unique(cnt.astype(np.int64) * base + nobs.astype(np.int64), return_inverse=True)
        ucnt, unobs = pair // base, pair % base
        lower, upper = scipy.stats.beta.interval(1 - confidence_alpha, ucnt + 0.5, unobs - ucnt + 0.5)
        weights_df["lower_ci"] = np.asarray(lower)[inverse]
        weights_df["upper_ci"] = np.asarray(upper)[inverse]
    if relative:
        for nt in ["A", "C", "G", "T", "N"]:
            weights_df[[nt]] = rel[[nt]]
    return weights_df.round(dict(consensus=3, lower_ci=3, upper_ci=3, shannon=3))


def variants(bam_path: "path to SAM/BAM file", abs_threshold: "absolute frequency above which to call variants" = 1,
             rel_threshold: "relative frequency (0.0-1.0) above which to call variants" = 0.01,
             only_variants: "exclude invariant sites from output" = False,
             absolute: "report absolute variant frequencies" = False, devices=None, min_base_quality=0, min_mapq=0,
             exclude_flags=0, primers=None, mask_overlaps=False, normalise=None, dedup=False):
    """EXTENSION -- not in the reference snapshot.  The reference's README (README.md:106-107) lists a `variants`
    sub-command ("Output variants exceeding specified absolute and relative frequency thresholds") but its code
    (kindel/kindel.py, kindel/cli.py) has no such function, so there is nothing to be bit-exact with: parity
    unpinned (SURVEY.md section 8c).  Defined here as a filter over the same integer table `weights` reports: per
    site, every allele (A, C, G, T, N, deletion) other than the site's most frequent one whose count exceeds
    `abs_threshold` AND whose share of the depth (A+C+G+T+N+deletions, as in `weights`) exceeds `rel_threshold`
    (variant_alleles).  Columns: chrom, pos, depth, consensus (allele letter, `-` = deletion), then one column per
    allele holding its relative (default) or absolute frequency where it is a variant and 0 elsewhere.  With
    only_variants the sites are selected on the device (K6, variant_sites) and only they are copied back.  primers,
    mask_overlaps, normalise, dedup: extensions, see pileup_run."""
    run = pileup_run(bam_path, devices, 1, min_base_quality, min_mapq, exclude_flags, primers=primers,
                     mask_overlaps=mask_overlaps, normalise=normalise, dedup=dedup)[0]
    return variants_from_run(run, abs_threshold, rel_threshold, only_variants, absolute)


_ALLELE_LETTERS = np.array(list("ACGTN-"))


def variant_alleles(t, abs_threshold, rel_threshold):
    """The rule of `variants` (extension) over count columns t (int64 [6, n]: A, C, G, T, N, deletions) ->
    (depth, top, share, is_var): depth = the sum of the six, top = the first most frequent allele, share = each
    count's true-division share of the depth (0 at depth 0), and is_var [6, n] = count > abs_threshold and
    share > rel_threshold and not the top allele.  K6 (kindel_b200/csrc/variants.cu) evaluates the same rule on the
    device."""
    depth = t.sum(axis=0)
    top = t.argmax(axis=0)                                        # first maximum in A,C,G,T,N,del order
    with np.errstate(invalid="ignore", divide="ignore"):
        share = np.where(depth > 0, t / np.maximum(depth, 1), 0.0)
    is_var = (t > abs_threshold) & (share > rel_threshold) & (np.arange(6)[:, None] != top[None, :])
    return depth, top, share, is_var


def variant_sites(run, abs_threshold=1, rel_threshold=0.01):
    """The sites of `variants --only-variants` (extension): (slot int64[n], counts int32[6, n], mask uint8[n]) in
    ascending slot order, bit k of mask set where allele k (A, C, G, T, N, deletions) is a variant.  A device run
    selects them with K6 and copies back only the sites; host tables (e.g. a multi-GPU result) go through
    variant_alleles."""
    batch = run.batch
    if run.counts is not None:
        return engine.variant_sites(run.counts, batch.contig_slot, batch.contig_len, abs_threshold, rel_threshold)
    tab = run.host_counts
    slots, counts, masks = [], [], []
    for c in range(batch.n_contigs):
        s, e = run.contig_slice(c)
        t = tab[0:6, s:e - 1].astype(np.int64)
        is_var = variant_alleles(t, abs_threshold, rel_threshold)[3]
        at = np.flatnonzero(is_var.any(axis=0))
        slots.append(s + at)
        counts.append(tab[0:6, s + at])
        masks.append((is_var[:, at].astype(np.uint8) << np.arange(6, dtype=np.uint8)[:, None]).sum(axis=0,
                                                                                               dtype=np.uint8))
    if not slots:
        return np.zeros(0, dtype=np.int64), np.zeros((6, 0), dtype=np.int32), np.zeros(0, dtype=np.uint8)
    return (np.concatenate(slots).astype(np.int64), np.concatenate(counts, axis=1).astype(np.int32),
            np.concatenate(masks).astype(np.uint8))


def _variants_frame(chrom, pos, t, abs_threshold, rel_threshold, absolute):
    """The `variants` rows of positions pos (1-based) of one contig with count columns t, and their is_var."""
    import pandas as pd

    depth, top, share, is_var = variant_alleles(t, abs_threshold, rel_threshold)
    value = np.where(is_var, t if absolute else np.round(share, 4), 0)
    df = pd.DataFrame({"chrom": [chrom] * pos.shape[0], "pos": pos, "depth": depth,
                       "consensus": np.where(depth > 0, _ALLELE_LETTERS[top], "N")})
    for k, a in enumerate(["A", "C", "G", "T", "N", "deletions"]):
        df[a] = value[k]
    return df, is_var


def variants_from_run(run, abs_threshold=1, rel_threshold=0.01, only_variants=False, absolute=False):
    """Host half of `variants` (extension; see there).  only_variants: the rows of variant_sites (K6 on a device run:
    only the sites leave the device), else every position from the whole table."""
    import pandas as pd

    alleles = ["A", "C", "G", "T", "N", "deletions"]
    frames = []
    if only_variants:
        site_slot, site_counts, _ = variant_sites(run, abs_threshold, rel_threshold)
        for c, chrom in enumerate(run.batch.contig_names):
            s, e = run.contig_slice(c)
            lo, hi = np.searchsorted(site_slot, [s, e - 1])
            if e - 1 == s:  # an empty contig, as below
                frames.append(_variants_frame(chrom, np.zeros(0, dtype=np.int64), np.zeros((6, 0), dtype=np.int64),
                                              abs_threshold, rel_threshold, absolute)[0])
                continue
            # one more row (an all-zero column, sliced off again) so that pandas infers every column's dtype from a
            # non-empty column even for a contig without sites, as it does for the per-position frame filtered below
            pos = np.append(site_slot[lo:hi] - s + 1, 0).astype(np.int64)
            t = np.zeros((6, hi - lo + 1), dtype=np.int64)
            t[:, :hi - lo] = site_counts[:, lo:hi]
            frames.append(_variants_frame(chrom, pos, t, abs_threshold, rel_threshold, absolute)[0].iloc[:hi - lo])
    else:
        tab = run.host_counts
        for c, chrom in enumerate(run.batch.contig_names):
            s, e = run.contig_slice(c)
            L = e - s - 1
            t = tab[0:6, s:s + L].astype(np.int64)                    # [6, L]
            frames.append(_variants_frame(chrom, np.arange(1, L + 1, dtype=np.int64), t, abs_threshold,
                                          rel_threshold, absolute)[0])
    cols = ["chrom", "pos", "depth", "consensus"] + alleles
    return pd.concat(frames, ignore_index=True) if frames else pd.DataFrame(columns=cols)


# ------------------------------------------------------------------------------------------------ VCF
# the VCF helpers under their kindel names (kindel_b200/vcf.py has them)
_strand_fields = vcf.strand_fields
check_max_sor = functools.partial(vcf.check_number, name="max_sor")
check_min_qual = functools.partial(vcf.check_number, name="min_qual")


def _vcf_header(run, abs_threshold, rel_threshold, filters, **options):
    """vcf.header of a run: its contigs, primers and mate masking; options: vcf.header's keywords."""
    normalised = getattr(run, "normalised", None)
    return vcf.header(run.batch.contig_names, run.batch.contig_len, abs_threshold, rel_threshold, filters,
                      getattr(run, "primers", None), getattr(run, "mask_overlaps", False),
                      normalise=None if normalised is None else normalised[0],
                      dedup=getattr(run, "deduplicated", None) is not None, **options)


def variants_vcf(bam_path, abs_threshold=1, rel_threshold=0.01, devices=None, min_base_quality=0, min_mapq=0,
                 exclude_flags=0, reference=None, strand=False, max_sor=None, primers=None, mask_overlaps=False,
                 samples=None, qual=False, min_qual=None, normalise=None, dedup=False, left_align=False) -> str:
    """Sites-only VCF 4.2 text of the sites of `variants --only-variants` (extension; `kindel variants --vcf`).

    kindel takes no reference sequence, so REF is the sample's own most frequent allele at the position: this is a
    file of the sample's minority variants, in the coordinates of the alignment's reference.  Per site: CHROM and the
    1-based POS; REF the top allele's letter (N when the top allele is N or a deletion, or the depth is 0); ALT the
    variant alleles among A, C, G, T and the deletion, in that order, the deletion written `*` (VCF 4.2: allele
    missing due to an upstream deletion, which is what the per-position deletion count is); ID and QUAL `.`, FILTER
    PASS; INFO DP (the depth A+C+G+T+N+deletions), AD (the REF count, then each ALT's) and AF (each ALT's share of the
    depth, rounded to 4 decimals: the value `variants` prints).  A site whose only variant allele is N is not
    written.  devices and the filters: extensions, see pileup_run.

    reference (extension: `--reference`): the FASTA the alignment was made against -- a path, or a Reference that
    reference.load_reference returned for this file's batch.  REF is then the reference's base, and the records are
    SNVs against it, deletions and insertions (variants_vcf_from_run has the rules).

    strand (extension: `--strand`): every record also carries ADF / ADR, the forward- and reverse-strand counts of REF
    and of each ALT, and SOR, the strand odds ratio of each ALT; max_sor (`--max-sor`, implies strand): FILTER `sor`
    where some ALT's SOR exceeds it.  vcf.strand_fields has the rules.

    primers (extension: `--primers`): see pileup_run; the records then count no primer base (the strand counts
    neither), and the header gets `##kindelPrimers=<the BED's file name>`.

    mask_overlaps (extension: `--mask-overlaps`): see pileup_run; DP, AD, AO and the strand counts then count each
    read pair once where its mates overlap, and the header gets `##kindelMateOverlaps=R2 masked where R1 covers`.

    bam_path a list or tuple of paths (extension: `kindel variants --vcf a.bam b.bam ...`): one VCF of all the
    samples, one FORMAT column each (DP:AD:AF), named by `samples` (unique, non-empty, no whitespace) or else by the
    files' names without their directories.  A record is written where some sample passes; INFO holds the values
    pooled over the samples, and without a reference REF is the pooled most frequent allele.  The options apply to
    every sample as they would to that sample alone; strand / max_sor are not available with a list (ValueError).
    kindel_b200/cohort.py has the layout and the union rules; a list of one path gives the data lines of that path
    alone in columns 1-8.

    qual (extension: `--qual`): a base-quality QUAL.  Every record with a base ALT (A, C, G or T) gets QUAL, the largest
    AQ of its base ALTs, and INFO ;BQ= (the mean Phred of the counted bases of REF and of each ALT, `.` where there is
    none or the allele is no base) and ;AQ= (per ALT, `.` for `*`).  min_qual (`--min-qual`, implies qual): FILTER
    `lowqual` where QUAL < min_qual.  A record without a base ALT (an indel, a `*`-only site) keeps QUAL `.`.  The
    qualities are summed on the device (K11, include/kindel_b200.h); vcf.allele_quality has the model.  Not available
    with several samples (ValueError); a kept read without qualities is a ValueError.

    normalise (extension: `--normalise N`, needs a named `primers` scheme): see pileup_run; every sample's reads are
    capped as it would be alone, and the header gets `##kindelNormalise=N` after `##kindelPrimers`.

    dedup (extension: `--dedup`): see pileup_run; every sample's duplicates are removed as they would be alone, and the
    header gets `##kindelDedup=fragment ends, base-quality score` after `##kindelPrimers`, before `##kindelNormalise`.

    left_align (extension: `--left-align`, needs `reference`; ValueError otherwise): every deletion and insertion event
    is moved to its leftmost place against the reference before the events are grouped and tested, so that one indel
    an aligner placed at several offsets of a repeat is one record with the count of all its placements
    (variants_vcf_from_run has the rule).  The header gets `##kindelLeftAlign=leftmost against the reference` after
    `##reference`."""
    left_align = check_left_align(left_align, reference)
    max_sor = check_max_sor(max_sor)
    strand = bool(strand) or max_sor is not None
    min_qual = check_min_qual(min_qual)
    qual = bool(qual) or min_qual is not None
    if isinstance(bam_path, (list, tuple)):
        if strand:
            raise ValueError("strand and max_sor are not available with several samples")
        if qual:
            raise ValueError("qual and min_qual are not available with several samples")
        from . import cohort

        return cohort.variants_vcf(bam_path, abs_threshold, rel_threshold, devices, min_base_quality, min_mapq,
                                   exclude_flags, reference=reference, primers=primers, mask_overlaps=mask_overlaps,
                                   samples=samples, normalise=normalise, dedup=dedup,
                                   **({"left_align": True} if left_align else {}))
    if samples is not None:
        raise ValueError("samples= names the columns of several samples: pass the alignment files as a list")
    filters = (min_base_quality, min_mapq, exclude_flags)
    run = pileup_run(bam_path, devices, 1, *filters, strand=strand, primers=primers, mask_overlaps=mask_overlaps,
                     qual=qual, normalise=normalise, dedup=dedup)[0]
    return variants_vcf_from_run(run, abs_threshold, rel_threshold, filters, reference=reference, strand=strand,
                                 max_sor=max_sor, qual=qual, min_qual=min_qual, left_align=left_align)


def check_left_align(left_align, reference) -> bool:
    """left_align as a bool; on without a reference raises ValueError (the shift is against its bases)."""
    if left_align and reference is None:
        raise ValueError("left_align needs a reference: the indels are moved against its bases")
    return bool(left_align)


def _quality_at(run, slots):
    """(qsum int64 [4, n], emass list of n ints) of the run's quality table at host slots."""
    import torch

    qsum, emass = run.quality_table()
    slots = np.asarray(slots, dtype=np.int64)
    if slots.size == 0:
        return np.zeros((4, 0), dtype=np.int64), []
    idx = torch.from_numpy(slots).to(qsum.device)
    q = qsum.index_select(1, idx).cpu().numpy().view(np.uint32).astype(np.int64)
    return q, [int(x) for x in emass.index_select(0, idx).cpu().numpy().view(np.uint64).tolist()]


def _rows_at(table, slots):
    """Columns 0-5 of a device table at host slots, int64 [6, n] on the host."""
    import torch

    slots = np.asarray(slots, dtype=np.int64)
    if slots.size == 0:
        return np.zeros((6, 0), dtype=np.int64)
    idx = torch.from_numpy(slots).to(table.device)
    return table[0:6].index_select(1, idx).cpu().numpy().astype(np.int64)


def _reverse_strand(run, slot, deletions, ins=None, ref=None):
    """The strand option of vcf.records from the run's reverse-strand reads: their rows at the sites and, with a
    reference (deletions given), their DPa at the sites, each deletion's reverse count and depth and each insertion
    string's reverse reads at a slot (the event rows whose read is reverse).  ins / ref (extension: left_align): the
    insertion table the records read (default: the run's) and the device reference codes the reverse reads'
    deletion events are left-aligned against (None: as the aligner placed them)."""
    rev_table, rev_batch = run.reverse_table()
    rows = _rows_at(rev_table, slot)
    if deletions is None:
        return rows, None, None, None, None
    batch = run.batch

    def strings_at(s):
        table = run.ins_table if ins is None else ins
        events = table.rows_at(s)
        out = {}
        for text, r in zip(table.strings_at(s), batch.reverse[events[:, 1].astype(np.int64)].tolist()):
            out[text] = out.get(text, 0) + r
        return out

    return (rows, _rows_at(rev_table, vcf.dpa_slots(batch, slot)).sum(axis=0),
            engine.deletion_counts(rev_batch, deletions[0], deletions[1], **({} if ref is None else {"ref": ref})),
            _rows_at(rev_table, deletions[0]).sum(axis=0), strings_at)


def variants_vcf_from_run(run, abs_threshold=1, rel_threshold=0.01, filters=None, reference=None, strand=False,
                          max_sor=None, qual=False, min_qual=None, left_align=False) -> str:
    """Host half of variants_vcf (see there): the VCF text of a finished pileup.  filters: (min_base_quality,
    min_mapq, exclude_flags) as the pileup applied them, for the header.  reference, strand, max_sor: see variants_vcf;
    vcf.records has the rules of the records.  Strand needs a run whose batch has `reverse`
    (ValueError otherwise).  A run piled with primers (extension) adds its `##kindelPrimers` line, one piled with
    mask_overlaps its `##kindelMateOverlaps` line, one piled with normalise its `##kindelNormalise` line, one piled
    with dedup its `##kindelDedup` line.

    Strand counts (ADF, ADR): without a reference they are the reverse table's counts of the record's AD columns and
    the total's minus those, so ADF + ADR == AD.  With one, an SNV's the same (REF 0 where the reference has no A, C,
    G or T); an indel's ALT entry is its reads on that strand (the reverse sub-batch's deletion events, the insertion
    events of reverse reads) and its REF entry max(DP_s - AO_s, 0), DP_s the record's DP taken from strand s's table,
    so ADF[1] + ADR[1] == AO.  qual / min_qual: see variants_vcf; needs a run whose batch has `qual8`.

    left_align (extension, needs a reference): with g the reference codes and s0 the contig's first slot, a deletion
    event (r, n) moves left while r > s0, g[r-1] is A, C, G or T and g[r-1] == g[r+n-1] (K15d, on the K7 groups, whose
    keys that meet are summed); an insertion event at p with string t moves left while p > s0, g[p-1] is a base and the
    last base of the string rotated so far equals it, the string rotating right by one each step (K15i, on every event
    row K10 did not drop; a base that is not A, C, G or T stops it).  The groups, the tests, DP / DPa, the strand
    counts and the records are then the rules above over the moved events; the strings at a slot are in the order of
    their rows.  The insertion candidates come from K6r over the table with column 6 replaced by K15i's per-slot count
    of moved rows.  Columns 0-6 of the table and the SNV records do not change."""
    left_align = check_left_align(left_align, reference)
    max_sor = check_max_sor(max_sor)
    strand = bool(strand) or max_sor is not None
    min_qual = check_min_qual(min_qual)
    qual = bool(qual) or min_qual is not None
    if strand and run.batch.reverse is None:
        raise ValueError("strand needs the reads' strands: decode the batch with strand=True")
    if qual and run.batch.qual8 is None:
        raise ValueError("qual needs the reads' qualities: decode the batch with qual=True")
    batch = run.batch
    ref = None
    if reference is not None:
        from .reference import Reference, load_reference

        ref = reference if isinstance(reference, Reference) else load_reference(reference, batch)
    lines = _vcf_header(run, abs_threshold, rel_threshold, filters, reference_name=None if ref is None else ref.name,
                        strand=strand, max_sor=max_sor, qual=qual, min_qual=min_qual, left_align=left_align)
    dpa = dels = codes = None
    ins = None  # the left-aligned insertion table (left_align), else the run's
    if ref is None:
        slot, site_counts, mask = variant_sites(run, abs_threshold, rel_threshold)
    else:
        # host tables (the multi-GPU result): the reduced table and the batch go to this process's GPU
        counts, dbatch = run.device_tables()
        sites_table, codes = counts, ref.codes
        if left_align:
            import torch

            codes = torch.from_numpy(np.ascontiguousarray(ref.codes, dtype=np.uint8)).to(counts.device)
            hist, ins = run.left_aligned_insertions(codes)
            sites_table = torch.empty((7, counts.shape[1]), dtype=torch.int32, device=counts.device)
            sites_table[0:6] = counts[0:6]
            sites_table[6] = hist
        slot, site_counts, dpa, mask = engine.variant_sites_ref(sites_table, batch.contig_slot, batch.contig_len,
                                                                codes, abs_threshold, rel_threshold)
        dpa = dpa[None]
        moved = {"ref": codes} if left_align else {}  # (the keyword only when on: the call stays as it was otherwise)
        d_slot, d_len, d_cnt, d_depth = engine.deletion_alleles(dbatch, counts, abs_threshold, rel_threshold, **moved)
        dels = d_slot, d_len, d_cnt[None], d_depth[None]
    lines += vcf.records(batch, abs_threshold, rel_threshold, slot, mask, site_counts[None, 0:6].astype(np.int64),
                         ref_codes=None if ref is None else ref.codes, dpa=dpa,
                         strings_at=lambda j, s: (run.ins_table if ins is None else ins).dict_at(s), deletions=dels,
                         strand=_reverse_strand(run, slot, dels, ins, codes if left_align else None) if strand else None,
                         max_sor=max_sor,
                         qual=_quality_at(run, slot) if qual else None, min_qual=min_qual)
    return "\n".join(lines) + "\n"


def features(bam_path: "path to SAM/BAM file", devices=None, min_base_quality=0, min_mapq=0, exclude_flags=0,
             primers=None, mask_overlaps=False, normalise=None, dedup=False):
    """DataFrame of relative per-site nucleotide frequencies, indels and entropy
    (reference kindel/kindel.py:633-664), including its indexing of `i`/`d` by global row number
    into the LAST contig's tables (IndexError on most multi-contig files, SURVEY.md A-14).
    devices, the filters, primers, mask_overlaps, normalise and dedup: extensions, see pileup_run."""
    return features_from_run(pileup_run(bam_path, devices, 1, min_base_quality, min_mapq, exclude_flags,
                                        primers=primers, mask_overlaps=mask_overlaps, normalise=normalise,
                                        dedup=dedup)[0])


def features_from_run(run):
    """Host half of `features`."""
    import pandas as pd
    import scipy.stats

    tab = run.host_counts
    frames = []
    last = None
    for c, chrom in enumerate(run.batch.contig_names):
        s, e = run.contig_slice(c)
        L = e - s - 1
        t = tab[:, s:e].astype(np.int64)
        last = t
        frames.append(pd.DataFrame({"chrom": [chrom] * L, "pos": np.arange(1, L + 1, dtype=np.int64),
                                    "A": t[0, :L], "C": t[1, :L], "G": t[2, :L], "T": t[3, :L], "N": t[4, :L]}))
    df = pd.concat(frames, ignore_index=True) if frames else pd.DataFrame(
        columns=["chrom", "pos", "A", "C", "G", "T", "N"])
    n_rows = len(df)
    if n_rows:
        if n_rows > last.shape[1]:
            raise IndexError("list index out of range")  # aln.insertions[pos], kindel.py:645
        df["i"] = last[6, :n_rows]
        df["d"] = last[5, :n_rows]
    else:
        df["i"] = []
        df["d"] = []
    df["depth"] = df[["A", "C", "G", "T", "N", "d"]].sum(axis=1)
    consensus_depths = df[["A", "C", "G", "T", "N"]].max(axis=1)
    df["consensus"] = consensus_depths.divide(df.depth)
    for nt in ["A", "C", "G", "T", "N", "i", "d"]:
        df[[nt]] = df[[nt]].divide(df.depth, axis=0)
    vals = df[["A", "C", "G", "T", "i", "d"]].values
    with np.errstate(invalid="ignore", divide="ignore"):
        df["shannon"] = scipy.stats.entropy(vals.astype(np.float64), axis=1) if n_rows else []
    return df.round(3)


def plotly_clips(bam_path):
    """Plotly HTML of depth / clip / indel traces of the first contig (reference kindel/kindel.py:667-703)."""
    import plotly.graph_objs as go
    import plotly.offline as py

    aln = list(parse_bam(bam_path).items())[0][1]
    aligned_depth = np.asarray(aln.weights.cols).sum(axis=0).tolist()
    ins = np.asarray(aln.table[6]).tolist()
    x_axis = list(range(1, len(aligned_depth) + 1))
    traces = [
        go.Scattergl(x=x_axis, y=aligned_depth, mode="lines", name="Aligned depth"),
        go.Scattergl(x=x_axis, y=aln.clip_depth, mode="lines", name="Soft clip total depth"),
        go.Scattergl(x=x_axis, y=aln.clip_start_depth, mode="lines", name="Soft clip start depth"),
        go.Scattergl(x=x_axis, y=aln.clip_end_depth, mode="lines", name="Soft clip end depth"),
        go.Scattergl(x=x_axis, y=aln.clip_starts, mode="markers", name="Soft clip starts"),
        go.Scattergl(x=x_axis, y=aln.clip_ends, mode="markers", name="Soft clip ends"),
        go.Scattergl(x=x_axis, y=ins, mode="markers", name="Insertions"),
        go.Scattergl(x=x_axis, y=aln.deletions, mode="markers", name="Deletions"),
    ]
    fig = go.Figure(data=traces, layout=go.Layout(xaxis=dict(type="linear", autorange=True),
                                                  yaxis=dict(type="linear", autorange=True)))
    out_fn = os.path.splitext(os.path.split(bam_path)[1])[0]
    py.plot(fig, filename=out_fn + ".plot.html")


# ------------------------------------------------------------------------------------- amplicons (extension)
AMPLICON_COLUMNS = ["sample", "contig", "amplicon", "pool", "start", "end", "insert_start", "insert_end", "reads",
                    "mean_depth", "lowest_depth", "covered", "status"]


def amplicon_label_counts(labels, n_amplicons):
    """int64 [3 + n_amplicons] on the device: the reads labelled -3, -2, -1, then those of each amplicon.  The classes
    are three reductions and only the assigned reads go through torch.bincount, so no bin takes millions of atomic
    adds: on cfg 4's 6.7 M reads, 74 % of them unprimed, this takes 0.49 ms where one bincount of all labels takes
    3.86 ms; on an amplicon batch of that size 0.86 ms against 0.51 ms (one H100 at 700 W,
    profiles/h100_bench_n1_cfg4_5Mb_200x_amplicons.json)."""
    import torch

    lab = labels.long()
    classes = torch.stack([(lab == k).sum() for k in (-3, -2, -1)])
    return torch.cat([classes, torch.bincount(lab[lab >= 0], minlength=n_amplicons)])


def amplicons_from_run(run, scheme, min_depth=20):
    """The amplicon table of one piled run (extension: `kindel amplicons`): a DataFrame with the columns of
    AMPLICON_COLUMNS but `sample`, one row per amplicon of `scheme` (primers.AmpliconScheme) on the run's contigs, in
    contig order, then start, then name.  K12 labels every read of the run's device batch (device_tables(), so a
    multi-GPU run too) and amplicon_label_counts counts them on the device; K12d reduces A+C+G+T of the count table over each
    insert.  `reads` = the reads K12 gives to the amplicon, `mean_depth` = the sum over the insert / its length,
    `lowest_depth` its minimum, `covered` = the share of its positions with A+C+G+T >= min_depth, `status` PASS or
    `dropout` (mean_depth < min_depth).  attrs["reads"] = (kept, assigned, unprimed, mispaired, ambiguous)."""
    import pandas as pd

    from .primers import AMBIGUOUS, amplicon_arrays

    batch = run.batch
    arrays = amplicon_arrays(scheme, batch.contig_names, batch.contig_len)
    counts, dbatch = run.device_tables()
    n = arrays.n_amplicons
    per = amplicon_label_counts(engine.assign_amplicons(dbatch, arrays), n).cpu().numpy()
    stats = engine.amplicon_depth(counts, arrays, min_depth, batch.contig_slot, batch.contig_len).cpu().numpy()
    idx = arrays.amplicon
    length = (arrays.insert_end - arrays.insert_start).astype(np.int64)
    mean = stats[:, 0] / np.maximum(length, 1) if n else np.zeros(0)
    df = pd.DataFrame({
        "contig": [batch.contig_names[c] for c in arrays.contig.tolist()],
        "amplicon": [scheme.names[j] for j in idx.tolist()],
        "pool": [scheme.pool[j] for j in idx.tolist()],
        "start": scheme.start[idx], "end": scheme.end[idx],
        "insert_start": arrays.insert_start.astype(np.int64), "insert_end": arrays.insert_end.astype(np.int64),
        "reads": per[-AMBIGUOUS:].astype(np.int64),
        "mean_depth": mean, "lowest_depth": stats[:, 1], "covered": stats[:, 2] / np.maximum(length, 1),
        "status": np.where(mean < min_depth, "dropout", "PASS") if n else np.zeros(0, dtype=object),
    }, columns=AMPLICON_COLUMNS[1:])
    df.attrs["reads"] = (int(batch.n_reads), int(per[-AMBIGUOUS:].sum()), int(per[2]), int(per[1]), int(per[0]))
    return df


def amplicons(bam_path, primers, min_depth=20, devices=None, min_base_quality=0, min_mapq=0, exclude_flags=0,
              mask_overlaps=False, samples=None, normalise=None, dedup=False):
    """Per sample and amplicon of a tiled primer scheme, its reads and the depth of its insert (extension: `kindel
    amplicons`; the reference has no such command).  bam_path: one alignment file or a list of them; primers: a named
    primer BED (primers.load_scheme) or an AmpliconScheme.  Each file is piled with `primers=` the scheme's rows, under
    the filters and mask_overlaps as in pileup_run, so the depths are the ones `consensus --primers` sees; files are
    piled one after the other, and samples are named by cohort.sample_names (`samples=` or the file names).  Returns
    a DataFrame with the columns AMPLICON_COLUMNS, in argument order of the samples, then amplicons_from_run's order;
    attrs["reads"] = {sample: (kept, assigned, unprimed, mispaired, ambiguous)}.  normalise (extension: `--normalise
    N`): each file's reads are capped first (pileup_run), so the reads and depths are those of the kept reads, and
    attrs["dropped"] = {sample: the reads over the cap}.  dedup (extension: `--dedup`): each file's duplicates are
    removed first (pileup_run), and attrs["duplicates"] = {sample: the reads removed}."""
    import pandas as pd

    from .cohort import sample_names
    from .primers import as_scheme

    scheme = as_scheme(primers)
    paths = [bam_path] if isinstance(bam_path, (str, os.PathLike)) else list(bam_path)
    names = sample_names(paths, samples)
    normalise = check_normalise(normalise)
    dedup = check_dedup(dedup)
    frames, reads, dropped, duplicates = [], {}, {}, {}
    for path, name in zip(paths, names):
        run, _ = pileup_run(path, devices, 1, min_base_quality, min_mapq, exclude_flags,
                            primers=scheme.primers if normalise is None else scheme, mask_overlaps=mask_overlaps,
                            normalise=normalise, dedup=dedup)
        df = amplicons_from_run(run, scheme, min_depth)
        reads[name] = df.attrs["reads"]
        if normalise is not None:
            dropped[name] = run.normalised[1]
        if dedup:
            pairs, singles, _, _ = run.deduplicated
            duplicates[name] = 2 * pairs + singles
        df.insert(0, "sample", name)
        frames.append(df)
        del run
    out = pd.concat(frames, ignore_index=True) if frames else pd.DataFrame(columns=AMPLICON_COLUMNS)
    out.attrs["reads"] = reads
    if normalise is not None:
        out.attrs["dropped"] = dropped
    if dedup:
        out.attrs["duplicates"] = duplicates
    return out
