"""Several samples in one VCF (extension: `kindel variants --vcf a.bam b.bam ...`, kindel.variants_vcf with a list).

The one place that knows the shared layout of a multi-sample VCF; it piles the samples and gathers what vcf.records
writes:

  layout    the union of the samples' batch contigs -- the first file's batch order, then each contig a later file
            shows first, in that file's order; a name given two @SQ lengths is an error -- laid out by
            bamio.layout_slots.  Contigs are only ever appended, so a contig's slot never moves while samples are
            added: the stacked table grows at its end.
  table     T, int32 [S][7][n_slots] on the device: columns 0-6 (A, C, G, T, N, deletions, insertion ops) of each
            sample's pileup gathered into its slice; zeros where a sample lacks a contig.  Each sample is piled by
            kindel.pileup_run as it would be alone and freed before the next one, so the device holds T and one
            sample's run: 28 * S * n_slots bytes plus one pileup.
  sites     K6m (engine.variant_sites_multi) over T: the slots where some sample passes, with the OR of the bits.
  records   vcf.records over every sample's rows at the sites, with FORMAT DP:AD:AF per sample: the deletions are
            engine.deletion_union's union of the (slot, length) keys that pass in some sample, the insertions the
            union of the samples' strings at a candidate slot (vcf.records has the rules).
  left_align  (extension) each sample's deletion groups (K15d) and insertion rows (K15i) are left-aligned against the
            reference in the sample's own slots before its run is dropped; T's column 6 is then K15i's per-slot count
            of the sample's moved rows, and the unions run over the moved keys and strings."""
from __future__ import annotations

import os

import numpy as np

from . import bamio, engine, vcf
from .insertions import decode_events

_LEN_BITS = engine._LEN_BITS
_CHUNK = 1 << 24  # int32 entries of T gathered to the host at once (64 MB)


def sample_names(paths, samples=None) -> list:
    """The VCF's column names: `samples` when given (one per path, unique, non-empty, no whitespace), else the files'
    names without their directories (two inputs with one file name: ValueError)."""
    if samples is not None:
        names = list(samples)
        if len(names) != len(paths):
            raise ValueError("samples= holds %d names for %d alignment files" % (len(names), len(paths)))
        for nm in names:
            if not isinstance(nm, str) or not nm or any(ch.isspace() for ch in nm):
                raise ValueError("sample name %r: a name must be a non-empty string without whitespace" % (nm,))
        seen = set()
        for nm in names:
            if nm in seen:
                raise ValueError("sample name %r is given twice" % nm)
            seen.add(nm)
        return names
    names, first = [], {}
    for p in paths:
        nm = os.path.basename(os.fspath(p))
        if nm in first:
            raise ValueError("%s and %s have the same file name %r: name the samples with samples=" % (first[nm], p, nm))
        first[nm] = os.fspath(p)
        names.append(nm)
    return names


class Layout:
    """The shared contig layout (the attributes reference.load_reference reads of a batch)."""

    def __init__(self):
        self.contig_names, self._len, self._owner = [], [], []
        self.contig_len = np.zeros(0, dtype=np.int64)
        self.contig_slot, self.n_slots = bamio.layout_slots(self.contig_len)

    def add(self, batch, path) -> np.ndarray:
        """Append the contigs of `batch` this layout lacks; the shared contig index of each of its contigs."""
        index = {nm: c for c, nm in enumerate(self.contig_names)}
        out = np.zeros(batch.n_contigs, dtype=np.int64)
        for c, (nm, L) in enumerate(zip(batch.contig_names, np.asarray(batch.contig_len).tolist())):
            k = index.get(nm)
            if k is None:
                k = index[nm] = len(self.contig_names)
                self.contig_names.append(nm)
                self._len.append(int(L))
                self._owner.append(os.fspath(path))
            elif self._len[k] != int(L):
                raise ValueError("contig %r has length %d in %s but %d in %s" % (nm, self._len[k], self._owner[k],
                                                                                  int(L), os.fspath(path)))
            out[c] = k
        self.contig_len = np.asarray(self._len, dtype=np.int64)
        self.contig_slot, self.n_slots = bamio.layout_slots(self.contig_len)
        return out


class Cohort:
    """The samples piled one by one into the stacked table T over the shared layout, with what the records need of
    each: its deletion groups (device) and its insertion events (host), both in shared slots."""

    def __init__(self, paths, devices=None, filters=(0, 0, 0), primers=None, mask_overlaps=False, normalise=None,
                 dedup=False, left_align=None):
        """left_align (extension): None, or a callable giving the reference codes (uint8 numpy) of a sample's batch
        from (batch, its shared slots of each contig slot, those slots) -- the samples are then left-aligned."""
        from .kindel import _normalise_scheme, check_dedup, check_normalise, pileup_run

        import torch

        self.layout = Layout()
        self.normalise = check_normalise(normalise)
        self.dedup = check_dedup(dedup)
        self.primers, self.scheme = _normalise_scheme(primers, self.normalise)  # (the scheme: normalise's, loaded once)
        self.mask_overlaps = bool(mask_overlaps)
        self.table = None
        self.deletions = []   # per sample: (key = shared slot << 28 | length, count), device, keys ascending
        self.insertions = []  # per sample: (shared slot int64[m] ascending, strings), first-seen order inside a slot
        S = len(paths)
        mbq, mapq, flags = filters
        for i, path in enumerate(paths):
            run = pileup_run(path, devices, 1, mbq, mapq, flags,
                             primers=self.primers if self.scheme is None else self.scheme,
                             mask_overlaps=self.mask_overlaps, normalise=self.normalise, dedup=self.dedup)[0]
            counts, dbatch = run.device_tables()
            batch = run.batch
            shared = self.layout.add(batch, path)
            dev = counts.device
            if self.table is None:
                self.table = torch.zeros((S, 7, self.layout.n_slots), dtype=torch.int32, device=dev)
            elif self.table.shape[2] < self.layout.n_slots:  # new contigs at the end: the table grows there
                grown = torch.zeros((S, 7, self.layout.n_slots), dtype=torch.int32, device=dev)
                grown[:, :, :self.table.shape[2]] = self.table
                self.table = grown
            src_slot = np.asarray(batch.contig_slot, dtype=np.int64)
            offset = self.layout.contig_slot[shared] - src_slot  # shared slot - sample slot, per sample contig
            span = np.asarray(batch.contig_len, dtype=np.int64) + 1
            src = np.concatenate([np.arange(s, s + n) for s, n in zip(src_slot.tolist(), span.tolist())]
                                 or [np.zeros(0, dtype=np.int64)]).astype(np.int64)
            dst = src + np.repeat(offset, span)
            columns, codes, ins = counts[0:7], None, run.ins_table if left_align is None else None
            if left_align is not None:
                codes = torch.from_numpy(np.ascontiguousarray(left_align(batch, src, dst), dtype=np.uint8)).to(dev)
                hist, ins = run.left_aligned_insertions(codes)
                columns = torch.cat([counts[0:6], hist[None]])
            if src.size:
                self.table[i, :, torch.from_numpy(dst).to(dev)] = columns.index_select(1, torch.from_numpy(src).to(dev))
            self.deletions.append(self._deletion_keys(dbatch, src_slot, offset, codes))
            ev_slot = ins.slots
            c_of = np.searchsorted(src_slot, ev_slot, side="right") - 1
            ins_slot = ev_slot + offset[c_of] if ev_slot.size else ev_slot
            order = np.argsort(ins_slot, kind="stable")
            strings = self._strings(ins)
            self.insertions.append((ins_slot[order], [strings[k] for k in order.tolist()]))
            del run, counts, dbatch  # the sample's device batch and table go before the next one is piled

    @staticmethod
    def _strings(ins) -> list:
        """The strings of every row of an insertion table, in its row order (rotated where it has rotations)."""
        strings = decode_events(ins.batch, ins.events)
        if ins.rot is None:
            return strings
        return [t[len(t) - k:] + t[:len(t) - k] if k else t for t, k in zip(strings, ins.rot.tolist())]

    @staticmethod
    def _deletion_keys(dbatch, src_slot, offset, codes=None):
        import torch

        key, cnt = engine._deletion_groups(dbatch, codes)
        if key.numel() == 0:
            return key, cnt
        slot = key >> _LEN_BITS
        cs = torch.from_numpy(src_slot).to(key.device)
        c = torch.searchsorted(cs, slot, right=True) - 1
        key = key + (torch.from_numpy(offset).to(key.device)[c] << _LEN_BITS)
        key, order = torch.sort(key)
        return key, cnt[order]

    # ------------------------------------------------------------------------------------------------ gathers
    def rows(self, slots) -> np.ndarray:
        """Columns 0-5 of every sample at host slots: int64 [S, 6, n], gathered from T in chunks."""
        import torch

        slots = np.asarray(slots, dtype=np.int64)
        S = self.table.shape[0]
        out = np.zeros((S, 6, slots.size), dtype=np.int64)
        step = max(1, _CHUNK // (6 * S))
        for lo in range(0, slots.size, step):
            idx = torch.from_numpy(slots[lo:lo + step]).to(self.table.device)
            out[:, :, lo:lo + step] = self.table[:, 0:6].index_select(2, idx).cpu().numpy()
        return out

    def strings_at(self, i, slot) -> dict:
        """{string: count} of sample i's insertion events at a shared slot, in first-seen order."""
        slots, strings = self.insertions[i]
        lo, hi = np.searchsorted(slots, [slot, slot + 1])
        out = {}
        for s in strings[lo:hi]:
            out[s] = out.get(s, 0) + 1
        return out


# ---------------------------------------------------------------------------------------------------- text
def variants_vcf(paths, abs_threshold=1, rel_threshold=0.01, devices=None, min_base_quality=0, min_mapq=0,
                 exclude_flags=0, reference=None, primers=None, mask_overlaps=False, samples=None,
                 normalise=None, dedup=False, left_align=False) -> str:
    """The multi-sample VCF of kindel.variants_vcf given a list of paths (see there for the rules).  left_align
    (extension) needs a reference (ValueError otherwise); a Reference given with it must be the one of the samples'
    shared layout."""
    from .reference import Reference, load_reference, read_fasta, reference_codes

    if left_align and reference is None:
        raise ValueError("left_align needs a reference: the indels are moved against its bases")
    paths = [os.fspath(p) for p in paths]
    if not paths:
        raise ValueError("variants_vcf needs at least one alignment file")
    names = sample_names(paths, samples)
    filters = (min_base_quality, min_mapq, exclude_flags)
    fasta = codes_of = None
    if left_align:
        if isinstance(reference, Reference):
            def codes_of(batch, src, dst):  # the shared layout's codes, gathered into the sample's slots
                out = np.full(int(batch.n_slots), 4, dtype=np.uint8)
                out[src] = reference.codes[dst]
                return out
        else:
            fasta = read_fasta(reference)  # one parse for every sample and the shared layout

            def codes_of(batch, src, dst):
                return reference_codes(fasta, batch, reference)
    cohort = Cohort(paths, devices, filters, primers, mask_overlaps, normalise, dedup, codes_of)
    lay = cohort.layout
    ref = None
    if isinstance(reference, Reference):
        ref = reference
    elif fasta is not None:
        ref = Reference(reference_codes(fasta, lay, reference), os.path.basename(os.fspath(reference)))
    elif reference is not None:
        ref = load_reference(reference, lay)
    lines = vcf.header(lay.contig_names, lay.contig_len, abs_threshold, rel_threshold, filters, cohort.primers,
                       cohort.mask_overlaps, reference_name=None if ref is None else ref.name, samples=names,
                       normalise=cohort.normalise, dedup=cohort.dedup, left_align=bool(left_align))
    return "\n".join(lines + records(cohort, None if ref is None else ref.codes, abs_threshold, rel_threshold)) + "\n"


def records(cohort, ref_codes, abs_threshold, rel_threshold) -> list:
    """The data lines of the cohort (vcf.records with FORMAT): K6m's sites, every sample's rows there (and at DPa's
    slots), its insertion strings and the deletions that pass in some sample."""
    lay = cohort.layout
    slot, mask = (x.cpu().numpy() for x in engine.variant_sites_multi(
        cohort.table, lay.contig_slot, lay.contig_len, ref_codes, abs_threshold, rel_threshold))
    dpa = dels = None
    if ref_codes is not None:
        if (mask & 64).any():
            dpa = cohort.rows(vcf.dpa_slots(lay, slot)).sum(axis=1)  # [S, n]
        dels = engine.deletion_union(cohort.deletions, cohort.table, abs_threshold, rel_threshold)
    return vcf.records(lay, abs_threshold, rel_threshold, slot, mask, cohort.rows(slot), ref_codes=ref_codes, dpa=dpa,
                       strings_at=cohort.strings_at, deletions=dels, per_sample=True)
