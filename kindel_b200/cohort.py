"""Several samples in one VCF (extension: `kindel variants --vcf a.bam b.bam ...`, kindel.variants_vcf with a list).

The one place that knows the shared layout and the union rules of a multi-sample VCF:

  layout    the union of the samples' batch contigs -- the first file's batch order, then each contig a later file
            shows first, in that file's order; a name given two @SQ lengths is an error -- laid out by
            bamio.layout_slots.  Contigs are only ever appended, so a contig's slot never moves while samples are
            added: the stacked table grows at its end.
  table     T, int32 [S][7][n_slots] on the device: columns 0-6 (A, C, G, T, N, deletions, insertion ops) of each
            sample's pileup gathered into its slice; zeros where a sample lacks a contig.  Each sample is piled by
            kindel.pileup_run as it would be alone and freed before the next one, so the device holds T and one
            sample's run: 28 * S * n_slots bytes plus one pileup.
  sites     K6m (engine.variant_sites_multi) over T: the slots where some sample passes, with the OR of the bits.
  records   the single-sample writer's records, with INFO pooled over the samples and FORMAT DP:AD:AF per sample;
            deletions are the union of the (slot, length) keys that pass in some sample, insertions the union of the
            strings at a candidate slot that pass in some sample (variants_vcf has the rules)."""
from __future__ import annotations

import os
import types

import numpy as np

from . import bamio, engine
from .insertions import decode_events
from .primers import as_primer_set

_LEN_BITS = engine._LEN_BITS
_CHUNK = 1 << 24  # int32 entries of T gathered to the host at once (64 MB)
_FORMAT = ['##FORMAT=<ID=DP,Number=1,Type=Integer,Description="The sample\'s depth: A + C + G + T + N + deletions '
           '(indels: the depth the allele is measured against)">',
           '##FORMAT=<ID=AD,Number=R,Type=Integer,Description="The sample\'s count of REF and of each ALT allele">',
           '##FORMAT=<ID=AF,Number=A,Type=Float,Description="The sample\'s share of DP of each ALT allele, rounded '
           'to 4 decimals">']


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

    def __init__(self, paths, devices=None, filters=(0, 0, 0), primers=None, mask_overlaps=False):
        from .kindel import pileup_run

        import torch

        self.layout = Layout()
        self.primers = as_primer_set(primers)
        self.mask_overlaps = bool(mask_overlaps)
        self.table = None
        self.deletions = []   # per sample: (key = shared slot << 28 | length, count), device, keys ascending
        self.insertions = []  # per sample: (shared slot int64[m] ascending, strings), first-seen order inside a slot
        S = len(paths)
        mbq, mapq, flags = filters
        for i, path in enumerate(paths):
            run = pileup_run(path, devices, 1, mbq, mapq, flags, primers=self.primers,
                             mask_overlaps=self.mask_overlaps)[0]
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
            if src.size:
                self.table[i, :, torch.from_numpy(dst).to(dev)] = counts[0:7].index_select(
                    1, torch.from_numpy(src).to(dev))
            self.deletions.append(self._deletion_keys(dbatch, src_slot, offset))
            ev = run.ins_table.events
            ev_slot = ev[:, 0].astype(np.int64)
            c_of = np.searchsorted(src_slot, ev_slot, side="right") - 1
            ins_slot = ev_slot + offset[c_of] if ev_slot.size else ev_slot
            order = np.argsort(ins_slot, kind="stable")
            strings = decode_events(batch, ev)
            self.insertions.append((ins_slot[order], [strings[k] for k in order.tolist()]))
            del run, counts, dbatch  # the sample's device batch and table go before the next one is piled

    @staticmethod
    def _deletion_keys(dbatch, src_slot, offset):
        import torch

        key, cnt = engine._deletion_groups(dbatch)
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

    def deletion_union(self, abs_threshold, rel_threshold):
        """The deletion keys that pass in some sample (count c > abs_threshold and c / depth(r) > rel_threshold, 0 at
        depth 0), on the device: (slot int64[n], length int64[n], counts int64[S, n], depths int64[S, n]) on the
        host, keys ascending; every sample's count (0 without the event) and six-allele depth at r."""
        import torch

        T = self.table
        dev = T.device
        a, r = engine.variant_abs_floor(abs_threshold), float(rel_threshold)
        zero = torch.zeros((), dtype=torch.float64, device=dev)
        passing = []
        for i, (key, cnt) in enumerate(self.deletions):
            if key.numel() == 0:
                continue
            depth = T[i, 0:6].index_select(1, key >> _LEN_BITS).to(torch.int64).sum(dim=0)
            share = torch.where(depth > 0, cnt.to(torch.float64) / depth.clamp(min=1).to(torch.float64), zero)
            passing.append(key[(cnt > a) & (share > r)])
        if not passing:
            z = np.zeros(0, dtype=np.int64)
            return z, z.copy(), np.zeros((T.shape[0], 0), dtype=np.int64), np.zeros((T.shape[0], 0), dtype=np.int64)
        union = torch.unique(torch.cat(passing), sorted=True)
        slot = union >> _LEN_BITS
        counts, depths = [], []
        for i, (key, cnt) in enumerate(self.deletions):
            if key.numel() == 0:
                counts.append(torch.zeros_like(union))
            else:
                at = torch.searchsorted(key, union).clamp(max=key.numel() - 1)
                counts.append(torch.where(key[at] == union, cnt[at], torch.zeros_like(cnt[at])))
            depths.append(T[i, 0:6].index_select(1, slot).to(torch.int64).sum(dim=0))
        return (slot.cpu().numpy(), (union & ((1 << _LEN_BITS) - 1)).cpu().numpy(),
                torch.stack(counts).cpu().numpy().astype(np.int64), torch.stack(depths).cpu().numpy())

    def strings_at(self, i, slot) -> dict:
        """{string: count} of sample i's insertion events at a shared slot, in first-seen order."""
        slots, strings = self.insertions[i]
        lo, hi = np.searchsorted(slots, [slot, slot + 1])
        out = {}
        for s in strings[lo:hi]:
            out[s] = out.get(s, 0) + 1
        return out


# ---------------------------------------------------------------------------------------------------- text
def _sample_fields(dp, ad) -> list:
    """FORMAT values DP:AD:AF of every sample: dp int64 [S], ad int64 [S, 1 + m] (REF, then each ALT); AF = each
    ALT's share of DP rounded to 4 decimals (0 at DP 0)."""
    dp = np.asarray(dp, dtype=np.int64)
    ad = np.asarray(ad, dtype=np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        af = np.round(np.where(dp[:, None] > 0, ad[:, 1:] / np.maximum(dp, 1)[:, None], 0.0), 4).tolist()
    return ["%d:%s:%s" % (d, ",".join(map(str, a)), ",".join(map(repr, f)))
            for d, a, f in zip(dp.tolist(), ad.tolist(), af)]


def variants_vcf(paths, abs_threshold=1, rel_threshold=0.01, devices=None, min_base_quality=0, min_mapq=0,
                 exclude_flags=0, reference=None, primers=None, mask_overlaps=False, samples=None) -> str:
    """The multi-sample VCF of kindel.variants_vcf given a list of paths (see there for the rules)."""
    from .kindel import _af, _vcf_header, _VCF_ALT, _ACGTN

    paths = [os.fspath(p) for p in paths]
    if not paths:
        raise ValueError("variants_vcf needs at least one alignment file")
    names = sample_names(paths, samples)
    filters = (min_base_quality, min_mapq, exclude_flags)
    cohort = Cohort(paths, devices, filters, primers, mask_overlaps)
    lay = cohort.layout
    ref = None
    if reference is not None:
        from .reference import Reference, load_reference

        ref = reference if isinstance(reference, Reference) else load_reference(reference, lay)
    like_run = types.SimpleNamespace(batch=lay, primers=cohort.primers, mask_overlaps=cohort.mask_overlaps)
    header = _vcf_header(like_run, abs_threshold, rel_threshold, filters,
                         reference_name=None if ref is None else ref.name)
    header = header[:-1] + _FORMAT + ["##kindelSamples=%d" % len(paths),
                                      "\t".join(["#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT"] + names)]
    lines = _records(cohort, None if ref is None else ref.codes, abs_threshold, rel_threshold, _af, _VCF_ALT, _ACGTN)
    return "\n".join(header + lines) + "\n"


def _records(cohort, ref_codes, abs_threshold, rel_threshold, _af, vcf_alt, acgtn) -> list:
    lay = cohort.layout
    T = cohort.table
    S = T.shape[0]
    contig_slot = np.asarray(lay.contig_slot, dtype=np.int64)
    contig_len = np.asarray(lay.contig_len, dtype=np.int64)
    slot_t, mask_t = engine.variant_sites_multi(T, contig_slot, contig_len, ref_codes, abs_threshold, rel_threshold)
    slot, mask = slot_t.cpu().numpy(), mask_t.cpu().numpy()
    contig = np.searchsorted(contig_slot, slot, side="right") - 1
    rows = cohort.rows(slot)                      # [S, 6, n]
    depth = rows.sum(axis=1)                      # [S, n]
    pooled = rows.sum(axis=0)                     # [6, n]
    recs = []  # (contig, POS, kind, deletion length, insertion slot, rank, line)

    if ref_codes is None:
        total = pooled.sum(axis=0)
        top = pooled.argmax(axis=0)
        for i in range(slot.shape[0]):
            m = int(mask[i])
            alts = [(k, letter) for k, letter in vcf_alt if m >> k & 1]
            if not alts:
                continue  # N alone
            c, tp, d = int(contig[i]), int(top[i]), int(total[i])
            ks = [tp] + [k for k, _ in alts]
            info = "DP={};AD={};AF={}".format(d, ",".join(str(int(pooled[k, i])) for k in ks),
                                              ",".join(_af(int(pooled[k, i]), d) for k, _ in alts))
            recs.append((c, int(slot[i] - contig_slot[c]) + 1, 0, 0, 0, 0, "\t".join(
                [lay.contig_names[c], str(int(slot[i] - contig_slot[c]) + 1), ".", "ACGT"[tp] if tp < 4 and d > 0
                 else "N", ",".join(letter for _, letter in alts), ".", "PASS", info, "DP:AD:AF"]
                + _sample_fields(depth[:, i], rows[:, ks, i]))))
        recs.sort(key=lambda x: x[:6])
        return [x[6] for x in recs]

    letters = np.frombuffer(b"ACGTN", dtype=np.uint8)[np.minimum(np.asarray(ref_codes), 4)].tobytes().decode("ascii")
    p_all = slot - contig_slot[contig] if slot.size else slot
    dpa = cohort.rows(np.where(p_all >= 1, slot - 1, slot)).sum(axis=1) if (mask & 64).any() else None  # [S, n]
    for i in range(slot.shape[0]):
        c, s, m = int(contig[i]), int(slot[i]), int(mask[i])
        s0, L, name = int(contig_slot[c]), int(contig_len[c]), lay.contig_names[c]
        p = s - s0
        if m & 15:
            alts = [k for k in range(4) if m >> k & 1]
            g = int(ref_codes[s])
            ad = np.zeros((S, 1 + len(alts)), dtype=np.int64)
            if g < 4:
                ad[:, 0] = rows[:, g, i]
            ad[:, 1:] = rows[:, alts, i].reshape(S, len(alts))
            tot, d = ad.sum(axis=0).tolist(), int(depth[:, i].sum())
            info = "DP={};AD={};AF={}".format(d, ",".join(map(str, tot)), ",".join(_af(x, d) for x in tot[1:]))
            recs.append((c, p + 1, 0, 0, 0, 0, "\t".join(
                [name, str(p + 1), ".", letters[s], ",".join("ACGT"[k] for k in alts), ".", "PASS", info, "DP:AD:AF"]
                + _sample_fields(depth[:, i], ad))))
        if m & 64 and L > 0:
            da = dpa[:, i]
            per = [cohort.strings_at(j, s) for j in range(S)]
            union = {}
            for d_j in per:  # first sample that has the string, then its first-seen rank there
                for text in d_j:
                    union.setdefault(text, len(union))
            for text, rank in union.items():
                if not text:
                    continue
                ao = np.array([d_j.get(text, 0) for d_j in per], dtype=np.int64)
                if not any(cnt > abs_threshold and (cnt / int(dj) if dj > 0 else 0.0) > rel_threshold
                           for cnt, dj in zip(ao.tolist(), da.tolist())):
                    continue
                tot_dp, tot_ao = int(da.sum()), int(ao.sum())
                info = "INDEL;DP={};AO={};AF={}".format(tot_dp, tot_ao, _af(tot_ao, tot_dp))
                alt_text = text.translate(acgtn)
                if p >= 1:
                    pos, rf, alt = p, letters[s - 1], letters[s - 1] + alt_text
                else:
                    pos, rf, alt = 1, letters[s0], alt_text + letters[s0]
                recs.append((c, pos, 2, 0, s, rank, "\t".join(
                    [name, str(pos), ".", rf, alt, ".", "PASS", info, "DP:AD:AF"]
                    + _sample_fields(da, np.stack([np.maximum(da - ao, 0), ao], axis=1)))))

    d_slot, d_len, d_cnt, d_depth = cohort.deletion_union(abs_threshold, rel_threshold)
    d_contig = np.searchsorted(contig_slot, d_slot, side="right") - 1
    for i in range(d_slot.shape[0]):
        c, s, n = int(d_contig[i]), int(d_slot[i]), int(d_len[i])
        s0, L, name = int(contig_slot[c]), int(contig_len[c]), lay.contig_names[c]
        r = s - s0
        if r >= 1:
            pos, rf, alt = r, letters[s - 1:s + n], letters[s - 1]
        elif n < L:
            pos, rf, alt = 1, letters[s0:s0 + n + 1], letters[s0 + n]
        else:
            continue  # the whole contig deleted: no base is left to anchor the record
        ao, dp = d_cnt[:, i], d_depth[:, i]
        tot_ao, tot_dp = int(ao.sum()), int(dp.sum())
        info = "INDEL;DP={};AO={};AF={}".format(tot_dp, tot_ao, _af(tot_ao, tot_dp))
        recs.append((c, pos, 1, n, 0, 0, "\t".join([name, str(pos), ".", rf, alt, ".", "PASS", info, "DP:AD:AF"]
                                                   + _sample_fields(dp, np.stack([np.maximum(dp - ao, 0), ao],
                                                                                 axis=1)))))
    recs.sort(key=lambda x: x[:6])
    return [x[6] for x in recs]
