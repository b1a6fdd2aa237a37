"""Independent restatement of `--mask-overlaps` (K10p / K10 / K10u, include/kindel_b200.h) for the tests.

Pairs by exact QNAME over the records oracle/samdecode.py decodes (RNEXT / PNEXT read by a small reader of its own:
samdecode keeps neither), with the eligibility of the rule; walks each R1 to its covered cursors (the reference's
cursor, kindel.py:40-81) and each R2 against them.  The tables are the C quality oracle's (oracle/kindel_qoracle.c)
with every masked base -- quality, primer and overlap -- read as N, minus the dropped deletions and insertions, and
the event rows without the dropped ones.  `ComposedMates` composes the same rule with oracle/py_cvoracle.py's
restatement of `variants --vcf` (filters, primers, reference, strand) and writes the whole VCF text.  Nothing here
imports kindel_b200: the batch handed to `pileup` is only the layout the C oracle walks.
"""
from __future__ import annotations

import gzip
import struct

import numpy as np

from . import py_cvoracle, py_poracle, samdecode
from .py_soracle import is_reverse

_M, _I, _D, _S = (0, 7, 8), 1, 2, 4
_LETTER = {c: i for i, c in enumerate("MIDNSHP=X")}


def mate_fields(path):
    """[(qname, RNEXT is the record's own contig, PNEXT - 1)] of every record, in file order."""
    with open(path, "rb") as fh:
        data = fh.read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)
    if data[:4] != b"BAM\x01":
        out = []
        for line in data.decode().splitlines():
            f = line.split("\t")
            if line.startswith("@") or len(f) < 11:
                continue
            try:
                pnext = int(f[7])
            except ValueError:
                pnext = -1
            out.append((f[0], f[6] == "=" or f[6] == f[2], pnext - 1 if 0 <= pnext < (1 << 31) else -1))
        return out
    l_text = struct.unpack_from("<i", data, 4)[0]
    p = 8 + l_text
    n_ref = struct.unpack_from("<i", data, p)[0]
    p += 4
    for _ in range(n_ref):
        p += 8 + struct.unpack_from("<i", data, p)[0]
    out = []
    while p + 4 <= len(data):
        bs = struct.unpack_from("<i", data, p)[0]
        ref_id, _, l_name = struct.unpack_from("<iiB", data, p + 4)
        next_ref, next_pos = struct.unpack_from("<ii", data, p + 24)
        out.append((data[p + 36:p + 36 + l_name - 1].decode(), next_ref == ref_id, next_pos))
        p += 4 + bs
    return out


def role(flag, same_contig):
    if not flag & 1 or flag & (0x8 | 0x100 | 0x800) or bool(flag & 0x40) == bool(flag & 0x80) or not same_contig:
        return 0
    return 1 if flag & 0x40 else 2


def _ops(rec):
    return [(int(n), _LETTER.get(op, 15) if op is not None else 15) for n, op in rec.cigars]


def is_hard(rec, L):
    """The engine's KDL_HARD class of a kept record (include/kindel_b200.h: neither simple nor tile-eligible)."""
    ops, lseq, start = _ops(rec), len(rec.seq), rec.pos - 1
    exotic = any(c.upper() not in "ACGTN" for c in rec.seq)
    if (len(ops) == 1 and ops[0][1] in _M and ops[0][0] == lseq and start >= 0 and start + lseq <= L
            and lseq <= 8192 and not exotic):
        return False
    q_span = sum(n for n, o in ops if o in _M or o in (_I, _S))
    r_span = sum(n for k, (n, o) in enumerate(ops) if o in _M or o == _D or (o == _S and k))
    lead = ops[0][0] if ops and ops[0][1] == _S else 0
    tile = (not exotic and len(ops) <= 64 and lseq <= 8192 and q_span <= lseq and start - lead - 1 >= 0
            and start + r_span <= L - 1 and r_span + 1 <= 1024 and lead + 1 <= 1024)
    return not tile


def kept(path, contig_names, min_mapq=0, exclude_flags=0):
    """({name: L}, [(contig name, record, QNAME, role, PNEXT - 1)]) in the engine's read order."""
    header, records = samdecode.read_alignment_file(path)
    mates = mate_fields(path)
    lengths = {sn[3:]: int(next(f for f in fl if f.startswith("LN:"))[3:]) for sn, fl in header["@SQ"].items()}
    groups = {}
    for r, (qn, same, pn) in zip(records, mates):
        groups.setdefault(r.rname, []).append((r, qn, role(r.flag, same), pn))
    out = []
    for nm in contig_names:
        for r, qn, ro, pn in groups.get(nm, []):
            if not r.mapped or len(r.seq) <= 1 or r.flag & exclude_flags or (min_mapq and r.mapq < min_mapq):
                continue
            out.append((nm, r, qn, ro, pn))
    return lengths, out


def pairs(lengths, recs):
    """{R2 index: R1 index} by exact QNAME."""
    by_name = {}
    for k, (nm, r, qn, ro, pn) in enumerate(recs):
        if ro:
            by_name.setdefault(qn, []).append(k)
    out = {}
    for ks in by_name.values():
        if len(ks) != 2:
            continue
        a, b = ks
        (na, ra, _, oa, pa), (nb, rb, _, ob, pb) = recs[a], recs[b]
        if {oa, ob} != {1, 2} or na != nb or ra.pos - 1 != pb or rb.pos - 1 != pa:
            continue
        if is_hard(ra, lengths[na]) or is_hard(rb, lengths[nb]):
            continue
        r1, r2 = (a, b) if oa == 1 else (b, a)
        out[r2] = r1
    return out


def covered(rec, masked):
    """The cursors R1 covers: M/=/X bases inside SEQ that are not N and not masked, and D ops (a right clip advances
    the cursor by its length: a paired read is never hard, so it never reaches the contig end)."""
    out = set()
    r, q = rec.pos - 1, 0
    for k, (n, op) in enumerate(_ops(rec)):
        if op in _M:
            for j in range(n):
                if q + j < len(rec.seq) and rec.seq[q + j].upper() != "N" and (q + j) not in masked:
                    out.add(r + j)
            r += n
            q += n
        elif op == _I:
            q += n
        elif op == _D:
            out.update(range(r, r + n))
            r += n
        elif op == _S:
            if k:
                r += n
            q += n
    return out


def overlap(rec, cover):
    """R2's (masked query offsets, dropped deletions [(cursor, len)], dropped insertions [(cursor, I-op number)])."""
    bases, dels, ins = [], [], []
    r, q, n_ins = rec.pos - 1, 0, 0
    for k, (n, op) in enumerate(_ops(rec)):
        if op in _M:
            bases += [q + j for j in range(n) if r + j in cover]
            r += n
            q += n
        elif op == _I:
            if r - 1 in cover and r in cover:
                ins.append((r, n_ins))
            n_ins += 1
            q += n
        elif op == _D:
            if r in cover:
                dels.append((r, n))
            r += n
        elif op == _S:
            if k:
                r += n
            q += n
    return bases, dels, ins


class Masked:
    """The rule over one file.  primer / quality masks: per kept record (engine order) its masked query offsets, as
    K9 and the decode make them (py_poracle.masked_by_read, bases below min_base_quality)."""

    def __init__(self, path, contig_names, min_mapq=0, exclude_flags=0, pre_masked=None):
        self.lengths, self.recs = kept(path, contig_names, min_mapq, exclude_flags)
        pre = pre_masked or [()] * len(self.recs)
        self.pre = [set(x) for x in pre]
        self.mate = pairs(self.lengths, self.recs)
        self.bases = [[] for _ in self.recs]
        self.dels, self.ins = {}, {}
        for r2, r1 in self.mate.items():
            b, d, i = overlap(self.recs[r2][1], covered(self.recs[r1][1], self.pre[r1]))
            self.bases[r2], self.dels[r2], self.ins[r2] = b, d, i
        ins_ops = [sum(1 for _, op in _ops(x[1]) if op == _I) for x in self.recs]
        self.evt_off = np.concatenate(([0], np.cumsum(ins_ops))).astype(np.int64)

    def stats(self):
        """(pairs, bases, deletions, insertions) as the REPORT line counts them."""
        return (len(self.mate), sum(len(x) for x in self.bases), sum(len(x) for x in self.dels.values()),
                sum(len(x) for x in self.ins.values()))

    def masked(self):
        """Per record, the sorted union of its own masked bases and its overlap bases: the list K10 writes."""
        return [sorted(p | set(b)) for p, b in zip(self.pre, self.bases)]

    def dropped_rows(self):
        return sorted(int(self.evt_off[r2]) + k for r2, xs in self.ins.items() for _, k in xs)

    def pileup(self, batch, slots):
        """(counts [19, n_slots], events) of `batch` -- the unmasked decode of the same records, whose layout the C
        oracle walks -- with every masked base read as N, the dropped deletions and insertions taken back and the
        dropped event rows left out.  slots: first slot of each contig name."""
        counts, events = py_poracle.pileup(batch, self.masked())
        for r2, xs in self.dels.items():
            s0 = slots[self.recs[r2][0]]
            for r, n in xs:
                counts[5, s0 + r:s0 + r + n] -= 1
        for r2, xs in self.ins.items():
            s0 = slots[self.recs[r2][0]]
            for r, _ in xs:
                counts[6, s0 + r] -= 1
        return counts, np.delete(events, self.dropped_rows(), axis=0)


def fragment_depth(path, contig_names):
    """Per contig, the number of distinct fragments (QNAMEs of kept paired records, else the record itself) with an
    M/=/X base over each position: the DP of a pileup that counts every fragment once, for fixtures without N bases,
    masks or indels."""
    lengths, recs = kept(path, contig_names)
    out = {nm: [set() for _ in range(lengths[nm])] for nm in contig_names}
    for k, (nm, r, qn, ro, pn) in enumerate(recs):
        key = qn if ro else ("#", k)
        cur, q = r.pos - 1, 0
        for n, op in _ops(r):
            if op in _M:
                for j in range(n):
                    if 0 <= cur + j < lengths[nm]:
                        out[nm][cur + j].add(key)
                cur += n
            elif op == _D:
                cur += n
    return {nm: np.array([len(s) for s in v], dtype=np.int64) for nm, v in out.items()}


class MatePile(py_cvoracle.Pile):
    """py_cvoracle's masked walk of one contig, with an R2's dropped ops left out: the D ops at the cursors in drop_d
    and the I ops (numbered in the record's op order) in drop_i add nothing at all."""

    def add(self, rec, masked, drop_d=(), drop_i=()):
        seq, L = rec.seq, self.L
        r, q, k_ins = rec.pos - 1, 0, 0
        for i, (n, op) in enumerate(rec.cigars):
            if op in ("M", "=", "X"):
                for _ in range(n):
                    if q not in masked:
                        self.weights[r][seq[q].upper()] += 1
                    r += 1
                    q += 1
            elif op == "I":
                if k_ins not in drop_i:
                    s = "".join("N" if k in masked else seq[k].upper() for k in range(q, min(q + n, len(seq))))
                    self.ins_ops[r] += 1
                    d = self.insertions[r]
                    d[s] = d.get(s, 0) + 1
                k_ins += 1
                q += n
            elif op == "D":
                if r not in drop_d:
                    if n >= 1 and r >= 0 and r + n <= L:
                        self.del_events[(r, n)] = self.del_events.get((r, n), 0) + 1
                    for k in range(n):
                        self.deletions[r + k] += 1
                r += n
            elif op == "S":
                if i == 0:
                    self.clip_ends[r] += 1
                    for g in range(n):
                        rel = r - n + g
                        if rel >= 0 and g not in masked:
                            self.cew[rel][seq[g].upper()] += 1
                    q += n
                else:
                    self.clip_starts[r - 1] += 1
                    for _ in range(n):
                        if r < L:
                            if q not in masked:
                                self.csw[r][seq[q].upper()] += 1
                            r += 1
                            q += 1


class ComposedMates(py_cvoracle.Composed):
    """py_cvoracle's composed restatement of `variants --vcf` (filters, primers, reference, strand) with
    `--mask-overlaps` on: pairs by exact QNAME over the kept records; each R1's covered cursors from its own quality and
    primer mask; each R2's overlap bases added to its mask and its dropped D / I ops left out of every pile (the total
    and its strand's).  The header gains the `##kindelMateOverlaps` line after `##kindelPrimers`."""

    def __init__(self, path, min_base_quality=0, min_mapq=0, exclude_flags=0, primer_rows=None):
        header, records = samdecode.read_alignment_file(path)
        lengths = {sn[3:]: int(next(f for f in fl if f.startswith("LN:"))[3:]) for sn, fl in header["@SQ"].items()}
        groups = {}
        for rec, mf in zip(records, mate_fields(path)):
            groups.setdefault(rec.rname, []).append((rec, mf))
        groups.pop("*", None)
        self.contigs = [(nm, lengths[nm]) for nm in groups]
        kept_recs = []  # (contig, record, QNAME, role, PNEXT - 1, mask)
        for nm, L in self.contigs:
            iv = py_poracle.contig_intervals(primer_rows, nm) if primer_rows is not None else None
            for rec, (qn, same, pn) in groups[nm]:
                if rec.flag & 0x4 or rec.mapq < min_mapq or rec.flag & exclude_flags or len(rec.seq) <= 1:
                    continue
                kept_recs.append((nm, rec, qn, role(rec.flag, same), pn,
                                  py_cvoracle.record_mask(rec, L, iv, min_base_quality)))
        mate = pairs(lengths, [x[:5] for x in kept_recs])
        drops, n_b, n_d, n_i = {}, 0, 0, 0
        for r2, r1 in mate.items():
            b, d, i = overlap(kept_recs[r2][1], covered(kept_recs[r1][1], kept_recs[r1][5]))
            kept_recs[r2][5].update(b)
            drops[r2] = ({r for r, _ in d}, {k for _, k in i})
            n_b, n_d, n_i = n_b + len(b), n_d + len(d), n_i + len(i)
        self.overlap_stats = (len(mate), n_b, n_d, n_i)
        self.piles = {nm: (MatePile(L), MatePile(L), MatePile(L)) for nm, L in self.contigs}
        for k, (nm, rec, _, _, _, m) in enumerate(kept_recs):
            dd, di = drops.get(k, ((), ()))
            piles = self.piles[nm]
            piles[0].add(rec, m, dd, di)
            piles[2 if is_reverse(rec) else 1].add(rec, m, dd, di)

    def vcf(self, *args, **kwargs):
        lines = super().vcf(*args, **kwargs).split("\n")
        at = next(k for k, x in enumerate(lines) if x.startswith("##kindelVariants="))
        if at + 1 < len(lines) and lines[at + 1].startswith("##kindelPrimers="):
            at += 1
        lines.insert(at + 1, "##kindelMateOverlaps=R2 masked where R1 covers")
        return "\n".join(lines)
