"""A seeded corpus that turns every consensus extension on at once, and the composed oracle it is checked against
(test infrastructure).

The corpus (`combo_case`) is a list of BAM-style records over three contigs, with real QUAL strings:
- "mix": two-haplotype mixed sites whose minor-allele share sits near the IUPAC thresholds 0.6 and 0.99, with the
  low-quality bases on the minor allele at some sites and on the major allele at others (masking flips the call: at
  0.6 both ways, at 0.99 from a code to a base);
  columns where every base is masked and columns that masking thins below a min_depth of 3; an insertion column whose
  inserted bases are partly masked; an insertion at the contig's last position; tile-eligible complex and hard reads.
- "gone": only reads that `exclude_flags=0x400` or `min_mapq=10` drop.  It comes second in the file but first in the
  header, so first-seen contig order matters, and with both filters on it has no reads at all.
- "edge": a replaced segment whose breakpoints clip the reads crossing them (`--realign` patches), uncovered runs at
  both ends (N for `trim_ends`).
Records without qualities (QUAL `*`), a spread of MAPQ values and the flags 0x100, 0x200 and 0x400 are mixed in.

The composed oracle (`Piled`) chains the existing restatements and never looks at the product's decoder output
beyond the read order of an UNMASKED, UNFILTERED batch:
  1. records that min_mapq / exclude_flags drop are rewritten as unmapped (flag | 4);
  2. `qoracle.pileup` over the unmasked batch and the records' QUAL does the masking itself;
  3. `coracle.vote` or `ioracle.vote_iupac`;
  4. the inserted strings are rendered here from SEQ and QUAL (a base with Q < threshold reads as N);
  5. `fqoracle.fastq` walks text and qualities, with the --realign patches of the host's CDR functions.
"""
from __future__ import annotations

import itertools
from collections import OrderedDict

import numpy as np

import helpers as H
from kindel_b200 import bamio
from oracle import coracle, fqoracle, ioracle, qoracle

CONTIGS = [("gone", 160), ("mix", 640), ("edge", 300)]
LOW_Q = (2, 10, 19)               # masked at 20 and 41
HIGH_Q = (20, 21, 30, 37, 40, 41)  # kept at 20; 20..40 masked at 41
MIX_SITES = ((40, 0.38, "minor"), (70, 0.42, "major"), (110, 0.35, None), (160, 0.03, "minor"),
             (190, 0.008, "major"), (230, 0.4, "minor"), (270, 0.3, "major"), (330, 0.42, None), (380, 0.011, "minor"),
             (450, 0.38, "major"), (500, 0.41, "minor"), (560, 0.02, "major"))
FULL_MASK = (95, 96, 97, 410)     # every base below Q20
THIN = (140, 141, 520)            # two bases at Q40, the rest below Q20
INS_SITE = 300


def _cigar(text):
    return bamio.parse_cigar_text(text)


def _qual(rng, n, low_frac=0.04):
    q = rng.choice(HIGH_Q, size=n)
    low = rng.random(n) < low_frac
    q[low] = rng.choice(LOW_Q, size=int(low.sum()))
    return q.astype(np.uint8)


def _fields(rng):
    """(flag, mapq) of an ordinary record: mostly kept, sometimes dropped by one of the two record filters."""
    flag = int(rng.choice([0, 0, 0, 16, 16, 0x100, 0x200, 0x400, 0x10 | 0x400]))
    mapq = int(rng.choice([60, 60, 60, 60, 30, 255, 10, 9, 5, 0]))
    return flag, mapq


def _mix_records(rng, L, ref, out):
    alt = {p: "ACGT"[("ACGT".index(ref[p]) + 1 + p % 3) % 4] for p, _, _ in MIX_SITES}
    starts = np.sort(rng.integers(0, L - 60, size=520))
    thin_seen = {p: 0 for p in THIN}
    for k, start in enumerate(starts.tolist()):
        rl = int(rng.integers(60, 110))
        end = min(L - 1, start + rl)  # position L-1 is only reached by the insertion reads below
        body = list(ref[start:end])
        q = _qual(rng, len(body))
        for p, f, low_on in MIX_SITES:
            if start <= p < end:
                minor = rng.random() < f
                if minor:
                    body[p - start] = alt[p]
                if (low_on == "minor" and minor and rng.random() < 0.7) or (
                        low_on == "major" and not minor and rng.random() < 0.3):
                    q[p - start] = rng.choice(LOW_Q)
                elif low_on is not None:
                    q[p - start] = rng.choice(HIGH_Q)
        for p in FULL_MASK:
            if start <= p < end:
                q[p - start] = rng.choice(LOW_Q)
        kept = False  # carries one of the two good bases of a thinned column: no filter may drop it
        for p in THIN:
            if start <= p < end:
                kept |= thin_seen[p] < 2
                q[p - start] = 40 if thin_seen[p] < 2 else rng.choice(LOW_Q)
                thin_seen[p] += 1
        if rng.random() < 0.01:
            body[int(rng.integers(0, len(body)))] = "N"
        seq = "".join(body)
        style = rng.random()
        if kept:
            cig = "%dM" % len(seq)
        elif start + 2 < INS_SITE < end - 2 and rng.random() < 0.85:  # the insertion column: "GT", partly masked
            cut = INS_SITE - start
            ins_q = np.where(rng.random(2) < 0.3, 10, 35).astype(np.uint8)
            cig = "%dM2I%dM" % (cut, len(seq) - cut)
            seq, q = seq[:cut] + "GT" + seq[cut:], np.concatenate([q[:cut], ins_q, q[cut:]])
        elif style < 0.08 and start > 20:  # leading / trailing soft clips: tile-eligible complex reads
            cl = int(rng.integers(3, 12))
            junk = "".join(rng.choice(list("ACGT"), size=cl))
            jq = _qual(rng, cl, 0.3)
            if rng.random() < 0.5:
                cig, seq, q = "%dS%dM" % (cl, len(seq)), junk + seq, np.concatenate([jq, q])
            else:
                cig, seq, q = "%dM%dS" % (len(seq), cl), seq + junk, np.concatenate([q, jq])
        elif style < 0.12 and len(seq) > 30:  # a small deletion
            cut, dl = int(rng.integers(10, len(seq) - 15)), int(rng.integers(1, 3))
            cig, seq, q = "%dM%dD%dM" % (cut, dl, len(seq) - cut - dl), seq[:cut] + seq[cut + dl:], \
                np.concatenate([q[:cut], q[cut + dl:]])
        elif style < 0.14 and len(seq) > 80:  # 70 CIGAR ops: a hard read (K1g)
            cig = "1M" * 68 + "%dM" % (len(seq) - 69) + "1M"
        else:
            cig = "%dM" % len(seq)
        flag, mapq = (0, 60) if kept else _fields(rng)
        # QUAL `*` is never masked: not on reads that cross the fully masked or thinned columns
        no_qual = rng.random() < 0.1 and not any(start <= p < end for p in FULL_MASK + THIN)
        out.append((1, start, flag, _cigar(cig), seq, "m%d" % k, mapq, None if no_qual else q))
    # an insertion at the last position (its d_next is the empty slot behind the contig): "CA", partly masked
    for k in range(5):
        n = int(rng.integers(30, 50))
        start = L - 1 - n
        seq = ref[start:L - 1] + "CA" + ref[L - 1]
        q = _qual(rng, len(seq))
        q[n:n + 2] = [[35, 35], [10, 35], [35, 10], [35, 35], [10, 10]][k]
        out.append((1, start, 0, _cigar("%dM2I1M" % n), seq, "t%d" % k, 60, q))


def _edge_records(rng, L, ref, out):
    b1, b2 = 130, 160
    z = "".join(rng.choice(list("ACGT"), size=18))
    for k in range(110):
        rl = int(rng.integers(25, 60))
        start = int(rng.integers(12, L - 12 - rl))  # positions 0..11 and L-12..L-1 stay uncovered
        end = start + rl
        if start < b1 < end and rng.random() < 0.8:
            tail = (z + ref[b2:])[: int(rng.integers(4, 25))]
            cig, seq = "%dM%dS" % (b1 - start, len(tail)), ref[start:b1] + tail
        elif start < b2 < end and rng.random() < 0.8:
            head = (ref[:b1] + z)[-int(rng.integers(4, 25)):]
            cig, seq, start = "%dS%dM" % (len(head), end - b2), head + ref[b2:end], b2
        else:
            cig, seq = "%dM" % rl, ref[start:end]
        q = _qual(rng, len(seq), 0.1)
        flag, mapq = _fields(rng)
        out.append((2, start, flag, _cigar(cig), seq, "e%d" % k, mapq, None if rng.random() < 0.15 else q))


def _gone_records(rng, L, ref, out):
    for k in range(24):
        start = int(rng.integers(0, L - 50))
        seq = ref[start:start + 50]
        flag, mapq = (0x400, 60) if k % 2 else (0, int(rng.choice([0, 5, 9])))
        out.append((0, start, flag, _cigar("50M"), seq, "g%d" % k, mapq, _qual(rng, 50)))


def combo_case(seed):
    """(contigs, records) of the corpus; a record is (ref_id, pos0, flag, cigar words, SEQ, QNAME, MAPQ, QUAL bytes or
    None), as bamio.write_bam takes it.  The file order is edge, gone, mix: first-seen order is not the header's."""
    rng = np.random.default_rng(seed)
    refs = ["".join(rng.choice(list("ACGT"), size=L)) for _, L in CONTIGS]
    mix, edge, gone = [], [], []
    _mix_records(rng, CONTIGS[1][1], refs[1], mix)
    _edge_records(rng, CONTIGS[2][1], refs[2], edge)
    _gone_records(rng, CONTIGS[0][1], refs[0], gone)
    edge.sort(key=lambda r: r[1])
    gone.sort(key=lambda r: r[1])
    mix.sort(key=lambda r: r[1])
    recs = [r[:7] + (None if r[7] is None else bytes(r[7].tolist()),) for r in edge + gone + mix]
    return list(CONTIGS), recs


def write_bam(path, contigs, records):
    bamio.write_bam(str(path), contigs, records)
    return str(path)


def sam_text(contigs, records):
    """The same records as SAM text."""
    lines = ["@HD\tVN:1.6\tSO:unsorted"] + ["@SQ\tSN:%s\tLN:%d" % c for c in contigs]
    for ref_id, pos, flag, cig, seq, name, mapq, qual in records:
        cig_text = "".join("%d%s" % (w >> 4, "MIDNSHP=X"[w & 15]) for w in cig)
        qtext = "*" if qual is None else "".join(chr(33 + x) for x in qual)
        lines.append("\t".join([name, str(flag), contigs[ref_id][0], str(pos + 1), str(mapq), cig_text, "*", "0", "0",
                                seq, qtext]))
    return "\n".join(lines) + "\n"


def excluded(record, min_mapq, exclude_flags):
    return record[6] < min_mapq or (record[2] & exclude_flags) != 0


def as_unmapped(records, min_mapq=0, exclude_flags=0):
    """The records with every one that the record filters drop rewritten as unmapped (flag | 4)."""
    return [r[:2] + (r[2] | 4,) + r[3:] if excluded(r, min_mapq, exclude_flags) else r for r in records]


# ------------------------------------------------------------------------------------------- composed oracle
class Piled:
    """The oracle's tables of one corpus at one (min_base_quality, min_mapq, exclude_flags)."""

    def __init__(self, contigs, records, path, min_base_quality=0, min_mapq=0, exclude_flags=0):
        self.q = int(min_base_quality)
        recs = as_unmapped(records, min_mapq, exclude_flags)
        write_bam(path, contigs, recs)
        self.path = str(path)
        self.batch = bamio.read_alignment(self.path)  # unmasked and unfiltered: only its read order is used
        by_name = OrderedDict((n, []) for n in self.batch.contig_names)
        for r in recs:
            if not (r[2] & 4) and r[4] != "*" and len(r[4]) > 1:
                by_name[contigs[r[0]][0]].append(r)
        self.reads = [r for group in by_name.values() for r in group]
        assert len(self.reads) == self.batch.n_reads
        assert [r[1] for r in self.reads] == self.batch.ref_start.tolist()
        assert [len(r[4]) for r in self.reads] == self.batch.seq_len.tolist()
        self.qual = np.frombuffer(b"".join(b"\xff" * len(r[4]) if r[7] is None else r[7] for r in self.reads),
                                  dtype=np.uint8)
        self.counts, self.events = qoracle.pileup(self.batch, self.qual, self.q)
        self.ins = self._insertions()

    def _insertions(self):
        """{slot: {string: count}} in first-seen order, each string from SEQ with its bases below Q read as N."""
        out = {}
        for slot, read, q0, n in self.events.tolist():
            r = self.reads[read]
            seq, qual = r[4].upper(), r[7]
            s = "".join("N" if qual is not None and qual[k] < self.q else seq[k]
                        for k in range(q0, min(q0 + n, len(seq))))
            d = out.setdefault(slot, OrderedDict())
            d[s] = d.get(s, 0) + 1
        return out

    def calls(self, t=None, min_depth=1):
        return coracle.vote(self.counts, min_depth) if t is None else ioracle.vote_iupac(self.counts, min_depth, t)

    def contigs(self):
        for c, name in enumerate(self.batch.contig_names):
            s0, L = int(self.batch.contig_slot[c]), int(self.batch.contig_len[c])
            yield c, name, s0, L, {s - s0: d for s, d in self.ins.items() if s0 <= s <= s0 + L}

    def patches(self, c, min_overlap=9, clip_decay_threshold=0.1, mask_ends=50):
        """The merged CDR patches of contig c by the host's CDR functions over the oracle's table."""
        from kindel_b200 import kindel as K

        run = K.PileupRun.from_host_tables(self.batch, self.counts, coracle.derive(self.counts), self.events)
        aln = run.alignment(c)
        return K.merge_cdrps(K.cdrp_consensuses(aln.weights, aln.deletions, aln.clip_start_weights,
                                                aln.clip_end_weights, aln.clip_start_depth, aln.clip_end_depth,
                                                clip_decay_threshold, mask_ends), min_overlap)

    def consensus(self, t=None, min_depth=1, realign=False, trim_ends=False, uppercase=False, min_overlap=9):
        """[(name, sequence, changes, qualities)] per contig."""
        calls = self.calls(t, min_depth)
        out = []
        for c, name, s0, L, ins_c in self.contigs():
            patches = self.patches(c, min_overlap) if realign else None
            seq, qual = fqoracle.fastq(self.counts, calls, s0, L, ins_c, patches, trim_ends, uppercase)
            out.append((name, seq, _unpatched(H.calls_to_changes(calls[s0:s0 + L]), patches), qual))
        return out


def _unpatched(changes, patches):
    """The change list of the positions the walk visits: a patch (the first Region starting at a position, when some
    Region starting there has a sequence) replaces its position and the end - start - 1 after it, which then keep
    no change; a negative skip ends the walk."""
    starts = {}
    for r in patches or []:
        if r.seq and 0 <= r.start < len(changes):
            starts.setdefault(r.start, next(x for x in patches if x.start == r.start))
    pos = 0
    while pos < len(changes):
        r = starts.get(pos)
        if r is None:
            pos += 1
            continue
        skip = r.end - r.start - 1
        hi = len(changes) if skip < 0 else min(len(changes), pos + 1 + skip)
        changes[pos:hi] = [None] * (hi - pos)
        pos = hi
    return changes


def option_matrix():
    """Rows of (iupac_threshold, min_base_quality, min_depth, realign, trim_ends, uppercase, (min_mapq, exclude_flags))
    such that every pair of values of every two options occurs in some row."""
    levels = [(None, 0.0, 0.6, 0.99, 1.0), (0, 20, 41), (1, 3), (False, True), (False, True), (False, True),
              ((0, 0), (10, 0x400))]
    want = {(i, a, j, b) for i, j in itertools.combinations(range(len(levels)), 2)
            for a in range(len(levels[i])) for b in range(len(levels[j]))}
    rows = []
    for x, y in itertools.product(range(5), range(3)):
        best = max(itertools.product(*[range(len(v)) for v in levels[2:]]),
                   key=lambda rest: len(_pairs((x, y) + rest) & want))
        row = (x, y) + best
        want -= _pairs(row)
        rows.append(row)
    while want:
        best = max(itertools.product(*[range(len(v)) for v in levels]), key=lambda r: len(_pairs(r) & want))
        want -= _pairs(best)
        rows.append(best)
    return [tuple(levels[i][v] for i, v in enumerate(r)) for r in rows]


def _pairs(row):
    return {(i, row[i], j, row[j]) for i, j in itertools.combinations(range(len(row)), 2)}
