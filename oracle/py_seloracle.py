"""TEST INFRASTRUCTURE ONLY -- which records of an alignment file reach the pileup when `--dedup` and `--normalise N`
(extensions) select the reads together, composed record by record from the single-stage oracles:

  1. the read filters: min_mapq / exclude_flags (oracle/py_moracle.kept, the engine's read order)
  2. `--dedup`: oracle/py_doracle.keep_loop over the kept records, the pairs of py_moracle.pairs (exact QNAME)
  3. labels: oracle/py_aoracle.label of every record the dedup kept, under the named scheme's rows
  4. `--normalise N`: oracle/py_noracle.keep_loop over those labels and strands, in the engine's read order

Contig order: the engine's contigs are the first-seen order of RNAME over every record of the file (`*` dropped), and
a record the filters, the dedup or the cap take out still counts for it, as a filtered record always has.  Neither
stage can empty a contig (each keeps the best of every duplicate set and the first N of every group), so the set of
contigs is the file's too.  A file that holds only the kept records therefore reports the same contigs in the same
order when every removed record stays in it as an unmapped placeholder (FLAG | 0x4, RNAME kept), which no read
counts but the first-seen order does.

Nothing here imports kindel_b200."""
from __future__ import annotations

from . import py_aoracle, py_doracle, py_moracle, py_noracle, samdecode


def contig_order(path):
    """The contigs of a file in first-seen RNAME order over all its records (`*` dropped)."""
    _, records = samdecode.read_alignment_file(path)
    seen = {}
    for r in records:
        if r.rname != "*":
            seen.setdefault(r.rname, None)
    return list(seen)


class Selection:
    """What the chain keeps.  contigs: the engine's contig order; before: the records the filters keep; dedup_removed
    / cap_dropped: file indices of the records the dedup / the cap removes; dedup_totals: (pairs removed, singles
    removed, singles shadowed by a pair end), None without the dedup; after_dedup, kept: the reads left after each
    stage."""

    def __init__(self, contigs, before, dedup_removed, dedup_totals, cap_dropped):
        self.contigs = contigs
        self.before = before
        self.dedup_removed = dedup_removed
        self.dedup_totals = dedup_totals
        self.cap_dropped = cap_dropped
        self.after_dedup = before - len(dedup_removed)
        self.kept = self.after_dedup - len(cap_dropped)

    @property
    def removed(self):
        return self.dedup_removed | self.cap_dropped


def select(path, min_mapq=0, exclude_flags=0, dedup=False, rows=None, normalise=None):
    """The Selection of the chain on a file.  rows: the named scheme's rows (chrom, start, end, amplicon, side), needed
    with normalise (an integer >= 1)."""
    contigs = contig_order(path)
    lengths, recs = py_moracle.kept(path, contigs, min_mapq, exclude_flags)
    index = py_doracle.read_order(path, contigs, min_mapq, exclude_flags)
    assert len(index) == len(recs)
    alive = list(range(len(recs)))
    totals, removed, dropped = None, set(), set()
    if dedup:
        keep, totals = py_doracle.keep_loop([nm for nm, *_ in recs], [py_doracle.end_of(r) for _, r, *_ in recs],
                                            [py_doracle.score_of(r) for _, r, *_ in recs],
                                            py_moracle.pairs(lengths, recs))
        removed = {index[k] for k in alive if not keep[k]}
        alive = [k for k in alive if keep[k]]
    if normalise is not None:
        table = py_aoracle.amplicon_table(rows, contigs)
        rows_of, amp_index = {}, {}
        for row in rows:
            rows_of.setdefault(row[0], []).append(row)
        for k, t in enumerate(table):
            amp_index.setdefault(t[0], {})[t[1]] = k
        labels = []
        for k in alive:
            nm, r = recs[k][0], recs[k][1]
            L = lengths[nm]
            labels.append(py_aoracle.label(py_aoracle.ends(r, L), L, rows_of.get(nm, []), amp_index.get(nm, {})))
        keep = py_noracle.keep_loop(labels, [1 if recs[k][1].flag & 0x10 else 0 for k in alive], normalise)
        dropped = {index[k] for k, ok in zip(alive, keep.tolist()) if not ok}
    return Selection(contigs, len(recs), removed, totals, dropped)
