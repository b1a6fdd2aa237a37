"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `--normalise N` (an extension: the reference has no such
option): keep at most N reads of each (amplicon, strand) group, the first ones in the engine's read order.

Per kept record (the read filters of oracle/py_aoracle.kept_records), in the engine's read order -- by contig in the
batch's contig order, file order inside a contig:
  label   py_aoracle.label of the record under the named scheme's rows (-1 unprimed, -2 mispaired, -3 ambiguous, else
          the amplicon's index)
  strand  FLAG & 0x10
  keep    label < 0, or fewer than N earlier records with the same (label, strand)

keep_loop is that rule as a dict of counters; keep_vectorised the same over numpy arrays (a stable sort by key, the
rank being the position minus the start of the key's run) for large batches.  Nothing here imports kindel_b200."""
from __future__ import annotations

import numpy as np

from . import py_aoracle, samdecode


def keep_loop(labels, reverse, cap):
    """uint8 keep flags of reads with these labels and strand bytes, in order."""
    seen, out = {}, []
    for lab, rev in zip(np.asarray(labels).tolist(), np.asarray(reverse).tolist()):
        if lab < 0:
            out.append(1)
            continue
        key = (lab, 1 if rev else 0)
        k = seen.get(key, 0)
        seen[key] = k + 1
        out.append(1 if k < cap else 0)
    return np.array(out, dtype=np.uint8)


def keep_vectorised(labels, reverse, cap):
    """keep_loop over large arrays: a stable argsort by key = 2 * label + strand, rank = position - group start."""
    lab = np.asarray(labels, dtype=np.int64)
    key = np.where(lab >= 0, 2 * lab + (np.asarray(reverse) != 0), -1)
    order = np.argsort(key, kind="stable")
    sk = key[order]
    n = sk.shape[0]
    starts = np.flatnonzero(np.concatenate(([True], sk[1:] != sk[:-1]))) if n else np.zeros(0, dtype=np.int64)
    group_start = np.repeat(starts, np.diff(np.append(starts, n)))
    rank = np.empty(n, dtype=np.int64)
    rank[order] = np.arange(n, dtype=np.int64) - group_start
    return ((key < 0) | (rank < cap)).astype(np.uint8)


def totals(labels, reverse, n_amplicons):
    """int64 [2 * n_amplicons]: the reads of each key."""
    lab = np.asarray(labels, dtype=np.int64)
    key = 2 * lab[lab >= 0] + (np.asarray(reverse)[lab >= 0] != 0)
    return np.bincount(key, minlength=2 * n_amplicons).astype(np.int64)


def records_in_read_order(path, contig_names, min_mapq=0, exclude_flags=0):
    """({name: L}, [(file index, contig name, record)]) of the kept records in the engine's read order."""
    header, records = samdecode.read_alignment_file(path)
    lengths = {}
    for sn, fields in header["@SQ"].items():
        ln = next(f for f in fields if f.startswith("LN:"))
        lengths[sn[3:]] = int(ln[3:])
    groups = {}
    for i, r in enumerate(records):
        if r.mapped and len(r.seq) > 1 and r.mapq >= min_mapq and not (r.flag & exclude_flags):
            groups.setdefault(r.rname, []).append((i, r))
    return lengths, [(i, nm, r) for nm in contig_names for i, r in groups.get(nm, [])]


def keep_by_record(path, contig_names, rows, cap, min_mapq=0, exclude_flags=0):
    """(keep uint8 in the engine's read order, the file indices of the dropped records), record by record."""
    lengths, recs = records_in_read_order(path, contig_names, min_mapq, exclude_flags)
    table = py_aoracle.amplicon_table(rows, list(contig_names))
    seen, keep, dropped = {}, [], set()
    for i, nm, r in recs:
        rows_c = [x for x in rows if x[0] == nm]
        idx = {t[1]: k for k, t in enumerate(table) if t[0] == nm}
        lab = py_aoracle.label(py_aoracle.ends(r, lengths[nm]), lengths[nm], rows_c, idx)
        ok = True
        if lab >= 0:
            key = (lab, 1 if r.flag & 0x10 else 0)
            ok = seen.get(key, 0) < cap
            seen[key] = seen.get(key, 0) + 1
        keep.append(1 if ok else 0)
        if not ok:
            dropped.add(i)
    return np.array(keep, dtype=np.uint8), dropped


def sam_without(sam_text, dropped):
    """The SAM text with the records of file indices `dropped` left out (header lines kept)."""
    out, k = [], 0
    for line in sam_text.splitlines(keepends=True):
        if line.startswith("@") or len(line.rstrip("\n").split("\t")) < 11:
            out.append(line)
            continue
        if k not in dropped:
            out.append(line)
        k += 1
    return "".join(out)
