"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `--dedup` (an extension: the reference has no such option):
duplicate reads and read pairs removed by fragment ends and base-quality score (include/kindel_b200.h K14).

Per kept record (the read filters), in the engine's read order -- by contig in the batch's contig order, file order
inside a contig:
  left alone  FLAG & 0x900, or no M/D/N/=/X op: never removed, nobody's duplicate
  end         (contig, u, strand): strand FLAG & 0x10; u = POS0 - the S/H ops before the first M/D/N/=/X op (forward),
              POS0 + the M/D/N/=/X lengths - 1 + the S/H ops after the last one (reverse)
  score       the sum of the Phred qualities >= 15 over SEQ (0 for QUAL `*`), at most 2^31 - 1
  pair        an R2 and its R1, paired by exact QNAME under K10's rule (oracle/py_moracle.py), neither left alone
  pairs       per (contig, E1 <= E2) the largest R1 + R2 score stays, ties to the smallest min(R1, R2) index
  singles     removed when a pair mate has their end; else per end the largest score stays, ties to the smallest index

keep_loop states it with dicts and Python ints; keep_vectorised does the same with np.lexsort over arrays, for bench
sizes.  Nothing here imports kindel_b200."""
from __future__ import annotations

import numpy as np

from . import py_moracle

SCORE_CAP = (1 << 31) - 1
_REF = "MDN=X"
_CLIP = "SH"


def end_of(rec):
    """(u, strand) of a record, or None when it is left alone."""
    if rec.flag & 0x900:
        return None
    ops = [(int(n), op) for n, op in rec.cigars if op is not None]
    at = [k for k, (_, op) in enumerate(ops) if op in _REF]
    if not at:
        return None
    pos0 = rec.pos - 1
    if rec.flag & 0x10:
        span = sum(n for n, op in ops if op in _REF)
        trail = sum(n for n, op in ops[at[-1] + 1:] if op in _CLIP)
        return pos0 + span - 1 + trail, 1
    return pos0 - sum(n for n, op in ops[:at[0]] if op in _CLIP), 0


def score_of(rec):
    """The duplicate score of a record: -1 for FLAG & 0x900 (the decode's dup_score)."""
    if rec.flag & 0x900:
        return -1
    return min(sum(q for q in rec.qual if q >= 15), SCORE_CAP) if rec.qual is not None else 0


def keep_loop(contig, ends, scores, pairs):
    """(keep uint8 [n], (pairs removed, singles removed, singles shadowed by a pair end)).  contig[r]: any hashable;
    ends[r]: (u, strand) or None (left alone); scores[r]: int; pairs: {R2: R1}."""
    n = len(ends)
    keep = [1] * n
    best_pair, pair_ends, mates = {}, set(), {}
    for r2, r1 in pairs.items():
        if ends[r1] is None or ends[r2] is None:
            continue
        mates[r1] = mates[r2] = True
        e1, e2 = sorted((ends[r1], ends[r2]))
        key = (contig[r2], e1, e2)
        cand = (scores[r1] + scores[r2], -min(r1, r2), r1, r2)
        if key not in best_pair or cand[:2] > best_pair[key][:2]:
            best_pair[key] = cand
        pair_ends.add((contig[r1], ends[r1]))
        pair_ends.add((contig[r2], ends[r2]))
    removed_pairs = 0
    for r2, r1 in pairs.items():
        if r1 in mates and r2 in mates:
            e1, e2 = sorted((ends[r1], ends[r2]))
            _, _, b1, b2 = best_pair[(contig[r2], e1, e2)]
            if (b1, b2) != (r1, r2):
                keep[r1] = keep[r2] = 0
                removed_pairs += 1
    best_single = {}
    singles = [r for r in range(n) if ends[r] is not None and r not in mates]
    for r in singles:
        key = (contig[r], ends[r])
        if key not in pair_ends and (key not in best_single or scores[r] > scores[best_single[key]]):
            best_single[key] = r
    removed = shadowed = 0
    for r in singles:
        key = (contig[r], ends[r])
        if key in pair_ends:
            keep[r] = 0
            removed += 1
            shadowed += 1
        elif best_single[key] != r:
            keep[r] = 0
            removed += 1
    return np.array(keep, dtype=np.uint8), (removed_pairs, removed, shadowed)


def _run_heads(*keys):
    """Start index of each element's run in arrays already sorted by `keys` (equal keys = one run)."""
    n = keys[0].shape[0]
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    change = np.zeros(n, dtype=bool)
    change[0] = True
    for k in keys:
        change[1:] |= k[1:] != k[:-1]
    return np.maximum.accumulate(np.where(change, np.arange(n), 0))


def keep_vectorised(contig, u, strand, alone, score, mate):
    """keep_loop over arrays: contig, u, strand (0 / 1), alone (bool), score (int) per read; mate[r] = R1 of an R2, -1
    elsewhere.  Returns the same (keep, totals)."""
    contig = np.asarray(contig, dtype=np.int64)
    n = contig.shape[0]
    e = 2 * np.asarray(u, dtype=np.int64) + np.asarray(strand, dtype=np.int64)
    alone = np.asarray(alone, dtype=bool)
    score = np.asarray(score, dtype=np.int64)
    mate = np.asarray(mate, dtype=np.int64)
    keep = np.ones(n, dtype=np.uint8)
    r2 = np.flatnonzero(mate >= 0)
    r1 = mate[r2]
    ok = ~alone[r2] & ~alone[r1]
    r1, r2 = r1[ok], r2[ok]
    paired = np.zeros(n, dtype=bool)
    paired[r1] = paired[r2] = True
    c, lo, hi = contig[r2], np.minimum(e[r1], e[r2]), np.maximum(e[r1], e[r2])
    first = np.minimum(r1, r2)
    order = np.lexsort((first, -(score[r1] + score[r2]), hi, lo, c))  # the best pair first in its key
    heads = _run_heads(c[order], lo[order], hi[order])
    lose = order[heads != np.arange(order.shape[0])]
    keep[r1[lose]] = keep[r2[lose]] = 0
    singles = np.flatnonzero(~alone & ~paired)
    # one list: every pair mate's end (domain 0, first in its end) and every single (domain 1, best first)
    mk = np.concatenate((r1, r2, singles))
    dom = np.concatenate((np.zeros(2 * r1.shape[0], dtype=np.int64), np.ones(singles.shape[0], dtype=np.int64)))
    sc = np.where(dom == 1, score[mk], 0)
    order = np.lexsort((mk, -sc, dom, e[mk], contig[mk]))
    heads = _run_heads(contig[mk][order], e[mk][order])
    pos = np.arange(order.shape[0])
    is_single = dom[order] == 1
    shadow = is_single & (dom[order][heads] == 0)
    lose_single = is_single & (shadow | (heads != pos))
    keep[mk[order][lose_single]] = 0
    return keep, (int(lose.shape[0]), int(lose_single.sum()), int(shadow.sum()))


def keep_by_record(path, contig_names, min_mapq=0, exclude_flags=0):
    """(keep uint8 in the engine's read order, totals, the file indices of the removed records), record by record
    over oracle/samdecode.py's records, paired by QNAME (py_moracle.pairs)."""
    lengths, recs = py_moracle.kept(path, contig_names, min_mapq, exclude_flags)
    pairs = py_moracle.pairs(lengths, recs)
    keep, totals = keep_loop([nm for nm, *_ in recs], [end_of(r) for _, r, *_ in recs],
                             [score_of(r) for _, r, *_ in recs], pairs)
    return keep, totals, _file_indices(path, contig_names, min_mapq, exclude_flags, keep)


def read_order(path, contig_names, min_mapq=0, exclude_flags=0):
    """The file indices of the kept records in the engine's read order (same filter and order as py_moracle.kept)."""
    from . import samdecode

    _, records = samdecode.read_alignment_file(path)
    groups = {}
    for i, r in enumerate(records):
        if r.mapped and len(r.seq) > 1 and not (r.flag & exclude_flags) and not (min_mapq and r.mapq < min_mapq):
            groups.setdefault(r.rname, []).append(i)
    return [i for nm in contig_names for i in groups.get(nm, [])]


def _file_indices(path, contig_names, min_mapq, exclude_flags, keep):
    """The file indices of the kept records with keep 0."""
    order = read_order(path, contig_names, min_mapq, exclude_flags)
    return {i for i, k in zip(order, keep.tolist()) if not k}
