"""A planted truth set for the quality vote (`consensus --quality-vote`) and a per-slot restatement of K2w (test
infrastructure; nothing here reads the engine).

One contig `v` of LEN bases.  Each block puts 4-base reads (4M, every base the same letter at the same Phred) on
positions [p, p + 4); the positions between blocks have no reads.  The blocks hold the columns of the issue's table:

    p   reads                       count vote   quality vote   Q
    4   6 A at Q5, 4 G at Q35       A            G              60
    12  3 A at Q10, 2 G at Q20      A            G              6
    20  5 A at Q30, 5 C at Q31      N (tie)      C              5
    28  3 A at Q0, 2 C at Q1        A            N              0
    36  5 N at Q30, 2 A at Q30      N            A              60
    44  5 T at Q30, 1 C at Q30      T            T              60
    52  2 A at Q30, 2 C at Q30      N (tie)      N (tie)        0
"""
from __future__ import annotations

import numpy as np

from kindel_b200.quality import WEIGHT

LEN = 64
BLOCKS = [
    (4, [("A", 5, 6), ("G", 35, 4)]),
    (12, [("A", 10, 3), ("G", 20, 2)]),
    (20, [("A", 30, 5), ("C", 31, 5)]),
    (28, [("A", 0, 3), ("C", 1, 2)]),
    (36, [("N", 30, 5), ("A", 30, 2)]),
    (44, [("T", 30, 5), ("C", 30, 1)]),
    (52, [("A", 30, 2), ("C", 30, 2)]),
]


def records():
    """(contigs, records) in the (ref_id, pos0, flag, cigar words, seq, name, mapq, qual) form of qual_cases.write."""
    recs = []
    for p, reads in BLOCKS:
        for base, q, n in reads:
            for j in range(n):
                recs.append((0, p, 0, [(4 << 4) | 0], base * 4, "b%d%s%d_%d" % (p, base, q, j), 60, bytes([q] * 4)))
    return [("v", LEN)], recs


def weight(q):
    return WEIGHT[min(int(q), 93)]


def vote_base(w):
    """(base code 0..4, Q) of four summed weights: the largest, N on a tie or an all-zero column."""
    best = max(w)
    if best == 0 or w.count(best) > 1:
        return 4, 0
    b = w.index(best)
    second = max(x for k, x in enumerate(w) if k != b)
    return b, min(60, (best - second) >> 16)


def expected(min_base_quality=0):
    """(count-vote text, quality-vote text, Q list, 1-based quality-vote sites, 1-based 'N' change sites) of the
    contig at min_depth 1, a base below min_base_quality not counted at all."""
    cols = [dict(A=0, C=0, G=0, T=0, N=0) for _ in range(LEN)]
    wsum = [[0] * 4 for _ in range(LEN)]
    for p, reads in BLOCKS:
        for base, q, n in reads:
            for s in range(p, p + 4):
                if q < min_base_quality:  # masked: not counted at all (K1q takes it back out of the N column)
                    continue
                if base == "N":
                    cols[s]["N"] += n
                    continue
                cols[s][base] += n
                wsum[s]["ACGT".index(base)] += n * weight(q)
    count, qual_text, quals, sites, n_sites = [], [], [], [], []
    for s, c in enumerate(cols):
        depth = c["A"] + c["C"] + c["G"] + c["T"]
        if depth < 1:
            count.append("N")
            qual_text.append("N")
            quals.append(0)
            n_sites.append(s + 1)
            continue
        order = [c[k] for k in "ATGCN"]  # consensus(): first maximum in A, T, G, C, N order; a tie emits N
        top = max(order)
        cv = "N" if order.count(top) > 1 else "ATGCN"[order.index(top)]
        b, q = vote_base(wsum[s])
        count.append(cv)
        qual_text.append("ACGTN"[b])
        quals.append(q)
        if cv != "ACGTN"[b]:
            sites.append(s + 1)
    return "".join(count), "".join(qual_text), quals, sites, n_sites


def restated_vote(counts, wsum, min_depth_ceil=1):
    """K2w slot by slot over a count table (>= 7 columns) and wsum [4][n] (Python ints): (calls, qual) uint8.  The
    D / N / I decisions are consensus_sequence's (kindel.py:402-424) in integers; the base is vote_base's."""
    n = counts.shape[1]
    cols = [[int(x) for x in counts[k]] for k in range(7)]
    ws = [[int(x) for x in wsum[k]] for k in range(4)]
    calls = np.zeros(n, dtype=np.uint8)
    qual = np.zeros(n, dtype=np.uint8)
    for s in range(n):
        a, c, g, t, _, dl, ins = (cols[k][s] for k in range(7))
        depth = a + c + g + t
        dn = sum(cols[k][s + 1] for k in range(4)) if s + 1 < n else 0
        if 2 * dl > depth:
            calls[s] = (1 << 4) | 4
        elif depth < min_depth_ceil:
            calls[s] = (2 << 4) | 4
        else:
            change = 3 if 2 * ins > min(depth, dn) else 0
            b, q = vote_base([ws[k][s] for k in range(4)])
            calls[s], qual[s] = (change << 4) | b, q
    return calls, qual
