"""Truth set of `--dedup` (include/kindel_b200.h K14): planted records, each with the verdict the rule gives it.

One SAM file over two contigs.  Scores come from the qualities: HIGH is ten Q40 bases (400), MID ten Q20 (200), LOW ten
Q2 (0: below 15) and `*` none (0).  `KEEP[k]` is the verdict of record k in file order; TOTALS the record's (pairs
removed, singles removed, singles a pair end shadowed)."""

HIGH, MID, LOW = "I" * 10, "5" * 10, "#" * 10
SEQ = "ACGTACGTAC"

# (QNAME, FLAG, RNAME, POS, CIGAR, RNEXT, PNEXT, QUAL, kept)
ROWS = [
    # a duplicate pair with a distinct best score: a2 stays
    ("a1", 99, "c0", 101, "10M", "=", 201, MID, 0), ("a1", 147, "c0", 201, "10M", "=", 101, MID, 0),
    ("a2", 99, "c0", 101, "10M", "=", 201, HIGH, 1), ("a2", 147, "c0", 201, "10M", "=", 101, HIGH, 1),
    # a score tie: the pair whose first mate comes first stays
    ("b1", 99, "c0", 301, "10M", "=", 401, MID, 1), ("b1", 147, "c0", 401, "10M", "=", 301, MID, 1),
    ("b2", 99, "c0", 301, "10M", "=", 401, MID, 0), ("b2", 147, "c0", 401, "10M", "=", 301, MID, 0),
    # an R1 / R2 swapped copy of the same fragment (c2's R1 is the reverse mate): one key
    ("c1", 99, "c0", 501, "10M", "=", 601, MID, 0), ("c1", 147, "c0", 601, "10M", "=", 501, MID, 0),
    ("c2", 83, "c0", 601, "10M", "=", 501, HIGH, 1), ("c2", 163, "c0", 501, "10M", "=", 601, HIGH, 1),
    # u = 700 on both strands: two ends, no duplicate
    ("d1", 0, "c0", 701, "10M", "*", 0, MID, 1), ("d2", 16, "c0", 692, "10M", "*", 0, MID, 1),
    # the same unclipped end at other POS: a soft clip against a hard clip (u 797), a right soft clip on the reverse
    # strand (u 859)
    ("e1", 0, "c0", 801, "3S7M", "*", 0, MID, 0), ("e2", 0, "c0", 799, "1H10M", "*", 0, HIGH, 1),
    ("e3", 16, "c0", 851, "7M3S", "*", 0, HIGH, 1), ("e4", 16, "c0", 851, "10M", "*", 0, MID, 0),
    # a reverse end across D and N ops: 900 + 15 - 1 = 914 = 905 + 10 - 1
    ("f1", 16, "c0", 901, "5M2D3N5M", "*", 0, MID, 0), ("f2", 16, "c0", 906, "10M", "*", 0, HIGH, 1),
    # a single on a pair's end is removed whatever its score; one base further on it is not
    ("g", 99, "c0", 1101, "10M", "=", 1201, MID, 1), ("g", 147, "c0", 1201, "10M", "=", 1101, MID, 1),
    ("gs1", 0, "c0", 1101, "10M", "*", 0, HIGH, 0), ("gs2", 0, "c0", 1102, "10M", "*", 0, MID, 1),
    # secondary and supplementary records are left alone and shadow nothing
    ("h1", 256, "c0", 1301, "10M", "*", 0, HIGH, 1), ("h2", 2048, "c0", 1301, "10M", "*", 0, HIGH, 1),
    ("h3", 0, "c0", 1301, "10M", "*", 0, MID, 1), ("h4", 0, "c0", 1301, "10M", "*", 0, LOW, 0),
    # mates on two contigs are two singles
    ("i", 99, "c0", 1401, "10M", "c1", 101, MID, 0), ("i2", 0, "c0", 1401, "10M", "*", 0, HIGH, 1),
    ("i", 147, "c1", 101, "10M", "c0", 1401, MID, 1),
    # three records of one name are three singles
    ("trio", 99, "c0", 1501, "10M", "=", 1601, MID, 0), ("trio", 147, "c0", 1601, "10M", "=", 1501, MID, 1),
    ("trio", 99, "c0", 1501, "10M", "=", 1601, HIGH, 1),
    # no qualities scores 0, as do qualities below 15: a tie, the first stays
    ("j1", 0, "c0", 1701, "10M", "*", 0, "*", 1), ("j2", 0, "c0", 1701, "10M", "*", 0, LOW, 0),
    # KDL_HARD reads (a clip reaching before the contig): u = -3 for both
    ("k1", 0, "c0", 1, "3S7M", "*", 0, MID, 0), ("k2", 0, "c0", 2, "4S6M", "*", 0, HIGH, 1),
    # no reference-consuming op: left alone
    ("l1", 0, "c0", 1801, "10S", "*", 0, MID, 1), ("l2", 0, "c0", 1801, "10S", "*", 0, MID, 1),
    # the same pair on two contigs: two keys
    ("n1", 99, "c0", 1901, "10M", "=", 1951, MID, 1), ("n1", 147, "c0", 1951, "10M", "=", 1901, MID, 1),
    ("n2", 99, "c1", 1901, "10M", "=", 1951, MID, 1), ("n2", 147, "c1", 1951, "10M", "=", 1901, MID, 1),
]

KEEP = [r[-1] for r in ROWS]
TOTALS = (3, 9, 1)
CONTIGS = ["c0", "c1"]


def sam_text(rows=ROWS):
    head = "@HD\tVN:1.6\tSO:unsorted\n@SQ\tSN:c0\tLN:2000\n@SQ\tSN:c1\tLN:2000\n"
    return head + "".join("%s\t%d\t%s\t%d\t60\t%s\t%s\t%d\t0\t%s\t%s\n" % (q, f, rn, pos, cig, nx, pn, SEQ, qual)
                          for q, f, rn, pos, cig, nx, pn, qual, _ in rows)


def engine_order(values, rows=ROWS):
    """Per-record values in the engine's read order (by contig in first-seen order, file order inside a contig)."""
    seen = []
    for r in rows:
        if r[2] not in seen:
            seen.append(r[2])
    return [v for c in seen for v, r in zip(values, rows) if r[2] == c]
