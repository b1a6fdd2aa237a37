"""An independent restatement of the variant sites of `variants --only-variants` and of the sites-only VCF (both
extensions: the reference has neither), as a per-position loop over plain Python ints and floats.

The rule: at each position of each contig (slots [contig_slot, contig_slot + L)), t = the counts of A, C, G, T, N and
deletions, depth = their sum, top = the first of them holding the maximum; allele k is a variant when t[k] >
abs_threshold, t[k] / depth > rel_threshold (0.0 at depth 0) and k != top.  Python's int / int true division is
correctly rounded, so the share is the float64 numpy computes; int-float comparisons are exact.  A site is a position
with a variant allele.

This file is test infrastructure; nothing in it is part of the product."""
from __future__ import annotations

import numpy as np

LETTERS = "ACGTN-"


def site_alleles(t, abs_threshold, rel_threshold):
    """(variant mask, depth, top) of one position's six counts."""
    depth = 0
    for v in t:
        depth += v
    top = 0
    for k in range(1, 6):
        if t[k] > t[top]:
            top = k
    mask = 0
    for k in range(6):
        share = t[k] / depth if depth > 0 else 0.0
        if k != top and t[k] > abs_threshold and share > rel_threshold:
            mask |= 1 << k
    return mask, depth, top


def sites(table, contig_slot, contig_len, abs_threshold, rel_threshold):
    """(slot int64[n], counts int32[6, n], mask uint8[n]) of every site, in ascending slot order."""
    cols = [np.asarray(table[k]).tolist() for k in range(6)]
    out_slot, out_counts, out_mask = [], [], []
    for s0, L in zip(np.asarray(contig_slot).tolist(), np.asarray(contig_len).tolist()):
        for s in range(s0, s0 + L):
            t = [cols[0][s], cols[1][s], cols[2][s], cols[3][s], cols[4][s], cols[5][s]]
            if not (t[0] or t[1] or t[2] or t[3] or t[4] or t[5]) and abs_threshold >= 0:
                continue  # nothing passes a non-negative count threshold at an empty position
            mask = site_alleles(t, abs_threshold, rel_threshold)[0]
            if mask:
                out_slot.append(s)
                out_counts.append(t)
                out_mask.append(mask)
    counts = np.array(out_counts, dtype=np.int32).reshape(-1, 6).T.copy()
    return np.array(out_slot, dtype=np.int64), counts, np.array(out_mask, dtype=np.uint8)


def vcf_records(names, contig_slot, slots, counts, masks, abs_threshold, rel_threshold):
    """The VCF data lines of the given sites: ALT = the variant alleles among A, C, G, T and the deletion (`*`), in
    that order; REF = the top allele's letter when it is A, C, G or T and the depth is not 0, else N; a site whose only
    variant is N has no line.  AF is the share rounded to 4 decimals as numpy rounds it."""
    starts = np.asarray(contig_slot).tolist()
    lines = []
    for s, t, m in zip(np.asarray(slots).tolist(), np.asarray(counts).T.tolist(), np.asarray(masks).tolist()):
        c = max(i for i, s0 in enumerate(starts) if s0 <= s)
        _, depth, top = site_alleles(t, abs_threshold, rel_threshold)
        alt = [k for k in (0, 1, 2, 3, 5) if m >> k & 1]
        if not alt:
            continue
        ref = LETTERS[top] if top < 4 and depth > 0 else "N"
        ad = [t[top]] + [t[k] for k in alt]
        af = [repr(float(np.round(np.float64(t[k] / depth if depth > 0 else 0.0), 4))) for k in alt]
        lines.append("%s\t%d\t.\t%s\t%s\t.\tPASS\tDP=%d;AD=%s;AF=%s" % (
            names[c], s - starts[c] + 1, ref, ",".join("*" if k == 5 else LETTERS[k] for k in alt), depth,
            ",".join(map(str, ad)), ",".join(af)))
    return lines
