"""TEST INFRASTRUCTURE ONLY -- the IUPAC vote (an extension) restated in Python over oracle/py_oracle.py's per-position
dicts, as an independent check of oracle/kindel_ioracle.c: the bases are taken in descending order of count, a tie
group at a time, until they hold at least t * depth (N excluded)."""
from __future__ import annotations

from .py_oracle import base_call

_IUPAC = {frozenset(k): v for k, v in (("A", "A"), ("C", "C"), ("G", "G"), ("T", "T"), ("AC", "M"), ("AG", "R"),
                                        ("AT", "W"), ("CG", "S"), ("CT", "Y"), ("GT", "K"), ("ACG", "V"), ("ACT", "H"),
                                        ("AGT", "D"), ("CGT", "B"), ("ACGT", "N"))}


def iupac_call(w, t):
    """The IUPAC letter of one base dict (keys A, C, G, T, N) at threshold t."""
    depth = w["A"] + w["C"] + w["G"] + w["T"]
    if depth == 0:
        return "N"
    taken, held = set(), 0
    for cnt in sorted((w[b] for b in "ACGT"), reverse=True):
        if cnt == 0 or (taken and held >= t * depth):
            break
        group = {b for b in "ACGT" if w[b] == cnt}
        if group <= taken:
            continue
        taken |= group
        held += cnt * len(group)
    return _IUPAC[frozenset(taken)]


def vote(p, min_depth, t):
    """py_oracle.vote (kindel.py:384-430 without patches / trim) with the IUPAC base: (sequence, changes)."""
    out, changes = [], [None] * len(p.weights)
    n = len(p.weights)
    for pos, w in enumerate(p.weights):
        ins = sum(p.insertions[pos].values()) if p.insertions[pos] else 0
        dele = p.deletions[pos]
        depth = w["A"] + w["C"] + w["G"] + w["T"]
        nxt = p.weights[pos + 1] if pos + 1 < n else None
        depth_next = (nxt["A"] + nxt["C"] + nxt["G"] + nxt["T"]) if nxt else 0
        if dele > depth * 0.5:
            changes[pos] = "D"
        elif depth < min_depth:
            out.append("N")
            changes[pos] = "N"
        else:
            if ins > min(depth * 0.5, depth_next * 0.5):
                key, _, tie = base_call(p.insertions[pos])
                out.append("N" if tie else key.lower())
                changes[pos] = "I"
            out.append(iupac_call(w, t))
    return "".join(out), changes
