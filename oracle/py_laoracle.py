"""TEST INFRASTRUCTURE ONLY -- an independent restatement of `variants --vcf --reference --left-align` (an extension):
every deletion and insertion event moved to its leftmost place against the reference, with a per-base loop over Python
strings, then grouped, tested and written by the composed oracles' rules (oracle/py_cvoracle.py, oracle/py_moracle.py
for `--mask-overlaps`).

  deletion (r, n)   while r > 0, ref[r-1] is A, C, G or T and ref[r-1] == ref[r+n-1]: r -= 1
  insertion (p, t)  while t, p > 0, ref[p-1] is A, C, G or T and t[-1] == ref[p-1]: p -= 1, t = t[-1] + t[:-1]

(ref = the contig's reference letters, upper case, anything but A, C, G, T read as N; positions are contig
positions.)  The piles' insertion dicts are rebuilt from the events in their walk order -- record order, then op
order -- so that the strings at a slot are in the first-seen order of the events moved there; the deletion groups are
summed per moved key.  The header gains `##kindelLeftAlign=leftmost against the reference` after `##reference`.
Nothing here imports kindel_b200."""
from __future__ import annotations

import contextlib
import copy

from . import py_cvoracle, py_moracle
from .py_rvoracle import ref_letters

_BASES = "ACGT"
HEADER = "##kindelLeftAlign=leftmost against the reference"


def left_deletion(ref, r, n):
    """The leftmost r of a deletion of n bases at r (ref: reference letters)."""
    while r > 0 and ref[r - 1] in _BASES and ref[r - 1] == ref[r + n - 1]:
        r -= 1
    return r


def left_insertion(ref, p, t):
    """(p, t) of an insertion of the string t before position p, moved to its leftmost place."""
    while t and p > 0 and ref[p - 1] in _BASES and t[-1] == ref[p - 1]:
        p -= 1
        t = t[-1] + t[:-1]
    return p, t


class _Logged(dict):
    """An insertion dict of one pile position that logs every string added to it, in order, to the pile's list."""

    def __init__(self, pos, log):
        super().__init__()
        self.pos, self.log = pos, log

    def __setitem__(self, key, value):
        self.log.append((self.pos, key))
        super().__setitem__(key, value)


def _logging(base):
    class Pile(base):
        def __init__(self, L):
            super().__init__(L)
            self.ins_log = []  # (position, string) of every insertion event, in walk order
            self.insertions = [_Logged(pos, self.ins_log) for pos in range(L + 1)]

    return Pile


@contextlib.contextmanager
def _piles_logged(module, name):
    """The composed oracles build their piles by a module-level class name: build logging ones instead."""
    base = getattr(module, name)
    setattr(module, name, _logging(base))
    try:
        yield
    finally:
        setattr(module, name, base)


def left_aligned_pile(pile, ref):
    """A copy of a logging pile whose insertion dicts and deletion groups hold the left-aligned events."""
    out = copy.copy(pile)
    out.insertions = [{} for _ in range(pile.L + 1)]
    for pos, s in pile.ins_log:
        p, t = left_insertion(ref, pos, s)
        out.insertions[p][t] = out.insertions[p].get(t, 0) + 1
    groups = {}
    for (r, n), c in pile.del_events.items():
        key = (left_deletion(ref, r, n), n)
        groups[key] = groups.get(key, 0) + c
    out.del_events = groups
    return out


class _LeftAligned:
    """The VCF of the composed oracle with the piles left-aligned against the reference."""

    def vcf(self, source, abs_threshold, rel_threshold, filters=(0, 0, 0), primers_name=None, reference=None,
            strand=False, max_sor=None, stats=None, left_align=True):
        if not left_align or reference is None:
            return super().vcf(source, abs_threshold, rel_threshold, filters, primers_name, reference, strand, max_sor,
                               stats)
        moved = copy.copy(self)
        moved.piles = {nm: tuple(left_aligned_pile(p, ref_letters(reference[1][nm])) for p in piles)
                       for nm, piles in self.piles.items()}
        text = super(_LeftAligned, moved).vcf(source, abs_threshold, rel_threshold, filters, primers_name, reference,
                                              strand, max_sor, stats)
        lines = text.split("\n")
        at = next(k for k, x in enumerate(lines) if x.startswith("##reference="))
        lines.insert(at + 1, HEADER)
        return "\n".join(lines)


class Composed(_LeftAligned, py_cvoracle.Composed):
    """py_cvoracle.Composed (filters, primers, reference, strand) with left_align."""

    def __init__(self, *args, **kwargs):
        with _piles_logged(py_cvoracle, "Pile"):
            super().__init__(*args, **kwargs)


class ComposedMates(_LeftAligned, py_moracle.ComposedMates):
    """py_moracle.ComposedMates (the same with `--mask-overlaps`) with left_align: the dropped events are left out
    before anything moves."""

    def __init__(self, *args, **kwargs):
        with _piles_logged(py_moracle, "MatePile"):
            super().__init__(*args, **kwargs)
