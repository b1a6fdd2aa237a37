"""Insertion strings from the event list the pileup kernel emits.

The reference keeps, per reference position, a dict {inserted string -> count} in first-seen order
(reference kindel/kindel.py:38,55-58).  The engine keeps the dense total per slot in count column 6
and one event row (slot, read, q_off, len) per I op, written in the reference's iteration order.
This module rebuilds, lazily and only where someone looks, the dict of a slot and its
`consensus()` (kindel.py:369-381: first maximum in first-seen order, tie = another key with the
same count) -- the vote needs that only at the few slots whose call carries change code 'I'
(kindel.py:419-422).
"""
from __future__ import annotations

import numpy as np

from .bamio import NIBBLES, ReadBatch

_LUT = np.frombuffer(NIBBLES.encode(), dtype=np.uint8)


def decode_events(batch: ReadBatch, rows: np.ndarray) -> list:
    """Upper-case inserted strings of event rows (slot, read, q_off, len), vectorised.
    A string is clipped at the end of SEQ exactly like Python slicing (kindel.py:56)."""
    if rows.shape[0] == 0:
        return []
    read = rows[:, 1].astype(np.int64)
    q0 = rows[:, 2].astype(np.int64)
    lseq = batch.seq_len[read].astype(np.int64)
    # simple reads store the op length in l_seq, but simple reads have no I ops, so lseq is SEQ's
    q1 = np.minimum(q0 + rows[:, 3].astype(np.int64), lseq)
    ln = np.maximum(q1 - q0, 0)
    total = int(ln.sum())
    if total == 0:
        return [""] * rows.shape[0]
    ends = np.cumsum(ln)
    starts = ends - ln
    within = np.arange(total, dtype=np.int64) - np.repeat(starts, ln)
    q = np.repeat(q0, ln) + within
    word = batch.seq4[np.repeat(batch.seq_off[read].astype(np.int64), ln) + (q >> 3)]
    nib = (word >> (28 - 4 * (q & 7)).astype(np.uint32)) & 0xF
    chars = _LUT[nib].tobytes().decode("ascii")
    return [chars[s:e] for s, e in zip(starts.tolist(), ends.tolist())]


class InsertionTable:
    """Events of one pileup, indexed by slot.

    slots / rot (extension: left-aligned insertions, K15i): each row's slot is then slots[i] instead of its column 0,
    and its string is the decoded one rotated right by rot[i]."""

    def __init__(self, batch: ReadBatch, events: np.ndarray, slots: np.ndarray = None, rot: np.ndarray = None):
        self.batch = batch
        events = np.ascontiguousarray(events, dtype=np.int32).reshape(-1, 4)
        slots = events[:, 0].astype(np.int64) if slots is None else np.asarray(slots, dtype=np.int64)
        order = np.argsort(slots, kind="stable")  # keep iteration order inside a slot
        self.events = events[order]
        self.slots = slots[order]
        self.rot = None if rot is None else np.asarray(rot, dtype=np.int64)[order]

    def _span(self, slot: int):
        return (np.searchsorted(self.slots, slot, side="left"), np.searchsorted(self.slots, slot, side="right"))

    def rows_at(self, slot: int) -> np.ndarray:
        lo, hi = self._span(slot)
        return self.events[lo:hi]

    def strings_at(self, slot: int) -> list:
        """The strings of the rows at a slot, in their order (rotated where the table has rotations)."""
        lo, hi = self._span(slot)
        texts = decode_events(self.batch, self.events[lo:hi])
        if self.rot is None:
            return texts
        return [t[len(t) - k:] + t[:len(t) - k] if k else t for t, k in zip(texts, self.rot[lo:hi].tolist())]

    def dict_at(self, slot: int) -> dict:
        """{string: count} in first-seen order (what `insertions[pos]` is in the reference)."""
        out = {}
        for s in self.strings_at(slot):
            out[s] = out.get(s, 0) + 1
        return out

    def consensus_at(self, slot: int):
        """(string, tie) = consensus(insertions[pos])[0], [3]  (kindel.py:369-381)."""
        return dict_consensus(self.dict_at(slot))

    def consensus_count_at(self, slot: int):
        """(string, tie, count): consensus_at and the chosen string's count in the slot's dict (0 when it is empty),
        the support of its quality (kindel_b200/quality.py)."""
        d = self.dict_at(slot)
        text, tie = dict_consensus(d)
        return text, tie, int(d.get(text, 0))


def dict_consensus(d: dict):
    if not d or not sum(d.values()):
        return "N", False
    best, freq = None, None
    for k, v in d.items():
        if freq is None or v > freq:
            best, freq = k, v
    tie = bool(freq) and any(v == freq for k, v in d.items() if k != best)
    return best, tie
