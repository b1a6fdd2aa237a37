"""Reference FASTA for `variants --vcf --reference` (extension): one base code per slot of a batch's slot space.

    load_reference(path, batch) -> Reference(codes uint8[n_slots], name)

Codes: 0-3 = A, C, G, T; 4 = anything else -- N, the IUPAC letters, the slot behind each contig and the padding.
The file is FASTA, plain or gzip (bgzip included), told apart by its magic bytes.  A record's id is its header text up
to the first whitespace; its sequence is its lines joined, with CR and every other whitespace dropped and case folded.
The FASTA must hold every contig of the batch, at the length of its `@SQ LN`, with letters only; an id may appear
once.  Each violation raises ValueError naming the contig.  Records of contigs the batch does not have are ignored.
Everything is vectorised numpy: a 6 Mb genome loads in well under a second.
"""
from __future__ import annotations

import gzip
import os
import re
from dataclasses import dataclass

import numpy as np

_CODE = np.full(256, 4, dtype=np.uint8)
for _i, _ch in enumerate(b"ACGT"):
    _CODE[_ch] = _i
    _CODE[_ch + 32] = _i  # lower case
_LETTER = np.zeros(256, dtype=bool)
_LETTER[ord("A"):ord("Z") + 1] = True
_LETTER[ord("a"):ord("z") + 1] = True
_SPACE = np.zeros(256, dtype=bool)
_SPACE[list(b" \t\r\n\v\f")] = True

LETTERS = "ACGTN"  # code -> letter


@dataclass(frozen=True)
class Reference:
    codes: np.ndarray  # uint8 [n_slots]
    name: str          # the FASTA's file name, without directories (the VCF's ##reference line)


def read_fasta(path) -> dict:
    """{id: raw sequence bytes (line breaks and other whitespace still in)} in file order; a repeated id raises."""
    with open(path, "rb") as fh:
        data = fh.read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)  # every member of a (b)gzip file
    heads = [m.start() for m in re.finditer(rb"^>", data, re.M)]
    if data.strip() and (not heads or data[:heads[0]].strip()):
        raise ValueError("%s: not a FASTA file (text before the first '>' header)" % path)
    out = {}
    for k, h in enumerate(heads):
        end = data.find(b"\n", h)
        end = len(data) if end < 0 else end
        fields = data[h + 1:end].split()
        if not fields:
            raise ValueError("%s: a FASTA header without an id" % path)
        name = fields[0].decode("utf-8", "replace")
        if name in out:
            raise ValueError("%s: contig %r appears twice in the FASTA" % (path, name))
        out[name] = data[end + 1:heads[k + 1] if k + 1 < len(heads) else len(data)]
    return out


def sequence_codes(raw: bytes, name: str) -> np.ndarray:
    """uint8 codes of one record's raw sequence bytes (whitespace dropped); a byte that is not a letter raises."""
    b = np.frombuffer(raw, dtype=np.uint8)
    b = b[~_SPACE[b]]
    bad = ~_LETTER[b]
    if bad.any():
        raise ValueError("contig %r: byte %r in its FASTA sequence is not a letter" % (name, bytes(b[bad][:1])))
    return _CODE[b]


def load_reference(path, batch) -> Reference:
    """Base codes of `batch`'s contigs from the FASTA at `path`, laid out over the batch's slots (see the module)."""
    return Reference(reference_codes(read_fasta(path), batch, path), os.path.basename(os.fspath(path)))


def reference_codes(records, batch, path) -> np.ndarray:
    """uint8 codes [n_slots] of `batch`'s contigs from read_fasta's `records` of the FASTA at `path` (see the module;
    one parse serves several layouts)."""
    codes = np.full(int(batch.n_slots), 4, dtype=np.uint8)
    for name, s0, L in zip(batch.contig_names, np.asarray(batch.contig_slot).tolist(),
                           np.asarray(batch.contig_len).tolist()):
        raw = records.get(name)
        if raw is None:
            raise ValueError("contig %r of the alignment is missing from the reference FASTA %s" % (name, path))
        c = sequence_codes(raw, name)
        if c.shape[0] != L:
            raise ValueError("contig %r: the reference FASTA holds %d bases, the alignment's @SQ LN is %d"
                             % (name, c.shape[0], L))
        codes[s0:s0 + L] = c
    return codes
