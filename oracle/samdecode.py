"""TEST INFRASTRUCTURE ONLY -- stdlib (gzip + struct) BAM/SAM decoder for the oracle side.

Produces record objects with exactly the attributes the reference's pileup consumes
(`.pos`, `.mapped`, `.seq`, `.cigars`: reference kindel/kindel.py:42-48; `.rname`: :145), plus `.flag`, `.mapq` and
`.qual` for the oracles of the record and base filters, and the
`header["@SQ"]` shape read at kindel/kindel.py:138-141. It is deliberately independent of the
product decoder `kindel_b200/bamio.py` (record-at-a-time struct.unpack, no numpy) so that the two
cross-check each other. Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
import it. It needs nothing from the reference tree.
"""
from __future__ import annotations

import gzip
import struct
from collections import OrderedDict, defaultdict

_CIGAR_OPS = "MIDNSHP=X"
_NIBBLES = "=ACMGRSVTWYHKDBN"


class Record:
    """simplesam.Sam look-alike: only what reference kindel/kindel.py:42-48,145 touches."""

    __slots__ = ("qname", "flag", "rname", "pos", "seq", "cigars", "mapq", "qual")

    def __init__(self, qname, flag, rname, pos, seq, cigars, mapq=255, qual=None):
        self.qname = qname
        self.flag = flag
        self.rname = rname
        self.pos = pos  # 1-based, SAM convention
        self.seq = seq
        self.cigars = cigars
        self.mapq = mapq
        self.qual = qual  # Phred values, one per base (a list of ints), or None for QUAL `*`

    @property
    def mapped(self):
        return not (self.flag & 0x4)


def _parse_cigar_text(text):
    if text == "*":
        return ((0, None),)
    out, num = [], 0
    for ch in text:
        if ch.isdigit():
            num = num * 10 + ord(ch) - 48
        else:
            out.append((num, ch))
            num = 0
    return tuple(out)


def _header_sq(text):
    """header["@SQ"] -> {"SN:<name>": ["LN:<len>", ...]} (shape consumed at kindel/kindel.py:138-141)."""
    hdr = defaultdict(OrderedDict)
    for line in text.splitlines():
        if line.startswith("@SQ"):
            fields = line.split("\t")[1:]
            sn = next(f for f in fields if f.startswith("SN:"))
            hdr["@SQ"][sn] = [f for f in fields if not f.startswith("SN:")]
    return hdr


def read_sam(path):
    header_lines, records = [], []
    with open(path, "rt") as fh:
        for line in fh:
            if line.startswith("@"):
                header_lines.append(line.rstrip("\n"))
                continue
            f = line.rstrip("\n").split("\t")
            if len(f) < 11:
                continue
            qual = None if f[10] == "*" else [ord(c) - 33 for c in f[10]]
            records.append(Record(f[0], int(f[1]), f[2], int(f[3]), f[9], _parse_cigar_text(f[5]), int(f[4]), qual))
    return _header_sq("\n".join(header_lines)), records


def read_bam(path):
    with gzip.open(path, "rb") as fh:  # BGZF is a series of gzip members
        data = fh.read()
    if data[:4] != b"BAM\x01":
        raise ValueError("not a BAM file: %s" % path)
    (l_text,) = struct.unpack_from("<i", data, 4)
    text = data[8 : 8 + l_text].split(b"\x00", 1)[0].decode()
    off = 8 + l_text
    (n_ref,) = struct.unpack_from("<i", data, off)
    off += 4
    names = []
    sq_lines = []
    for _ in range(n_ref):
        (l_name,) = struct.unpack_from("<i", data, off)
        off += 4
        name = data[off : off + l_name - 1].decode()
        off += l_name
        (l_ref,) = struct.unpack_from("<i", data, off)
        off += 4
        names.append(name)
        sq_lines.append("@SQ\tSN:%s\tLN:%d" % (name, l_ref))
    header = _header_sq(text) if "@SQ" in text else _header_sq("\n".join(sq_lines))
    records = []
    n = len(data)
    while off + 4 <= n:
        (block_size,) = struct.unpack_from("<i", data, off)
        off += 4
        end = off + block_size
        ref_id, pos, l_read_name, mapq, _bin, n_cigar, flag, l_seq, _nref, _npos, _tlen = struct.unpack_from(
            "<iiBBHHHiiii", data, off
        )
        p = off + 32
        qname = data[p : p + l_read_name - 1].decode()
        p += l_read_name
        cig = struct.unpack_from("<%dI" % n_cigar, data, p)
        p += 4 * n_cigar
        cigars = tuple((c >> 4, _CIGAR_OPS[c & 0xF]) for c in cig) if n_cigar else ((0, None),)
        packed = data[p : p + (l_seq + 1) // 2]
        if l_seq:
            chars = []
            for b in packed:
                chars.append(_NIBBLES[b >> 4])
                chars.append(_NIBBLES[b & 0xF])
            seq = "".join(chars[:l_seq])
        else:
            seq = "*"
        p += (l_seq + 1) // 2
        qual = list(data[p : p + l_seq]) if l_seq and data[p] != 0xFF else None
        rname = names[ref_id] if ref_id >= 0 else "*"
        records.append(Record(qname, flag, rname, pos + 1, seq, cigars, mapq, qual))
        off = end
    return header, records


def read_alignment_file(path):
    path = str(path)
    with open(path, "rb") as fh:
        magic = fh.read(2)
    if magic == b"\x1f\x8b":
        return read_bam(path)
    return read_sam(path)


