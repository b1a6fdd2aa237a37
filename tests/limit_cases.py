"""Alignments that sit exactly on the engine's own limits, and one step past them (test infrastructure).

The engine picks a kernel per read from a few fixed limits (include/kindel_b200.h) and every kernel has fixed
capacities (kindel_b200/csrc/pileup_tile.cu, tile_common.cuh).  The random generators (fuzz_cases.py, synth) reach
none of them except by chance, so each group here is built by hand to land ON a limit and one step PAST it:

  simple_len  simple reads of 8191 / 8192 / 8193 bases (KDL_FAST_MAXLEN), one ending on the contig's last base
  ops         complex reads of 64 and 65 CIGAR ops (KDL_TILE_MAXOPS), 64 and 65 consecutive M ops
  reach       reference span 1023 / 1024 (r_span + 1 <= KDL_TILE_MAXREACH), leading clip 1023 / 1024
  edges       a leading clip that ends on slot 0 / 1 / -1, spans that end on the last slot / one past it, POS 0
  long_ins    `a M b I c M` up to SEQ length 8192 / 8193 (KDL_LEN_MASK field; pieces whose virtual start lies
              up to 16 tiles left of the tile)
  items       tiles of exactly kRmax and kRmax + 1 reads, staged exactly full (kCapW words) and one word over
  pieces      10 reads of 64 M ops (640 pieces) + 32 = kPcap exactly, + 33 = one over, and 11 reads of 64
  carries     three 64-piece reads on one producer thread (its byte carry counters: PER * 64 <= 255)
  flush       248 / 255 / 256 / 257 identical reads on one slot, and 4x that (8 reads per lane and block, a flush
              every F_FLUSH_BLOCKS blocks)
  offsets     simple, clipped and deleting reads starting at every lane (mod 8) and window (mod 64) offset and
              at slots 511 / 512 / 513
  contigs     contigs of 510 / 511 / 512 / 1 / 2 bases (L + 1 = 511 / 512 / 513 slots) and contigs starting mid-tile
  mixed       a bit of every shape above in a background of plain 150M reads

Each read's name ends in the class the engine must give it: `_s` simple, `_t` tile-eligible complex, `_h` KDL_HARD.
QUAL is a deterministic lattice (`#` = Q2 below, `I` = Q40): the first and last base of every M op, some bases of long
insertions and of long leading clips, q mod 8 in {0, 7} of reads of 8192 bases, and every base of every 17th read.
It changes nothing unless a base-quality filter (threshold 3..40) is on.  Everything is seeded; nothing random can
move a case off its limit.  Every group piles without an exception in the reference."""
from __future__ import annotations

import random
import re

# The capacities the corpus targets, mirrored in one place; tests/test_limit_cases.py parses them out of the sources.
KDL_FAST_MAXLEN = 8192
KDL_TILE_MAXOPS = 64
KDL_TILE_MAXREACH = 1024
KDL_LEN_MASK = 0xFFFF
KDL_TILE = 512
F_WIN = 64
F_FLUSH_BLOCKS = 31
RMAX = {False: 512, True: 384}     # TileCfg<kCx>::kRmax (two stages)
CAPW = {False: 9728, True: 7680}   # TileCfg<kCx>::kCapW
PCAP = 672                         # TileCfg<true>::kPcap
W_PT = 128                         # producer threads of K1

MASK_QUAL = 20  # a threshold that masks exactly the lattice's `#` bases
_LOW, _HIGH = "#", "I"
_OPS = "MIDNSHP=X"


def _parse(cigar):
    return [(int(n), op) for n, op in re.findall(r"(\d+)([MIDNSHP=X])", cigar)]


def _qlen(cigar):
    return sum(n for n, op in _parse(cigar) if op in "MIS=X")


class _Group:
    def __init__(self, name):
        self.name = name
        self.rng = random.Random(sum(map(ord, name)) * 7919)
        self.contigs = []   # (name, length)
        self.reads = []     # (contig, pos0, cigar, seq, cls)

    def contig(self, length, name=None):
        name = name or "%s_%d" % (self.name, len(self.contigs))
        self.contigs.append((name, length))
        return name

    def read(self, contig, pos0, cigar, cls, seq=None):
        assert cls in "sth"
        if seq is None:
            seq = "".join(self.rng.choice("ACGT") for _ in range(_qlen(cigar)))
        self.reads.append((contig, pos0, cigar, seq, cls))

    def background(self, contig, length, step=61, lo=0, hi=None, read_len=150):
        hi = length if hi is None else hi
        for p in range(lo, hi - read_len + 1, step):
            self.read(contig, p, "%dM" % read_len, "s")

    def sam(self):
        lines = ["@HD\tVN:1.6\tSO:coordinate"] + ["@SQ\tSN:%s\tLN:%d" % c for c in self.contigs]
        order = {c[0]: k for k, c in enumerate(self.contigs)}
        reads = sorted(self.reads, key=lambda r: (order[r[0]], r[1]))  # stable: coordinate-sorted, ties in order
        for k, (contig, pos0, cigar, seq, cls) in enumerate(reads):
            lines.append("%s_%d_%s\t0\t%s\t%d\t60\t%s\t*\t0\t0\t%s\t%s"
                         % (self.name, k, cls, contig, pos0 + 1, cigar, seq, _quals(k, cigar, len(seq))))
        return "\n".join(lines) + "\n"


def _quals(k, cigar, lseq):
    """The masking lattice of read k (see the module docstring)."""
    low = set()
    if k % 17 == 0:
        low = set(range(lseq))
    q = 0
    for i, (n, op) in enumerate(_parse(cigar)):
        if op in "M=X":
            low.update((q, q + n - 1))
        elif op == "I" and n >= 64:
            low.update(range(q, q + n, 97))
            low.update((q, q + n - 1))
        elif op == "S" and i == 0 and n >= 1000:
            low.update(range(q, q + n, 3))
        if op in "MIS=X":
            q += n
    if lseq == KDL_FAST_MAXLEN:
        low.update(x for x in range(lseq) if x % 8 in (0, 7))
    return "".join(_LOW if x in low else _HIGH for x in range(lseq))


# ---------------------------------------------------------------------------------------------------------------
def _simple_len():
    g = _Group("simple_len")
    L = 8600
    c = g.contig(L)
    g.background(c, L, step=97)
    g.read(c, 3, "%dM" % (KDL_FAST_MAXLEN - 1), "s")
    g.read(c, 100, "%dM" % KDL_FAST_MAXLEN, "s")
    g.read(c, 101, "%d=" % KDL_FAST_MAXLEN, "s")
    g.read(c, 102, "%dX" % KDL_FAST_MAXLEN, "s")
    g.read(c, 200, "%dM" % (KDL_FAST_MAXLEN + 1), "h")       # one past: never simple, too long for the tile kernel
    g.read(c, L - KDL_FAST_MAXLEN, "%dM" % KDL_FAST_MAXLEN, "s")  # ends on the contig's last base
    g.read(c, L - KDL_FAST_MAXLEN - 1, "%dM" % (KDL_FAST_MAXLEN + 1), "h")
    return g


def _ops():
    g = _Group("ops")
    L = 4000
    c = g.contig(L)
    g.background(c, L)
    at = iter(range(40, 3000, 37))
    g.read(c, next(at), "4S" + "3M1I" * 31 + "4S", "t")               # 64 ops
    g.read(c, next(at), "4S" + "3M1I" * 31 + "3M4S", "h")             # 65
    g.read(c, next(at), "3M1I" * 32, "t")                              # 64
    g.read(c, next(at), "3M1I" * 32 + "2M", "h")                       # 65
    g.read(c, next(at), "2M" * 64, "t")                                # 64 consecutive M ops = 64 pieces
    g.read(c, next(at), "2M" * 65, "h")
    g.read(c, next(at), "2=2X" * 32, "t")
    g.read(c, next(at), "2=2X" * 32 + "1=", "h")
    g.read(c, next(at), "3M1D" * 32, "t")
    g.read(c, next(at), "1S" + "1M" * 62 + "1S", "t")
    g.read(c, next(at), "3M1N" * 32, "t")                              # N: counted as an op, moves nothing
    g.read(c, next(at), "3M1H" * 32 + "1M", "h")
    return g


def _reach():
    g = _Group("reach")
    L = 6000
    c = g.contig(L)
    g.background(c, L, step=71)
    R = KDL_TILE_MAXREACH - 1  # the longest reference span a tile-eligible read may have
    for k, (cig, cls) in enumerate([
            ("10M%dD10M" % (R - 20), "t"), ("10M%dD10M" % (R - 19), "h"),
            ("%dM23S" % (R - 23), "t"), ("%dM24S" % (R - 23), "h"),
            ("500M100N%dM" % (R - 500), "t"), ("500M100N%dM" % (R - 499), "h"),
            ("%dM" % R + "1I", "t"), ("%dM" % (R + 1) + "1I", "h"),
            ("%dS50M" % R, "t"), ("%dS50M" % (R + 1), "h"),
            ("%dS%dM" % (R, R), "t"), ("%dS%dM1S" % (R, R), "h"),
            ("%dS1000M23S" % R, "t"), ("%dS1000M1I23S" % R, "t")]):
        g.read(c, 1100 + 211 * k, cig, cls)
    return g


def _edges():
    g = _Group("edges")
    L = 3000
    c = g.contig(L)
    g.background(c, L, step=83, lo=200, hi=L - 200)
    g.read(c, 30, "30S20M", "h")        # the clip ends on slot 0 (start - lead - 1 = -1)
    g.read(c, 31, "30S20M", "t")        # ... on slot 1
    g.read(c, 29, "30S20M", "h")        # one clip base falls off the contig
    g.read(c, 0, "5S10M", "h")
    g.read(c, 1023, "1023S20M", "h")
    g.read(c, 1024, "1023S20M", "t")
    g.read(c, 0, "20M", "s")
    g.read(c, -1, "10M", "h")           # POS 0: weights[-1] wraps to the contig's last position
    g.read(c, 1, "1M1I5M", "t")
    g.read(c, 0, "1M1I5M", "h")         # (start - lead - 1 >= 0 fails at start 0)
    for d in (0, 1):                    # reference span ending on the last slot (L - 1) / on slot L
        g.read(c, L - 25 + d, "20M4D", "t" if d == 0 else "h")
        g.read(c, L - 31 + d, "20M10S", "t" if d == 0 else "h")
        g.read(c, L - 21 + d, "10M1I10M", "t" if d == 0 else "h")
        g.read(c, L - 1024 + d, "%dM3D" % 1020, "t" if d == 0 else "h")
    g.read(c, L - 25, "20M10S", "h")    # a right clip running past the contig end
    g.read(c, L - 20, "20M", "s")       # the last 20 bases
    g.read(c, L - 20, "10M1D9M", "h")
    return g


def _long_ins():
    g = _Group("long_ins")
    L = 9600
    c = g.contig(L)
    g.background(c, L, step=53)
    sizes = (1, 7, 8, 9, 63, 64, 65, 511, 512, 513, 1000, 4095, 7000, 7992)
    for k, b in enumerate(sizes):
        g.read(c, 1030 + 13 * k, "100M%dI100M" % b, "t")
    g.read(c, 1300, "100M7993I100M", "h")            # SEQ of 8193 bases
    g.read(c, 1301, "100M7992I100M", "t")            # 8192: the longest complex read the tile kernel takes
    g.read(c, 1302, "5S100M7000I100M", "t")
    g.read(c, 1303, "1S%dM" % (KDL_FAST_MAXLEN - 1), "h")  # 8192 bases, but a reference span of 8191
    g.read(c, 1304, "20M3000I20M3000I20M2000I20M", "t")
    g.read(c, 1305, "1000S20M3000I20M3000I20M2000I1000S", "h")  # 10080 bases
    return g


def _items():
    """Tiles of lean-size items (19-word reads: 512 x 19 = kCapW) and kCx-size ones (20-word reads: 384 x 20)."""
    g = _Group("items")
    tiles = [[150] * 512,                      # exactly kRmax (lean) reads, exactly kCapW (lean) words
             [150] * 511 + [160],              # 512 reads, one word over
             [150] * 513,                      # kRmax + 1 reads (and over in words); 9747 words: realigned
             [160] * 384,                      # exactly kRmax and kCapW of the kCx instantiation
             [160] * 383 + [165],              # one word over
             [160] * 382 + [165] * 3,          # kRmax + 1 (kCx); realigned
             ]
    L = KDL_TILE * (len(tiles) + 1)
    c = g.contig(L)
    for t, lens in enumerate(tiles):
        n = len(lens)
        span = KDL_TILE - 166                  # no read leaves its tile, none reaches into the next tile's range
        for i, rl in enumerate(lens):
            g.read(c, KDL_TILE * t + 1 + i * span // n, "%dM" % rl, "s")
    # the last tile: 385 short reads, every 7th a tile-eligible complex read (kCx cuts at 384)
    for i in range(385):
        g.read(c, KDL_TILE * len(tiles) + 1 + i, "5M1I4M" if i % 7 == 3 else "10M", "t" if i % 7 == 3 else "s")
    return g


def _pieces():
    """Every read has n M ops of 2 bases; reads stay inside their tile (r_span 2n <= 130, away from its ends)."""
    g = _Group("pieces")
    plan = [[64] * 10 + [32], [64] * 10 + [33], [64] * 11, [64] * 10 + [2]]
    c = g.contig(KDL_TILE * len(plan) + 1)
    for t, counts in enumerate(plan):
        for i, n in enumerate(counts):
            g.read(c, KDL_TILE * t + 2 + 30 * i, "2M" * n, "t")
    return g


def _carries():
    """One item of 300 reads; reads 0, 128 and 256 (the same producer thread) have 64 M ops, one of which is long."""
    g = _Group("carries")
    c = g.contig(2 * KDL_TILE)
    for i in range(300):
        if i % W_PT == 0:
            g.read(c, 2 + i // 16, "1M" * 30 + "%dM" % (320 + i) + "1M" * 33, "t")
        else:
            g.read(c, 2 + i // 16, "40M", "s")
    return g


def _flush():
    """Stacks of identical reads on one slot, one stack per tile."""
    g = _Group("flush")
    stacks = (8 * F_FLUSH_BLOCKS, 255, 256, 257, 4 * 8 * F_FLUSH_BLOCKS, 1020, 1024, 1025, 1100)
    c = g.contig(KDL_TILE * len(stacks) + 1)
    for t, n in enumerate(stacks):
        seq = "".join(g.rng.choice("ACGT") for _ in range(20))
        for _ in range(n):
            g.read(c, KDL_TILE * t + 30 + 7 * t, "20M", "s", seq=seq)
    return g


def _offsets():
    g = _Group("offsets")
    L = 1700
    c = g.contig(L)
    starts = list(range(0, 130)) + list(range(500, 530)) + list(range(1015, 1030))
    for s in starts:
        g.read(c, s, "17M", "s")
        if s >= 4:
            g.read(c, s, "3S9M1I5M", "t")
        g.read(c, s + 1, "6M2D6M", "t")
    return g


def _contigs():
    g = _Group("contigs")
    for L in (510, 511, 512, 1, 2, 300, 700, 513):
        c = g.contig(L)
        if L == 1:                          # (a read of one base is dropped, as the reference drops it)
            g.read(c, 0, "1M1S", "h")
            g.read(c, 0, "1S1M", "h")
            g.read(c, 0, "1M1I", "h")
            continue
        if L == 2:
            g.read(c, 0, "2M", "s")
            g.read(c, 1, "1M1S", "h")
            g.read(c, 1, "1S1M1D", "h")     # span ends on slot L
            g.read(c, 0, "1M1I1M", "h")
            continue
        g.read(c, 0, "%dM" % L, "s")           # the whole contig
        g.read(c, 1, "%dM" % (L - 2), "s")
        g.read(c, 1, "1S%dM1S" % (L - 3), "h")  # the leading clip ends on slot 0
        g.read(c, 2, "1S%dM1S" % (L - 4), "t")
        g.read(c, 5, "3S%dM2I%dM" % (L // 2, L // 2 - 20), "t")
        g.read(c, L - 10, "10M", "s")
        g.read(c, L - 11, "5M1D4M", "t")
    return g


def _mixed():
    g = _Group("mixed")
    L = 12000
    c = g.contig(L)
    g.background(c, L, step=23)
    rng = random.Random(5)
    cases = [("100M%dI100M" % b, "t") for b in (7000, 4000, 900, 64)] + \
            [("2M" * 64, "t"), ("2M" * 65, "h"), ("1023S50M", "t"), ("1024S50M", "h"), ("10M1003D10M", "t"),
             ("10M1004D10M", "h"), ("%dM" % KDL_FAST_MAXLEN, "s"), ("3M1I" * 32, "t"), ("3M1I" * 32 + "1M", "h")]
    for k in range(60):
        cig, cls = cases[k % len(cases)]
        start = 1100 + 180 * k + rng.randrange(8)
        r_span = sum(n for n, op in _parse(cig) if op in "M=XD") + sum(n for n, op in _parse(cig)[1:] if op == "S")
        if start + r_span <= L - 2:  # (every leading clip here is shorter than 1100)
            g.read(c, start, cig, cls)
    return g


GROUPS = {f.__name__[1:]: f for f in (_simple_len, _ops, _reach, _edges, _long_ins, _items, _pieces, _carries, _flush,
                                      _offsets, _contigs, _mixed)}


def group(name):
    return GROUPS[name]()


def sam_text(name):
    return group(name).sam()


def expected_classes(name):
    """The class letter of every read, in the order the decoders keep them (coordinate order per contig)."""
    out = []
    for line in sam_text(name).splitlines():
        if not line.startswith("@"):
            out.append(line.split("\t")[0].rsplit("_", 1)[1])
    return out
