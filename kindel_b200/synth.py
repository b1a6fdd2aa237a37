"""Seeded synthetic alignments of the BASELINE.json shapes, built directly in the flattened layout.

    simple_reads(...)    coordinate-sorted `nM` short reads over one or more random contigs
                         (configs 2, 4, 5: 30 kb x 2000x, 5 Mb x 200x, 64 x 100 kb x 500x)
    complex_reads(...)   indel- and soft-clip-heavy CIGARs plus a tail of edge-case reads (config 3)
    strands(...)         seeded strand bytes, with reads that must lie on one strand (alleles carried by one strand)
    tiled_scheme(...)    a tiled amplicon primer scheme as BED rows (`--primers`)
    amplicon_reads(...)  tiled-amplicon reads: every read starts or ends at an amplicon end, in a primer

Reads copy the contig's bases on M segments with a substitution rate (to A/C/G/T/N uniformly);
inserted and clipped bases are random.  Everything is vectorised numpy so the 5 Mb x 200x case
(6.7 M reads, 10^9 aligned bases) is generated in well under a minute; generation is not part of
any timed region.  `to_records` turns a (small) batch back into BAM-writer records so tests can
push the same data through a real .bam file.
"""
from __future__ import annotations

import numpy as np

from . import bamio

_CODE = np.array([1, 2, 4, 8, 15], dtype=np.uint8)  # A C G T N nibbles


def random_contig(rng, length: int) -> np.ndarray:
    """uint8 nibble codes (1,2,4,8) of a uniform random ACGT contig."""
    return _CODE[rng.integers(0, 4, size=length, dtype=np.uint8)]


def _pack_rows(nib: np.ndarray) -> np.ndarray:
    """[n, w] nibble codes (w % 8 == 0) -> [n, w/8] uint32 words, first base in the top nibble."""
    return bamio.pack_nibbles(nib)


def simple_reads(seed: int, contig_lens, depth: float, read_len: int = 150, sub_rate: float = 0.01,
                 chunk: int = 1 << 18, start_frac=None, read_seed=None) -> bamio.ReadBatch:
    """`read_len`M reads, uniformly placed, sorted by start inside each contig.

    start_frac=(f0, f1) places the (same number of) reads only in that fraction of every contig's
    start range -- a weak-scaling shard: rank r of N uses (r/N, (r+1)/N) and a read_seed of its own
    while `seed` (the contigs' bases) stays common, so the ranks pile N x deeper on disjoint slices."""
    rng = np.random.default_rng(seed)
    rrng = rng if read_seed is None else np.random.default_rng(read_seed)
    contig_lens = [int(x) for x in contig_lens]
    words = (read_len + 7) // 8
    ref_start_all, seq_rows, read_off = [], [], [0]
    for L in contig_lens:
        n = int(round(depth * L / read_len))
        ref = random_contig(rng, L)
        ref_pad = np.concatenate([ref, np.zeros(words * 8, dtype=np.uint8)])
        span = L - read_len + 1
        s_lo, s_hi = (0, span) if start_frac is None else (int(span * start_frac[0]), max(int(span * start_frac[1]),
                                                                                         int(span * start_frac[0]) + 1))
        starts = np.sort(rrng.integers(s_lo, s_hi, size=n, dtype=np.int64))
        for s0 in range(0, n, chunk):
            st = starts[s0:s0 + chunk]
            idx = st[:, None] + np.arange(words * 8, dtype=np.int64)[None, :]
            nib = ref_pad[idx]
            nib[:, read_len:] = 0
            if sub_rate > 0:
                n_sub = rrng.binomial(st.shape[0] * read_len, sub_rate)
                rr = rrng.integers(0, st.shape[0], size=n_sub)
                cc = rrng.integers(0, read_len, size=n_sub)
                nib[rr, cc] = _CODE[rrng.integers(0, 5, size=n_sub)]
            seq_rows.append(_pack_rows(nib))
        ref_start_all.append(starts)
        read_off.append(read_off[-1] + n)
    ref_start = np.concatenate(ref_start_all)
    n = ref_start.shape[0]
    seq4 = np.concatenate(seq_rows).reshape(-1)
    seq_off = np.arange(n, dtype=np.int64) * words
    l_seq = np.full(n, read_len, dtype=np.int64)
    cig_off = np.arange(n + 1, dtype=np.int64)
    cigar = np.full(n, read_len << 4, dtype=np.int64)
    names = ["ctg%d" % i for i in range(len(contig_lens))]
    return bamio.finalize(names, np.array(contig_lens), np.array(read_off), ref_start, seq_off, l_seq, cig_off,
                          cigar, seq4, n_records=n)


def complex_reads(seed: int, contig_len: int, depth: float, read_len: int = 150, sub_rate: float = 0.01,
                  edge_tail: bool = True, unsorted_tail: bool = False, start_frac=None, read_seed=None,
                  ref_seed=None) -> bamio.ReadBatch:
    """Config-3 shape: per read p=0.5 leading soft clip (1-29), p=0.5 trailing soft clip (1-29),
    0-3 indel events (I or D, length 1-4) between M segments; query length is always `read_len`.
    With edge_tail a few hundred reads using N / = / X / H / P ops, H-then-S, clips overhanging
    both contig ends and POS == 0 are added (all legal for the reference, no exceptions); unsorted_tail leaves them
    at the end of the batch (an unsorted file: the order-independent kernels take it)."""
    rng = np.random.default_rng(seed if read_seed is None else read_seed)
    L = int(contig_len)
    n = int(round(depth * L / read_len))
    lead = np.where(rng.random(n) < 0.5, rng.integers(1, 30, size=n), 0)
    trail = np.where(rng.random(n) < 0.5, rng.integers(1, 30, size=n), 0)
    n_ev = rng.integers(0, 4, size=n)
    ev_is_ins = rng.random((n, 3)) < 0.5
    ev_len = rng.integers(1, 5, size=(n, 3))
    ev_on = np.arange(3)[None, :] < n_ev[:, None]
    ins_total = (ev_len * (ev_is_ins & ev_on)).sum(axis=1)
    del_total = (ev_len * (~ev_is_ins & ev_on)).sum(axis=1)
    m_total = read_len - lead - trail - ins_total  # aligned bases
    # split m_total into n_ev + 1 segments, each >= 10
    cuts = np.sort(rng.random((n, 3)), axis=1)
    cuts = np.where(ev_on, cuts, 1.0)
    spare = m_total - 10 * (n_ev + 1)
    bounds = np.concatenate([np.zeros((n, 1)), cuts, np.ones((n, 1))], axis=1)
    seg = np.floor(np.diff(bounds, axis=1) * spare[:, None]).astype(np.int64)
    seg_on = np.arange(4)[None, :] <= n_ev[:, None]
    seg = np.where(seg_on, seg + 10, 0)
    seg[np.arange(n), n_ev] += m_total - seg.sum(axis=1)  # rounding remainder into the last segment
    ref_span = m_total + del_total
    span = max(int(L - ref_span.max() - 1), 1)  # start_frac: a weak-scaling shard's share of the start range
    s_lo, s_hi = (0, span) if start_frac is None else (int(span * start_frac[0]),
                                                       max(int(span * start_frac[1]), int(span * start_frac[0]) + 1))
    start = np.sort(rng.integers(s_lo, s_hi, size=n))

    # ops as an [n, 9] grid: S, M0, E0, M1, E1, M2, E2, M3, S
    op_len = np.zeros((n, 9), dtype=np.int64)
    op_code = np.zeros((n, 9), dtype=np.int64)
    op_len[:, 0], op_code[:, 0] = lead, 4
    op_len[:, 8], op_code[:, 8] = trail, 4
    for k in range(4):
        op_len[:, 1 + 2 * k] = seg[:, k]
    for k in range(3):
        op_len[:, 2 + 2 * k] = np.where(ev_on[:, k], ev_len[:, k], 0)
        op_code[:, 2 + 2 * k] = np.where(ev_is_ins[:, k], 1, 2)
    on = op_len > 0
    n_ops = on.sum(axis=1)
    cigar = ((op_len << 4) | op_code)[on]
    cig_off = np.concatenate([[0], np.cumsum(n_ops)])

    # bases: random everywhere, reference copy (+ substitutions) on M segments
    ref = random_contig(rng if ref_seed is None else np.random.default_rng(ref_seed), L)
    words = (read_len + 7) // 8
    nib = _CODE[rng.integers(0, 4, size=(n, words * 8), dtype=np.uint8)]
    nib[:, read_len:] = 0
    consumes_q = np.isin(op_code, (0, 1, 4))
    consumes_r = np.isin(op_code, (0, 2))
    q_begin = np.cumsum(np.where(consumes_q, op_len, 0), axis=1) - np.where(consumes_q, op_len, 0)
    r_begin = start[:, None] + np.cumsum(np.where(consumes_r, op_len, 0), axis=1) - np.where(consumes_r, op_len, 0)
    for k in range(4):
        col = 1 + 2 * k
        ln = op_len[:, col]
        rows = np.repeat(np.arange(n), ln)
        within = np.arange(ln.sum()) - np.repeat(np.cumsum(ln) - ln, ln)
        nib[rows, np.repeat(q_begin[:, col], ln) + within] = ref[np.repeat(r_begin[:, col], ln) + within]
    n_sub = rng.binomial(n * read_len, sub_rate)
    nib[rng.integers(0, n, size=n_sub), rng.integers(0, read_len, size=n_sub)] = _CODE[rng.integers(0, 5, size=n_sub)]
    seq_rows = [_pack_rows(nib)]
    ref_start = [start]
    l_seq = [np.full(n, read_len, dtype=np.int64)]
    cig_parts = [cigar]
    cig_counts = [n_ops]

    if edge_tail:
        tail = []  # (pos0, [(len, op)], seq length)
        for k in range(64):
            p = int(rng.integers(100, L - 400))
            tail += [
                (p, [(20, 0), (7, 3), (30, 0)], 50),                # N is a no-op
                (p, [(5, 5), (10, 7), (3, 8), (20, 0), (4, 5)], 33),  # H = X M H
                (p, [(3, 5), (6, 4), (25, 0)], 31),                 # H then S: treated as right clip
                (p, [(12, 0), (2, 6), (12, 0), (5, 4)], 29),        # P no-op, trailing S
                (p, [(10, 0), (4, 4), (10, 0)], 24),                # mid-CIGAR S
            ]
        tail += [(-1, [(30, 0)], 30), (0, [(25, 4), (30, 0)], 55), (3, [(25, 4), (30, 0)], 55),
                 (L - 20, [(20, 0), (15, 4)], 35), (L - 10, [(10, 0), (1, 1), (9, 4)], 20),
                 (L - 5, [(5, 0), (2, 1)], 7), (L - 30, [(28, 0), (2, 2)], 28), (-1, [(3, 1), (4, 4)], 7)]
        t_start = np.array([t[0] for t in tail], dtype=np.int64)
        t_len = np.array([t[2] for t in tail], dtype=np.int64)
        t_words = (int(t_len.max()) + 7) // 8
        t_nib = _CODE[rng.integers(0, 5, size=(len(tail), t_words * 8), dtype=np.uint8)]
        t_nib[np.arange(t_words * 8)[None, :] >= t_len[:, None]] = 0
        packed = _pack_rows(t_nib)
        if t_words < words:
            packed = np.concatenate([packed, np.zeros((len(tail), words - t_words), dtype=np.uint32)], axis=1)
        elif t_words > words:
            raise ValueError("edge-tail reads longer than read_len are not laid out here")
        seq_rows.append(packed)
        ref_start.append(t_start)
        l_seq.append(t_len)
        cig_parts.append(np.array([(ln << 4) | op for t in tail for ln, op in t[1]], dtype=np.int64))
        cig_counts.append(np.array([len(t[1]) for t in tail], dtype=np.int64))

    ref_start = np.concatenate(ref_start)
    l_seq = np.concatenate(l_seq)
    n_all = ref_start.shape[0]
    counts = np.concatenate(cig_counts)
    cig_off = np.concatenate([[0], np.cumsum(counts)])
    seq4 = np.concatenate(seq_rows).reshape(-1)
    seq_off = np.arange(n_all, dtype=np.int64) * words
    batch = bamio.finalize(["ctg0"], np.array([L]), np.array([0, n_all]), ref_start, seq_off, l_seq, cig_off,
                           np.concatenate(cig_parts), seq4, n_records=n_all)
    if edge_tail and not unsorted_tail:  # the tail goes where a coordinate-sorted file would have it
        batch = bamio.select_reads(batch, np.argsort(ref_start, kind="stable"))
    return batch


def on_contig(batch: bamio.ReadBatch, names, contig_lens, c: int) -> bamio.ReadBatch:
    """A single-contig batch re-homed as contig `c` of a multi-contig layout (same length required)."""
    assert batch.n_contigs == 1 and int(batch.contig_len[0]) == int(contig_lens[c])
    read_off = np.zeros(len(names) + 1, dtype=np.int64)
    read_off[c + 1:] = batch.n_reads
    words = (batch.seq_len.astype(np.int64) + 7) // 8
    bases = bamio._ragged_gather(batch.seq4, batch.seq_off, words)
    return bamio.finalize(names, np.asarray(contig_lens), read_off, batch.ref_start, np.cumsum(words) - words,
                          batch.seq_len, batch.cig_off, batch.cigar, bases, n_records=batch.n_reads)


def mixed_reads(seed: int, contig_lens, depth: float, complex_frac: float, read_len: int = 150, start_frac=None,
                read_seed=None) -> bamio.ReadBatch:
    """What a real short-read alignment looks like: coordinate-sorted `read_len`M reads with a fraction of clipped /
    indel reads (the config-3 generator without its edge-case tail) mixed in at the same depth profile.
    start_frac / read_seed: as in simple_reads (a weak-scaling shard)."""
    contig_lens = [int(x) for x in contig_lens]
    names = ["ctg%d" % i for i in range(len(contig_lens))]
    parts = [simple_reads(seed, contig_lens, depth * (1.0 - complex_frac), read_len=read_len, start_frac=start_frac,
                          read_seed=read_seed)]
    for c, L in enumerate(contig_lens):
        rs = None if read_seed is None else list(np.atleast_1d(read_seed)) + [7, c]
        cx = complex_reads(seed * 131 + c, L, depth * complex_frac, read_len=read_len, edge_tail=False,
                           start_frac=start_frac, read_seed=rs)
        parts.append(on_contig(cx, names, contig_lens, c))
    return bamio.merge_batches(parts)


def tiled_scheme(seed: int, contig_names, contig_lens, spacing: int = 200, overlap: int = 50):
    """A tiled amplicon primer scheme (ARTIC-like) as BED rows [(chrom, start, end)]: amplicon k of a contig spans
    [k * spacing, k * spacing + spacing + overlap), with a left primer at its start and a right primer at its end, each
    22-30 bp long; both rows of every pair."""
    rng = np.random.default_rng(seed)
    rows = []
    for name, L in zip(contig_names, (int(x) for x in contig_lens)):
        for a in range(0, L - spacing - overlap + 1, spacing):
            b = a + spacing + overlap
            rows.append((name, a, a + int(rng.integers(22, 31))))
            rows.append((name, b - int(rng.integers(22, 31)), b))
    return rows


def amplicon_reads(seed: int, contig_len: int, depth: float, read_len: int = 150, spacing: int = 200,
                   overlap: int = 50, sub_rate: float = 0.01):
    """Tiled-amplicon sequencing of one random contig: (batch, scheme rows).  Every read starts at the start of an
    amplicon of tiled_scheme(seed, ...) or ends at its end (half each), so every read begins or ends in a primer;
    `read_len`M reads, sorted by start."""
    rng = np.random.default_rng(seed)
    rows = tiled_scheme(seed, ["ctg0"], [contig_len], spacing, overlap)
    amp_lo = np.array([a for _, a, _ in rows[0::2]], dtype=np.int64)
    amp_hi = np.array([b for _, _, b in rows[1::2]], dtype=np.int64)
    n = int(round(depth * contig_len / read_len))
    words = (read_len + 7) // 8
    k = rng.integers(0, amp_lo.shape[0], size=n)
    starts = np.sort(np.where(rng.random(n) < 0.5, amp_lo[k], amp_hi[k] - read_len))
    ref = random_contig(rng, contig_len)
    ref_pad = np.concatenate([ref, np.zeros(words * 8, dtype=np.uint8)])
    rows_packed = []
    for s0 in range(0, n, 1 << 18):
        st = starts[s0:s0 + (1 << 18)]
        nib = ref_pad[st[:, None] + np.arange(words * 8, dtype=np.int64)[None, :]]
        nib[:, read_len:] = 0
        n_sub = rng.binomial(st.shape[0] * read_len, sub_rate)
        nib[rng.integers(0, st.shape[0], size=n_sub), rng.integers(0, read_len, size=n_sub)] = \
            _CODE[rng.integers(0, 5, size=n_sub)]
        rows_packed.append(_pack_rows(nib))
    seq4 = np.concatenate(rows_packed).reshape(-1) if rows_packed else np.zeros(0, dtype=np.uint32)
    batch = bamio.finalize(["ctg0"], np.array([contig_len]), np.array([0, n]), starts,
                           np.arange(n, dtype=np.int64) * words, np.full(n, read_len, dtype=np.int64),
                           np.arange(n + 1, dtype=np.int64), np.full(n, read_len << 4, dtype=np.int64), seq4,
                           n_records=n)
    return batch, rows


def to_records(batch: bamio.ReadBatch):
    """(contigs, records) for bamio.write_bam -- small batches only (Python loop)."""
    contigs = list(zip(batch.contig_names, (int(x) for x in batch.contig_len)))
    recs = []
    for c in range(batch.n_contigs):
        for r in range(int(batch.contig_read_off[c]), int(batch.contig_read_off[c + 1])):
            words = batch.cigar[int(batch.cig_off[r]):int(batch.cig_off[r + 1])].tolist()
            lseq = int(batch.seq_len[r])
            base = int(batch.seq_off[r])
            nib = bamio.unpack_nibbles(batch.seq4[base:base + (lseq + 7) // 8])[:lseq]
            flag = 0 if batch.reverse is None else 16 * int(batch.reverse[r])
            recs.append((c, int(batch.ref_start[r]), flag, words, "".join(bamio.NIBBLES[x] for x in nib.tolist())))
    return contigs, recs


def write_simple_bam(path, batch: bamio.ReadBatch, level: int = 1, threads: int = 8):
    """Vectorised BAM writer for an all-simple, uniform-read-length batch (the config 2/4/5 shapes):
    lets tests and tools push 10^5..10^7 synthetic reads through the real decode path quickly."""
    import struct
    from concurrent.futures import ThreadPoolExecutor

    n = batch.n_reads
    lens = np.unique(batch.l_seq)
    if batch.n_complex or lens.shape[0] != 1:
        raise ValueError("write_simple_bam needs simple reads of one length")
    L = int(lens[0])
    words = (L + 7) // 8
    n_seq = (L + 1) // 2
    name = b"r\x00"
    rec_len = 32 + len(name) + 4 + n_seq + L
    rec = np.zeros((n, 4 + rec_len), dtype=np.uint8)

    def put(col, values, dtype):
        v = np.ascontiguousarray(values, dtype=dtype).view(np.uint8).reshape(n, -1)
        rec[:, col:col + v.shape[1]] = v

    ref_id = np.repeat(np.arange(batch.n_contigs, dtype=np.int32), np.diff(batch.contig_read_off))
    put(0, np.full(n, rec_len), "<i4")
    put(4, ref_id, "<i4")
    put(8, batch.ref_start, "<i4")
    rec[:, 12] = len(name)
    rec[:, 13] = 60
    put(14, np.full(n, 4680), "<u2")
    put(16, np.ones(n), "<u2")            # n_cigar_op
    put(18, np.zeros(n) if batch.reverse is None else 16 * batch.reverse.astype(np.int64), "<u2")  # flag
    put(20, np.full(n, L), "<i4")
    put(24, np.full(n, -1), "<i4")
    put(28, np.full(n, -1), "<i4")
    put(32, np.zeros(n), "<i4")
    rec[:, 36:36 + len(name)] = np.frombuffer(name, dtype=np.uint8)
    put(36 + len(name), np.full(n, L << 4), "<u4")
    seq_be = batch.seq4.reshape(n, words).astype(">u4").view(np.uint8).reshape(n, words * 4)[:, :n_seq]
    rec[:, 40 + len(name):40 + len(name) + n_seq] = seq_be
    rec[:, 40 + len(name) + n_seq:] = 0xFF
    header_text = ("@HD\tVN:1.6\tSO:coordinate\n" + "".join(
        "@SQ\tSN:%s\tLN:%d\n" % (nm, ln) for nm, ln in zip(batch.contig_names, batch.contig_len))).encode()
    head = bytearray(b"BAM\x01" + struct.pack("<i", len(header_text)) + header_text + struct.pack("<i", batch.n_contigs))
    for nm, ln in zip(batch.contig_names, batch.contig_len):
        nb = nm.encode() + b"\x00"
        head += struct.pack("<i", len(nb)) + nb + struct.pack("<i", int(ln))
    body = bytes(head) + rec.tobytes()
    chunks = [body[s:s + 65280] for s in range(0, len(body), 65280)]
    with ThreadPoolExecutor(max_workers=threads) as pool:
        blocks = list(pool.map(lambda c: bamio._bgzf_block(c, level), chunks, chunksize=32))
    with open(path, "wb") as fh:
        for blk in blocks:
            fh.write(blk)
        fh.write(bamio._bgzf_block(b"", level))


def strands(seed: int, n: int, p: float = 0.5, forward=None, reverse=None) -> np.ndarray:
    """Seeded strand bytes of n reads (1 = reverse, FLAG 0x10): each read reverse with probability p, except the
    reads listed in `forward` (all forward) and in `reverse` (all reverse) -- how a truth set plants alleles that only
    one strand carries."""
    out = (np.random.default_rng(seed).random(n) < p).astype(np.uint8)
    if forward is not None:
        out[np.asarray(forward, dtype=np.int64)] = 0
    if reverse is not None:
        out[np.asarray(reverse, dtype=np.int64)] = 1
    return out


def with_strands(batch: bamio.ReadBatch, seed: int, p: float = 0.5) -> bamio.ReadBatch:
    """`batch` with seeded strands (strands(seed, n_reads, p)); the read data is shared."""
    import dataclasses

    return dataclasses.replace(batch, reverse=strands(seed, batch.n_reads, p))


def qualities(seed: int, seq_len, low_frac: float = 0.05, chunk: int = 1 << 26) -> np.ndarray:
    """Seeded Phred qualities, one byte per base, concatenated in read order: about `low_frac` of the bases are below
    Q20 (Q2..Q19), weighted toward the 3' end (the chance grows linearly along the read, averaging low_frac); the rest
    are Q20..Q41.  Built in chunks of reads, so 10^9 bases need 1 GB and no more."""
    lens = np.asarray(seq_len, dtype=np.int64)
    out = np.empty(int(lens.sum()), dtype=np.uint8)
    rng = np.random.default_rng(seed)
    ends = np.cumsum(lens)
    r0, b0 = 0, 0
    while r0 < lens.shape[0]:
        r1 = int(np.searchsorted(ends, b0 + chunk, side="right"))
        r1 = max(r1, r0 + 1)
        ln = lens[r0:r1]
        n = int(ln.sum())
        q = np.arange(n, dtype=np.int64) - np.repeat(np.cumsum(ln) - ln, ln)   # offset inside the read
        frac = (2.0 * low_frac) * (q + 0.5) / np.repeat(np.maximum(ln, 1), ln)   # linear ramp, mean low_frac
        low = rng.random(n, dtype=np.float32) < frac
        out[b0:b0 + n] = np.where(low, rng.integers(2, 20, n, dtype=np.uint8), rng.integers(20, 42, n, dtype=np.uint8))
        r0, b0 = r1, b0 + n
    return out


def mapq_flags(seed: int, n: int):
    """Seeded MAPQ (mostly 60, some 0..30 and 255) and FLAG mixes (secondary, supplementary, duplicate, QC-fail,
    reverse) for `n` records."""
    rng = np.random.default_rng(seed)
    mapq = rng.choice(np.array([60, 60, 60, 60, 0, 1, 5, 20, 30, 255]), n).astype(np.int64)
    flag = rng.choice(np.array([0, 0, 0, 16, 16, 256, 2048, 1024, 512, 16 | 1024]), n).astype(np.int64)
    return mapq, flag


def with_qualities(batch: bamio.ReadBatch, seed: int, min_base_quality: int = 20, low_frac: float = 0.05):
    """(masked batch, qualities): `batch` with the bases of the seeded quality model below `min_base_quality`
    masked, as the decoders would mask them, and the qualities themselves (for the checkers)."""
    qual = qualities(seed, batch.seq_len, low_frac)
    counts, qpos = bamio.low_quality_mask(qual, batch.seq_len, min_base_quality)
    return bamio.with_mask(batch, counts, qpos), qual
