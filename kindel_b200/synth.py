"""Seeded synthetic alignments of the BASELINE.json shapes, built directly in the flattened layout.

    simple_reads(...)    coordinate-sorted `nM` short reads over one or more random contigs
                         (configs 2, 4, 5: 30 kb x 2000x, 5 Mb x 200x, 64 x 100 kb x 500x)
    complex_reads(...)   indel- and soft-clip-heavy CIGARs plus a tail of edge-case reads (config 3)
    strands(...)         seeded strand bytes, with reads that must lie on one strand (alleles carried by one strand)
    tiled_scheme(...)    a tiled amplicon primer scheme as BED rows (`--primers`)
    amplicon_reads(...)  tiled-amplicon reads: every read starts or ends at an amplicon end, in a primer
    paired_reads(...)    Illumina-style read pairs (`--mask-overlaps`): both mates of every fragment, names, flags and
                         mate positions, both orientations, some fragments with an indel the mates share
    amplicon_pairs(...)  read pairs of tiled amplicons: both mates of a fragment start or end in its primers
    simple_pairs(...)    paired_reads / amplicon_pairs at the sizes of the bench lines, vectorised, without indels

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


def named_scheme_bed(rows) -> str:
    """tiled_scheme's rows as a named primer BED (`kindel amplicons`): per contig the k-th pair is `amp_<k>_LEFT` and
    `amp_<k>_RIGHT`, pools 1 and 2 alternating, strands + and -."""
    out, k_of = [], {}
    for i in range(0, len(rows), 2):
        (c, a, b), (_, x, y) = rows[i], rows[i + 1]
        k = k_of.get(c, 0)
        k_of[c] = k + 1
        out.append("%s\t%d\t%d\tamp_%d_LEFT\t%d\t+\n" % (c, a, b, k, 1 + k % 2))
        out.append("%s\t%d\t%d\tamp_%d_RIGHT\t%d\t-\n" % (c, x, y, k, 1 + k % 2))
    return "".join(out)


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


def write_simple_bam(path, batch: bamio.ReadBatch, level: int = 1, threads: int = 8, names=None, flag=None,
                     next_pos=None, qual=None):
    """Vectorised BAM writer for an all-simple, uniform-read-length batch (the config 2/4/5 shapes):
    lets tests and tools push 10^5..10^7 synthetic reads through the real decode path quickly.  names (uint8 [n, k]
    fixed-width QNAMEs), flag (per read) and next_pos (PNEXT - 1 per read, RNEXT then the read's own contig): paired
    reads (write_paired_bam); by default every read is "r", FLAG 0 or 16 by strand, RNEXT / PNEXT -1.  qual: the
    reads' Phred qualities concatenated in read order (qualities()); by default none (0xff)."""
    import struct
    from concurrent.futures import ThreadPoolExecutor

    n = batch.n_reads
    lens = np.unique(batch.l_seq)
    if batch.n_complex or lens.shape[0] != 1:
        raise ValueError("write_simple_bam needs simple reads of one length")
    L = int(lens[0])
    words = (L + 7) // 8
    n_seq = (L + 1) // 2
    name = b"r\x00" if names is None else b"\x00" * (names.shape[1] + 1)
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
    if flag is None:
        flag = np.zeros(n) if batch.reverse is None else 16 * batch.reverse.astype(np.int64)
    put(18, flag, "<u2")  # flag
    put(20, np.full(n, L), "<i4")
    put(24, np.full(n, -1) if next_pos is None else ref_id, "<i4")
    put(28, np.full(n, -1) if next_pos is None else next_pos, "<i4")
    put(32, np.zeros(n), "<i4")
    if names is None:
        rec[:, 36:36 + len(name)] = np.frombuffer(name, dtype=np.uint8)
    else:
        rec[:, 36:36 + names.shape[1]] = names
        rec[:, 36 + names.shape[1]] = 0
    put(36 + len(name), np.full(n, L << 4), "<u4")
    seq_be = batch.seq4.reshape(n, words).astype(">u4").view(np.uint8).reshape(n, words * 4)[:, :n_seq]
    rec[:, 40 + len(name):40 + len(name) + n_seq] = seq_be
    if qual is None:
        rec[:, 40 + len(name) + n_seq:] = 0xFF
    else:
        rec[:, 40 + len(name) + n_seq:] = np.asarray(qual, dtype=np.uint8).reshape(n, L)
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


_NAME_DIGITS = 9  # paired read names: "p" + the fragment number, zero-padded


def pair_names(frag) -> np.ndarray:
    """The QNAMEs of fragments `frag` as fixed-width bytes rows (uint8 [n, 1 + _NAME_DIGITS])."""
    frag = np.asarray(frag, dtype=np.int64)
    digits = (frag[:, None] // (10 ** np.arange(_NAME_DIGITS - 1, -1, -1, dtype=np.int64))[None, :]) % 10
    return np.concatenate([np.full((frag.shape[0], 1), ord("p"), dtype=np.uint8),
                           (digits + ord("0")).astype(np.uint8)], axis=1)


def _fnv_rows(rows: np.ndarray) -> np.ndarray:
    """64-bit FNV-1a of every bytes row (bamio.name_hash, vectorised)."""
    h = np.full(rows.shape[0], 0xCBF29CE484222325, dtype=np.uint64)
    with np.errstate(over="ignore"):
        for k in range(rows.shape[1]):
            h = (h ^ rows[:, k].astype(np.uint64)) * np.uint64(0x100000001B3)
    return h


def _pair_batch(names, contig_lens, contig_of, starts, mate_starts, flags, cigars, seqs, frag):
    """ReadBatch (mates included) of reads given one by one: contig, start, CIGAR words, nibble codes."""
    order = np.lexsort((starts, contig_of))
    n = len(order)
    seq_len = np.array([len(seqs[i]) for i in order], dtype=np.int64)
    words = (seq_len + 7) // 8
    seq4 = np.concatenate([_pack_rows(np.concatenate([seqs[i], np.zeros((-len(seqs[i])) % 8, np.uint8)])[None, :])
                           .reshape(-1) for i in order]) if n else np.zeros(0, dtype=np.uint32)
    cig = [cigars[i] for i in order]
    cig_off = np.concatenate(([0], np.cumsum([len(c) for c in cig]))).astype(np.int64)
    read_off = np.concatenate(([0], np.cumsum(np.bincount(np.asarray(contig_of)[order], minlength=len(names)))))
    flag = np.asarray(flags)[order]
    same = np.ones(n, dtype=bool)
    roles = np.array([bamio.pair_role(int(f), bool(x)) for f, x in zip(flag, same)], dtype=np.uint8)
    mates = (_fnv_rows(pair_names(np.asarray(frag)[order])), np.asarray(mate_starts)[order], roles)
    batch = bamio.finalize(names, np.asarray(contig_lens), read_off, np.asarray(starts)[order],
                           np.cumsum(words) - words, seq_len, cig_off,
                           np.array([w for c in cig for w in c], dtype=np.int64), seq4, n_records=n,
                           reverse=((flag & 0x10) != 0).astype(np.uint8), mates=mates)
    return batch, flag.astype(np.uint16), np.asarray(frag)[order]


def paired_reads(seed: int, contig_lens, depth: float, read_len: int = 150, insert_mean: float = 300,
                 insert_sd: float = 40, indel_frac: float = 0.05, sub_rate: float = 0.01, names=None, refs=None):
    """Paired-end reads of random contigs: (batch, flag uint16[n], frag int64[n]).  Every fragment of length
    ~N(insert_mean, insert_sd) (at least read_len) gives two `read_len` reads, one from each end: the left mate
    forward, the right one reverse, and which of them is the first mate (FLAG 0x40) is random.  A share indel_frac of
    the fragments carries one insertion or deletion that both mates read where they cover it, so pairs with I / D in
    their overlap occur.  The batch has its mates (name_hash of "p<fragment>", mate_start, pair_role) and strands;
    write_paired_bam writes it with QNAME, RNEXT and PNEXT.  refs: a dict that receives each contig's sequence."""
    rng = np.random.default_rng(seed)
    names = names or ["ctg%d" % i for i in range(len(contig_lens))]
    contig_of, starts, mstarts, flags, cigars, seqs, frag = [], [], [], [], [], [], []
    nf = 0
    for c, L in enumerate(contig_lens):
        ref = random_contig(rng, int(L))
        if refs is not None:
            refs[names[c]] = "".join("ACGTN"[int(x).bit_length() - 1] if x != 15 else "N" for x in ref)
        n_frag = int(round(depth * L / (2 * read_len)))
        ins = np.clip(np.round(rng.normal(insert_mean, insert_sd, n_frag)), read_len, L - 2).astype(np.int64)
        fs = rng.integers(1, np.maximum(L - ins, 2))
        kind = np.where(rng.random(n_frag) < indel_frac, rng.integers(1, 3, n_frag), 0)  # 1 = D, 2 = I
        first_left = rng.random(n_frag) < 0.5
        for k in range(n_frag):
            s0, ln = int(fs[k]), int(ins[k])
            mol = ref[s0:s0 + ln].copy()
            ops_pos = None
            if kind[k]:  # an indel in the middle of the fragment, where the mates most likely overlap
                at = ln // 2 + int(rng.integers(-10, 11))
                size = int(rng.integers(1, 6))
                if kind[k] == 1 and at + size < ln - 1:
                    mol = np.concatenate([mol[:at], mol[at + size:]])
                    ops_pos = ("D", at, size)
                elif kind[k] == 2:
                    mol = np.concatenate([mol[:at], random_contig(rng, size), mol[at:]])
                    ops_pos = ("I", at, size)
            sub = rng.random(mol.shape[0]) < sub_rate
            mol[sub] = _CODE[rng.integers(0, 5, int(sub.sum()))]
            m = mol.shape[0]
            rl = min(read_len, m)
            for left in (True, False):
                q0 = 0 if left else m - rl  # the read's bases mol[q0 : q0 + rl]
                cig, r0 = _window_cigar(q0, rl, ops_pos)
                contig_of.append(c)
                starts.append(s0 + r0)
                seqs.append(mol[q0:q0 + rl])
                cigars.append(cig)
                frag.append(nf + k)
                first = left == bool(first_left[k])
                flags.append(0x1 | 0x2 | (0x40 if first else 0x80) | (0x20 if left else 0x10))
            # each mate's PNEXT is the other's start
            mstarts += [starts[-1], starts[-2]]
        nf += n_frag
    return _pair_batch(names, contig_lens, contig_of, starts, mstarts, flags, cigars, seqs, frag)


def _window_cigar(q0: int, n: int, event):
    """(CIGAR words, reference offset of its start within the fragment) of the molecule bases [q0, q0 + n) when the
    molecule is the fragment with `event` = None, ("D", at, size) or ("I", at, size) at molecule offset `at`."""
    M, I, D = 0, 1, 2
    if event is None:
        return [n << 4 | M], q0
    kind, at, size = event
    if kind == "D":  # molecule offset x >= at sits at fragment offset x + size
        r0 = q0 if q0 < at else q0 + size
        if q0 < at < q0 + n:
            return [(at - q0) << 4 | M, size << 4 | D, (q0 + n - at) << 4 | M], r0
        return [n << 4 | M], r0
    # insertion: molecule [at, at + size) is inserted; x >= at + size sits at fragment offset x - size
    lo, hi = max(q0, at), min(q0 + n, at + size)
    if lo >= hi:
        return [n << 4 | M], q0 if q0 < at else q0 - size
    ops = []
    if lo > q0:
        ops.append((lo - q0) << 4 | M)
    ops.append((hi - lo) << 4 | (I if (lo > q0 and hi < q0 + n) else 4))  # at a read end the inserted bases are a clip
    if hi < q0 + n:
        ops.append((q0 + n - hi) << 4 | M)
    r0 = q0 if q0 < at else at
    return ops, r0


def amplicon_pairs(seed: int, contig_len: int, depth: float, read_len: int = 150, spacing: int = 200,
                   overlap: int = 50, sub_rate: float = 0.01):
    """Tiled-amplicon read pairs of one random contig: (batch, flag, frag, scheme rows).  Each fragment is one whole
    amplicon of tiled_scheme(seed, ...), so one mate starts in its left primer and the other ends in its right
    primer; the mates overlap in the amplicon's middle when it is shorter than two reads."""
    rng = np.random.default_rng(seed)
    rows = tiled_scheme(seed, ["ctg0"], [contig_len], spacing, overlap)
    amp_lo = np.array([a for _, a, _ in rows[0::2]], dtype=np.int64)
    amp_hi = np.array([b for _, _, b in rows[1::2]], dtype=np.int64)
    ref = random_contig(rng, contig_len)
    n_frag = int(round(depth * contig_len / (2 * read_len)))
    k = rng.integers(0, amp_lo.shape[0], size=n_frag)
    first_left = rng.random(n_frag) < 0.5
    contig_of, starts, mstarts, flags, cigars, seqs, frag = [], [], [], [], [], [], []
    for j in range(n_frag):
        a, b = int(amp_lo[k[j]]), int(amp_hi[k[j]])
        rl = min(read_len, b - a)
        for left in (True, False):
            s0 = a if left else b - rl
            bases = ref[s0:s0 + rl].copy()
            sub = rng.random(rl) < sub_rate
            bases[sub] = _CODE[rng.integers(0, 5, int(sub.sum()))]
            contig_of.append(0)
            starts.append(s0)
            seqs.append(bases)
            cigars.append([rl << 4])
            frag.append(j)
            first = left == bool(first_left[j])
            flags.append(0x1 | 0x2 | (0x40 if first else 0x80) | (0x20 if left else 0x10))
        mstarts += [starts[-1], starts[-2]]
    batch, flag, fr = _pair_batch(["ctg0"], [contig_len], contig_of, starts, mstarts, flags, cigars, seqs, frag)
    return batch, flag, fr, rows


def paired_records(batch: bamio.ReadBatch, flag, frag):
    """(contigs, records) for bamio.write_bam of a paired batch: QNAME "p<fragment>", its FLAG, RNEXT = its own
    contig and PNEXT = mate_start -- small batches only (Python loop)."""
    contigs, recs = to_records(batch)
    names = pair_names(frag)
    out = []
    for r, (ref_id, pos0, _, words, seq) in enumerate(recs):
        out.append((ref_id, pos0, int(flag[r]), words, seq, names[r].tobytes().decode(), 60, None, ref_id,
                    int(batch.mate_start[r])))
    return contigs, out


def write_paired_bam(path, batch: bamio.ReadBatch, flag, frag, level: int = 1, threads: int = 8):
    """A paired batch as a BAM file with QNAME, FLAG, RNEXT and PNEXT: vectorised for an all-simple batch of one read
    length (write_simple_bam), record by record otherwise."""
    if batch.n_complex == 0 and np.unique(batch.l_seq).shape[0] == 1:
        write_simple_bam(path, batch, level, threads, names=pair_names(frag), flag=flag,
                         next_pos=batch.mate_start)
        return
    bamio.write_bam(path, *paired_records(batch, flag, frag), level=level)


def simple_pairs(seed: int, contig_len: int, depth: float, read_len: int = 150, insert_mean: float = 300,
                 insert_sd: float = 40, sub_rate: float = 0.01, amplicons=None):
    """paired_reads for large sizes, vectorised: one contig, `read_len`M mates without indels, sorted by start.
    amplicons: scheme rows (tiled_scheme); each fragment is then one whole amplicon, so one mate starts in its left
    primer and the other ends in its right one.  Returns (batch, flag, frag)."""
    rng = np.random.default_rng(seed)
    n_frag = int(round(depth * contig_len / (2 * read_len)))
    if amplicons is None:
        ins = np.clip(np.round(rng.normal(insert_mean, insert_sd, n_frag)), read_len, contig_len - 2).astype(np.int64)
        lo = rng.integers(1, np.maximum(contig_len - ins, 2))
    else:
        a = np.array([x for _, x, _ in amplicons[0::2]], dtype=np.int64)
        b = np.array([y for _, _, y in amplicons[1::2]], dtype=np.int64)
        k = rng.integers(0, a.shape[0], size=n_frag)
        lo, ins = a[k], np.maximum(b[k] - a[k], read_len)
    first_left = rng.random(n_frag) < 0.5
    frag = np.repeat(np.arange(n_frag, dtype=np.int64), 2)
    left = np.tile(np.array([True, False]), n_frag)
    start = np.where(left, np.repeat(lo, 2), np.repeat(lo + ins - read_len, 2))
    mate_start = np.where(left, np.repeat(lo + ins - read_len, 2), np.repeat(lo, 2))
    first = left == np.repeat(first_left, 2)
    flag = (0x1 | 0x2 | np.where(first, 0x40, 0x80) | np.where(left, 0x20, 0x10)).astype(np.uint16)
    order = np.argsort(start, kind="stable")
    start, mate_start, flag, frag = start[order], mate_start[order], flag[order], frag[order]
    n = start.shape[0]
    words = (read_len + 7) // 8
    ref = random_contig(rng, contig_len)
    ref_pad = np.concatenate([ref, np.zeros(words * 8, dtype=np.uint8)])
    parts = []
    for s0 in range(0, n, 1 << 18):
        st = start[s0:s0 + (1 << 18)]
        nib = ref_pad[st[:, None] + np.arange(words * 8, dtype=np.int64)[None, :]]
        nib[:, read_len:] = 0
        n_sub = rng.binomial(st.shape[0] * read_len, sub_rate)
        nib[rng.integers(0, st.shape[0], size=n_sub), rng.integers(0, read_len, size=n_sub)] = \
            _CODE[rng.integers(0, 5, size=n_sub)]
        parts.append(_pack_rows(nib))
    seq4 = np.concatenate(parts).reshape(-1) if parts else np.zeros(0, dtype=np.uint32)
    roles = np.where((flag & 0x40) != 0, 1, 2).astype(np.uint8)
    mates = (_fnv_rows(pair_names(frag)), mate_start, roles)
    batch = bamio.finalize(["ctg0"], np.array([contig_len]), np.array([0, n]), start,
                           np.arange(n, dtype=np.int64) * words, np.full(n, read_len, dtype=np.int64),
                           np.arange(n + 1, dtype=np.int64), np.full(n, read_len << 4, dtype=np.int64), seq4,
                           n_records=n, reverse=((flag & 0x10) != 0).astype(np.uint8), mates=mates)
    return batch, flag, frag


def dup_pairs(seed: int, contig_len: int, depth: float, read_len: int = 150, insert_mean: float = 300,
              insert_sd: float = 40, dup_frac: float = 0.2, clip_frac: float = 0.3, sub_rate: float = 0.01,
              amplicons=None, want_qual: bool = False):
    """Shotgun read pairs with planted PCR duplicates (`--dedup`), vectorised: simple_pairs' fragments, of which a
    seeded share `dup_frac` is copied 1-5 more times, so many that the pairs, copies included, make `depth`.  Each copy is a fragment of its own (QNAME, qualities) over the
    same two ends: which mate is first (FLAG 0x40) is drawn afresh, and with probability `clip_frac` each mate soft-clips
    1-20 bases of its 5' end (the left mate's start moves right by the clip, the right mate's M shrinks), which leaves
    its unclipped end where it was.  amplicons: scheme rows; every fragment is then one whole amplicon (the extreme
    case: thousands of copies of one key).  The batch has strands, mates and `dup_score` (the sum of its seeded
    qualities >= 15, synth.qualities).  Returns (batch, flag, frag, qual): qual the concatenated qualities in read order
    when want_qual, else None."""
    rng = np.random.default_rng(seed)
    n0 = int(round(depth * contig_len / (2 * read_len) / (1 + 3 * dup_frac)))  # 3 copies on average: depth overall
    if amplicons is None:
        ins0 = np.clip(np.round(rng.normal(insert_mean, insert_sd, n0)), read_len, contig_len - 2).astype(np.int64)
        lo0 = rng.integers(1, np.maximum(contig_len - ins0, 2))
    else:
        a = np.array([x for _, x, _ in amplicons[0::2]], dtype=np.int64)
        b = np.array([y for _, _, y in amplicons[1::2]], dtype=np.int64)
        k = rng.integers(0, a.shape[0], size=n0)
        lo0, ins0 = a[k], np.maximum(b[k] - a[k], read_len)
    copies = np.where(rng.random(n0) < dup_frac, rng.integers(1, 6, n0), 0)
    src = np.repeat(np.arange(n0), 1 + copies)
    n_frag = src.shape[0]
    lo, ins = lo0[src], ins0[src]
    is_copy = np.concatenate(([False], src[1:] == src[:-1]))
    clip = np.where(is_copy[:, None] & (rng.random((n_frag, 2)) < clip_frac), rng.integers(1, 21, (n_frag, 2)), 0)
    first_left = rng.random(n_frag) < 0.5
    L = read_len
    frag = np.repeat(np.arange(n_frag, dtype=np.int64), 2)
    left = np.tile(np.array([True, False]), n_frag)
    win = np.where(left, np.repeat(lo, 2), np.repeat(lo + ins - L, 2))  # the mate's SEQ is ref[win : win + L]
    cl = np.where(left, np.repeat(clip[:, 0], 2), np.repeat(clip[:, 1], 2))  # the mate's 5' soft clip
    start = win + np.where(left, cl, 0)
    mate_start = np.where(left, np.repeat(lo + ins - L, 2), np.repeat(lo + clip[:, 0], 2))
    first = left == np.repeat(first_left, 2)
    flag = (0x1 | 0x2 | np.where(first, 0x40, 0x80) | np.where(left, 0x20, 0x10)).astype(np.uint16)
    order = np.argsort(start, kind="stable")
    start, mate_start, flag, frag, win, cl, left = (x[order] for x in (start, mate_start, flag, frag, win, cl, left))
    n = start.shape[0]
    n_ops = np.where(cl > 0, 2, 1)
    cig_off = np.concatenate(([0], np.cumsum(n_ops)))
    cigar = np.empty(int(cig_off[-1]), dtype=np.int64)
    at = cig_off[:-1]
    m_len = L - cl
    cigar[at] = np.where((cl > 0) & left, (cl << 4) | 4, m_len << 4)
    two = np.flatnonzero(cl > 0)
    cigar[at[two] + 1] = np.where(left[two], m_len[two] << 4, (cl[two] << 4) | 4)
    words = (L + 7) // 8
    ref = random_contig(rng, contig_len)
    ref_pad = np.concatenate([ref, np.zeros(words * 8, dtype=np.uint8)])
    parts, scores, quals = [], [], []
    for s0 in range(0, n, 1 << 18):
        w = win[s0:s0 + (1 << 18)]
        nib = ref_pad[w[:, None] + np.arange(words * 8, dtype=np.int64)[None, :]]
        nib[:, L:] = 0
        n_sub = rng.binomial(w.shape[0] * L, sub_rate)
        nib[rng.integers(0, w.shape[0], size=n_sub), rng.integers(0, L, size=n_sub)] = _CODE[rng.integers(0, 5, size=n_sub)]
        parts.append(_pack_rows(nib))
        q = qualities(seed * 1000003 + s0, np.full(w.shape[0], L)).reshape(-1, L)
        scores.append(np.where(q >= 15, q, 0).sum(axis=1, dtype=np.int64).astype(np.int32))
        if want_qual:
            quals.append(q.reshape(-1))
    seq4 = np.concatenate(parts).reshape(-1) if parts else np.zeros(0, dtype=np.uint32)
    roles = np.where((flag & 0x40) != 0, 1, 2).astype(np.uint8)
    mates = (_fnv_rows(pair_names(frag)), mate_start, roles)
    batch = bamio.finalize(["ctg0"], np.array([contig_len]), np.array([0, n]), start,
                           np.arange(n, dtype=np.int64) * words, np.full(n, L, dtype=np.int64), cig_off, cigar, seq4,
                           n_records=n, reverse=((flag & 0x10) != 0).astype(np.uint8), mates=mates,
                           dup_score=np.concatenate(scores) if scores else np.zeros(0, dtype=np.int32))
    qual = (np.concatenate(quals) if quals else np.zeros(0, dtype=np.uint8)) if want_qual else None
    return batch, flag, frag, qual
