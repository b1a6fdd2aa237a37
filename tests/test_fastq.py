"""Per-base consensus qualities (`qualities=True`, `kindel consensus --fastq`; an extension: the reference has none),
without a GPU.

There is no reference to pin them against, so two restatements written in different forms are held against each
other: oracle/kindel_fqoracle.c (`fqoracle`: a linear search over q per slot, then a sequential walk over the
positions writing text and qualities side by side) and oracle/py_fqoracle.py (numpy: all 61 q at once per slot).  The
host assembly of the product (kindel.assemble_consensus with qualities) must reproduce the C walk, and K2q / K5q run
from their CUDA source under the host emulator (tests/emu/emu_api.cpp) and must reproduce the C oracle."""
import math
import os
import re
from decimal import Decimal, getcontext

import numpy as np
import pytest

import emu_harness as E
import helpers as H
from kindel_b200 import _ffi, cli, quality
from kindel_b200 import kindel as K
from oracle import coracle, fqoracle, ioracle, py_fqoracle
from oracle.py_oracle import base_call
from test_iupac import MIN_DEPTHS, _adversarial, _contigs, _piled, _table

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
THRESHOLDS = (0.0, 0.6, 0.99)
WORKED = [  # (D, k, Q) of the definition, two of them exact equalities of the product and the bound
    (8, 8, 10), (98, 98, 20), (1, 1, 4), (10, 10, 10), (100, 100, 20), (1000, 1000, 30), (100, 90, 9), (30, 29, 12),
    (100, 55, 3), (10 ** 6, 10 ** 6, 60),
]


def _hex_table(path, start):
    src = open(os.path.join(H.ROOT, path)).read()
    body = src[src.index(start) + len(start):]
    body = body[:body.index("}")]
    return [float.fromhex(h) for h in re.findall(r"0x[0-9a-fA-F.]+p[+-]\d+", body)]


def _votes(counts, md):
    yield "majority", coracle.vote(counts, md)
    for t in THRESHOLDS:
        yield "iupac%s" % t, ioracle.vote_iupac(counts, md, t)


# ------------------------------------------------------------------------------------------------ the rule
def test_ten_table_is_one_table():
    """TEN is parsed out of the CUDA source; the C oracle, the numpy oracle and the product's host copy hold the same 61
    doubles, each within half an ulp of 10^(q/10) (60 decimal digits), and nothing computes a logarithm."""
    cuda = _hex_table("kindel_b200/csrc/assemble.cu", "kQualTen[61] = {")
    assert len(cuda) == 61
    assert _hex_table("oracle/kindel_fqoracle.c", "TEN[61] = {") == cuda
    assert list(py_fqoracle.TEN) == cuda
    assert list(quality.TEN) == cuda
    getcontext().prec = 60
    for q, v in enumerate(cuda):
        exact = Decimal(10) ** (Decimal(q) / 10)
        assert abs(Decimal(v) - exact) <= Decimal(math.ulp(v)) / 2, q
    for path in ("kindel_b200/csrc/assemble.cu", "kindel_b200/quality.py", "oracle/kindel_fqoracle.c",
                 "oracle/py_fqoracle.py"):
        assert "log10" not in open(os.path.join(H.ROOT, path)).read(), path


def test_worked_values():
    for d, k, q in WORKED:
        assert fqoracle.phred(d, k) == q, (d, k)
        assert quality.phred(d, k) == q, (d, k)
        assert int(py_fqoracle._q(np.array([d]), np.array([k]))[0]) == q, (d, k)
    assert 1 * quality.TEN[10] == 10.0 and 1 * quality.TEN[20] == 100.0  # the two exact equalities
    # the same values from a table and its call bytes: A alone (single-base call), and an IUPAC R at 55 A / 45 G
    cols = [[k for _, k, _ in WORKED] + [55], [0] * 11, [d - k for d, k, _ in WORKED] + [45], [0] * 11]
    tab = _table(cols)
    calls = np.zeros(tab.shape[1], dtype=np.uint8)
    calls[10] = 0x80 | 0x5  # R = A/G
    want = np.array([q for _, _, q in WORKED] + [20], dtype=np.uint8)
    assert np.array_equal(fqoracle.qual(tab, calls)[:11], want)
    assert np.array_equal(py_fqoracle.qual(tab, calls)[:11], want)
    if E.available():
        assert np.array_equal(E.consensus_qual(tab, calls)[:11], want)


def _boundary_tables():
    """k = 0 in every form (N call, tie, zero depth, 'D', min-depth 'N', the IUPAC set of all four); depths near 2^33
    from four columns near 2^31; every IUPAC set; exact equalities of the product and the bound."""
    big = (1 << 31) - 1
    cols = np.array([
        [5, 3, 0, 0, 5, 7, big, big, big - 5, big, 0, 9, 8, 98, 1 << 30, big, 40, 40, 40, 40, 40, 40, 40, 40],
        [0, 3, 0, 0, 0, 7, big, big, big - 3, 0, 0, 0, 0, 0, 1 << 30, big, 30, 30, 30, 30, 30, 30, 30, 30],
        [0, 0, 0, 9, 0, 7, big, big, 1, 0, 0, 0, 0, 0, 1 << 30, big, 20, 20, 20, 20, 20, 20, 20, 20],
        [0, 0, 0, 0, 0, 7, big, 0, 0, 0, 0, 0, 0, 0, 1 << 30, 3, 10, 10, 10, 10, 10, 10, 10, 10],
    ], dtype=np.int64)
    calls = np.array([0x24, 0x04, 0x04, 0x14, 0x00, 0x8F, 0x00, 0x83, 0x81, 0x00, 0x04, 0x00, 0x00, 0x00, 0x8F, 0x87,
                      0x83, 0x85, 0x89, 0x86, 0x8A, 0x8C, 0x87, 0x8E], dtype=np.uint8)
    return _table(cols), calls


def test_boundaries():
    tab, calls = _boundary_tables()
    n = calls.shape[0]
    full = np.zeros(tab.shape[1], dtype=np.uint8)
    full[:n] = calls
    got = fqoracle.qual(tab, full)
    assert np.array_equal(got, py_fqoracle.qual(tab, full))
    assert (got[[0, 1, 2, 3, 5, 10, 14]] == 0).all()  # every k = 0 form
    w = tab[:4, :n].astype(np.int64)
    for s in range(n):
        c = int(full[s])
        if c & 0x80:
            k = 0 if c & 15 == 15 else int(sum(w[b, s] for b in range(4) if c >> b & 1))
        else:
            k = int(w[c & 7, s]) if c & 7 < 4 else 0
        assert got[s] == quality.phred(int(w[:, s].sum()), k), s
    assert got[6] == quality.phred(4 * ((1 << 31) - 1), (1 << 31) - 1) > 0  # D near 2^33
    assert got[12] == 10 and got[13] == 20
    if E.available():
        assert np.array_equal(E.consensus_qual(tab, full), got)


def test_insertion_rule():
    d, dn, k = np.array([10, 10, 3, 100, 0, 7]), np.array([4, 10, 9, 100, 0, 7]), np.array([4, 10, 3, 55, 1, -1])
    want = [quality.insertion_phred(int(a), int(b), int(max(c, 0)), c < 0) for a, b, c in zip(d, dn, k)]
    assert list(py_fqoracle.insertion_qual(d, dn, k)) == want
    assert want[1] == quality.phred(10, 10) == 10 and want[-1] == 0
    assert want[4] == quality.phred(1, 1)  # D = max(min(0, 0), 1)


# ------------------------------------------------------------------------------------- oracle vs oracle
def _ins_qual(counts, s0, ins_c):
    """{position: Q} of the insertion dicts of one contig, by the numpy oracle."""
    pos = sorted(ins_c)
    if not pos:
        return {}
    w = counts[:4].astype(np.int64).sum(axis=0)
    w = np.concatenate([w, [0]])
    slots = np.array(pos, dtype=np.int64) + s0
    k = []
    for p in pos:
        _, cnt, tie = base_call(ins_c[p])
        k.append(-1 if tie else cnt)
    q = py_fqoracle.insertion_qual(w[slots], w[slots + 1], np.array(k))
    return dict(zip(pos, q.tolist()))


def _check_contig(name, counts, calls, s0, L, ins_c, patches=None, trim_ends=False, uppercase=False):
    qual = py_fqoracle.qual(counts, calls)
    iq = _ins_qual(counts, s0, ins_c)
    lookup = lambda p: K.dict_consensus(ins_c.get(p, {}))  # noqa: E731
    seq, changes, quals = K.assemble_consensus(calls[s0:s0 + L], lookup, patches, trim_ends, uppercase,
                                               qual=qual[s0:s0 + L], ins_qual=lambda p: iq[p])
    plain, plain_changes = K.assemble_consensus(calls[s0:s0 + L], lookup, patches, trim_ends, uppercase)
    assert seq == plain and list(changes) == list(plain_changes), name
    assert len(quals) == len(seq), name
    want = fqoracle.fastq(counts, calls, s0, L, ins_c, patches, trim_ends, uppercase)
    assert (seq, quals) == want, name
    return quals


def test_restatements_agree(manifest, tmp_path):
    """On the golden fixtures, the 96 clip cases and the fuzz cases that pile without an error, with both votes at three
    min_depths: the C and numpy Q per slot are equal, and the product's host assembly with qualities gives the C walk's
    text and qualities (and the text and changes of the assembly without them)."""
    n_files = n_chars = 0
    seen = set()
    for name, batch, counts, events in _piled(manifest, tmp_path):
        n_files += 1
        contigs = list(_contigs(batch, counts, events))
        for md in MIN_DEPTHS:
            for vote, calls in _votes(counts, md):
                assert np.array_equal(fqoracle.qual(counts, calls), py_fqoracle.qual(counts, calls)), (name, vote)
                for s0, L, ins_c in contigs:
                    quals = _check_contig((name, vote, md), counts, calls, s0, L, ins_c)
                    n_chars += len(quals)
                    seen.update(quals)
    assert n_files > 100 and n_chars > 100_000
    assert {"!", "+", "5", "?"} <= seen  # Q0, 10, 20, 30


def test_clip_cases_with_realign_trim_and_uppercase(tmp_path):
    """The 96 clip cases with --realign patches (Q0), trim_ends and uppercase: the C walk equals the host assembly."""
    from clip_cases import clip_case

    n_patched = 0
    for seed in range(96):
        p = tmp_path / ("clip%d.sam" % seed)
        p.write_text(clip_case(seed))
        from kindel_b200 import bamio

        batch = bamio.read_alignment(p)
        try:
            counts, events = coracle.pileup(batch)
        except (IndexError, KeyError):
            continue
        run = K.PileupRun.from_host_tables(batch, counts, coracle.derive(counts), events)
        for c, (s0, L, ins_c) in enumerate(_contigs(batch, counts, events)):
            aln = run.alignment(c)
            cdrps = K.cdrp_consensuses(aln.weights, aln.deletions, aln.clip_start_weights, aln.clip_end_weights,
                                       aln.clip_start_depth, aln.clip_end_depth, 0.1, 50)
            patches = K.merge_cdrps(cdrps, 7)
            for md in (1, 3):
                for vote, calls in _votes(counts, md):
                    for trim, upper in ((False, False), (True, False), (True, True)):
                        quals = _check_contig((seed, vote), counts, calls, s0, L, ins_c, patches, trim, upper)
                        n_patched += int(any(r.seq for r in patches)) and quals.count("!") > 0
    assert n_patched > 20


def test_adversarial_tables():
    """Ties, counts near 2^29 with random deletion / insertion columns and the rounding tables of the IUPAC vote."""
    for seed in (1, 2):
        for tab in _adversarial(seed):
            for md in MIN_DEPTHS:
                for vote, calls in _votes(tab, md):
                    q = fqoracle.qual(tab, calls)
                    assert np.array_equal(q, py_fqoracle.qual(tab, calls)), (seed, vote, md)
                    assert q.max() <= 60


# ------------------------------------------------------------------------------------------ kernels
@needs_emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 1)])
def test_emulated_k2q_equals_oracle(schedule, seed, tmp_path):
    from fuzz_cases import random_case
    from kindel_b200 import bamio

    E.set_schedule(schedule, seed)
    try:
        tables = _adversarial(seed + 21) + [_boundary_tables()[0]]
        for s in range(0, 400, 16):
            p = tmp_path / ("fuzz%d.sam" % s)
            p.write_text(random_case(s))
            try:
                tables.append(coracle.pileup(bamio.read_alignment(p))[0])
            except (ValueError, KeyError, IndexError):
                continue
        for tab in tables:
            for md in (0, 7):
                for vote, calls in _votes(tab, md):
                    np.testing.assert_array_equal(E.consensus_qual(tab, calls), fqoracle.qual(tab, calls),
                                                  err_msg="%s %s md=%d" % (schedule, vote, md))
    finally:
        E.set_schedule("forward")


@needs_emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 2)])
def test_emulated_k5q_equals_oracle(schedule, seed, manifest, tmp_path):
    """K5 then K5q from their source: every contig's text and qualities equal the C walk -- insertion slots, 'D' calls,
    contig ends and multi-contig slot spaces included."""
    E.set_schedule(schedule, seed)
    n_ins = n_del = n_multi = 0
    try:
        for k, (name, batch, counts, events) in enumerate(_piled(manifest, tmp_path)):
            if k % 3 and batch.n_contigs == 1:
                continue
            n_multi += batch.n_contigs > 1
            run = K.PileupRun.from_host_tables(batch, counts, coracle.derive(counts), events)
            contigs = list(_contigs(batch, counts, events))
            for vote, calls in list(_votes(counts, 1))[:2]:
                qual = fqoracle.qual(counts, calls)
                slots = K._insertion_slots(batch, calls)
                strings, iq = [], []
                allq = {}
                for s0, L, ins_c in contigs:
                    allq.update({s0 + p: q for p, q in _ins_qual(counts, s0, ins_c).items()})
                for sl in slots.tolist():
                    text, tie = run.ins_table.consensus_at(sl)
                    strings.append("N" if tie else text.lower())
                    iq.append(allq[sl])
                texts, quals = E.assemble_qual(calls, qual, batch, slots, strings, iq)
                n_ins += len(strings)
                n_del += int(np.count_nonzero(((calls >> 4) & 3) == 1))
                for c, (s0, L, ins_c) in enumerate(contigs):
                    assert (texts[c], quals[c]) == fqoracle.fastq(counts, calls, s0, L, ins_c), (name, vote, c)
    finally:
        E.set_schedule("forward")
    assert n_ins > 50 and n_del > 50 and n_multi >= 1


# --------------------------------------------------------------------------------------- host / CLI
def test_trim_and_patches_keep_lengths():
    calls = np.array([0x24, 0x00, 0x34, 0x14, 0x02, 0x24], dtype=np.uint8)
    qual = np.array([0, 30, 0, 0, 12, 0], dtype=np.uint8)
    lookup = lambda p: ("TT", False)  # noqa: E731
    seq, _, q = K.assemble_consensus(calls, lookup, qual=qual, ins_qual=lambda p: 7)
    assert (seq, q) == ("NAttNGN", "!?((!-!")
    seq, _, q = K.assemble_consensus(calls, lookup, trim_ends=True, uppercase=True, qual=qual, ins_qual=lambda p: 7)
    assert (seq, q) == ("ATTNG", "?((!-")
    patch = [K.Region(1, 3, "ACGT", None)]
    seq, _, q = K.assemble_consensus(calls, lookup, patch, qual=qual, ins_qual=lambda p: 7)
    assert (seq, q) == ("NacgtG" + "N", "!!!!!-!")
    assert K.assemble_consensus(calls, lookup)[0] == "NAttNGN"
    assert K._trim_n("NNN", "!!!") == ("", "") and K._trim_n("NaN", None) == ("a", None)


def test_seqrecord_and_cli_flag():
    assert K.consensus_seqrecord("AC", "x").qualities is None
    assert K.consensus_seqrecord("AC", "x", "!+").qualities == "!+"
    p = cli.build_parser()
    assert p.parse_args(["consensus", "x.bam"]).fastq is False
    assert p.parse_args(["consensus", "x.bam", "--fastq"]).fastq is True


def test_abi_entry_points():
    """Exported, bound, and refusing bad arguments before they launch anything."""
    lib = _ffi.load()
    for name in ("kdl_consensus_qual", "kdl_assemble_qual"):
        assert name in _ffi.EXPORTED_SYMBOLS and getattr(lib, name)
    buf = np.zeros(4 * 8, dtype=np.int32)
    calls = np.zeros(8, dtype=np.uint8)
    assert lib.kdl_consensus_qual(buf.ctypes.data, calls.ctypes.data, 6, calls.ctypes.data, None) == 1
    assert lib.kdl_consensus_qual(None, calls.ctypes.data, 8, calls.ctypes.data, None) == 1
    assert lib.kdl_assemble_qual(None, calls.ctypes.data, 8, None, None, 0, calls.ctypes.data, None) == 1
    assert lib.kdl_assemble_qual(buf.ctypes.data, calls.ctypes.data, 8, None, None, 2, calls.ctypes.data, None) == 1
