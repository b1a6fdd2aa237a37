"""`variants --vcf --reference` (extension) without a GPU: the FASTA loader, a truth set of planted SNVs, insertions and
deletions that pins the oracle (oracle/py_rvoracle.py), K6r and K7 from their CUDA source under the host emulator
(tests/emu/emu_variants_ref.cpp) against the oracle, and the host VCF writer over the emulated kernels.

The truth set (`truth_set`) is generated here: a random reference, alleles planted at chosen fractions -- at the first
and last positions, next to each other, several at one locus -- and error-free reads whose CIGARs are taken from the
edits, with the generator's own count of the reads carrying each allele."""
import gzip

import numpy as np
import pytest

import emu_variants_ref_harness as ER
import limit_cases as LC
from fuzz_cases import random_case
from kindel_b200 import bamio, cli, engine, _ffi
from kindel_b200 import kindel as K
from kindel_b200.reference import Reference, load_reference
from oracle import coracle, samdecode
from oracle import py_oracle as PO
from oracle import py_rvoracle as RV
from test_variants_vcf import GRID, adversarial

needs_emu = pytest.mark.skipif(not ER.available(), reason="needs g++ and the CUDA headers")
NAN = float("nan")
OPS = "MIDNSHP=X"


# ------------------------------------------------------------------------------------------------ truth set
def _loci(L, high):
    """Allele groups of one contig: (kind, where, [(allele, fraction)]).  Alleles of a group exclude each other in a
    read; groups do not overlap (a deletion may end where an insertion sits, an SNV may touch either)."""
    f = (lambda lo: lo) if not high else (lambda lo: 0.6 + lo / 10)
    m = L // 2
    # (above one half an insertion before a deleted base would not reach the consensus: kindel's vote skips the
    # insertion check at a deleted position)
    return [
        ("snv", 0, [("G", f(0.3))]),              # POS 1
        ("ins", 0, [("TT", f(0.2))]),             # before the first base
    ] + ([] if high else [
        ("ins", 1, [("CA", f(0.25))]),            # POS 1, next to the SNV and the deletion
    ]) + [
        ("del", 1, [(1, f(0.3))]),                # POS 1, REF ref[0..1]
        ("snv", 2, [("T", f(0.15))]),             # POS 3
        ("snv", m, [("A", 0.2), ("C", 0.15)] if not high else [("A", 0.7)]),
        ("ins", m + 1, [("GA", 0.2), ("T", 0.1), ("GA", 0.05)] if not high else [("GAC", 0.65)]),
        ("del", m + 3, [(1, 0.1), (4, 0.25)] if not high else [(4, 0.8)]),
        ("snv", L - 2, [("C", f(0.35))]),         # POS L - 1
        ("del", L - 1, [(1, f(0.2))]),            # the last base
        ("ins", L, [("AAG", f(0.3))]),            # behind the last base (slot L)
    ]


def truth_set(seed, L=160, n_full=40, n_plain=25, high=False):
    """(ref text, reads [(pos0, cigar [(n, op)], seq)], planted [(kind, where, allele, count)]).  Every full read
    spans the contig and carries at most one allele per group; plain reads are reference copies of random spans."""
    rng = np.random.default_rng(seed)
    ref = "".join("ACGT"[i] for i in rng.integers(0, 4, L))
    loci = _loci(L, high)
    for kind, where, alleles in loci:  # SNV alleles must differ from the reference base
        if kind == "snv":
            alleles[:] = [(b if b != ref[where] else "ACGT"[("ACGT".index(b) + 1) % 4], fr) for b, fr in alleles]
    carried = [dict() for _ in range(n_full)]
    planted = []
    for g, (kind, where, alleles) in enumerate(loci):
        order = rng.permutation(n_full)
        k = 0
        for a, fr in alleles:
            n = int(round(fr * n_full))
            for r in order[k:k + n]:
                carried[r][g] = a
            k += n
        counts = {}
        for a, _ in alleles:
            counts[a] = sum(1 for c in carried if c.get(g) == a)
        for a in counts:  # (the same string twice in a group is one allele)
            planted.append((kind, where, a, counts[a]))
    reads = []
    for c in carried:
        ops, seq, p = [], [], 0
        ins = {loci[g][1]: a for g, a in c.items() if loci[g][0] == "ins"}
        dels = {loci[g][1]: a for g, a in c.items() if loci[g][0] == "del"}
        snv = {loci[g][1]: a for g, a in c.items() if loci[g][0] == "snv"}

        def op(n, o):
            if ops and ops[-1][1] == o:
                ops[-1] = (ops[-1][0] + n, o)
            else:
                ops.append((n, o))

        while True:
            if p in ins:
                op(len(ins[p]), "I")
                seq.append(ins[p])
            if p == L:
                break
            if p in dels:
                op(dels[p], "D")
                p += dels[p]
                continue
            op(1, "M")
            seq.append(snv.get(p, ref[p]))
            p += 1
        reads.append((0, ops, "".join(seq)))
    for _ in range(n_plain):
        a = int(rng.integers(0, L - 20))
        b = int(rng.integers(a + 10, L + 1))
        reads.append((a, [(b - a, "M")], ref[a:b]))
    return ref, reads, planted


def expected_alleles(ref, planted):
    """{(POS, REF, ALT): count} the VCF must list for the planted alleles (the rules of §5 of the design)."""
    out = {}
    for kind, w, a, n in planted:
        if kind == "snv":
            key = (w + 1, ref[w], a)
        elif kind == "del":
            key = (w, ref[w - 1:w + a], ref[w - 1]) if w >= 1 else (1, ref[0:a + 1], ref[a])
        else:
            key = (w, ref[w - 1], ref[w - 1] + a) if w >= 1 else (1, ref[0], a + ref[0])
        out[key] = n
    return out


def _recs(reads):
    return [PO.Rec(p + 1, True, seq, tuple(ops)) for p, ops, seq in reads]


def bam_records(reads, ref_id=0):
    return [(ref_id, p, 0, [(n << 4) | OPS.index(o) for n, o in ops], seq) for p, ops, seq in reads]


def _parse(lines):
    """{(POS, REF, ALT): (count of the allele, INFO dict)} of one-contig VCF lines (AD's second value for an SNV)."""
    out = {}
    for ln in lines:
        f = ln.split("\t")
        info = dict(kv.split("=") if "=" in kv else (kv, True) for kv in f[7].split(";"))
        for j, alt in enumerate(f[4].split(",")):
            n = int(info["AO"]) if "INDEL" in info else int(info["AD"].split(",")[1 + j])
            out[(int(f[1]), f[3], alt)] = (n, info)
    return out


@pytest.mark.parametrize("seed,high", [(1, False), (2, False), (3, True)])
def test_oracle_lists_exactly_the_planted_alleles(seed, high):
    ref, reads, planted = truth_set(seed, high=high, n_plain=0 if high else 25)
    lines = RV.vcf_lines([("t", ref, _recs(reads))], 0, 0.0)
    got = _parse(lines)
    want = expected_alleles(ref, planted)
    assert {k: v[0] for k, v in got.items()} == want
    # POS order, SNV before deletion before insertion at one POS
    keys = [(int(ln.split("\t")[1]), 0 if "INDEL" not in ln else (1 if len(ln.split("\t")[3]) > 1 else 2))
            for ln in lines]
    assert keys == sorted(keys)
    # thresholds: above every count nothing is left
    assert RV.vcf_lines([("t", ref, _recs(reads))], 10 ** 6, 0.0) == []


# --------------------------------------------------------------------------------------------------- FASTA
def _batch(names, lens):
    slots, n_slots = bamio.layout_slots(np.asarray(lens))
    return type("B", (), dict(contig_names=list(names), contig_len=np.asarray(lens, dtype=np.int32),
                              contig_slot=slots, n_slots=n_slots, n_contigs=len(lens)))()


def test_fasta_loader(tmp_path):
    b = _batch(["c1", "c2"], [10, 7])
    text = ">c2 second contig\r\nACG\r\ntnR\r\nk\r\n>other\nNNNN\n>c1\nACGTA\nCGTAC\n"
    plain = tmp_path / "r.fa"
    plain.write_bytes(text.encode())
    gz = tmp_path / "r.fa.gz"
    gz.write_bytes(gzip.compress(text.encode()))
    a, g = load_reference(plain, b), load_reference(gz, b)
    assert isinstance(a, Reference) and a.name == "r.fa" and g.name == "r.fa.gz"
    np.testing.assert_array_equal(a.codes, g.codes)
    s1, s2 = int(b.contig_slot[0]), int(b.contig_slot[1])
    assert a.codes.dtype == np.uint8 and a.codes.shape == (b.n_slots,)
    assert a.codes[s1:s1 + 10].tolist() == [0, 1, 2, 3, 0, 1, 2, 3, 0, 1]
    assert a.codes[s2:s2 + 7].tolist() == [0, 1, 2, 3, 4, 4, 4]  # lower case folded; N and IUPAC are 4
    others = np.ones(b.n_slots, dtype=bool)
    others[s1:s1 + 10] = others[s2:s2 + 7] = False
    assert (a.codes[others] == 4).all()  # slot L and the padding


@pytest.mark.parametrize("text,needle", [
    (">c1\nACGTACGTAC\n", "'c2'"),                                   # missing contig
    (">c1\nACGTACGTAC\n>c2\nACGTAC\n", "'c2'"),                      # length differs from LN
    (">c1\nACGTACGTAC\n>c2\nACGTACG\n>c1\nA\n", "'c1'"),             # duplicate id
    (">c1\nACGTA-GTAC\n>c2\nACGTACG\n", "'c1'"),                     # not a letter
    (">c1\nACGTACGTAC\n>c2\nACG4ACG\n", "'c2'"),
])
def test_fasta_loader_errors(tmp_path, text, needle):
    p = tmp_path / "bad.fa"
    p.write_text(text)
    with pytest.raises(ValueError, match=needle):
        load_reference(p, _batch(["c1", "c2"], [10, 7]))


def test_fasta_loader_speed(tmp_path):
    import time

    rng = np.random.default_rng(0)
    seq = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, 6_000_000)].tobytes()
    p = tmp_path / "big.fa"
    p.write_bytes(b">big\n" + b"\n".join(seq[i:i + 80] for i in range(0, len(seq), 80)) + b"\n")
    t0 = time.perf_counter()
    ref = load_reference(p, _batch(["big"], [6_000_000]))
    assert time.perf_counter() - t0 < 1.0
    lut = np.zeros(256, dtype=np.uint8)
    lut[list(b"ACGT")] = [0, 1, 2, 3]
    np.testing.assert_array_equal(ref.codes[:6_000_000], lut[np.frombuffer(seq, np.uint8)])


# -------------------------------------------------------------------------------------------- corpora
def _groups(path):
    header, records = samdecode.read_alignment_file(path)
    lens = {sn[3:]: int(f[0][3:]) for sn, f in header["@SQ"].items()}
    groups = {}
    for r in records:
        groups.setdefault(r.rname, []).append(r)
    groups.pop("*", None)
    return lens, groups


def _random_ref(rng, batch):
    """Codes with A, C, G, T and some 4 (N) at the positions; 4 elsewhere."""
    codes = np.full(batch.n_slots, 4, dtype=np.uint8)
    for s0, L in zip(batch.contig_slot.tolist(), batch.contig_len.tolist()):
        codes[s0:s0 + L] = rng.choice(np.array([0, 1, 2, 3, 4], dtype=np.uint8), L, p=[0.24, 0.24, 0.24, 0.24, 0.04])
    return codes


def corpus(tmp_path, seeds=range(400), limits=True):
    """(name, batch, table, ref codes, {contig: records}) of the fuzz cases and the limit cases that the reference's
    loop accepts."""
    out = []
    paths = []
    for seed in seeds:
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(random_case(seed))
        paths.append(("fuzz%d" % seed, p))
    if limits:
        for name in LC.GROUPS:
            p = tmp_path / ("limit_%s.sam" % name)
            p.write_text(LC.sam_text(name))
            paths.append(("limit_" + name, p))
    for k, (name, p) in enumerate(paths):
        try:
            batch = bamio.read_alignment(p)
            table, _ = coracle.pileup(batch)
            lens, groups = _groups(p)
            for nm in batch.contig_names:  # the oracle's own walk must accept them too
                PO.pileup(lens[nm], groups.get(nm, []))
        except (ValueError, KeyError, IndexError):
            continue
        out.append((name, batch, table, _random_ref(np.random.default_rng(k), batch), groups))
    return out


def ref_adversarial(seed):
    """test_variants_vcf.adversarial's tables (counts in slot L and the padding, ties, zero depth, near 2^31) with an
    insertion column and reference codes that put 4 at some positions and every code in slot L and the padding."""
    table, cs, cl = adversarial(seed)
    rng = np.random.default_rng(seed)
    n = table.shape[1]
    table[6] = rng.integers(0, 6, n)
    table[6, rng.random(n) < 0.05] = (1 << 31) - 1
    codes = rng.integers(0, 5, n).astype(np.uint8)
    return table, cs, cl, codes


def _sites_equal(got, want, what):
    for g, w, name in zip(got, want, ("slot", "counts", "dpa", "mask")):
        assert g.dtype == w.dtype, (what, name, g.dtype, w.dtype)
        np.testing.assert_array_equal(g, w, err_msg="%s: %s" % (what, name))


# ---------------------------------------------------------------------------------------------- K6r, K7
@needs_emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 3)])
def test_emulated_k6r_equals_oracle(schedule, seed, tmp_path):
    """K6r from its source == RV.sites: adversarial tables over the whole threshold grid, the fuzz and limit tables
    at two grid points each and the default thresholds."""
    ER.set_schedule(schedule, seed)
    try:
        n_sites = 0
        for s in (1, 2):
            table, cs, cl, codes = ref_adversarial(s + seed)
            for a, r in GRID:
                want = RV.sites(table, cs, cl, codes, a, r)
                got = ER.variant_sites_ref(table, cs, cl, codes, engine.variant_abs_floor(a), r)
                _sites_equal(got, want, (schedule, s, a, r))
                n_sites += len(want[0])
        for j, (name, batch, table, codes, _) in enumerate(corpus(tmp_path, range(seed, 400, 4))):
            for a, r in [GRID[(7 * j + i) % len(GRID)] for i in range(2)] + [(1, 0.01), (0, 0.0)]:
                want = RV.sites(table, batch.contig_slot, batch.contig_len, codes, a, r)
                got = ER.variant_sites_ref(table, batch.contig_slot, batch.contig_len, codes,
                                           engine.variant_abs_floor(a), r)
                _sites_equal(got, want, (schedule, name, a, r))
                n_sites += len(want[0])
        assert n_sites > 20_000
    finally:
        ER.set_schedule("forward")


def _oracle_events(batch, groups):
    """RV.deletion_events of every contig, as (slot, length) in the batch's contig order."""
    out = []
    for c, nm in enumerate(batch.contig_names):
        s0 = int(batch.contig_slot[c])
        out += [(s0 + r, n) for r, n in RV.deletion_events(int(batch.contig_len[c]), groups.get(nm, []))]
    return out


@needs_emu
@pytest.mark.parametrize("schedule,seed", [("forward", 0), ("reverse", 0), ("random", 5)])
def test_emulated_k7_equals_oracle(schedule, seed, tmp_path):
    """K7 from its source: the events of every fuzz and limit case (POS 0, mid-read S, D past the end) in read order
    == the oracle's walk over the decoded records, and on an unsorted copy of a batch the same events."""
    ER.set_schedule(schedule, seed)
    try:
        n = 0
        for name, batch, _, _, groups in corpus(tmp_path, range(400) if schedule == "forward" else range(seed, 400, 3)):
            slot, length = ER.deletion_events(batch)
            got = list(zip(slot.tolist(), length.tolist()))
            assert got == _oracle_events(batch, groups), name
            n += len(got)
        assert n > (200 if schedule == "forward" else 50)
        ref, reads, _ = truth_set(7)
        p = tmp_path / "truth.bam"
        bamio.write_bam(p, [("t", len(ref))], bam_records(reads[::-1]))  # reversed: not coordinate-sorted
        batch = bamio.read_alignment(p)
        slot, length = ER.deletion_events(batch)
        assert sorted(zip(slot.tolist(), length.tolist())) == sorted(
            (r, n) for r, n in RV.deletion_events(len(ref), _recs(reads[::-1])))
    finally:
        ER.set_schedule("forward")


# ------------------------------------------------------------------------------------------- host VCF
class _Emulated:
    """engine.variant_sites_ref / engine.deletion_alleles over the emulated kernels (host tables), so that the host
    half of the VCF runs without a GPU."""

    def __init__(self, batch):
        self.batch = batch

    def sites(self, counts, contig_slot, contig_len, ref, a, r):
        return ER.variant_sites_ref(counts, contig_slot, contig_len, ref, engine.variant_abs_floor(a), r)

    def deletions(self, dbatch, counts, a, r):
        slot, length = ER.deletion_events(self.batch)
        groups = {}
        for key in zip(slot.tolist(), length.tolist()):
            groups[key] = groups.get(key, 0) + 1
        out = []
        for (s, n), c in sorted(groups.items()):
            d = int(np.asarray(counts)[0:6, s].astype(np.int64).sum())
            if c > engine.variant_abs_floor(a) and (c / d if d > 0 else 0.0) > r:
                out.append((s, n, c, d))
        arr = np.array(out, dtype=np.int64).reshape(-1, 4)
        return tuple(arr[:, k].copy() for k in range(4))


def host_vcf(monkeypatch, batch, table, events, ref, a, r):
    run = K.PileupRun.from_host_tables(batch, table, coracle.derive(table), events)
    run.counts, run.dbatch = table, batch  # host stand-ins: the patched engine calls take them as they are
    emu = _Emulated(batch)
    monkeypatch.setattr(engine, "variant_sites_ref", emu.sites)
    monkeypatch.setattr(engine, "deletion_alleles", emu.deletions)
    return K.variants_vcf_from_run(run, a, r, reference=ref)


def oracle_vcf_lines(batch, groups, ref_text, a, r):
    return RV.vcf_lines([(nm, ref_text[nm], groups.get(nm, [])) for nm in batch.contig_names], a, r)


def _texts(batch, codes):
    return {nm: "".join("ACGTN"[x] for x in codes[s0:s0 + L].tolist())
            for nm, s0, L in zip(batch.contig_names, batch.contig_slot.tolist(), batch.contig_len.tolist())}


@needs_emu
def test_host_vcf_equals_oracle_text(monkeypatch, tmp_path):
    """variants_vcf_from_run(reference=...) over oracle tables and the emulated kernels == the oracle's VCF lines, on
    the fuzz and limit corpora and on truth sets, at several thresholds; the header carries the reference's name."""
    items = []
    for name, batch, table, codes, groups in corpus(tmp_path, range(0, 400, 2)):
        items.append((name, batch, table, codes, groups))
    for seed in (1, 2, 3):
        ref, reads, _ = truth_set(seed, high=seed == 3, n_plain=0 if seed == 3 else 25)
        p = tmp_path / ("truth%d.bam" % seed)
        bamio.write_bam(p, [("t", len(ref))], bam_records(reads))
        batch = bamio.read_alignment(p)
        table, _ = coracle.pileup(batch)
        codes = load_reference_text(tmp_path, batch, {"t": ref})
        items.append(("truth%d" % seed, batch, table, codes, _groups(p)[1]))
    n = 0
    for name, batch, table, codes, groups in items:
        events = coracle.pileup(batch)[1]
        ref = Reference(codes, "ref.fa")
        for a, r in ((1, 0.01), (0, 0.0), (2, 0.2)):
            text = host_vcf(monkeypatch, batch, table, events, ref, a, r)
            lines = text.splitlines()
            body = [ln for ln in lines if not ln.startswith("#")]
            assert lines[3] == "##reference=ref.fa" and lines[len(lines) - len(body) - 1].startswith("#CHROM")
            assert body == oracle_vcf_lines(batch, groups, _texts(batch, codes), a, r), (name, a, r)
            n += len(body)
    assert n > 2000


def load_reference_text(tmp_path, batch, texts):
    p = tmp_path / "ref.fa"
    p.write_text("".join(">%s\n%s\n" % (nm, texts[nm]) for nm in batch.contig_names))
    return load_reference(p, batch).codes


@needs_emu
def test_truth_set_vcf_lists_the_planted_alleles(monkeypatch, tmp_path):
    ref, reads, planted = truth_set(11)
    p = tmp_path / "truth.bam"
    bamio.write_bam(p, [("t", len(ref))], bam_records(reads))
    batch = bamio.read_alignment(p)
    table, events = coracle.pileup(batch)
    codes = load_reference_text(tmp_path, batch, {"t": ref})
    text = host_vcf(monkeypatch, batch, table, events, Reference(codes, "ref.fa"), 0, 0.0)
    got = _parse([ln for ln in text.splitlines() if not ln.startswith("#")])
    assert {k: v[0] for k, v in got.items()} == expected_alleles(ref, planted)
    header = text.splitlines()
    assert '##INFO=<ID=INDEL,Number=0,Type=Flag,Description="The record is an insertion or a deletion">' in header
    assert any(h.startswith("##INFO=<ID=AO,Number=A,Type=Integer") for h in header)


def test_vcf_without_reference_is_unchanged():
    """No reference: the header and records are the ones of the sites-only VCF (the pinned test in
    test_variants_vcf.py covers the lines); reference=None is the default."""
    import inspect

    assert inspect.signature(K.variants_vcf).parameters["reference"].default is None
    assert inspect.signature(K.variants_vcf_from_run).parameters["reference"].default is None


# ------------------------------------------------------------------------------------------------- CLI
def test_cli_reference_option(monkeypatch, capsys):
    p = cli.build_parser()
    a = p.parse_args(["variants", "--vcf", "--reference", "r.fa", "x.bam"])
    assert a.reference == "r.fa" and a.rel_threshold == 0.01
    assert p.parse_args(["variants", "x.bam"]).reference is None
    seen = {}

    def fake_vcf(path, a, r, devices=None, reference=None, **filters):
        seen["vcf"] = (path, a, r, devices, reference, filters)
        return "##fileformat=VCFv4.2\n"

    monkeypatch.setattr(K, "variants_vcf", fake_vcf)
    assert cli.main(["variants", "--vcf", "--reference", "g/r.fa", "-r", "0.2", "x.bam"]) == 0
    assert capsys.readouterr().out == "##fileformat=VCFv4.2\n"
    assert seen["vcf"] == ("x.bam", 1, 0.2, None, "g/r.fa", dict(min_base_quality=0, min_mapq=0, exclude_flags=0))


@pytest.mark.parametrize("args", [["--reference", "r.fa"], ["-o", "--reference", "r.fa"]])
def test_cli_reference_needs_vcf(args, capsys):
    with pytest.raises(SystemExit) as e:
        cli.main(["variants", *args, "x.bam"])
    assert e.value.code == 2
    assert "--reference" in capsys.readouterr().err


# ------------------------------------------------------------------------------------------------- ABI
def test_abi_entry_points_refuse_bad_arguments():
    lib = _ffi.load()
    for name in ("kdl_variant_ref_count", "kdl_variant_ref_scatter", "kdl_deletion_scratch_words",
                 "kdl_deletion_count", "kdl_deletion_scatter"):
        assert name in _ffi.EXPORTED_SYMBOLS and getattr(lib, name)
    assert lib.kdl_deletion_scratch_words(0) == 1 and lib.kdl_deletion_scratch_words(256) == 2
    assert lib.kdl_deletion_scratch_words(257) == 3
    buf = np.zeros(19 * 8, dtype=np.int32)
    cs, cl = np.zeros(1, dtype=np.int64), np.full(1, 4, dtype=np.int32)
    ref = np.zeros(16, dtype=np.uint8)
    sums = np.zeros(4, dtype=np.uint32)
    out = np.zeros(64, dtype=np.int64)

    def count(n_slots, r=ref.ctypes.data, abs_floor=1):
        return lib.kdl_variant_ref_count(buf.ctypes.data, n_slots, cs.ctypes.data, cl.ctypes.data, 1, r, abs_floor,
                                         0.01, sums.ctypes.data, None)

    def scatter(n_slots, n_sites, r=ref.ctypes.data):
        return lib.kdl_variant_ref_scatter(buf.ctypes.data, n_slots, cs.ctypes.data, cl.ctypes.data, 1, r, 1, 0.01,
                                           sums.ctypes.data, n_sites, out.ctypes.data, out.ctypes.data,
                                           out.ctypes.data, out.ctypes.data, None)

    for rc in (count(6), count(0), count(8, r=None), count(8, r=ref.ctypes.data + 1), count(8, abs_floor=-2),
               scatter(8, -1), scatter(8, 9), scatter(8, 1, r=None)):
        assert rc == 1
    bad = _ffi.KdlBatch()
    bad.n_reads = -1
    import ctypes as C

    assert lib.kdl_deletion_count(C.byref(bad), sums.ctypes.data, None) == 1
    assert lib.kdl_deletion_scatter(C.byref(bad), sums.ctypes.data, 0, None, None, None) == 1
