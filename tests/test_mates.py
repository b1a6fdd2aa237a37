"""`--mask-overlaps` without a GPU: the mates' decode, K10p / K10 / K10u under the kernel emulator against the
independent restatement oracle/py_moracle.py, and the product's own Python over the emulated kernels."""
import contextlib
import dataclasses
import os
import types

import numpy as np
import pytest
import torch

import emu_harness as E
import mate_cases as MC
from kindel_b200 import __version__, _ffi, bamio, cli, distributed, engine, synth
from kindel_b200 import kindel as K
from oracle import coracle, py_oracle
from oracle import py_moracle as MO

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("mates")
    sam = MC.lattice_sam(str(d / "lattice.sam"))
    b = bamio.read_alignment(sam, mates=True)
    bam = str(d / "lattice.bam")
    # the same records as BAM (QNAME, RNEXT, PNEXT from the text)
    recs = []
    with open(sam) as fh:
        names = {"c0": 0, "c1": 1}
        for line in fh:
            if line.startswith("@"):
                continue
            f = line.rstrip("\n").split("\t")
            rn = names[f[2]] if f[6] == "=" else names.get(f[6], -1)
            recs.append((names[f[2]], int(f[3]) - 1, int(f[1]), bamio.parse_cigar_text(f[5]), f[9], f[0], int(f[4]),
                         None if f[10] == "*" else bytes(ord(c) - 33 for c in f[10]), rn, int(f[7]) - 1))
    bamio.write_bam(bam, [("c0", MC.L), ("c1", 100)], recs)
    pbam = MC.paired_bam(str(d / "pairs.bam"))
    return dict(sam=sam, bam=bam, pairs=pbam, dir=d, batch=b)


# ------------------------------------------------------------------------------------------------ decode
def test_fnv1a_is_the_reference_hash():
    assert bamio.name_hash("") == 0xCBF29CE484222325
    assert bamio.name_hash("a") == 0xAF63DC4C8601EC8C
    assert bamio.name_hash(b"foobar") == 0x85944171F73967E8


@pytest.mark.parametrize("which", ["bam", "sam_cpp", "sam_py"])
def test_decoders_give_the_mates(files, which):
    path = files["bam"] if which == "bam" else files["sam"]
    b = bamio.read_sam(path, mates=True) if which == "sam_py" else bamio.read_bam(path, mates=True)
    lengths, recs = MO.kept(files["sam"], b.contig_names)
    assert [bamio.name_hash(qn) for _, _, qn, _, _ in recs] == b.name_hash.tolist()
    assert [ro for _, _, _, ro, _ in recs] == b.pair_role.tolist()
    assert [pn for _, _, _, _, pn in recs] == b.mate_start.tolist()
    roles = dict(zip([qn for _, _, qn, _, _ in recs], b.pair_role.tolist()))
    assert roles["twoContigs"] == 0 and roles["disjoint"] in (1, 2)


def test_role_rule():
    assert bamio.pair_role(0x1 | 0x40, True) == 1 and bamio.pair_role(0x1 | 0x80, True) == 2
    for flag in (0x40, 0x1 | 0x40 | 0x8, 0x1 | 0x40 | 0x100, 0x1 | 0x40 | 0x800, 0x1, 0x1 | 0x40 | 0x80):
        assert bamio.pair_role(flag, True) == 0
    assert bamio.pair_role(0x1 | 0x40, False) == 0


def test_off_decodes_nothing(files):
    b = bamio.read_alignment(files["bam"])
    assert b.mates is None and b.name_hash is None
    assert bamio.read_sam(files["sam"]).mates is None


def test_batches_carry_the_mates(files, tmp_path):
    b = files["batch"]
    sub = bamio.select_reads(b, [3, 1, 4])
    assert sub.name_hash.tolist() == b.name_hash[[3, 1, 4]].tolist()  # (the given order inside a contig)
    m = bamio.merge_batches([sub, bamio.select_reads(b, [0, 2])])
    assert sorted(m.name_hash.tolist()) == sorted(b.name_hash[:5].tolist())
    bamio.save_batch(str(tmp_path / "b"), b)
    back = bamio.load_batch(str(tmp_path / "b"))
    for f in ("name_hash", "mate_start", "pair_role"):
        assert np.array_equal(getattr(back, f), getattr(b, f))
    bamio.save_batch(str(tmp_path / "b"), bamio.read_alignment(files["bam"]))
    assert bamio.load_batch(str(tmp_path / "b")).mates is None


def test_write_bam_default_records_are_unchanged(tmp_path):
    recs = [(0, 5, 0, [10 << 4], "ACGTACGTAC"), (0, 7, 16, [10 << 4], "ACGTACGTAC", "x", 30, None, None, None)]
    bamio.write_bam(str(tmp_path / "a.bam"), [("c", 50)], recs[:1] + [recs[1][:7]])
    bamio.write_bam(str(tmp_path / "b.bam"), [("c", 50)], recs)
    assert open(tmp_path / "a.bam", "rb").read() == open(tmp_path / "b.bam", "rb").read()


# ------------------------------------------------------------------------------------------------ K10p
def _oracle_mate(path, b, **filters):
    lengths, recs = MO.kept(path, b.contig_names, **filters)
    want = np.full(b.n_reads, -1)
    for r2, r1 in MO.pairs(lengths, recs).items():
        want[r2] = r1
    return want


@needs_emu
def test_k10p_planted_cases(files):
    b = files["batch"]
    _, _, _, mate = MC.emu_overlaps(b)
    want = _oracle_mate(files["sam"], b)
    assert mate.tolist() == want.tolist()
    names = [qn for _, _, qn, _, _ in MO.kept(files["sam"], b.contig_names)[1]]
    paired = {qn for k, qn in enumerate(names) if mate[k] >= 0 or (mate == k).any()}
    for qn in ("disjoint", "abut", "partial", "contained", "same", "r2left", "delPast", "clips", "supp"):
        assert qn in paired, qn
    for qn in ("three", "twoR1", "offby1", "hard", "lone", "twoContigs"):
        assert qn not in paired, qn
    # file order of the mates does not matter (`partial` is written R2 first), nor the order inside a hash group
    idx = np.flatnonzero(b.pair_role)
    order = idx[np.lexsort((-idx, b.name_hash[idx]))]
    assert MC.emu_overlaps(b, order=order)[3].tolist() == mate.tolist()


@needs_emu
def test_k10p_a_mate_filtered_by_mapq_leaves_a_singleton(files):
    b = bamio.read_alignment(files["sam"], mates=True, min_mapq=30)
    mate = MC.emu_overlaps(b)[3]
    assert mate.tolist() == _oracle_mate(files["sam"], b, min_mapq=30).tolist()
    names = [qn for _, _, qn, _, _ in MO.kept(files["sam"], b.contig_names, min_mapq=30)[1]]
    assert mate[names.index("lowmapq")] == -1


@needs_emu
def test_k10p_planted_hash_collision_leaves_the_group_alone(files):
    """Two names that hash alike are one group on the device: a collision planted through the ABI makes two proper
    pairs a group of four, which stays unpaired (the one known gap of pairing by hash, DESIGN.md)."""
    b = files["batch"]
    names = [qn for _, _, qn, _, _ in MO.kept(files["sam"], b.contig_names)[1]]
    h = b.name_hash.copy()
    h[[k for k, qn in enumerate(names) if qn == "same"]] = h[names.index("partial")]
    mate = MC.emu_overlaps(dataclasses.replace(b, name_hash=h))[3]
    for qn in ("same", "partial"):
        assert all(mate[k] == -1 and not (mate == k).any() for k, x in enumerate(names) if x == qn)
    assert mate[names.index("disjoint")] >= 0 or (mate == names.index("disjoint")).any()


# ------------------------------------------------------------------------------------------------ K10 + pileup + K10u
def _check_tables(path, mbq=0, mapq=0):
    b = bamio.read_alignment(path, mates=True, min_base_quality=mbq, min_mapq=mapq)
    plain = bamio.read_alignment(path, min_mapq=mapq)
    counts, events, drops, tot, mate, masked = MC.emu_tables(b)
    o = MO.Masked(path, b.contig_names, min_mapq=mapq, pre_masked=MC.mask_lists(b))
    assert MC.mask_lists(masked) == o.masked()
    assert tuple(int(x) for x in tot[3:7]) == o.stats()
    want, wev = o.pileup(plain, dict(zip(b.contig_names, b.contig_slot.tolist())))
    np.testing.assert_array_equal(counts, want)
    np.testing.assert_array_equal(events, wev)
    return b, counts, mate, drops, o


def _sam_with_quals(files, seed=3):
    rng = np.random.default_rng(seed)
    out = []
    for line in open(files["sam"]).read().splitlines():
        f = line.split("\t")
        if not line.startswith("@") and f[10] == "*":
            f[10] = "".join(chr(33 + int(q)) for q in rng.choice([5, 30, 40], len(f[9]), p=[.15, .45, .4]))
        out.append("\t".join(f))
    p = files["dir"] / "quals.sam"
    p.write_text("\n".join(out) + "\n")
    return str(p)


@needs_emu
@pytest.mark.parametrize("schedule", ["forward", "reverse", "random"])
def test_k10_lattice_against_the_oracle(files, schedule):
    E.set_schedule(schedule, 7)
    try:
        b, counts, mate, drops, o = _check_tables(files["sam"])
        assert o.stats()[2] >= 2 and o.stats()[3] >= 2  # dropped deletions and insertions
        _check_tables(_sam_with_quals(files), mbq=20)
        _check_tables(files["sam"], mapq=30)
    finally:
        E.set_schedule("forward")


@needs_emu
@pytest.mark.parametrize("seed", [1, 2])
def test_k10_synthetic_pairs_against_the_oracle(files, seed):
    path = MC.paired_bam(str(files["dir"] / ("p%d.bam" % seed)), seed=seed, contig_lens=(2500, 1800), depth=25)
    _, _, _, _, o = _check_tables(path)
    assert o.stats()[0] > 100 and o.stats()[2] > 0 and o.stats()[3] > 0


@needs_emu
def test_k10_invariant_per_pair_and_position(files):
    """Per pair and position, the counts the pair adds to columns 0-3 and 5 and its insertion events: at most one.
    (These mates have no N base and no mask, and both read a fragment's indel alike, so none of the exceptions at the
    edges of R1's information -- DESIGN.md section 1 -- arises.)"""
    b = bamio.read_alignment(files["pairs"], mates=True)
    masked, drops, tot, mate = MC.emu_overlaps(b)
    for r2 in np.flatnonzero(mate >= 0)[:200]:
        r1 = int(mate[r2])
        sub = bamio.select_reads(masked, [r1, r2])
        t, ev = E.pileup_pipeline(sub)
        E.unmask(sub, t)
        mine = drops[drops[:, 2] == r2].copy()
        mine[:, 2] = 1
        MC.untake(mine, t)
        assert (t[0:4].sum(axis=0) + t[5] <= 1).all(), (r1, r2)
        assert (t[6] <= 1).all()


# ------------------------------------------------------------------------------------------------ the product's Python
def on_the_emulator(monkeypatch):
    """The engine's kdl_* calls on the kernel emulator, over CPU tensors (the upload copies seq4: K9 and K10 write
    it in place, as on the device)."""
    lib = E.load()
    lib.emu_set_sm_count(E.SM_COUNT)
    cpu = torch.device("cpu")
    upload = engine.upload
    emu_ffi = types.ModuleType("emu_ffi")
    emu_ffi.__dict__.update(vars(_ffi))
    emu_ffi.load = lambda: lib
    monkeypatch.setattr(engine, "_ffi", emu_ffi)
    monkeypatch.setattr(engine, "require_cuda", lambda device=None: cpu)
    monkeypatch.setattr(engine, "_stream_ptr", lambda device: None)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    monkeypatch.setattr(engine, "upload", lambda host, device=None, non_blocking=False: upload(
        dataclasses.replace(host, seq4=np.array(host.seq4, dtype=np.uint32, copy=True)), cpu))


@needs_emu
def test_product_run_equals_the_oracle(files, monkeypatch):
    on_the_emulator(monkeypatch)
    for path in (files["sam"], files["pairs"]):
        run, _ = K.pileup_run(path, strand=True, mask_overlaps=True)
        b = run.batch
        o = MO.Masked(path, b.contig_names)
        want, wev = o.pileup(bamio.read_alignment(path), dict(zip(b.contig_names, b.contig_slot.tolist())))
        np.testing.assert_array_equal(run.host_counts, want)
        got_ev = run.ins_table.events
        want_ev = wev[np.argsort(wev[:, 0], kind="stable")]
        np.testing.assert_array_equal(got_ev, want_ev)
        assert run.overlap_stats == o.stats()
        # the reverse table: its drops are those of reverse R2s; forward + reverse adds up
        rev, sub = run.reverse_table()
        keep = np.flatnonzero(b.reverse)
        o_rev = _reverse_oracle(o, b, keep, path)
        np.testing.assert_array_equal(rev.numpy(), o_rev)


def _reverse_oracle(o, b, keep, path):
    """The oracle's table of the reverse reads alone: the same masks and drops, restricted to them."""
    plain = bamio.select_reads(bamio.read_alignment(path), keep)
    sub = MO.Masked.__new__(MO.Masked)
    sub.recs = [o.recs[k] for k in keep]
    sub.pre = [o.pre[k] for k in keep]
    sub.bases = [o.bases[k] for k in keep]
    pos = {int(k): j for j, k in enumerate(keep)}
    sub.dels = {pos[r]: v for r, v in o.dels.items() if r in pos}
    sub.ins = {pos[r]: v for r, v in o.ins.items() if r in pos}
    sub.mate = {}
    ins_ops = [sum(1 for _, op in MO._ops(x[1]) if op == 1) for x in sub.recs]
    sub.evt_off = np.concatenate(([0], np.cumsum(ins_ops))).astype(np.int64)
    return sub.pileup(plain, dict(zip(b.contig_names, b.contig_slot.tolist())))[0]


@needs_emu
def test_vcf_and_report_of_the_product(files, monkeypatch):
    on_the_emulator(monkeypatch)
    path = files["pairs"]
    fa = str(files["dir"] / "ref.fa")
    b = bamio.read_alignment(path)
    rng = np.random.default_rng(0)
    with open(fa, "w") as fh:
        for nm, L in zip(b.contig_names, b.contig_len):
            fh.write(">%s\n%s\n" % (nm, "".join("ACGT"[x] for x in rng.integers(0, 4, int(L)))))
    off = K.variants_vcf(path, 0, 0.0, reference=fa, strand=True)
    assert off == K.variants_vcf(path, 0, 0.0, reference=fa, strand=True, mask_overlaps=False)
    on = K.variants_vcf(path, 0, 0.0, reference=fa, strand=True, mask_overlaps=True)
    assert "##kindelMateOverlaps=R2 masked where R1 covers" in on and "kindelMateOverlaps" not in off
    o = MO.Masked(path, b.contig_names)
    want, _ = o.pileup(b, dict(zip(b.contig_names, b.contig_slot.tolist())))
    n_rec = 0
    for line in on.splitlines():
        if line.startswith("#"):
            continue
        f = line.split("\t")
        info = dict(x.split("=") for x in f[7].split(";") if "=" in x)
        c = b.contig_names.index(f[0])
        if "INDEL" in f[7]:
            continue
        s = int(b.contig_slot[c]) + int(f[1]) - 1
        assert int(info["DP"]) == int(want[0:6, s].sum())
        adf, adr = ([int(x) for x in info[k].split(",")] for k in ("ADF", "ADR"))
        ad = [int(x) for x in info["AD"].split(",")]
        assert [x + y for x, y in zip(adf, adr)] == ad
        n_rec += 1
    assert n_rec > 0
    for line in on.splitlines():  # ADF[1] + ADR[1] == AO on the indel records
        if "INDEL" in line and not line.startswith("#"):
            info = dict(x.split("=") for x in line.split("\t")[7].split(";") if "=" in x)
            assert int(info["ADF"].split(",")[1]) + int(info["ADR"].split(",")[1]) == int(info["AO"])
    res_on = K.bam_to_consensus(path, mask_overlaps=True)
    res_off = K.bam_to_consensus(path)
    rep = res_on.refs_reports[b.contig_names[0]]
    assert "- mate overlaps: %d pairs, %d bases, %d deletions, %d insertions masked" % o.stats() in rep
    assert "mate overlaps" not in res_off.refs_reports[b.contig_names[0]]
    assert K.bam_to_consensus(path, mask_overlaps=False).refs_reports == res_off.refs_reports


@needs_emu
@pytest.mark.parametrize("row", [(0, 0, 0, False, False), (20, 0, 0, True, False), (0, 30, 0x400, False, True),
                                 (20, 30, 0, True, True)])
def test_option_matrix_off_is_unchanged_and_on_is_stable(files, monkeypatch, row):
    """Over filters x primers x reference x strand: with mask_overlaps=False every output is the one without the
    keyword, and on it runs through every public entry point."""
    on_the_emulator(monkeypatch)
    bq, mq, ex, primers, strand = row
    path = files["pairs"]
    kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex)
    if primers:
        b = bamio.read_alignment(path)
        rows = synth.tiled_scheme(1, b.contig_names, [int(x) for x in b.contig_len])
        bed = files["dir"] / "s.bed"
        bed.write_text("".join("%s\t%d\t%d\n" % r for r in rows))
        kw["primers"] = str(bed)
    for fn, args in ((K.variants_vcf, dict(strand=strand)), (K.weights, {}), (K.features, {}), (K.variants, {})):
        a = fn(path, **kw, **args)
        b_ = fn(path, **kw, **args, mask_overlaps=False)
        if isinstance(a, str):
            assert a == b_
        else:
            assert a.equals(b_)
        fn(path, **kw, **args, mask_overlaps=True)
    c = K.bam_to_consensus(path, **kw)
    d = K.bam_to_consensus(path, **kw, mask_overlaps=False)
    assert [x.sequence for x in c.consensuses] == [x.sequence for x in d.consensuses]
    assert c.refs_reports == d.refs_reports
    K.bam_to_consensus(path, **kw, mask_overlaps=True)


@needs_emu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_ranks_add_up_to_one_gpu(files, monkeypatch, world):
    """Mates split across shards: the parent masks the whole batch once (K9, K10p, K10), every rank piles its shard
    of the masked host batch and takes back its own R2s' drop rows; the ranks' tables add up to one GPU's, and the
    merged events without the dropped rows are one GPU's insertion table."""
    on_the_emulator(monkeypatch)
    path = files["pairs"]
    batch = bamio.read_alignment(path, mates=True, strand=True)
    one = K.PileupRun(batch, mask_overlaps=True)
    shards, drops, _ = K._masked_for_shards(batch, None, True)
    for plan in ("reads", "contigs"):
        total, evs, idxs = 0, [], []
        for rank in range(world):
            idx = distributed.shard_indices(shards, rank, world, plan)
            db = engine.upload(bamio.select_reads(shards, idx))
            db = dataclasses.replace(db, drops=torch.from_numpy(distributed.shard_drops(drops, idx)))
            counts, events = engine.pileup(db)
            total = total + counts.numpy().astype(np.int64)
            evs.append(events.numpy())
            idxs.append(idx)
        np.testing.assert_array_equal(total, one.host_counts)
        dropped = np.sort(drops[drops[:, 3] >= 0, 3])
        host = K.PileupRun.from_host_tables(batch, total, one.host_derived, distributed.merge_events(evs, idxs),
                                            mask_overlaps=True, dropped_events=dropped)
        np.testing.assert_array_equal(host.ins_table.events, one.ins_table.events)


def test_cli_takes_mask_overlaps_on_every_pileup_command():
    parser = cli.build_parser()
    for cmd in (["consensus"], ["weights"], ["features"], ["variants"], ["variants", "--vcf", "--strand"]):
        a = parser.parse_args(cmd + ["x.bam", "--mask-overlaps", "--primers", "s.bed"])
        assert cli._filters(a)["mask_overlaps"] is True
        assert "mask_overlaps" not in cli._filters(parser.parse_args(cmd + ["x.bam"]))


def test_report_line():
    rep = K.build_report("c", K.DepthRange(1, 2), [], [], "x.bam", False, 1, 9, 0.1, False, False,
                         overlaps=(3, 40, 1, 2))
    assert "- mate overlaps: 3 pairs, 40 bases, 1 deletions, 2 insertions masked" in rep
    assert "mate overlaps" not in K.build_report("c", K.DepthRange(1, 2), [], [], "x.bam", False, 1, 9, 0.1, False,
                                                 False)


def test_synthetic_pairs_roundtrip(tmp_path):
    b, flag, frag = synth.paired_reads(4, [2000], 15, read_len=80, insert_mean=150, indel_frac=0.2)
    assert b.n_complex > 0 and (b.pair_role == 1).sum() == (b.pair_role == 2).sum() == b.n_reads // 2
    synth.write_paired_bam(str(tmp_path / "p.bam"), b, flag, frag)
    c = bamio.read_alignment(str(tmp_path / "p.bam"), mates=True, strand=True)
    for f in ("name_hash", "mate_start", "pair_role", "ref_start", "seq4", "l_seq", "reverse"):
        assert np.array_equal(getattr(c, f), getattr(b, f)), f
    a, aflag, afrag, rows = synth.amplicon_pairs(2, 3000, 20)
    lo = {a_ for _, a_, _ in rows[0::2]}
    hi = {b_ for _, _, b_ in rows[1::2]}
    for r in range(a.n_reads):  # each read starts at an amplicon start or ends at an amplicon end
        assert int(a.ref_start[r]) in lo or int(a.ref_start[r]) + int(a.seq_len[r]) in hi


# ------------------------------------------------------------------------------------------------ composed oracle
SOURCE = "kindel {}".format(__version__)


@pytest.fixture(scope="module")
def combo(tmp_path_factory):
    return MC.combo_files(tmp_path_factory.mktemp("mates_combo"))


def laid_out(batch, tables):
    """py_cvoracle-style per-contig tables as one int32 [19, n_slots] table in the batch's slot layout."""
    out = np.zeros((19, batch.n_slots), dtype=np.int32)
    for nm, cols, _ in tables:
        s = int(batch.contig_slot[batch.contig_names.index(nm)])
        out[:, s:s + len(cols[0])] = np.array(cols, dtype=np.int32)
    return out


def oracle_vcf(files, row):
    bq, mq, ex, pr, ref, strand, (a, r) = row
    o = MO.ComposedMates(files["bam"], bq, mq, ex, files["rows"] if pr else None)
    return o.vcf(SOURCE, a, r, (bq, mq, ex), os.path.basename(files["bed"]) if pr else None,
                 (os.path.basename(files["fa"]), files["refs"]) if ref else None, strand)


def product_vcf(path, files, row, **extra):
    bq, mq, ex, pr, ref, strand, (a, r) = row
    kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, strand=strand, mask_overlaps=True, **extra)
    if pr:
        kw["primers"] = files["bed"]
    if ref:
        kw["reference"] = files["fa"]
    return K.variants_vcf(path, a, r, **kw)


def test_composed_oracle_is_pinned_to_the_per_record_oracle(files):
    """ComposedMates' total table is Masked's (the C quality walk minus the drops) on the lattice, with and without
    the lattice's primer."""
    b = bamio.read_alignment(files["sam"])
    slots = dict(zip(b.contig_names, b.contig_slot.tolist()))
    want, _ = MO.Masked(files["sam"], b.contig_names).pileup(b, slots)
    np.testing.assert_array_equal(laid_out(b, MO.ComposedMates(files["sam"]).tables(0)), want)


def test_mate_oracle_without_pairs_is_the_plain_oracle(tmp_path):
    """On reads without pairs (no FLAG 0x1) py_moracle masks and drops nothing: its table and events are the C
    oracle's, and its weights and deletions py_oracle's."""
    b, _, _ = synth.paired_reads(3, [3000], 20, read_len=80, insert_mean=140, indel_frac=0.3)
    contigs, recs = synth.to_records(b)  # (FLAG 0 or 16: no read is paired)
    path = str(tmp_path / "single.bam")
    bamio.write_bam(path, contigs, recs)
    plain = bamio.read_alignment(path)
    o = MO.Masked(path, plain.contig_names)
    assert o.stats() == (0, 0, 0, 0)
    got, ev = o.pileup(plain, dict(zip(plain.contig_names, plain.contig_slot.tolist())))
    want, wev = coracle.pileup(plain)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(ev, wev)
    L, s0 = int(plain.contig_len[0]), int(plain.contig_slot[0])
    p = py_oracle.pileup(L, py_oracle.records_of(plain))
    for k, b_ in enumerate("ACGTN"):
        assert got[k, s0:s0 + L].tolist() == [w[b_] for w in p.weights]
    assert got[5, s0:s0 + L + 1].tolist() == list(p.deletions)


@needs_emu
def test_primer_masked_first_mate_covers_nothing(files, monkeypatch):
    """K9 runs before K10: where the first mate's bases are primer bases, the second mate's are counted.  The product
    run (every engine call emulated) equals the composed oracle with the lattice's primer, and `primerR1`'s second
    mate has counts inside the primer."""
    on_the_emulator(monkeypatch)
    bed = files["dir"] / "lattice.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in MC.PRIMERS))
    run, _ = K.pileup_run(files["sam"], primers=str(bed), mask_overlaps=True, strand=True)
    o = MO.ComposedMates(files["sam"], primer_rows=MC.PRIMERS)
    np.testing.assert_array_equal(run.host_counts, laid_out(run.batch, o.tables(0)))
    np.testing.assert_array_equal(run.reverse_table()[0].numpy(), laid_out(run.batch, o.tables(2)))
    assert run.overlap_stats == o.overlap_stats
    s0 = int(run.batch.contig_slot[0])
    plain = MO.ComposedMates(files["sam"])  # without the primer R1 covers [225, 240) and R2 is masked there
    assert (run.host_counts[0:4, s0 + 225:s0 + 240].sum(axis=0)
            > laid_out(run.batch, plain.tables(0))[0:4, s0 + 225:s0 + 240].sum(axis=0) - 2).all()


@needs_emu
def test_composed_vcf_matrix_emulated(combo, monkeypatch):
    """variants_vcf with mask_overlaps on -- decode, K9, K10p, K10, the pileup, K1q, K10u, K8's reverse table, K7's
    deletion groups with the drops subtracted, the insertion table without the dropped rows -- equals the composed
    oracle byte for byte, deletion AO and ADF / ADR included, over filters x primers x reference x strand, from BAM and
    from SAM text."""
    on_the_emulator(monkeypatch)
    n_indel = 0
    for k, row in enumerate(MC.mates_matrix()):
        want = oracle_vcf(combo, row)
        got = product_vcf(combo["sam"] if k % 3 == 2 else combo["bam"], combo, row)
        assert got == want, row
        n_indel += got.count("INDEL;")
    assert n_indel > 20


@needs_emu
def test_composed_vcf_from_host_tables(combo, monkeypatch):
    """The multi-GPU result: the parent masks once, two ranks pile their shards with their own drop rows, and the VCF
    of those host tables equals the composed oracle's."""
    on_the_emulator(monkeypatch)
    row = MC.mates_matrix()[-1]
    bq, mq, ex, pr, ref, strand, (a, r) = row
    batch = bamio.read_alignment(combo["bam"], min_base_quality=bq, min_mapq=mq, exclude_flags=ex, strand=True,
                                 mates=True)
    from kindel_b200 import primers as P

    ps = P.load_primers(combo["bed"])
    shards, drops, stats = K._masked_for_shards(batch, ps, True)
    total, evs, idxs = 0, [], []
    for rank in range(2):
        idx = distributed.shard_indices(shards, rank, 2, "reads")
        db = engine.upload(bamio.select_reads(shards, idx))
        db = dataclasses.replace(db, drops=torch.from_numpy(distributed.shard_drops(drops, idx)))
        counts, events = engine.pileup(db)
        total = total + counts.numpy().astype(np.int64)
        evs.append(events.numpy())
        idxs.append(idx)
    dropped = np.sort(drops[drops[:, 3] >= 0, 3])
    run = K.PileupRun.from_host_tables(batch, total, np.zeros((5, batch.n_slots), np.int32),
                                       distributed.merge_events(evs, idxs), primers=ps, mask_overlaps=True,
                                       dropped_events=dropped, overlap_stats=stats)
    assert run.overlap_stats == stats and run._device is None  # the REPORT's numbers need no re-upload
    got = K.variants_vcf_from_run(run, a, r, (bq, mq, ex), reference=combo["fa"], strand=strand)
    assert got == oracle_vcf(combo, row)
