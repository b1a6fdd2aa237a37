"""`variants --vcf` with its options together, without a GPU: base and read filters, primers, reference and strand on
one corpus (tests/vcf_combo_cases.py) against one composed oracle (oracle/py_cvoracle.py).

- The oracle is pinned: unmasked it writes the records of py_voracle, py_rvoracle and py_soracle; masked, its tables
  and insertion dicts are those of the C quality walk (oracle/kindel_qoracle.c) fed py_poracle's primer bases.
- The emulated kernel chain K9, K0 + K1 (+ K1e / K1g), K1q, then K8 over the reverse bytes and the same pileup gives
  the oracle's total and reverse tables, and K8's sub-batch carries the merged mask list.
- The product's own `variants_vcf` -- decode, PileupRun, reverse_table, device_tables, the engine's Python -- runs
  with every kdl_* entry point taken from the kernel emulator, and its text equals the oracle's byte for byte over a
  pairwise-covering option matrix, over every combination of the four masking inputs, and from host tables (the
  multi-GPU result, re-uploaded and masked again by device_tables).
- Every rank of a sharded run masks its own shard, and the shard tables add up to the oracle's."""
import contextlib
import dataclasses
import os
import types

import numpy as np
import pytest
import torch

import emu_harness as E
import helpers as H
import primer_cases as PC
import strand_cases as S
import vcf_combo_cases as VC
from kindel_b200 import __version__, _ffi, bamio, distributed, engine
from kindel_b200 import kindel as K
from kindel_b200 import primers as P
from kindel_b200.insertions import InsertionTable
from oracle import coracle, py_cvoracle as CV, py_poracle as PO, py_rvoracle as RV, py_soracle as SO
from oracle import py_voracle as V
from oracle import samdecode

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
SOURCE = "kindel {}".format(__version__)
INPUTS = os.path.join(H.ROOT, "tests", "golden", "inputs")


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("vcf_combo")
    bam, sam, fa, bed, contigs, recs, refs, rows = VC.write(d)
    return dict(bam=str(bam), sam=str(sam), fa=str(fa), bed=str(bed), contigs=contigs, recs=recs, refs=refs, rows=rows,
                dir=d, composed={})


def composed(corpus, bq, mq, ex, primers):
    key = (bq, mq, ex, primers)
    if key not in corpus["composed"]:
        corpus["composed"][key] = CV.Composed(corpus["bam"], bq, mq, ex, corpus["rows"] if primers else None)
    return corpus["composed"][key]


def oracle_text(corpus, row, stats=None):
    bq, mq, ex, pr, ref, strand, (a, r) = row
    return composed(corpus, bq, mq, ex, pr).vcf(
        SOURCE, a, r, (bq, mq, ex), os.path.basename(corpus["bed"]) if pr else None,
        (os.path.basename(corpus["fa"]), corpus["refs"]) if ref else None, strand != "off",
        strand if isinstance(strand, float) else None, stats)


def laid_out(batch, tables):
    """The oracle's per-contig columns [(name, cols, ...)] as one table [19, n_slots] over the batch's slots."""
    out = np.zeros((19, int(batch.n_slots)), dtype=np.int32)
    for c, (nm, cols, _) in enumerate(tables):
        assert nm == batch.contig_names[c]
        s0 = int(batch.contig_slot[c])
        out[:, s0:s0 + len(cols[0])] = np.array(cols, dtype=np.int32)
    return out


def _body(text):
    return [ln for ln in text.splitlines() if not ln.startswith("#")]


# ------------------------------------------------------------------------------------------- oracle pins
def _groups(path):
    _, records = samdecode.read_alignment_file(path)
    out = {}
    for rec in records:
        out.setdefault(rec.rname, []).append(rec)
    out.pop("*", None)
    return out


def test_unmasked_oracle_equals_the_single_option_oracles(corpus, tmp_path):
    """No filter, no primer: the data lines are py_voracle's (over the C oracle's table), py_rvoracle's and
    py_soracle's, with and without strand, on fixtures, the strand truth set and this corpus."""
    bam, fa, ref, _ = S.write(tmp_path)
    cases = [(os.path.join(INPUTS, "mm2_gp120.bam"), os.path.join(INPUTS, "hxb2-gp120-mutated.fa")),
             (os.path.join(INPUTS, "bwa_1_1.bam"), None), (str(bam), str(fa)), (corpus["bam"], corpus["fa"])]
    n = 0
    for path, fasta in cases:
        batch = bamio.read_alignment(path)
        groups = _groups(path)
        oracle = CV.Composed(path)
        assert [nm for nm, _ in oracle.contigs] == batch.contig_names
        table, _ = coracle.pileup(batch)
        texts = None
        if fasta:
            from kindel_b200.reference import load_reference
            codes = load_reference(fasta, batch).codes
            texts = {nm: "".join("ACGTN"[x] for x in codes[s0:s0 + L].tolist()) for nm, s0, L in
                     zip(batch.contig_names, batch.contig_slot.tolist(), batch.contig_len.tolist())}
        for a, r, max_sor in ((1, 0.01, None), (0, 0.0, 3.0), (2, 0.2, 1.5)):
            sites = V.sites(table, batch.contig_slot, batch.contig_len, a, r)
            assert _body(oracle.vcf(SOURCE, a, r)) == V.vcf_records(batch.contig_names, batch.contig_slot, *sites, a, r)
            plain = [(nm, L, groups.get(nm, [])) for nm, L in zip(batch.contig_names, batch.contig_len.tolist())]
            got = _body(oracle.vcf(SOURCE, a, r, max_sor=max_sor, strand=True))
            assert got == SO.vcf_lines(plain, a, r, max_sor), (path, a, r)
            n += len(got)
            if texts:
                with_ref = [(nm, texts[nm], groups.get(nm, [])) for nm in batch.contig_names]
                assert _body(oracle.vcf(SOURCE, a, r, reference=("x.fa", texts))) == RV.vcf_lines(with_ref, a, r)
                assert _body(oracle.vcf(SOURCE, a, r, reference=("x.fa", texts), strand=True, max_sor=max_sor)) == \
                    SO.vcf_lines(with_ref, a, r, max_sor, reference=True)
    assert n > 500


def _c_walk(corpus, tmp_path, bq, mq, ex, primers):
    """(batch, counts, {slot: {string: count}}) of the C quality walk over the corpus with the records that the record
    filters drop rewritten as unmapped, fed py_poracle's primer bases; inserted strings rendered from SEQ and QUAL."""
    recs = [r[:2] + (r[2] | 4,) + r[3:] if r[6] < mq or r[2] & ex else r for r in corpus["recs"]]
    path = tmp_path / "rewritten.bam"
    bamio.write_bam(str(path), corpus["contigs"], recs)
    batch = bamio.read_alignment(path)
    by_name = {nm: [] for nm in batch.contig_names}
    for r in recs:
        if not r[2] & 4 and len(r[4]) > 1:
            by_name[corpus["contigs"][r[0]][0]].append(r)
    reads = [r for nm in batch.contig_names for r in by_name[nm]]
    qual = np.frombuffer(b"".join(b"\xff" * len(r[4]) if r[7] is None else r[7] for r in reads), dtype=np.uint8)
    prim = PO.masked_by_read(str(path), batch.contig_names, corpus["rows"]) if primers else [[]] * len(reads)
    counts, events = PO.pileup(batch, prim, qual, bq)
    ins = {}
    for slot, read, q0, n in events.tolist():
        seq, q = reads[read][4].upper(), reads[read][7]
        s = "".join("N" if q is not None and q[k] < bq else seq[k] for k in range(q0, min(q0 + n, len(seq))))
        d = ins.setdefault(slot, {})
        d[s] = d.get(s, 0) + 1
    return batch, counts, ins


def test_masked_oracle_equals_the_c_quality_walk(corpus, tmp_path):
    """Two independent masked walks agree: the composed oracle's 19 columns and insertion dicts (first-seen order
    included) == oracle/kindel_qoracle.c fed py_poracle.quality_vector, at every combination of the masking inputs."""
    masked_strings = 0
    for bq, mq, ex, pr, _, _, _ in VC.masking_product():
        batch, counts, ins = _c_walk(corpus, tmp_path, bq, mq, ex, pr)
        oracle = composed(corpus, bq, mq, ex, pr)
        tables = oracle.tables()
        np.testing.assert_array_equal(laid_out(batch, tables), counts, err_msg=str((bq, mq, ex, pr)))
        got = {}
        for c, (_, _, dicts) in enumerate(tables):
            for p, d in enumerate(dicts):
                if d:
                    got[int(batch.contig_slot[c]) + p] = d
        assert {s: list(d.items()) for s, d in got.items()} == {s: list(d.items()) for s, d in ins.items()}
        masked_strings += sum("N" in s for d in got.values() for s in d)
    assert masked_strings > 10


# ------------------------------------------------------------------------------------------- the emulated device
def on_the_emulator(monkeypatch):
    """Point the engine at the kernel emulator: every kdl_* call of engine.py runs the CUDA source on the host, over
    CPU tensors (the decoders keep the real library).  The upload copies seq4, because K9 writes it in place and a device upload is a copy too."""
    lib = E.load()
    lib.emu_set_sm_count(E.SM_COUNT)
    cpu = torch.device("cpu")
    upload = engine.upload
    emu_ffi = types.ModuleType("emu_ffi")  # the engine's _ffi, loading the emulator's library
    emu_ffi.__dict__.update(vars(_ffi))
    emu_ffi.load = lambda: lib
    monkeypatch.setattr(engine, "_ffi", emu_ffi)
    monkeypatch.setattr(engine, "require_cuda", lambda device=None: cpu)
    monkeypatch.setattr(engine, "_stream_ptr", lambda device: None)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    monkeypatch.setattr(engine, "upload", lambda host, device=None, non_blocking=False: upload(
        dataclasses.replace(host, seq4=np.array(host.seq4, dtype=np.uint32, copy=True)), cpu))


@needs_emu
def test_emulated_chain_equals_the_oracle_tables(corpus):
    """K9 (primer_cases.emu_primers), then the pileup and K1q, give the oracle's total; K8 over the masked batch's
    reverse bytes gives bamio.select_reads of the masked host batch -- the merged mask list, not the decode one -- and
    its pileup and K1q give the oracle's reverse table.  Both with all 19 columns."""
    n_primer_listed = 0
    for bq, mq, ex, pr, _, _, _ in VC.masking_product():
        batch = bamio.read_alignment(corpus["bam"], min_mapq=mq, exclude_flags=ex, min_base_quality=bq, strand=True)
        masked = batch
        if pr:
            masked, tot = PC.emu_primers(batch, PC.arrays_for(batch, corpus["rows"]))
            n_primer_listed += int(tot[3])
            assert masked.n_masked > batch.n_masked
        oracle = composed(corpus, bq, mq, ex, pr)
        counts, events = E.pileup_pipeline(masked)
        np.testing.assert_array_equal(E.unmask(masked, counts), laid_out(batch, oracle.tables(0)))
        keep = masked.reverse
        got = E.select(masked, keep)
        want = bamio.select_reads(masked, np.flatnonzero(keep))
        S.assert_equal(got, S.fields(want), (bq, mq, ex, pr))
        sub = dataclasses.replace(want, **{f: got[f] for f in ("ref_start", "seq_off", "l_seq", "seq4",
                                                                "contig_read_off", "complex_idx", "hard_idx",
                                                                "mask_read", "mask_off", "mask_qpos")})
        rev, _ = E.pileup_pipeline(sub)
        np.testing.assert_array_equal(E.unmask(sub, rev), laid_out(batch, oracle.tables(2)), err_msg=str((bq, pr)))
        # the strings the VCF groups by: the host's InsertionTable over the product's decode
        table = InsertionTable(batch, events)
        for c, (_, _, dicts) in enumerate(oracle.tables(0)):
            for p, d in enumerate(dicts):
                if d:
                    assert list(table.dict_at(int(batch.contig_slot[c]) + p).items()) == list(d.items())
    assert n_primer_listed > 1000


def _kwargs(corpus, row):
    bq, mq, ex, pr, ref, strand, _ = row
    return dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, primers=corpus["bed"] if pr else None,
                reference=corpus["fa"] if ref else None, strand=strand != "off",
                max_sor=strand if isinstance(strand, float) else None)


def test_option_matrix_covers_every_pair():
    rows = VC.option_matrix()
    assert len(rows) <= 16
    for i in range(len(VC.LEVELS)):
        for j in range(i + 1, len(VC.LEVELS)):
            assert {(r[i], r[j]) for r in rows} == {(a, b) for a in VC.LEVELS[i][1] for b in VC.LEVELS[j][1]}


@needs_emu
def test_variants_vcf_on_the_emulator_equals_the_oracle(corpus, monkeypatch):
    """K.variants_vcf -- the whole product path, its kernels emulated -- == the composed oracle's text, header included,
    over the pairwise option matrix and over every combination of the four masking inputs with everything else on."""
    on_the_emulator(monkeypatch)
    n = 0
    for row in VC.option_matrix() + VC.masking_product():
        path = corpus["sam"] if n % 3 == 2 else corpus["bam"]
        got = K.variants_vcf(path, *row[6], **_kwargs(corpus, row))
        want = oracle_text(corpus, row)
        assert got == want, row
        n += 1


def _sharded_tables(batch, primers, world, plan, tmp_path):
    """Every rank's shard (distributed.shard_indices), masked by the primer arrays as the ranks receive them (saved
    beside the batch and loaded again) and piled on the emulated engine: (the ranks' summed counts, merged events)."""
    total, evs, idx_all = None, [], []
    arrays = None
    if primers is not None:
        pth = str(tmp_path / "primers.npz")
        P.save_arrays(pth, P.primer_arrays(primers, batch.contig_names, batch.contig_len))
        arrays = P.load_arrays(pth)
    for rank in range(world):
        idx = distributed.shard_indices(batch, rank, world, plan)
        db = engine.upload(bamio.select_reads(batch, idx))
        if arrays is not None:
            db = engine.mask_primers(db, arrays)
        counts, events = engine.pileup(db)
        total = counts.numpy().astype(np.int64) if total is None else total + counts.numpy()
        evs.append(events.numpy())
        idx_all.append(idx)
    return total.astype(np.int32), distributed.merge_events(evs, idx_all)


@needs_emu
def test_shards_mask_their_own_reads(corpus, monkeypatch, tmp_path):
    """Each rank masks its own shard: the shard tables add up to the oracle's masked table, for 2 and 3 ranks and both
    plans, and host tables (the multi-GPU result) give the oracle's VCF -- device_tables re-uploads the batch and masks
    its primer bases again, and the reverse table comes from that copy."""
    on_the_emulator(monkeypatch)
    ps = P.load_primers(corpus["bed"])
    for row in (VC.masking_product()[-1], (20, 0, 0x500, True, False, "on", (0, 0)),
                (20, 30, 0, True, True, "on", (2, 0.2))):
        bq, mq, ex, pr, ref, strand, (a, r) = row
        batch = bamio.read_alignment(corpus["bam"], min_mapq=mq, exclude_flags=ex, min_base_quality=bq, strand=True)
        oracle = composed(corpus, bq, mq, ex, pr)
        for world, plan in ((2, "reads"), (3, "reads"), (2, "contigs")):
            counts, events = _sharded_tables(batch, ps, world, plan, tmp_path)
            np.testing.assert_array_equal(counts, laid_out(batch, oracle.tables(0)), err_msg=str((row, world, plan)))
        run = K.PileupRun.from_host_tables(batch, counts, E.derive(counts), events, primers=ps)
        got = K.variants_vcf_from_run(run, a, r, (bq, mq, ex), reference=corpus["fa"] if ref else None,
                                      strand=True, max_sor=strand if isinstance(strand, float) else None)
        assert got == oracle_text(corpus, row), row


@needs_emu
def test_a_masked_exotic_base_raises_nothing(monkeypatch, tmp_path):
    """One read with a low-quality R in an M op and a low-quality Y in a soft clip: masked, the VCF equals the
    oracle's; unmasked, the product and the oracle both raise the same KeyError."""
    on_the_emulator(monkeypatch)
    bam, sam, fa, bed, contigs, recs, refs, rows = VC.write(tmp_path, exotic=True)
    row = (20, 0, 0, True, True, 3.0, (1, 0.01))
    want = CV.Composed(str(bam), 20, 0, 0, rows).vcf(SOURCE, 1, 0.01, (20, 0, 0), bed.name, (fa.name, refs), True, 3.0)
    corpus = dict(bed=str(bed), fa=str(fa))
    assert K.variants_vcf(str(bam), 1, 0.01, **_kwargs(corpus, row)) == want
    with pytest.raises(KeyError) as oracle_exc:
        CV.Composed(str(bam), 0, 0, 0, rows)
    with pytest.raises(KeyError) as product_exc:
        K.variants_vcf(str(bam), 1, 0.01, **_kwargs(corpus, (0,) + row[1:]))
    assert product_exc.value.args == oracle_exc.value.args


# ------------------------------------------------------------------------------------------- the corpus
def test_corpus_is_not_vacuous(corpus):
    """Over the option matrix: masking changes a record's line and removes a record; the indel strand clamp
    max(DP_s - AO_s, 0) is hit; FILTER sor is set; an insertion string holds a masked N; a site lies on a contig that
    follows an all-filtered contig.  And the shapes the corpus is for are there."""
    seen = dict(changed=0, removed=0, clamp=0, sor=0, masked_n=0, after_filtered=0)
    for row in VC.option_matrix() + VC.masking_product():
        stats = {}
        text = oracle_text(corpus, row, stats)
        seen["clamp"] += stats.get("clamp", 0)
        body = _body(text)
        seen["sor"] += sum(ln.split("\t")[6] == "sor" for ln in body)
        bq, mq, ex, pr = row[:4]
        seen["masked_n"] += composed(corpus, bq, mq, ex, pr).piles["main"][0].masked_n_inserts
        if bq or pr:
            plain = {tuple(ln.split("\t")[:5]): ln for ln in _body(oracle_text(corpus, (0, mq, ex, False) + row[4:]))}
            mine = {tuple(ln.split("\t")[:5]): ln for ln in body}
            seen["removed"] += len(set(plain) - set(mine))
            seen["changed"] += sum(plain[k] != v for k, v in mine.items() if k in plain)
        if mq >= 30:
            names = [nm for nm, _ in composed(corpus, bq, mq, ex, pr).contigs]
            assert composed(corpus, bq, mq, ex, pr).piles["lowmq"][0].depth(40) == 0
            later = set(names[names.index("lowmq") + 1:])
            seen["after_filtered"] += sum(ln.split("\t")[0] in later for ln in body)
    assert all(seen.values()), seen
    batch = bamio.read_alignment(corpus["bam"], min_mapq=30, strand=True)
    assert "lowmq" in batch.contig_names and "nohits" not in batch.contig_names
    c = batch.contig_names.index("lowmq")
    assert batch.contig_read_off[c] == batch.contig_read_off[c + 1]
    assert [nm for nm, _ in corpus["contigs"]] != batch.contig_names
    tiny = [batch.contig_names.index(nm) for nm, _ in VC.TINY]
    assert len({int(batch.contig_slot[t]) // 512 for t in tiny}) == 1
    assert {1, 2, 513} <= set(batch.contig_len.tolist()) and 0 < batch.reverse.mean() < 1
    flags = {r[2] for r in corpus["recs"]}
    assert any(f & 0x400 for f in flags) and any(f & 0x100 for f in flags)
    assert any(r[7] is None for r in corpus["recs"]) and 200 < len(corpus["recs"]) < 5000
    assert any(ch not in "ACGT" for ch in corpus["refs"]["edge"])
