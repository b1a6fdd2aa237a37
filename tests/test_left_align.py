"""`variants --vcf --reference --left-align` without a GPU: K15d / K15i on the kernel emulator against the left-aligning
oracle (oracle/py_laoracle.py), and the product's own variants_vcf with every engine call emulated.

- The truth set (tests/left_align_cases.py) rests on no shared code: every placement keeps its haplotype, cannot move
  further and moves nowhere a second time; each repeat gives one record with the reads of all its placements at the
  leftmost POS; no two records share POS, REF and ALT.
- K15d and K15i in three thread orders over the truth set, the fuzz corpus and the limit corpus, against the oracle's
  per-base loops, the per-slot count H included.
- The product's text equals the oracle's byte for byte over filters x primers x strand, with mask_overlaps, from 2- and
  3-rank host tables and for several samples; left_align=False is the keyword absent; on indels that are already
  leftmost only the header line differs; the CLI and the API refuse left-align without a reference."""
import contextlib
import ctypes as C
import dataclasses
import os
import random
import types

import numpy as np
import pytest
import torch

import emu_harness as E
import helpers as H
import left_align_cases as LA
import limit_cases as LC
import mate_cases as MC
import vcf_combo_cases as VC
from fuzz_cases import random_case
from kindel_b200 import __version__, _ffi, bamio, cli, distributed, engine
from kindel_b200 import kindel as K
from oracle import py_laoracle as LO

needs_emu = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")
SOURCE = "kindel {}".format(__version__)
ORDERS = ("forward", "reverse", "random")


def on_the_emulator(monkeypatch):
    """The engine's kdl_* calls on the kernel emulator, over CPU tensors (the upload copies seq4: K9 and K10 write it
    in place, as on the device)."""
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


@pytest.fixture(scope="module")
def truth(tmp_path_factory):
    d = tmp_path_factory.mktemp("left_align")
    bam, fa = LA.write(d)
    lead_bam, _ = LA.write(d, leftmost_only=True)
    return dict(bam=str(bam), fa=str(fa), leftmost=str(lead_bam), dir=d)


# ------------------------------------------------------------------------------------------------ the truth set
def test_truth_set_placements():
    """Every placement keeps its haplotype, cannot move further, and moves nowhere a second time; the oracle's loops
    give the brute-force placement; each repeat not split by an N is one group per kind."""
    per_repeat = {}
    for k, kind, nm, at, x in LA.placements():
        ref = LA.REFS[nm]
        if kind == "D":
            r = LA.leftmost_deletion(ref, at, x)
            assert LA.deletion_haplotype(ref, r, x) == LA.deletion_haplotype(ref, at, x)
            assert not (r > 0 and ref[r - 1] in "ACGT" and ref[r - 1] == ref[r + x - 1])
            assert LA.leftmost_deletion(ref, r, x) == r == LO.left_deletion(ref, at, x)
            per_repeat.setdefault((k, kind), set()).add(r)
        else:
            p, t = LA.leftmost_insertion(ref, at, x)
            assert LA.insertion_haplotype(ref, p, t) == LA.insertion_haplotype(ref, at, x)
            assert not (p > 0 and ref[p - 1] in "ACGT" and t[-1] == ref[p - 1])
            assert LA.leftmost_insertion(ref, p, t) == (p, t) == LO.left_insertion(ref, at, x)
            per_repeat.setdefault((k, kind), set()).add((p, t))
    assert all(len(v) == 1 for v in per_repeat.values())
    assert {("D", "head", 0, 1), ("I", "head", 0, "T"), ("I", "rep", 107, "G")} <= set(LA.expected())


def _records(text):
    return [ln.split("\t") for ln in text.splitlines() if not ln.startswith("#")]


def _indel_ao(fields):
    return int(dict(kv.split("=") for kv in fields[7].split(";") if "=" in kv)["AO"])


def _expected_lines(ref, key):
    """(POS, REF, ALT) of a truth-set group as vcf.records anchors it."""
    kind, nm, at, x = key
    if kind == "D":
        return (at, ref[at - 1:at + x], ref[at - 1]) if at >= 1 else (1, ref[:x + 1], ref[x])
    return (at, ref[at - 1], ref[at - 1] + x) if at >= 1 else (1, ref[0], x + ref[0])


def check_truth_text(text):
    """The truth set's VCF: one record per group, AO the reads of all its placements, no duplicate records."""
    recs = _records(text)
    keys = [(f[0], int(f[1]), f[3], f[4]) for f in recs]
    assert len(keys) == len(set(keys))
    got = {k: _indel_ao(f) for k, f in zip(keys, recs)}
    want = {}
    for key, n in LA.expected().items():
        want[(key[1],) + _expected_lines(LA.REFS[key[1]], key)] = n
    assert got == want


@needs_emu
def test_truth_set_on_the_emulator(truth, monkeypatch):
    """The product's VCF of the truth set: one record per repeat and kind, AO of all placements, no duplicate; without
    left_align the head repeat's r = 0 / r = 1 deletions are two records with one POS, REF and ALT."""
    on_the_emulator(monkeypatch)
    text = K.variants_vcf(truth["bam"], 0, 0, reference=truth["fa"], left_align=True)
    check_truth_text(text)
    want = LO.Composed(truth["bam"]).vcf(SOURCE, 0, 0, reference=("left_align.fa", LA.REFS), left_align=True)
    assert text == want
    plain = _records(K.variants_vcf(truth["bam"], 0, 0, reference=truth["fa"]))
    keys = [(f[0], f[1], f[3], f[4]) for f in plain]
    assert len(keys) > len(set(keys))


# ------------------------------------------------------------------------------------------------ the kernels
def _aligned_rows(events):
    """int32 [n, 4] rows on a 16-byte boundary (the entry point's requirement)."""
    n = int(np.asarray(events).reshape(-1, 4).shape[0])
    buf = np.zeros(4 * n + 4, dtype=np.int32)
    at = (-buf.ctypes.data % 16) // 4
    out = buf[at:at + 4 * n].reshape(n, 4)
    out[:] = np.asarray(events).reshape(-1, 4)
    return out


def emu_insertions(batch, events, codes, dead=None):
    """K15i (kdl_left_align_insertions) over host arrays: (norm_slot, rot, hist); writes past the rows are checked."""
    lib = E.load()
    st, keep = engine.host_struct(batch)
    rows = _aligned_rows(events)
    n = rows.shape[0]
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    slot = np.full(n + 1, -7, dtype=np.int64)
    rot = np.full(n + 1, -7, dtype=np.int32)
    hist = np.zeros(int(batch.n_slots) + 1, dtype=np.int32)
    hist[-1] = -7
    dead = None if dead is None else np.ascontiguousarray(dead, dtype=np.uint8)
    rc = lib.kdl_left_align_insertions(C.byref(st), rows.ctypes.data if n else None, n,
                                       dead.ctypes.data if dead is not None else None, codes.ctypes.data,
                                       slot.ctypes.data, rot.ctypes.data, hist.ctypes.data, None)
    assert rc == 0, lib.kdl_status_string(rc)
    assert slot[n] == -7 and rot[n] == -7 and hist[-1] == -7, "K15i wrote past its outputs"
    del keep
    return slot[:n], rot[:n], hist[:-1]


def emu_deletions(keys, contig_slot, codes):
    lib = E.load()
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    out = np.full(keys.size + 1, -7, dtype=np.int64)
    cs = np.ascontiguousarray(contig_slot, dtype=np.int64)
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    rc = lib.kdl_left_align_deletions(keys.ctypes.data if keys.size else None, keys.size, cs.ctypes.data, cs.size,
                                      codes.ctypes.data, out.ctypes.data, None)
    assert rc == 0 and out[-1] == -7
    return out[:-1]


def repeat_codes(batch, seed):
    """Reference codes for a batch: runs of one base (1-6 long), now and then a two-base unit repeated or an N."""
    rng = random.Random(seed)
    codes = np.full(int(batch.n_slots), 4, dtype=np.uint8)
    for s0, L in zip(np.asarray(batch.contig_slot).tolist(), np.asarray(batch.contig_len).tolist()):
        out = []
        while len(out) < L:
            u = rng.random()
            if u < 0.05:
                out.append(4)
            elif u < 0.2:
                a, b = rng.randrange(4), rng.randrange(4)
                out += [a, b] * rng.randint(2, 4)
            else:
                out += [rng.randrange(4)] * rng.randint(1, 6)
        codes[s0:s0 + L] = out[:L]
    return codes


def oracle_insertions(batch, events, codes):
    """(norm_slot, rotated strings, hist) of event rows by the oracle's per-base loop."""
    letters = "".join("ACGTN"[c] for c in np.asarray(codes).tolist())
    cs = np.asarray(batch.contig_slot, dtype=np.int64)
    slots, texts = [], []
    hist = np.zeros(int(batch.n_slots), dtype=np.int32)
    for slot, read, q_off, length in np.asarray(events).reshape(-1, 4).tolist():
        s0 = int(cs[np.searchsorted(cs, slot, side="right") - 1])
        p, t = LO.left_insertion(letters[s0:slot], slot - s0, H.event_string(batch, read, q_off, length))
        slots.append(s0 + p)
        texts.append(t)
        hist[s0 + p] += 1
    return np.array(slots, dtype=np.int64), texts, hist


def check_kernels(batch, events, codes, what):
    want_slot, want_text, want_hist = oracle_insertions(batch, events, codes)
    for order in ORDERS:
        E.set_schedule(order, 7)
        slot, rot, hist = emu_insertions(batch, events, codes)
        np.testing.assert_array_equal(slot, want_slot, err_msg=str((what, order)))
        np.testing.assert_array_equal(hist, want_hist, err_msg=str((what, order)))
        for row, k, t in zip(np.asarray(events).reshape(-1, 4).tolist(), rot.tolist(), want_text):
            s = H.event_string(batch, *row[1:])
            assert (s[len(s) - k:] + s[:len(s) - k] if k else s) == t, (what, row)
    ev_slot, ev_len = E.deletion_events(batch)
    keys = (ev_slot.astype(np.int64) << 28) | ev_len.astype(np.int64)
    letters = "".join("ACGTN"[c] for c in np.asarray(codes).tolist())
    cs = np.asarray(batch.contig_slot, dtype=np.int64)
    want = []
    for r, n in zip(ev_slot.tolist(), ev_len.tolist()):
        s0 = int(cs[np.searchsorted(cs, r, side="right") - 1])
        want.append(((s0 + LO.left_deletion(letters[s0:r + n], r - s0, n)) << 28) | n)
    for order in ORDERS:
        E.set_schedule(order, 3)
        np.testing.assert_array_equal(emu_deletions(keys, cs, codes), np.array(want, dtype=np.int64).reshape(-1),
                                      err_msg=str((what, order)))
    return len(events), int((np.asarray(want_slot) != np.asarray(events).reshape(-1, 4)[:, 0]).sum())


@needs_emu
def test_kernels_on_the_truth_set(truth):
    batch = bamio.read_alignment(truth["bam"])
    codes = load_codes(truth["fa"], batch)
    _, events = E.pileup_pipeline(batch)
    n, moved = check_kernels(batch, events, codes, "truth")
    assert n and moved > n // 2


def load_codes(fa, batch):
    from kindel_b200.reference import load_reference

    return load_reference(fa, batch).codes


@needs_emu
def test_kernels_on_the_fuzz_corpus(tmp_path):
    n_rows = 0
    for seed in range(400):
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            batch = bamio.read_alignment(str(p))
            _, events = E.pileup_pipeline(batch)
        except (IndexError, KeyError):
            continue
        n_rows += check_kernels(batch, events, repeat_codes(batch, seed), seed)[0]
    assert n_rows > 10


@needs_emu
@pytest.mark.parametrize("name", list(LC.GROUPS))
def test_kernels_on_the_limit_corpus(name, tmp_path):
    p = tmp_path / (name + ".sam")
    p.write_text(LC.sam_text(name))
    batch = bamio.read_alignment(str(p))
    _, events = E.pileup_pipeline(batch)
    check_kernels(batch, events, repeat_codes(batch, len(name)), name)


@needs_emu
def test_dead_rows_count_nowhere(truth):
    batch = bamio.read_alignment(truth["bam"])
    codes = load_codes(truth["fa"], batch)
    _, events = E.pileup_pipeline(batch)
    dead = np.zeros(len(events), dtype=np.uint8)
    dead[::3] = 1
    slot, rot, hist = emu_insertions(batch, events, codes, dead)
    _, _, all_hist = emu_insertions(batch, events, codes)
    assert (slot[::3] == -1).all() and (rot[::3] == 0).all()
    assert hist.sum() == len(events) - dead.sum() and (hist <= all_hist).all()


# ------------------------------------------------------------------------------------------------ the product
@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("la_combo")
    bam, sam, fa, bed, contigs, recs, refs, rows = VC.write(d)
    return dict(bam=str(bam), sam=str(sam), fa=str(fa), bed=str(bed), refs=refs, rows=rows)


def oracle_text(corpus, row, cls=LO.Composed, left_align=True):
    bq, mq, ex, pr, _, strand, (a, r) = row
    o = cls(corpus["bam"], bq, mq, ex, corpus["rows"] if pr else None)
    return o.vcf(SOURCE, a, r, (bq, mq, ex), os.path.basename(corpus["bed"]) if pr else None,
                 (os.path.basename(corpus["fa"]), corpus["refs"]), strand not in ("off", False),
                 strand if isinstance(strand, float) else None, left_align=left_align)


def _kwargs(corpus, row):
    bq, mq, ex, pr, _, strand, _ = row
    return dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, primers=corpus["bed"] if pr else None,
                reference=corpus["fa"], strand=strand not in ("off", False),
                max_sor=strand if isinstance(strand, float) else None)


def _rows():
    return [r for r in VC.option_matrix() if r[4]] + VC.masking_product()


@needs_emu
def test_variants_vcf_matrix_on_the_emulator(corpus, monkeypatch):
    """filters x primers x strand x thresholds with left_align: the product's text is the oracle's; left_align=False
    is the keyword absent; the corpus's indels move."""
    on_the_emulator(monkeypatch)
    n_moved = 0
    for k, row in enumerate(_rows()):
        path = corpus["sam"] if k % 3 == 2 else corpus["bam"]
        got = K.variants_vcf(path, *row[6], left_align=True, **_kwargs(corpus, row))
        assert got == oracle_text(corpus, row), row
        off = K.variants_vcf(path, *row[6], left_align=False, **_kwargs(corpus, row))
        assert off == K.variants_vcf(path, *row[6], **_kwargs(corpus, row))
        n_moved += got.replace(LO.HEADER + "\n", "") != off
    assert n_moved > 3


@pytest.fixture(scope="module")
def combo(tmp_path_factory):
    return MC.combo_files(tmp_path_factory.mktemp("la_mates"))


@needs_emu
def test_mask_overlaps_on_the_emulator(combo, monkeypatch):
    """With mask_overlaps the dropped events are left out before anything moves: the product's text is the
    oracle's over the mates matrix rows with a reference."""
    on_the_emulator(monkeypatch)
    n = 0
    for row in MC.mates_matrix():
        bq, mq, ex, pr, ref, strand, (a, r) = row
        if not ref:
            continue
        kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, strand=strand, mask_overlaps=True,
                  reference=combo["fa"], left_align=True, primers=combo["bed"] if pr else None)
        got = K.variants_vcf(combo["bam"], a, r, **kw)
        o = LO.ComposedMates(combo["bam"], bq, mq, ex, combo["rows"] if pr else None)
        want = o.vcf(SOURCE, a, r, (bq, mq, ex), os.path.basename(combo["bed"]) if pr else None,
                     (os.path.basename(combo["fa"]), combo["refs"]), strand, left_align=True)
        assert got == want, row
        n += 1
    assert n >= 2


def _host_run(batch, world, plan, **kw):
    """A run from the summed host tables of `world` ranks, each shard piled on the emulated engine."""
    total, evs, idx_all = None, [], []
    for rank in range(world):
        idx = distributed.shard_indices(batch, rank, world, plan)
        counts, events = engine.pileup(engine.upload(bamio.select_reads(batch, idx)))
        total = counts.numpy().astype(np.int64) if total is None else total + counts.numpy()
        evs.append(events.numpy())
        idx_all.append(idx)
    counts = total.astype(np.int32)
    return K.PileupRun.from_host_tables(batch, counts, E.derive(counts), distributed.merge_events(evs, idx_all), **kw)


@needs_emu
@pytest.mark.parametrize("world", [2, 3])
def test_host_tables_on_the_emulator(corpus, truth, monkeypatch, world):
    """2- and 3-rank host tables (the multi-GPU result): the event rows go up next to the batch, and the text is the
    one GPU's."""
    on_the_emulator(monkeypatch)
    for path, fa, a, r in ((corpus["bam"], corpus["fa"], 1, 0.01), (truth["bam"], truth["fa"], 0, 0)):
        batch = bamio.read_alignment(path, strand=True)
        run = _host_run(batch, world, "reads")
        got = K.variants_vcf_from_run(run, a, r, (0, 0, 0), reference=fa, strand=True, left_align=True)
        assert got == K.variants_vcf(path, a, r, reference=fa, strand=True, left_align=True)


@needs_emu
def test_several_samples_on_the_emulator(truth, corpus, monkeypatch, tmp_path):
    """Each sample is left-aligned before its batch goes: a list of one path gives the single-sample data lines in
    columns 1-8, and two copies of the truth set give one record per group with twice its reads."""
    on_the_emulator(monkeypatch)
    for path, fa in ((truth["bam"], truth["fa"]), (corpus["bam"], corpus["fa"])):
        one = K.variants_vcf([path], 0, 0, reference=fa, left_align=True)
        single = K.variants_vcf(path, 0, 0, reference=fa, left_align=True)
        assert [ln.split("\t")[:8] for ln in one.splitlines() if not ln.startswith("#")] == _records(single)
        assert LO.HEADER in one.splitlines()
    copy = tmp_path / "copy.bam"
    copy.write_bytes(open(truth["bam"], "rb").read())
    two = _records(K.variants_vcf([truth["bam"], str(copy)], 0, 0, reference=truth["fa"], left_align=True))
    single = _records(K.variants_vcf(truth["bam"], 0, 0, reference=truth["fa"], left_align=True))
    assert [f[:5] for f in two] == [f[:5] for f in single]
    assert [_indel_ao(f) for f in two] == [2 * _indel_ao(f) for f in single]


@needs_emu
def test_leftmost_indels_change_only_the_header(truth, monkeypatch):
    on_the_emulator(monkeypatch)
    on = K.variants_vcf(truth["leftmost"], 0, 0, reference=truth["fa"], strand=True, left_align=True)
    off = K.variants_vcf(truth["leftmost"], 0, 0, reference=truth["fa"], strand=True)
    lines = on.splitlines()
    assert lines[lines.index(LO.HEADER) - 1].startswith("##reference=")
    assert "\n".join(x for x in lines if x != LO.HEADER) + "\n" == off
    assert on.count("INDEL;") > 10


def test_left_align_needs_a_reference(truth):
    with pytest.raises(ValueError, match="reference"):
        K.variants_vcf(truth["bam"], left_align=True)
    with pytest.raises(ValueError, match="reference"):
        K.variants_vcf([truth["bam"], truth["bam"]], samples=["a", "b"], left_align=True)
    with pytest.raises(ValueError, match="reference"):
        K.variants_vcf_from_run(None, left_align=True)
    for argv in (["variants", "--left-align", truth["bam"]],
                 ["variants", "--vcf", "--left-align", truth["bam"]],
                 ["variants", "--reference", truth["fa"], "--left-align", truth["bam"]]):
        with pytest.raises(SystemExit) as e:
            cli.main(argv)
        assert e.value.code == 2
    a = cli.build_parser().parse_args(["variants", "--vcf", "--reference", truth["fa"], "--left-align", truth["bam"]])
    assert a.left_align
