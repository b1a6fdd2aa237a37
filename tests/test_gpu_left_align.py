"""`variants --vcf --reference --left-align` (extension) on the GPU: K15d / K15i on the device against the left-aligning
oracle (oracle/py_laoracle.py) on the truth set, the fuzz corpus and a config-4-sized batch with planted repeats (the
sha256 of the moved keys and of H); variants_vcf and the CLI against the oracle's text byte for byte with every
compatible option; several samples; two GPUs against one."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
import left_align_cases as LA
import mate_cases as MC
import vcf_combo_cases as VC
from fuzz_cases import random_case
from kindel_b200 import __version__, bamio, engine
from kindel_b200 import kindel as K
from kindel_b200.reference import load_reference
from oracle import py_laoracle as LO
from test_left_align import _records, check_truth_text, oracle_insertions, repeat_codes

pytestmark = pytest.mark.gpu
SOURCE = "kindel {}".format(__version__)


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def truth(tmp_path_factory):
    d = tmp_path_factory.mktemp("left_align_gpu")
    bam, fa = LA.write(d)
    return dict(bam=str(bam), fa=str(fa), dir=d)


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("la_combo_gpu")
    bam, sam, fa, bed, contigs, recs, refs, rows = VC.write(d)
    return dict(bam=str(bam), sam=str(sam), fa=str(fa), bed=str(bed), refs=refs, rows=rows)


def device_moves(batch, codes):
    """(moved deletion keys, norm_slot, rot, hist) of a batch on the device, as numpy."""
    db = engine.upload(batch)
    _, events = engine.pileup(db)
    t_codes = _dev(codes)
    slot, length = engine.deletion_events(db)
    keys = (slot << 28) | length.long()
    cnt = keys.new_ones(keys.shape)
    moved, _ = engine.left_align_deletions(keys, cnt, t_codes, db.tensors["contig_slot"], batch.n_contigs)
    norm_slot, rot, hist = engine.left_align_insertions(db, events, t_codes)
    return moved.cpu().numpy(), norm_slot.cpu().numpy(), rot.cpu().numpy(), hist.cpu().numpy(), events.cpu().numpy()


def oracle_keys(batch, codes, slot, length):
    letters = "".join("ACGTN"[c] for c in np.asarray(codes).tolist())
    cs = np.asarray(batch.contig_slot, dtype=np.int64)
    out = set()
    for r, n in zip(np.asarray(slot).tolist(), np.asarray(length).tolist()):
        s0 = int(cs[np.searchsorted(cs, r, side="right") - 1])
        out.add(((s0 + LO.left_deletion(letters[s0:r + n], r - s0, n)) << 28) | n)
    return np.array(sorted(out), dtype=np.int64)


def check_device(batch, codes):
    moved, norm_slot, rot, hist, events = device_moves(batch, codes)
    want_slot, want_text, want_hist = oracle_insertions(batch, events, codes)
    np.testing.assert_array_equal(norm_slot, want_slot)
    np.testing.assert_array_equal(hist, want_hist)
    for row, k, t in zip(events.tolist(), rot.tolist(), want_text):
        s = H.event_string(batch, *row[1:])
        assert (s[len(s) - k:] + s[:len(s) - k] if k else s) == t
    slot, length = engine.deletion_events(engine.upload(batch))
    np.testing.assert_array_equal(moved, oracle_keys(batch, codes, slot.cpu().numpy(), length.cpu().numpy()))
    return len(events)


def test_kernels_on_the_truth_set_and_the_fuzz_corpus(truth, tmp_path):
    batch = bamio.read_alignment(truth["bam"])
    assert check_device(batch, load_reference(truth["fa"], batch).codes) > 50
    n = 0
    for seed in range(400):
        p = tmp_path / ("fuzz%d.sam" % seed)
        p.write_text(random_case(seed))
        try:
            batch = bamio.read_alignment(str(p))
            engine.pileup(engine.upload(batch))
        except (IndexError, KeyError):
            continue
        n += check_device(batch, repeat_codes(batch, seed))
    assert n > 10


def test_truth_set_vcf(truth):
    text = K.variants_vcf(truth["bam"], 0, 0, reference=truth["fa"], left_align=True)
    check_truth_text(text)
    assert text == LO.Composed(truth["bam"]).vcf(SOURCE, 0, 0, reference=("left_align.fa", LA.REFS), left_align=True)


def test_variants_vcf_matrix(corpus):
    for row in [r for r in VC.option_matrix() if r[4]] + VC.masking_product():
        bq, mq, ex, pr, _, strand, (a, r) = row
        kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, primers=corpus["bed"] if pr else None,
                  reference=corpus["fa"], strand=strand != "off", max_sor=strand if isinstance(strand, float) else None)
        got = K.variants_vcf(corpus["bam"], a, r, left_align=True, **kw)
        o = LO.Composed(corpus["bam"], bq, mq, ex, corpus["rows"] if pr else None)
        want = o.vcf(SOURCE, a, r, (bq, mq, ex), os.path.basename(corpus["bed"]) if pr else None,
                     (os.path.basename(corpus["fa"]), corpus["refs"]), strand != "off",
                     strand if isinstance(strand, float) else None, left_align=True)
        assert got == want, row
        assert K.variants_vcf(corpus["bam"], a, r, left_align=False, **kw) == K.variants_vcf(corpus["bam"], a, r, **kw)


def test_mask_overlaps(tmp_path):
    combo = MC.combo_files(tmp_path)
    for row in MC.mates_matrix():
        bq, mq, ex, pr, ref, strand, (a, r) = row
        if not ref:
            continue
        got = K.variants_vcf(combo["bam"], a, r, min_base_quality=bq, min_mapq=mq, exclude_flags=ex, strand=strand,
                             mask_overlaps=True, reference=combo["fa"], left_align=True,
                             primers=combo["bed"] if pr else None)
        want = LO.ComposedMates(combo["bam"], bq, mq, ex, combo["rows"] if pr else None).vcf(
            SOURCE, a, r, (bq, mq, ex), os.path.basename(combo["bed"]) if pr else None,
            (os.path.basename(combo["fa"]), combo["refs"]), strand, left_align=True)
        assert got == want, row


def test_several_samples(truth, tmp_path):
    copy = tmp_path / "copy.bam"
    copy.write_bytes(open(truth["bam"], "rb").read())
    one = K.variants_vcf([truth["bam"]], 0, 0, reference=truth["fa"], left_align=True)
    single = K.variants_vcf(truth["bam"], 0, 0, reference=truth["fa"], left_align=True)
    assert [f[:8] for f in _records(one)] == _records(single)
    two = _records(K.variants_vcf([truth["bam"], str(copy)], 0, 0, reference=truth["fa"], left_align=True))
    assert [f[:5] for f in two] == [f[:5] for f in _records(single)]


def test_cli(corpus):
    """The CLI with every compatible flag equals the API."""
    argv = ["variants", "--vcf", "--reference", corpus["fa"], "--left-align", "--strand", "--max-sor", "3",
            "--primers", corpus["bed"], "--min-base-quality", "20", "--min-mapq", "30", "--mask-overlaps", "--dedup",
            "-a", "1", "-r", "0.01", corpus["bam"]]
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    got = subprocess.run([sys.executable, "-m", "kindel_b200"] + argv, capture_output=True, text=True, env=env,
                         cwd=H.ROOT)
    assert got.returncode == 0, got.stderr
    want = K.variants_vcf(corpus["bam"], 1, 0.01, reference=corpus["fa"], left_align=True, strand=True, max_sor=3.0,
                          primers=corpus["bed"], min_base_quality=20, min_mapq=30, mask_overlaps=True, dedup=True)
    assert got.stdout == want


def test_two_gpus_equal_one(corpus, truth):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for path, fa in ((corpus["bam"], corpus["fa"]), (truth["bam"], truth["fa"])):
        one = K.variants_vcf(path, 0, 0, reference=fa, strand=True, left_align=True)
        assert K.variants_vcf(path, 0, 0, reference=fa, strand=True, left_align=True, devices=2) == one


def planted_reference(length, seed=4, every=997):
    """The config-4 contig's text with a homopolymer or a dinucleotide repeat planted every `every` bases."""
    sys.path.insert(0, os.path.join(H.ROOT, "tools"))
    from bench_variants_ref import contig_text

    text = list(contig_text(seed, length))
    rng = np.random.default_rng(seed)
    for at in range(50, length - 20, every):
        a, b = "ACGT"[rng.integers(4)], "ACGT"[rng.integers(4)]
        text[at:at + 12] = list(a * 12 if rng.random() < 0.5 else (a + b) * 6)
    return "".join(text)


def test_config4_sized_batch(tmp_path):
    """bench.py's config-4 batch against a reference with planted repeats: the sha256 of K15d's moved keys (grouped)
    and of K15i's H equal the oracle's."""
    sys.path.insert(0, H.ROOT)
    import bench

    batch = bench.gen_reads("cfg4_5Mb_200x")
    fa = tmp_path / "planted.fa"
    fa.write_text(">%s\n%s\n" % (batch.contig_names[0], planted_reference(int(batch.contig_len[0]))))
    codes = load_reference(str(fa), batch).codes
    moved, norm_slot, _, hist, events = device_moves(batch, codes)
    want_slot, _, want_hist = oracle_insertions(batch, events, codes)
    slot, length = engine.deletion_events(engine.upload(batch))
    want_keys = oracle_keys(batch, codes, slot.cpu().numpy(), length.cpu().numpy())
    digest = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()  # noqa: E731
    assert digest(np.unique(moved)) == digest(want_keys)
    assert digest(hist) == digest(want_hist)
    assert digest(norm_slot) == digest(want_slot)
    assert (norm_slot != events[:, 0]).sum() > 100
