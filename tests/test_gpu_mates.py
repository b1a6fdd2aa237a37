"""`--mask-overlaps` (an extension) on the GPU: K10p / K10 / K10u through the real library against the independent
restatement (oracle/py_moracle.py), the product's API and CLI with the other options, config 4's shape as read
pairs against the oracle's table by sha256, and two GPUs against one."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import helpers as H
import mate_cases as MC
from kindel_b200 import __version__, bamio, engine, synth
from kindel_b200 import kindel as K
from oracle import py_moracle as MO

pytestmark = pytest.mark.gpu
SOURCE = "kindel {}".format(__version__)


def _sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("gpu_mates")
    return dict(sam=MC.lattice_sam(str(d / "lattice.sam")), pairs=MC.paired_bam(str(d / "pairs.bam")), dir=d)


def _oracle(path, b):
    o = MO.Masked(path, b.contig_names, pre_masked=MC.mask_lists(b))
    return o, o.pileup(bamio.read_alignment(path), dict(zip(b.contig_names, b.contig_slot.tolist())))


@pytest.mark.parametrize("which", ["sam", "pairs"])
def test_device_chain_against_the_oracle(files, which):
    path = files[which]
    run = K.PileupRun(bamio.read_alignment(path, mates=True, strand=True), mask_overlaps=True)
    o, (want, wev) = _oracle(path, run.batch)
    np.testing.assert_array_equal(run.host_counts, want)
    np.testing.assert_array_equal(run.ins_table.events, wev[np.argsort(wev[:, 0], kind="stable")])
    assert run.overlap_stats == o.stats()
    rev, sub = run.reverse_table()
    total = run.host_counts
    assert (rev.cpu().numpy()[0:7] <= total[0:7]).all()


def test_device_pairing_with_a_torch_sort_equals_numpy_order(files):
    b = bamio.read_alignment(files["pairs"], mates=True)
    db = engine.upload(b)
    got = engine.pair_mates(db).cpu().numpy()
    idx = np.flatnonzero(b.pair_role)
    order = torch.from_numpy(idx[np.argsort(b.name_hash[idx], kind="stable")].astype(np.int32))
    assert np.array_equal(got, engine.pair_mates(db, order).cpu().numpy())
    lengths, recs = MO.kept(files["pairs"], b.contig_names)
    want = np.full(b.n_reads, -1)
    for r2, r1 in MO.pairs(lengths, recs).items():
        want[r2] = r1
    assert got.tolist() == want.tolist()


@pytest.fixture(scope="module")
def combo(tmp_path_factory):
    return MC.combo_files(tmp_path_factory.mktemp("gpu_mates_combo"))


def _oracle_vcf(files, row):
    bq, mq, ex, pr, ref, strand, (a, r) = row
    o = MO.ComposedMates(files["bam"], bq, mq, ex, files["rows"] if pr else None)
    return o.vcf(SOURCE, a, r, (bq, mq, ex), os.path.basename(files["bed"]) if pr else None,
                 (os.path.basename(files["fa"]), files["refs"]) if ref else None, strand)


@pytest.mark.parametrize("k", range(len(MC.mates_matrix())))
def test_option_matrix_on_the_device(combo, k):
    """variants_vcf with mask_overlaps on equals the composed oracle byte for byte (deletion AO, ADF / ADR included)
    over filters x primers x reference x strand; off it equals the call without the keyword."""
    row = MC.mates_matrix()[k]
    bq, mq, ex, pr, ref, strand, (a, r) = row
    kw = dict(min_base_quality=bq, min_mapq=mq, exclude_flags=ex, strand=strand)
    if pr:
        kw["primers"] = combo["bed"]
    if ref:
        kw["reference"] = combo["fa"]
    path = combo["sam"] if k % 3 == 2 else combo["bam"]
    assert K.variants_vcf(path, a, r, mask_overlaps=True, **kw) == _oracle_vcf(combo, row)
    assert K.variants_vcf(path, a, r, **kw) == K.variants_vcf(path, a, r, mask_overlaps=False, **kw)


def test_cli_with_every_flag(combo, tmp_path):
    """`variants --vcf --reference --primers --strand --mask-overlaps` prints the composed oracle's VCF; without
    `--mask-overlaps` it prints the call without the keyword; the other commands run with it."""
    path = combo["bam"]
    base = [sys.executable, "-m", "kindel", "variants", "--vcf", "--reference", combo["fa"], "--primers", combo["bed"],
            "--strand", path]
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    off = subprocess.run(base, capture_output=True, text=True, cwd=H.ROOT, env=env)
    on = subprocess.run(base + ["--mask-overlaps"], capture_output=True, text=True, cwd=H.ROOT, env=env)
    assert off.returncode == 0 and on.returncode == 0, on.stderr
    assert on.stdout == _oracle_vcf(combo, (0, 0, 0, True, True, True, (1, 0.01)))
    assert off.stdout == K.variants_vcf(path, reference=combo["fa"], primers=combo["bed"], strand=True)
    one = MC.paired_bam(str(tmp_path / "one.bam"))  # (features raises the reference's IndexError on two contigs)
    for cmd in (["consensus"], ["weights"], ["features"]):
        r = subprocess.run([sys.executable, "-m", "kindel"] + cmd + [one, "--mask-overlaps"], capture_output=True,
                           text=True, cwd=H.ROOT, env=env)
        assert r.returncode == 0, r.stderr


def test_cli_dp_and_ad_are_fragment_counts(tmp_path):
    """On pairs without indels, substitutions or masks, the full command's DP and AD at every SNV record are the
    number of fragments over the position (`variants --vcf --reference --strand --mask-overlaps`)."""
    refs = {}
    b, flag, frag = synth.paired_reads(9, [4000], 40, read_len=100, insert_mean=160, indel_frac=0.0, sub_rate=0.0,
                                       refs=refs)
    path = str(tmp_path / "f.bam")
    synth.write_paired_bam(path, b, flag, frag)
    fa = tmp_path / "f.fa"
    # a reference with a different base every 50 positions: an SNV record there whose ALT count is the depth
    ref = "".join(("C" if c != "C" else "G") if k % 50 == 25 else c for k, c in enumerate(refs["ctg0"]))
    fa.write_text(">ctg0\n%s\n" % ref)
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    out = subprocess.run([sys.executable, "-m", "kindel", "variants", "--vcf", "--reference", str(fa), "--strand",
                          "--mask-overlaps", path], capture_output=True, text=True, cwd=H.ROOT, env=env)
    assert out.returncode == 0, out.stderr
    want = MO.fragment_depth(path, b.contig_names)["ctg0"]
    n = 0
    for line in out.stdout.splitlines():
        if line.startswith("#"):
            continue
        f = line.split("\t")
        info = dict(x.split("=") for x in f[7].split(";") if "=" in x)
        pos = int(f[1]) - 1
        assert int(info["DP"]) == want[pos] and info["AD"] == "0,%d" % want[pos], line
        n += 1
    assert n >= 70


def test_dp_equals_fragment_counts(tmp_path):
    """On pairs without indels, Ns or masks, a site's DP is the number of fragments over it."""
    b, flag, frag = synth.paired_reads(9, [4000], 40, read_len=100, insert_mean=160, indel_frac=0.0, sub_rate=0.0)
    path = str(tmp_path / "f.bam")
    synth.write_paired_bam(path, b, flag, frag)
    run = K.PileupRun(bamio.read_alignment(path, mates=True), mask_overlaps=True)
    want = MO.fragment_depth(path, b.contig_names)
    s = int(b.contig_slot[0])
    np.testing.assert_array_equal(run.host_counts[0:6, s:s + 4000].sum(axis=0), want["ctg0"])


def test_config4_shape_as_pairs(tmp_path):
    """Config 4's depth and read length (200x of 2 x 150 bp on ~300 bp inserts) over a 100 kb contig, a fiftieth of
    its size: the table's sha256 against the oracle's."""
    b, flag, frag = synth.paired_reads(4, [100_000], 200, read_len=150, insert_mean=300, insert_sd=40,
                                       indel_frac=0.01)
    path = str(tmp_path / "cfg4.bam")
    synth.write_paired_bam(path, b, flag, frag)
    run = K.PileupRun(bamio.read_alignment(path, mates=True), mask_overlaps=True)
    o, (want, wev) = _oracle(path, run.batch)
    assert _sha(run.host_counts) == _sha(want)
    assert run.overlap_stats == o.stats() and o.stats()[0] > 50_000


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus_equal_one(files):
    path = files["pairs"]
    one = K.variants_vcf(path, 0, 0.0, strand=True, mask_overlaps=True)
    two = K.variants_vcf(path, 0, 0.0, strand=True, mask_overlaps=True, devices=2)
    assert one == two
    a = K.bam_to_consensus(path, mask_overlaps=True)
    c = K.bam_to_consensus(path, mask_overlaps=True, devices=2)
    assert [x.sequence for x in a.consensuses] == [x.sequence for x in c.consensuses]
