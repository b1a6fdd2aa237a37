"""Several samples in one VCF on the H100: K6m against the multi-sample oracle's sites, variants_vcf over lists of
paths and the CLI against the oracle's text, a tenth of config 4 split into 4 samples with planted alleles, and two
GPUs against one."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import cohort_cases as CO
import helpers as H
from kindel_b200 import __version__, bamio, engine
from kindel_b200 import kindel as K
from oracle import coracle
from oracle import py_msoracle as MS
from test_cohort import as_named, k6m_cases, kwargs, matrix, oracle_text
from test_variants_vcf import GRID

pytestmark = pytest.mark.gpu
SOURCE = "kindel {}".format(__version__)


def test_k6m_on_the_device_equals_the_oracle_sites():
    import torch

    n = 0
    for S, T, cs, cl, ref, samples in k6m_cases():
        texts = CO.ref_texts(ref, cs, cl)
        dT = torch.from_numpy(T).cuda()
        for a, r in GRID[S % 4::6]:
            for mode in ("pooled", "reference"):
                slot, mask = engine.variant_sites_multi(dT, cs, cl, ref if mode == "reference" else None, a, r)
                got = as_named(slot.cpu().numpy(), mask.cpu().numpy(), cs, cl)
                assert got == MS.site_bits(samples, a, r, texts if mode == "reference" else None), (S, a, r, mode)
                n += len(got)
    assert n > 5000


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    d = tmp_path_factory.mktemp("cohort_gpu")
    paths, fa, bed, rows, refs = CO.split_corpus(d)
    return dict(paths=paths, fa=fa, bed=bed, rows=rows, refs=refs, oracle={})


def test_variants_vcf_of_samples_on_the_device(split):
    for k, row in enumerate(matrix()):
        a, r = ((1, 0.01), (0, 0.0), (2, 0.2))[k % 3]
        got = K.variants_vcf(split["paths"], a, r, samples=["s0", "s1", "s2"], **kwargs(split, row))
        assert got == oracle_text(split, row, ["s0", "s1", "s2"], a, r), row


def test_cli_with_several_files(split):
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    for ref in (False, True):
        cmd = [sys.executable, "-m", "kindel_b200", "variants", "--vcf", *split["paths"]]
        if ref:
            cmd += ["--reference", split["fa"]]
        out = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=H.ROOT, check=True).stdout
        assert out == oracle_text(split, (0, 0, 0, False, ref, False), ["s0.bam", "s1.bam", "s2.bam"])


def test_a_tenth_of_config_4_in_four_samples(tmp_path):
    """500 kb at 200x (a tenth of config 4's contig), as 4 samples of 50x with reads and planted alleles of their own:
    the pooled VCF's sha256 equals the oracle's, over the C oracle's tables."""
    samples = CO.synthetic_samples(tmp_path, 4, 500_000, 50)
    paths = [p for p, _ in samples]
    got = K.variants_vcf(paths, 1, 0.05)
    oracle = []
    for p, _ in samples:
        b = bamio.read_alignment(p)
        t, _ = coracle.pileup(b)
        oracle.append(MS.Sample.from_table(b.contig_names, b.contig_len, b.contig_slot, t))
    want = MS.vcf(oracle, [os.path.basename(p) for p in paths], SOURCE, 1, 0.05)
    assert hashlib.sha256(got.encode()).hexdigest() == hashlib.sha256(want.encode()).hexdigest()
    body = [ln for ln in got.splitlines() if not ln.startswith("#")]
    assert len(body) >= 16  # every planted allele is a record


def test_two_gpus_equal_one(split):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for row in ((0, 0, 0, False, True, False), (20, 30, 0x500, True, False, True)):
        one = K.variants_vcf(split["paths"], 1, 0.01, devices=1, **kwargs(split, row))
        assert K.variants_vcf(split["paths"], 1, 0.01, devices=2, **kwargs(split, row)) == one
