"""`variants --vcf` with its options together on the GPU: the VCF of base and read filters, primers, reference and
strand against the composed oracle (oracle/py_cvoracle.py) byte for byte over the option matrix of
tests/test_vcf_combined.py, several GPUs against one, the CLI with every flag, and a tenth of config 4 whose masked
reverse and forward tables equal the C quality walk."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
import primer_cases as PC
import vcf_combo_cases as VC
from kindel_b200 import bamio, synth
from kindel_b200 import kindel as K
from oracle import py_poracle as PO
from test_vcf_combined import _kwargs, oracle_text

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("vcf_combo_gpu")
    bam, sam, fa, bed, contigs, recs, refs, rows = VC.write(d)
    return dict(bam=str(bam), sam=str(sam), fa=str(fa), bed=str(bed), contigs=contigs, recs=recs, refs=refs, rows=rows,
                dir=d, composed={})


def test_variants_vcf_equals_the_composed_oracle(corpus):
    rows = VC.option_matrix() + VC.masking_product()
    for k, row in enumerate(rows):
        path = corpus["sam"] if k % 3 == 2 else corpus["bam"]
        assert K.variants_vcf(path, *row[6], devices=1, **_kwargs(corpus, row)) == oracle_text(corpus, row), row


def test_two_gpus_equal_one(corpus):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    for row in (VC.masking_product()[-1],) + tuple(VC.option_matrix()[:2]):
        one = K.variants_vcf(corpus["bam"], *row[6], devices=1, **_kwargs(corpus, row))
        assert K.variants_vcf(corpus["bam"], *row[6], devices=2, **_kwargs(corpus, row)) == one, row
        assert one == oracle_text(corpus, row), row


def test_cli_with_every_flag(corpus):
    args = ["variants", "--vcf", "--reference", corpus["fa"], "--strand", "--max-sor", "3", "--primers", corpus["bed"],
            "--min-base-quality", "20", "--min-mapq", "30", "--exclude-flags", "0x500", corpus["bam"]]
    res = subprocess.run([sys.executable, "-m", "kindel_b200", *args], capture_output=True, text=True, cwd=H.ROOT,
                         timeout=900)
    assert res.returncode == 0, res.stderr[-2000:]
    row = (20, 30, 0x500, True, True, 3.0, (1, 0.01))
    assert res.stdout == K.variants_vcf(corpus["bam"], 1, 0.01, **_kwargs(corpus, row)) == oracle_text(corpus, row)


def _sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.int32).tobytes()).hexdigest()


def test_masked_strand_tables_of_a_tenth_of_config4():
    """Quality mask at Q20, a tiled primer scheme and seeded strands: the reverse table == the C quality walk over the
    reverse reads with their qualities and primer bases, and total - reverse == the same over the forward reads."""
    plain = synth.with_strands(synth.mixed_reads(4, [500_000], 200, 0.01), 3)
    batch, qual = synth.with_qualities(plain, 5)
    batch = synth.with_strands(batch, 3)
    rows = synth.tiled_scheme(1, batch.contig_names, batch.contig_len)
    run = K.PileupRun(batch, primers=PC.primer_set(rows))
    rev = run.reverse_table()[0].cpu().numpy()
    fwd = run.counts.cpu().numpy().astype(np.int64) - rev
    per_base = np.repeat(plain.reverse, plain.seq_len)
    for strand, got in ((1, rev), (0, fwd)):
        sub = bamio.select_reads(plain, np.flatnonzero(plain.reverse == strand))
        want, _ = PO.pileup(sub, PO.masked_arrays(sub, rows), qual[per_base == strand], 20)
        assert want[0:5].sum() > 0 and _sha(got[0:19]) == _sha(want[0:19]), strand
