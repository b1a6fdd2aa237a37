"""`variants --vcf --strand` (extension) on the GPU: K8 equals bamio.select_reads field for field, the reverse table
plus the forward table is the total, and the VCF equals oracle/py_soracle.py byte for byte."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
import strand_cases as S
from kindel_b200 import bamio, engine, synth
from kindel_b200 import kindel as K
from kindel_b200.reference import load_reference
from oracle import py_soracle as SO
from oracle import samdecode

pytestmark = pytest.mark.gpu

INPUTS = os.path.join(H.ROOT, "tests", "golden", "inputs")
FIXTURES = sorted(f for f in os.listdir(INPUTS) if f.endswith((".bam", ".sam")))


def _keeps(batch, seed):
    rng = np.random.default_rng(seed)
    n = batch.n_reads
    out = [batch.reverse, 1 - batch.reverse, np.zeros(n, np.uint8), np.ones(n, np.uint8),
           (rng.random(n) < 0.3).astype(np.uint8)]
    if batch.n_contigs > 1:  # a contig with no kept read
        k = np.ones(n, np.uint8)
        k[int(batch.contig_read_off[0]):int(batch.contig_read_off[1])] = 0
        out.append(k)
    return out


def _check_select(batch, db, seed, what):
    import torch

    for j, keep in enumerate(_keeps(batch, seed)):
        keep = np.ascontiguousarray(keep, dtype=np.uint8)
        sub = engine.select_reads(db, torch.from_numpy(keep))
        want = bamio.select_reads(batch, np.flatnonzero(keep))
        S.assert_equal(engine.download_fields(sub), S.fields(want), (what, j))
        got_t, got_e = engine.pileup(sub)
        want_t, want_e = engine.pileup(engine.upload(want))
        assert np.array_equal(got_t.cpu().numpy(), want_t.cpu().numpy()), (what, j)
        assert np.array_equal(got_e.cpu().numpy(), want_e.cpu().numpy()), (what, j)


@pytest.mark.parametrize("name", FIXTURES)
def test_k8_equals_select_reads_on_fixtures(name):
    path = os.path.join(INPUTS, name)
    for mbq in (0, 20):
        try:
            batch = bamio.read_alignment(path, strand=True, min_base_quality=mbq)
        except ValueError:
            continue
        _check_select(batch, engine.upload(batch), 7, (name, mbq))


@pytest.mark.parametrize("masked", [False, True])
def test_k8_on_a_tenth_of_config4(masked):
    batch = synth.mixed_reads(4, [500_000], 200, 0.01)
    if masked:
        batch = synth.with_qualities(batch, 5)[0]
    batch = synth.with_strands(batch, 3)
    _check_select(batch, engine.upload(batch), 11, ("cfg4/10", masked))


def test_reverse_plus_forward_is_the_total():
    for batch in (synth.with_strands(synth.mixed_reads(6, [200_000, 3_000], 100, 0.05), 1),
                  bamio.read_alignment(os.path.join(INPUTS, "mm2_multi.bam"), strand=True, min_base_quality=20)):
        run = K.PileupRun(batch)
        rev = run.reverse_table()[0].cpu().numpy()
        fwd = engine.pileup(engine.upload(bamio.select_reads(batch, np.flatnonzero(batch.reverse == 0))))[0]
        total = run.counts.cpu().numpy()
        assert rev.shape == total.shape == (19, batch.n_slots)
        assert np.array_equal(rev.astype(np.int64) + fwd.cpu().numpy(), total)  # all 19 columns, bit for bit
        assert rev.any() and fwd.cpu().numpy().any()


def _groups(path):
    header, records = samdecode.read_alignment_file(path)
    groups = {}
    for rec in records:
        groups.setdefault(rec.rname, []).append(rec)
    groups.pop("*", None)
    return groups


def _body(text):
    return [ln for ln in text.splitlines() if not ln.startswith("#")]


def _ad_sums_hold(lines):
    for ln in lines:
        info = dict(kv.split("=") for kv in ln.split("\t")[7].split(";") if "=" in kv)
        adf = [int(x) for x in info["ADF"].split(",")]
        adr = [int(x) for x in info["ADR"].split(",")]
        if "AO" in info:
            assert adf[1] + adr[1] == int(info["AO"]), ln
        else:
            assert [a + b for a, b in zip(adf, adr)] == [int(x) for x in info["AD"].split(",")], ln
        assert all(float(x) >= 0 for x in info["SOR"].split(",")), ln  # (> 0, but "%.3f" may round to 0)


@pytest.mark.parametrize("name", ["mm2_gp120.bam", "mm2_multi.bam", "bwa_1_1.bam", "seg_2_1.bam", "ext_2_bc63.sam"])
def test_vcf_equals_oracle_on_fixtures(name):
    path = os.path.join(INPUTS, name)
    batch = bamio.read_alignment(path)
    groups = _groups(path)
    for a, r, max_sor in ((1, 0.01, None), (0, 0.0, 3.0), (2, 0.2, 1.5)):
        text = K.variants_vcf(path, a, r, strand=True, max_sor=max_sor)
        want = SO.vcf_lines([(nm, int(L), groups.get(nm, [])) for nm, L in zip(batch.contig_names, batch.contig_len)],
                            a, r, max_sor)
        assert _body(text) == want, (name, a, r)
        assert all(h in text.splitlines() for h in SO.header_lines(max_sor))
        _ad_sums_hold(want)
        # with strand off the file is what it was, and the strand fields are all that was added
        plain = K.variants_vcf(path, a, r)
        assert "ADF" not in plain and "kindelStrand" not in plain
        assert [ln.split("\t")[:6] for ln in _body(plain)] == [ln.split("\t")[:6] for ln in want]


def test_vcf_against_reference_equals_oracle(tmp_path):
    bam, fa, ref, reads = S.write(tmp_path)
    cases = [(str(bam), str(fa), {"t": S.oracle_records(reads)}),
             (os.path.join(INPUTS, "mm2_gp120.bam"), os.path.join(INPUTS, "hxb2-gp120-mutated.fa"), None)]
    for path, fasta, groups in cases:
        batch = bamio.read_alignment(path)
        groups = groups or _groups(path)
        codes = load_reference(fasta, batch).codes
        texts = {nm: "".join("ACGTN"[x] for x in codes[s0:s0 + L].tolist())
                 for nm, s0, L in zip(batch.contig_names, batch.contig_slot.tolist(), batch.contig_len.tolist())}
        for a, r, max_sor in ((1, 0.01, 3.0), (0, 0.0, None)):
            text = K.variants_vcf(path, a, r, reference=fasta, strand=True, max_sor=max_sor)
            want = SO.vcf_lines([(nm, texts[nm], groups.get(nm, [])) for nm in batch.contig_names], a, r, max_sor,
                                reference=True)
            assert _body(text) == want, (path, a, r)
            _ad_sums_hold(want)
            plain = K.variants_vcf(path, a, r, reference=fasta)
            assert [ln.split("\t")[:6] for ln in _body(plain)] == [ln.split("\t")[:6] for ln in want]


def test_truth_set_on_the_gpu(tmp_path):
    bam, fa, ref, reads = S.write(tmp_path)
    got = S.parse(_body(K.variants_vcf(str(bam), reference=str(fa), strand=True, max_sor=3)))
    one = {k: v for k, v in got.items() if v[0] == "sor"}
    assert {k[0] for k in one} == {S.SNV_ONE + 1, S.INS_AT, S.DEL_AT}
    bal = [v for k, v in got.items() if k[0] == S.SNV_BAL + 1]
    assert bal and bal[0][0] == "PASS" and bal[0][1]["SOR"] == "0.693"


def test_two_gpus_equal_one(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    bam, fa, _, _ = S.write(tmp_path)
    for path, fasta in ((str(bam), str(fa)), (os.path.join(INPUTS, "mm2_gp120.bam"),
                                              os.path.join(INPUTS, "hxb2-gp120-mutated.fa"))):
        for extra in ({}, dict(reference=fasta)):
            assert (K.variants_vcf(path, devices=2, strand=True, max_sor=3, **extra)
                    == K.variants_vcf(path, devices=1, strand=True, max_sor=3, **extra))


def test_cli_end_to_end(tmp_path):
    bam, fa, _, _ = S.write(tmp_path)
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    res = subprocess.run([sys.executable, "-m", "kindel", "variants", "--vcf", "--strand", "--max-sor", "3", str(bam)],
                         capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout == K.variants_vcf(str(bam), strand=True, max_sor=3.0)
    assert "\tsor\t" in res.stdout and "##FILTER=<ID=sor" in res.stdout


def test_bench_strand_parity():
    import json

    res = subprocess.run([sys.executable, os.path.join(H.ROOT, "tools", "bench_strand.py"), "--steps", "3",
                          "--warmup", "1"], capture_output=True, text=True, timeout=3000)
    assert res.returncode == 0, res.stderr[-2000:]
    line = json.loads(res.stdout.strip().splitlines()[-1])
    assert line["parity"] is True, line["parity_detail"]
    assert line["strand_ms"]["k8_select"]["median"] > 0
