"""The variant sites (`variants --only-variants`) and the sites-only VCF (`variants --vcf`; extensions) on the GPU: K6
equals the per-position restatement (oracle/py_voracle.py) on fuzz and adversarial tables, one by one and concatenated
into one launch, and on the full config-4 table; a device run gives the host code's frame and VCF over the oracle's
tables; the CLI writes the API's VCF; K6 adds exactly its three launches to `variants -o`; two GPUs equal one."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

import combo_cases as CC
import helpers as H
from conftest import golden_input
from kindel_b200 import _ffi, bamio, engine, synth
from kindel_b200 import kindel as K
from oracle import coracle, py_voracle as V
from test_variants_vcf import GRID, _fuzz_runs, _oracle_run, _sites_equal, adversarial, combo_run

pytestmark = pytest.mark.gpu
NAN = float("nan")


def _device_sites(table, cs, cl, a, r):
    import torch

    t = torch.from_numpy(np.ascontiguousarray(table, dtype=np.int32)).cuda()
    return engine.variant_sites(t, cs, cl, a, r)


def _tables(tmp_path):
    out = [(n, r.host_counts, r.batch.contig_slot, r.batch.contig_len) for n, r in _fuzz_runs(tmp_path)]
    out += [("adversarial%d" % s,) + adversarial(s) for s in (1, 2, 3, 4)]
    out.append(("empty", np.zeros((19, 2052), dtype=np.int32), np.array([0, 1030]), np.array([1000, 1020])))
    return out


def test_k6_equals_restatement_on_fuzz_and_adversarial_tables(tmp_path):
    tables = _tables(tmp_path)
    # all of them in one launch: the contig layouts shifted by each table's offset in the concatenation
    parts, cs_all, cl_all, off = [], [], [], 0
    for _, t, cs, cl in tables:
        n = (t.shape[1] + 3) // 4 * 4
        part = np.zeros((19, n), dtype=np.int32)
        part[:, :t.shape[1]] = t
        parts.append(part)
        cs_all.append(np.asarray(cs, dtype=np.int64) + off)
        cl_all.append(np.asarray(cl, dtype=np.int64))
        off += n
    big, cs_all, cl_all = np.concatenate(parts, axis=1), np.concatenate(cs_all), np.concatenate(cl_all)
    n_sites = 0
    for a, r in GRID:
        want = V.sites(big, cs_all, cl_all, a, r)
        _sites_equal(_device_sites(big, cs_all, cl_all, a, r), want, ("concatenated", a, r))
        n_sites += len(want[0])
    assert n_sites > 100_000
    for name, t, cs, cl in tables:
        for a, r in GRID[::4]:
            _sites_equal(_device_sites(t, cs, cl, a, r), V.sites(t, cs, cl, a, r), (name, a, r))


def test_k6_on_the_full_config4_table():
    """cfg 4 (5 Mb x 200x, 1 % substitutions, ~1 % indel / clip reads) at the default and a high rel threshold."""
    batch = synth.mixed_reads(4, [5_000_000], 200, 0.01)
    counts, _ = engine.pileup(engine.upload(batch))
    host = counts.cpu().numpy()
    n = []
    for a, r in ((1, 0.01), (2, 0.05)):
        got = engine.variant_sites(counts, batch.contig_slot, batch.contig_len, a, r)
        _sites_equal(got, V.sites(host, batch.contig_slot, batch.contig_len, a, r), ("cfg4", a, r))
        n.append(len(got[0]))
    assert n[0] > 1_000_000 and n[1] > 0


def _paths(manifest, tmp_path):
    """(path, filters, the oracle's host run) of the golden fixtures and the combo corpus, the latter with and without
    the filters."""
    out = [(golden_input(e), (0, 0, 0), None) for e in manifest["files"].values()]
    for seed in (0, 1):
        contigs, recs = CC.combo_case(seed)
        path = CC.write_bam(tmp_path / ("combo%d.bam" % seed), contigs, recs)
        for flt in ((0, 0, 0), (20, 10, 0x400)):
            out.append((path, flt, combo_run(contigs, recs, path, flt, tmp_path / ("piled%d.bam" % seed))))
    return out


def _host(path, flt, run):
    return run if run is not None else _oracle_run(bamio.read_alignment(path))


def _kw(filters):
    return dict(min_base_quality=filters[0], min_mapq=filters[1], exclude_flags=filters[2])


def test_only_variants_on_device_equals_host_tables(manifest, tmp_path):
    n = 0
    for k, (path, flt, run) in enumerate(_paths(manifest, tmp_path)):
        host = _host(path, flt, run)
        for a, r in ((1, 0.01), (0, 0.2), (-1, -0.5))[: 3 if k % 4 == 0 else 2]:
            for absolute in (False, True):
                got = K.variants(path, a, r, True, absolute, **_kw(flt))
                pd.testing.assert_frame_equal(got, K.variants_from_run(host, a, r, True, absolute))
                n += len(got)
    assert n > 1000


def test_vcf_on_device_equals_host_tables(manifest, tmp_path):
    for path, flt, run in _paths(manifest, tmp_path):
        host = _host(path, flt, run)
        for a, r in ((1, 0.01), (2, 0.25)):
            assert K.variants_vcf(path, a, r, **_kw(flt)) == K.variants_vcf_from_run(host, a, r, flt), (path, flt)


def test_cli(manifest, tmp_path):
    path = golden_input(next(iter(manifest["files"].values())))
    env = dict(os.environ, PYTHONPATH=H.ROOT)

    def run(*args):
        res = subprocess.run([sys.executable, "-m", "kindel", "variants", *args, path], capture_output=True, text=True,
                             env=env, timeout=900)
        assert res.returncode == 0, res.stderr[-2000:]
        return res.stdout

    assert run("--vcf") == K.variants_vcf(path)
    assert run("--vcf", "-a", "2", "-r", "0.2", "--min-mapq", "1") == K.variants_vcf(path, 2, 0.2, min_mapq=1)
    host = _host(path, (0, 0, 0), None)
    assert run("-o") == K.variants_from_run(host, 1, 0.01, True).to_csv(sep="\t", index=False)
    assert run("-o", "--absolute", "--gpus", "1") == K.variants_from_run(host, 1, 0.01, True, True).to_csv(
        sep="\t", index=False)


def test_launch_count(manifest):
    """`variants -o` = the pileup's launches + K6's three (sums, scan, scatter), sites or not; the VCF the same."""
    lib = _ffi.load()
    path = golden_input(next(iter(manifest["files"].values())))

    def launches(fn):
        fn()  # warm
        n0 = lib.kdl_launch_count()
        fn()
        return lib.kdl_launch_count() - n0

    pileup = launches(lambda: K.pileup_run(path))
    assert launches(lambda: K.variants(path, only_variants=True)) == pileup + 3
    assert launches(lambda: K.variants(path, 10 ** 12, 0.5, only_variants=True)) == pileup + 3  # no site
    assert launches(lambda: K.variants_vcf(path)) == pileup + 3


def test_two_gpus_equal_one(manifest, tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    for path, flt, _ in _paths(manifest, tmp_path)[-3:]:
        assert K.variants_vcf(path, devices=2, **_kw(flt)) == K.variants_vcf(path, devices=1, **_kw(flt))
