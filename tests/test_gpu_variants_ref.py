"""`variants --vcf --reference` (extension) on the GPU: K6r and K7 equal oracle/py_rvoracle.py on the fuzz corpus
(K6r over all its tables concatenated into one launch) and on the full config-4 table with its regenerated FASTA;
variants_vcf(path, reference=...) and the CLI equal the oracle's VCF byte for byte on synthetic BAMs with indels and on
mm2_gp120.bam with its reference; on a truth set with every planted fraction above 0.5 the VCF lists the planted
alleles and, applied to the FASTA, gives bam_to_consensus's sequence; two GPUs equal one."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
from kindel_b200 import bamio, engine, synth
from kindel_b200 import kindel as K
from kindel_b200.reference import load_reference
from oracle import py_oracle as PO
from oracle import py_rvoracle as RV
from test_variants_ref import (_groups, _parse, _sites_equal, bam_records, corpus, expected_alleles, ref_adversarial,
                               truth_set)
from test_variants_vcf import GRID

pytestmark = pytest.mark.gpu
GP120 = os.path.join(H.ROOT, "tests", "golden", "inputs")


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_k6r_and_k7_on_the_fuzz_corpus(tmp_path):
    items = corpus(tmp_path)
    tables = [(name, table, b.contig_slot, b.contig_len, codes) for name, b, table, codes, _ in items]
    tables += [("adversarial%d" % s,) + ref_adversarial(s)[:3] + (ref_adversarial(s)[3],) for s in (1, 2)]
    parts, cparts, cs_all, cl_all, off = [], [], [], [], 0
    for _, t, cs, cl, codes in tables:
        n = (t.shape[1] + 3) // 4 * 4
        part = np.zeros((19, n), dtype=np.int32)
        part[:, :t.shape[1]] = t
        cp = np.full(n, 4, dtype=np.uint8)
        cp[:t.shape[1]] = codes
        parts.append(part)
        cparts.append(cp)
        cs_all.append(np.asarray(cs, dtype=np.int64) + off)
        cl_all.append(np.asarray(cl, dtype=np.int64))
        off += n
    big, codes = np.concatenate(parts, axis=1), np.concatenate(cparts)
    cs_all, cl_all = np.concatenate(cs_all), np.concatenate(cl_all)
    t_big, t_codes = _dev(big), _dev(codes)
    n_sites = 0
    for a, r in GRID[::3] + [(1, 0.01), (0, 0.0)]:
        want = RV.sites(big, cs_all, cl_all, codes, a, r)
        _sites_equal(engine.variant_sites_ref(t_big, cs_all, cl_all, t_codes, a, r), want, ("concatenated", a, r))
        n_sites += len(want[0])
    assert n_sites > 50_000
    n_events = 0
    for name, batch, _, _, groups in items:  # K7: the events in read order, then op order
        slot, length = engine.deletion_events(engine.upload(batch))
        want = []
        for c, nm in enumerate(batch.contig_names):
            s0 = int(batch.contig_slot[c])
            want += [(s0 + r, n) for r, n in RV.deletion_events(int(batch.contig_len[c]), groups.get(nm, []))]
        assert list(zip(slot.cpu().tolist(), length.cpu().tolist())) == want, name
        n_events += len(want)
    assert n_events > 200


def cfg4_reference_text():
    """The config-4 contig as synth.simple_reads draws it from seed 4: its first draw from default_rng(4)."""
    nib = synth.random_contig(np.random.default_rng(4), 5_000_000)
    return np.frombuffer(bamio.NIBBLES.encode(), dtype=np.uint8)[nib].tobytes().decode("ascii")


def test_k6r_and_k7_on_the_full_config4_table(tmp_path):
    batch = synth.mixed_reads(4, [5_000_000], 200, 0.01)
    fa = tmp_path / "cfg4.fa"
    fa.write_text(">ctg0\n" + cfg4_reference_text() + "\n")
    ref = load_reference(fa, batch)
    db = engine.upload(batch)
    counts, _ = engine.pileup(db)
    host = counts.cpu().numpy()
    n = []
    for a, r in ((1, 0.01), (2, 0.05)):
        got = engine.variant_sites_ref(counts, batch.contig_slot, batch.contig_len, ref.codes, a, r)
        _sites_equal(got, RV.sites(host, batch.contig_slot, batch.contig_len, ref.codes, a, r), ("cfg4", a, r))
        n.append(len(got[0]))
    assert n[0] > 10_000 and n[1] > 0
    # K7 + the grouping against the oracle's walk over the complex reads' records (simple reads have no D op)
    groups = {}
    for r in np.asarray(batch.complex_idx).tolist():
        for ev in RV.deletion_events(5_000_000, PO.records_of(batch, r, r + 1)):
            groups[ev] = groups.get(ev, 0) + 1
    for a, r in ((0, 0.0), (1, 0.001)):
        got = engine.deletion_alleles(db, counts, a, r)
        want = sorted((s, n, c, int(host[0:6, s].astype(np.int64).sum())) for (s, n), c in groups.items()
                      if c > a and c / int(host[0:6, s].astype(np.int64).sum()) > r)
        assert list(zip(*[x.tolist() for x in got])) == want
        assert len(want) > (40_000 if a == 0 else 0)


def _oracle_body(path, fasta, a, r):
    lens, groups = _groups(path) if str(path).endswith(".sam") else _bam_groups(path)
    batch = bamio.read_alignment(path)
    codes = load_reference(fasta, batch).codes
    texts = {nm: "".join("ACGTN"[x] for x in codes[s0:s0 + L].tolist())
             for nm, s0, L in zip(batch.contig_names, batch.contig_slot.tolist(), batch.contig_len.tolist())}
    return RV.vcf_lines([(nm, texts[nm], groups.get(nm, [])) for nm in batch.contig_names], a, r)


def _bam_groups(path):
    from oracle import samdecode

    header, records = samdecode.read_alignment_file(path)
    groups = {}
    for rec in records:
        groups.setdefault(rec.rname, []).append(rec)
    groups.pop("*", None)
    return None, groups


def _inputs(tmp_path):
    """(BAM path, FASTA path) of the synthetic indel BAMs and of mm2_gp120.bam."""
    out = []
    for seed, high in ((1, False), (2, False), (3, True)):
        ref, reads, _ = truth_set(seed, high=high, n_plain=0 if high else 25)
        bam, fa = tmp_path / ("truth%d.bam" % seed), tmp_path / ("truth%d.fa" % seed)
        bamio.write_bam(bam, [("t", len(ref))], bam_records(reads))
        fa.write_text(">t description\n" + "\n".join(ref[i:i + 60] for i in range(0, len(ref), 60)) + "\n")
        out.append((bam, fa))
    cx = synth.complex_reads(9, 3000, 30)  # clips, indels and the edge tail (POS 0, N / H / P ops, mid-read S)
    contigs, recs = synth.to_records(cx)
    bam, fa = tmp_path / "complex.bam", tmp_path / "complex.fa.gz"
    bamio.write_bam(bam, contigs, recs)
    import gzip

    text = cfg4_reference_text()[:3000]
    fa.write_bytes(gzip.compress((">ctg0\n" + text + "\n").encode()))
    out.append((bam, fa))
    out.append((os.path.join(GP120, "mm2_gp120.bam"), os.path.join(GP120, "hxb2-gp120-mutated.fa")))
    return out


def test_vcf_and_cli_equal_the_oracle(tmp_path):
    env = dict(os.environ, PYTHONPATH=H.ROOT)
    n = 0
    for k, (bam, fa) in enumerate(_inputs(tmp_path)):
        for a, r in ((1, 0.01), (0, 0.0), (2, 0.2)):
            text = K.variants_vcf(str(bam), a, r, reference=str(fa))
            lines = text.splitlines()
            body = [ln for ln in lines if not ln.startswith("#")]
            assert "##reference=" + os.path.basename(str(fa)) in lines
            assert body == _oracle_body(bam, fa, a, r), (bam, a, r)
            assert text.endswith("\n")
            n += len(body)
        res = subprocess.run([sys.executable, "-m", "kindel", "variants", "--vcf", "--reference", str(fa), str(bam)],
                             capture_output=True, text=True, env=env, timeout=900)
        assert res.returncode == 0, res.stderr[-2000:]
        assert res.stdout == K.variants_vcf(str(bam), reference=str(fa))
    assert n > 300
    # without --reference the VCF is the sites-only one, whatever reference mode did before it
    bam = os.path.join(GP120, "mm2_gp120.bam")
    assert "##reference" not in K.variants_vcf(bam) and "INDEL" not in K.variants_vcf(bam)


def _apply(ref, alleles):
    """The reference with alleles (kind, where, allele) applied: an SNV at a position, an insertion before the base of
    a slot, a deletion of `allele` bases from a position."""
    L = len(ref)
    base, ins = list(ref), [""] * (L + 1)
    for kind, w, a in alleles:
        if kind == "snv":
            base[w] = a
        elif kind == "ins":
            ins[w] += a
        else:
            for p in range(w, w + a):
                base[p] = ""
    return "".join(ins[p] + base[p] for p in range(L)) + ins[L]


def test_truth_set_above_one_half(tmp_path):
    ref, reads, planted = truth_set(3, high=True, n_plain=0)
    bam, fa = tmp_path / "t.bam", tmp_path / "t.fa"
    bamio.write_bam(bam, [("t", len(ref))], bam_records(reads))
    fa.write_text(">t\n" + ref + "\n")
    text = K.variants_vcf(str(bam), 0, 0.0, reference=str(fa))
    body = [ln for ln in text.splitlines() if not ln.startswith("#")]
    got = _parse(body)
    want = expected_alleles(ref, planted)
    assert {k: v[0] for k, v in got.items()} == want
    # every record has AF > 0.5; applied to the FASTA they give the consensus.  (The VCF equals the planted alleles,
    # so they are applied in the generator's terms.)  kindel's consensus never emits the insertions behind the last
    # base (slot L), so that one is left out.
    assert all(float(info["AF"]) > 0.5 for _, info in got.values())
    res = K.bam_to_consensus(str(bam), uppercase=True)
    alleles = [(kind, w, a) for kind, w, a, _ in planted if not (kind == "ins" and w == len(ref))]
    assert _apply(ref, alleles) == res.consensuses[0].sequence


def test_two_gpus_equal_one(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    for bam, fa in _inputs(tmp_path)[-3:]:
        assert K.variants_vcf(str(bam), devices=2, reference=str(fa)) == K.variants_vcf(str(bam), devices=1,
                                                                                        reference=str(fa))
