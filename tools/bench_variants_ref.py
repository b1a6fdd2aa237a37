"""Bench line of `variants --vcf --reference` (K6r, K7; an extension): BASELINE.json configs[3] (`cfg4_5Mb_200x`, as
bench.py builds it), bench.py's single-GPU step, then K6r and K7 over its last table and batch.

    python tools/bench_variants_ref.py [--steps K] [--warmup W]      # one JSON line on stdout

The timed step is bench.py's.  On top of bench.py's fields the line carries:
  `variant_ref_ms`  K6r's three launches (kdl_variant_ref_count + kdl_variant_ref_scatter), K7's three with the
                    torch grouping and the copy back of the kept deletions (engine.deletion_alleles), K6 and K2, over
                    the last step's table, in 7 alternating rounds of 20 launches, at abs 1 / rel 0.01;
  `e2e_vcf`         variants_vcf(path, reference=fa) against variants_vcf(path) on a 10^6-read BAM, best of 3;
  `gpu`             the card's name and power limit, read in the same run;
  `parity`          K6r's sites equal oracle/py_rvoracle.py's over the host table, K7's kept deletions equal the
                    oracle's walk over the complex reads, and the step's calls equal the C oracle's.
The config-4 contig's FASTA is regenerated from the synthetic generator's seed.  Writes nothing into the tree."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from bench_fastq import alternate  # noqa: E402

WORKLOAD = "cfg4_5Mb_200x"


def contig_text(seed, length):
    from kindel_b200 import bamio, synth

    nib = synth.random_contig(np.random.default_rng(seed), length)
    return np.frombuffer(bamio.NIBBLES.encode(), dtype=np.uint8)[nib].tobytes().decode("ascii")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "power_limit": None, "error": str(e)}


def e2e_vcf(rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub = synth.simple_reads(4, [750_000], 200)  # 10^6 reads, as bench.py's host block
    with tempfile.TemporaryDirectory() as tmp:
        path, fa = os.path.join(tmp, "slice.bam"), os.path.join(tmp, "slice.fa")
        synth.write_simple_bam(path, sub)
        with open(fa, "w") as fh:
            fh.write(">ctg0\n" + contig_text(4, 750_000) + "\n")
        K.variants_vcf(path, reference=fa), K.variants_vcf(path)  # warm
        best = {"reference": None, "sites_only": None}
        for _ in range(rounds):
            for key, fn in (("reference", lambda: K.variants_vcf(path, reference=fa)),
                            ("sites_only", lambda: K.variants_vcf(path))):
                t0 = time.perf_counter()
                text = fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
                if key == "reference":
                    n_ref = text.count("\n") - sum(1 for ln in text.splitlines() if ln.startswith("#"))
    return {"reference_s": best["reference"], "sites_only_s": best["sites_only"], "records": n_ref,
            "reads": int(sub.n_reads), "note": "variants_vcf(path, reference=fa) vs variants_vcf(path), best of %d, "
                                              "alternating" % rounds}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import _ffi, engine
    from kindel_b200.reference import load_reference
    from oracle import coracle
    from oracle import py_oracle as PO
    from oracle import py_rvoracle as RV

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _ffi.load()
    gpu = gpu_info()
    batch = bench.gen_reads(WORKLOAD)
    n_slots = batch.n_slots
    db = engine.upload(batch, dev)
    table = engine.CountTable(n_slots, dev)
    calls_buf = torch.empty(n_slots, dtype=torch.uint8, device=dev)

    def step(timers=None):
        if timers:
            timers[0].record()
        engine.pileup(db, check=False, table=table)
        if timers:
            timers[1].record()
        out = engine.vote(table.t, 1, out=calls_buf)
        if timers:
            timers[2].record()
        return out

    tm = bench.time_steps(step, args.steps, args.warmup, torch, None, 1, dev)
    calls = tm["out"].cpu().numpy()

    with tempfile.TemporaryDirectory() as tmp:
        fa = os.path.join(tmp, "cfg4.fa")
        with open(fa, "w") as fh:
            fh.write(">ctg0\n" + contig_text(4, int(batch.contig_len[0])) + "\n")
        ref = load_reference(fa, batch)
    t_ref = torch.from_numpy(ref.codes).to(dev)
    t_slot = torch.from_numpy(np.asarray(batch.contig_slot, dtype=np.int64)).to(dev)
    t_len = torch.from_numpy(np.asarray(batch.contig_len, dtype=np.int32)).to(dev)
    sums = torch.empty(int(lib.kdl_variant_scratch_words(n_slots)), dtype=torch.int32, device=dev)
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    a, r = 1, 0.01
    fl = engine.variant_abs_floor(a)
    sites = engine.variant_sites_ref(table.t, batch.contig_slot, batch.contig_len, t_ref, a, r)
    n = len(sites[0])
    k6n = len(engine.variant_sites(table.t, batch.contig_slot, batch.contig_len, a, r)[0])
    o_slot = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    o_cnt = torch.empty((7, max(n, 1)), dtype=torch.int32, device=dev)
    o_dpa = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    o_mask = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    o6_slot = torch.empty(max(k6n, 1), dtype=torch.int64, device=dev)
    o6_cnt = torch.empty((6, max(k6n, 1)), dtype=torch.int32, device=dev)
    o6_mask = torch.empty(max(k6n, 1), dtype=torch.uint8, device=dev)
    vote_buf = torch.empty(n_slots, dtype=torch.uint8, device=dev)

    def k6r():
        base = (table.t.data_ptr(), n_slots, t_slot.data_ptr(), t_len.data_ptr(), batch.n_contigs, t_ref.data_ptr(),
                fl, r, sums.data_ptr())
        lib.kdl_variant_ref_count(*base, st)
        lib.kdl_variant_ref_scatter(*base, n, o_slot.data_ptr(), o_cnt.data_ptr(), o_dpa.data_ptr(),
                                    o_mask.data_ptr(), st)

    def k6():
        base = (table.t.data_ptr(), n_slots, t_slot.data_ptr(), t_len.data_ptr(), batch.n_contigs, fl, r,
                sums.data_ptr())
        lib.kdl_variant_count(*base, st)
        lib.kdl_variant_scatter(*base, k6n, o6_slot.data_ptr(), o6_cnt.data_ptr(), o6_mask.data_ptr(), st)

    timing = alternate((("k2_vote", lambda: engine.vote(table.t, 1, out=vote_buf)), ("k6_variants", k6),
                        ("k6r_variants_ref", k6r),
                        ("k7_deletions", lambda: engine.deletion_alleles(db, table.t, a, r))), torch)
    dels = engine.deletion_alleles(db, table.t, a, r)
    timing.update(abs_threshold=a, rel_threshold=r, k6r_sites=n, k6_sites=k6n, deletions_kept=int(len(dels[0])),
                  k6r_bytes=2 * 29 * n_slots + n * 49,
                  # K7: l_seq of every read, [n_ops][evt_off][ops] of every complex read
                  k7_bytes=4 * int(batch.n_reads) + int(
                      (8 + 4 * np.diff(np.asarray(batch.cig_off, dtype=np.int64))[np.asarray(batch.complex_idx)]).sum()),
                  note="k7_deletions includes the 4-byte read-back of the event total, the torch grouping and the "
                       "copy back of the kept deletions")
    e2e = e2e_vcf()

    host = table.t.cpu().numpy()
    parity_sites = all(np.array_equal(x, y) for x, y in zip(
        sites, RV.sites(host, batch.contig_slot, batch.contig_len, ref.codes, a, r)))
    groups = {}
    for rd in np.asarray(batch.complex_idx).tolist():
        for ev in RV.deletion_events(int(batch.contig_len[0]), PO.records_of(batch, rd, rd + 1)):
            groups[ev] = groups.get(ev, 0) + 1
    want = sorted((s, ln, c, int(host[0:6, s].astype(np.int64).sum())) for (s, ln), c in groups.items())
    want = [w for w in want if w[2] > a and w[2] / w[3] > r]
    parity_dels = list(zip(*[x.tolist() for x in dels])) == want
    want_calls = coracle.vote(coracle.pileup(batch)[0], 1)
    parity = bool(parity_sites and parity_dels and np.array_equal(calls, want_calls))
    ms_per_step = tm["total_ms"] / tm["reps"]
    line = {
        "metric": bench.METRIC, "value": batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": parity, "parity_detail": {"k6r_sites": bool(parity_sites), "k7_deletions": bool(parity_dels)},
        "config": {"workload": WORKLOAD, "reads_per_rank": int(batch.n_reads),
                   "complex_reads_per_rank": int(batch.n_complex), "aligned_bases_total": int(batch.aligned_bases),
                   "tool": "tools/bench_variants_ref.py",
                   "parity_oracle": "oracle/py_rvoracle.py over the host table and the complex reads' records; the "
                                    "step's calls against oracle/kindel_oracle.c"},
        "gpu": gpu, "variant_ref_ms": timing, "e2e_vcf": e2e, "e2e": None,
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
