#!/usr/bin/env python
"""Multi-sample VCF (`kindel variants --vcf a.bam b.bam ...`) on one GPU: one JSON line per workload.

Workloads (synthetic, seeded; every sample has reads of its own over one shared contig and four planted alleles of
its own, tests/cohort_cases.py):
  plate96_30kb_1000x   96 samples of 30 kb at 1 000x   (a viral plate)
  bact8_5Mb_100x       8 samples of 5 Mb at 100x       (a bacterial set)

Fields beside bench.py's shape (`value` = aligned bases/s through variants_vcf(paths), `ms_per_step` its time):
  cohort_ms.kernels        K6m's count pass over the stacked table T, pooled and reference mode, against S count
                           passes of K6 / K6r over the same tables (medians of alternating rounds, CUDA events);
                           bytes read per pass: 24 * S (pooled) or 29 * S (reference, + 1 B of reference) per slot
  cohort_ms.phases_s       pileups (pileup_run of every sample), stack (Cohort's build minus its pileups), deletion
                           union, records + text (K6m, the gathers, the formatting)
  cohort_ms.e2e_s          variants_vcf(paths) against a loop of variants_vcf(path) in one process -- which leaves
                           out each `kindel` call's own start-up (torch import, CUDA context, library load), so it
                           understates what one call instead of S saves
  parity                   plate: the VCF's sha256 against oracle/py_msoracle.py over the C oracle's tables;
                           bacterial set: K6m's sites against a vectorised numpy restatement of the pooled rule
Card name and power limit are read in the same run.  Writes nothing into the tree (samples go to a temporary
directory); --out DIR writes one file per workload there."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

WORKLOADS = {"plate96_30kb_1000x": (96, 30_000, 1000), "bact8_5Mb_100x": (8, 5_000_000, 100)}
HBM_TBPS = 3.35  # H100 SXM data sheet


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "power_limit": None, "error": str(e)}


def contig_text(seed, length):
    from kindel_b200 import bamio, synth

    nib = synth.random_contig(np.random.default_rng(seed), length)
    return np.frombuffer(bamio.NIBBLES.encode(), dtype=np.uint8)[nib].tobytes().decode("ascii")


def _stats(xs):
    return {"min": float(min(xs)), "median": float(np.median(xs)), "max": float(max(xs))}


def kernel_times(cohort, ref_codes, rounds=7, reps=10):
    """K6m vs S x K6 (pooled) and vs S x K6r (reference) over T, alternating, CUDA events; ms per selection."""
    import torch

    from kindel_b200 import _ffi, engine

    lib = _ffi.load()
    T = cohort.table
    S, _, n = T.shape
    lay = cohort.layout
    dev = T.device
    ref = torch.from_numpy(ref_codes).to(dev)
    t_slot, t_len, n_contigs = engine._device_layout(lay.contig_slot, lay.contig_len, dev)
    sums = torch.empty(int(lib.kdl_variant_scratch_words(n)), dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    a, r = 1, 0.01
    per = {}

    def sites_count(fn):
        fn()
        torch.cuda.synchronize()
        return int(sums[-1].item())

    def k6m(refp):
        return lambda: lib.kdl_variant_multi_count(T.data_ptr(), S, n, t_slot.data_ptr(), t_len.data_ptr(), n_contigs,
                                                   refp, a, r, sums.data_ptr(), st)

    def k6_loop():
        for i in range(S):
            lib.kdl_variant_count(T[i].data_ptr(), n, t_slot.data_ptr(), t_len.data_ptr(), n_contigs, a, r,
                                  sums.data_ptr(), st)

    def k6r_loop():
        for i in range(S):
            lib.kdl_variant_ref_count(T[i].data_ptr(), n, t_slot.data_ptr(), t_len.data_ptr(), n_contigs,
                                      ref.data_ptr(), a, r, sums.data_ptr(), st)

    # the count pass is what is timed: the scatter pass reads the same bytes again and writes the few sites
    fns = {"k6m_pooled": k6m(None), "k6_loop": k6_loop, "k6m_reference": k6m(ref.data_ptr()), "k6r_loop": k6r_loop}
    n_sites = {k: sites_count(f) for k, f in fns.items() if k.startswith("k6m")}
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, f in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                f()
            e1.record()
            e1.synchronize()
            per.setdefault(k, []).append(e0.elapsed_time(e1) / reps)
    out = {k: _stats(v) for k, v in per.items()}
    for mode, b in (("pooled", 24), ("reference", 29)):
        bytes_ = b * S * n
        ms = out["k6m_" + mode]["median"]
        out["k6m_%s_bytes_per_pass" % mode] = bytes_
        out["k6m_%s_tb_per_s" % mode] = bytes_ / (ms * 1e-3) / 1e12
        out["k6m_%s_share_of_datasheet_hbm" % mode] = bytes_ / (ms * 1e-3) / 1e12 / HBM_TBPS
    out["sites"] = n_sites
    out["n_slots"] = n
    out["note"] = ("count pass (per-CTA sums + scan) of each selection, ms per selection; the share is of the "
                   "H100 SXM data sheet's %.2f TB/s, not a measured peak" % HBM_TBPS)
    return out


def run_workload(name, tmp):
    import pathlib

    import torch

    import cohort_cases as CO
    from kindel_b200 import __version__, bamio, cohort, engine
    from kindel_b200 import kindel as K

    S, L, depth = WORKLOADS[name]
    d = pathlib.Path(tmp) / name
    d.mkdir()
    t0 = time.perf_counter()
    samples = CO.synthetic_samples(d, S, L, depth, progress=True)
    gen_s = time.perf_counter() - t0
    print("%s: %d samples written in %.1f s" % (name, S, gen_s), file=sys.stderr, flush=True)
    paths = [p for p, _ in samples]
    bases = int(sum(int(np.asarray(b.l_seq).sum()) for _, b in samples))
    fa = str(d / "ref.fa")
    with open(fa, "w") as fh:
        fh.write(">ctg0\n" + contig_text(4, L) + "\n")
    K.variants_vcf(paths[:2]), K.variants_vcf(paths[0])  # warm: modules, allocator

    # phases
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for p in paths:
        run = K.pileup_run(p)[0]
        run.device_tables()
        del run
    torch.cuda.synchronize()
    pile_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    co = cohort.Cohort(paths)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    from kindel_b200.reference import load_reference

    ref_codes = load_reference(fa, co.layout).codes
    t0 = time.perf_counter()
    engine.deletion_union(co.deletions, co.table, 1, 0.01)
    union_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    pooled_lines = cohort.records(co, None, 1, 0.01)
    text_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    cohort.records(co, ref_codes, 1, 0.01)
    text_ref_s = time.perf_counter() - t0
    kern = kernel_times(co, ref_codes)
    peak = torch.cuda.max_memory_allocated() / 1e9

    print("%s: phases and kernels timed" % name, file=sys.stderr, flush=True)
    # end to end, alternating
    e2e = {"joint": [], "loop": []}
    for _ in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        joint = K.variants_vcf(paths)
        e2e["joint"].append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        for p in paths:
            K.variants_vcf(p)
        e2e["loop"].append(time.perf_counter() - t0)

    # parity
    if name.startswith("plate"):
        from oracle import coracle
        from oracle import py_msoracle as MS

        oracle = []
        for p in paths:
            b = bamio.read_alignment(p)
            t, _ = coracle.pileup(b)
            oracle.append(MS.Sample.from_table(b.contig_names, b.contig_len, b.contig_slot, t))
        want = MS.vcf(oracle, [os.path.basename(p) for p in paths], "kindel {}".format(__version__), 1, 0.01)
        parity = hashlib.sha256(joint.encode()).hexdigest() == hashlib.sha256(want.encode()).hexdigest()
        parity_detail = {"vcf_sha256": hashlib.sha256(joint.encode()).hexdigest(), "oracle": "oracle/py_msoracle.py "
                         "over oracle/kindel_oracle.c tables", "records": len(pooled_lines)}
    else:
        passes = np.zeros((6, L), dtype=bool)
        pooled = np.zeros((6, L), dtype=np.int64)
        for i in range(S):  # one contig at slot 0
            t = co.table[i, 0:6, :L].cpu().numpy().astype(np.int64)
            depth = t.sum(axis=0)
            with np.errstate(invalid="ignore", divide="ignore"):
                share = np.where(depth > 0, t / np.maximum(depth, 1), 0.0)
            passes |= (t > 1) & (share > 0.01)
            pooled += t
        top = pooled.argmax(axis=0)
        passes[top, np.arange(L)] = False
        want_slot = np.flatnonzero(passes.any(axis=0))
        want_mask = (passes[:, want_slot].astype(np.uint8) << np.arange(6, dtype=np.uint8)[:, None]).sum(
            axis=0, dtype=np.uint8)
        slot, mask = engine.variant_sites_multi(co.table, co.layout.contig_slot, co.layout.contig_len, None, 1, 0.01)
        parity = bool(np.array_equal(slot.cpu().numpy(), want_slot) and np.array_equal(mask.cpu().numpy(), want_mask))
        parity_detail = {"k6m_sites": int(want_slot.size), "oracle": "numpy restatement of the pooled site rule over "
                         "T copied to the host", "records": len(pooled_lines)}
    joint_s = float(np.median(e2e["joint"]))
    return {
        "metric": "aligned bases/sec through variants_vcf(paths)", "value": bases / joint_s,
        "unit": "aligned_bases/s", "n_gpus": 1, "ms_per_step": joint_s * 1e3, "higher_is_better": True,
        "data": "synthetic", "parity": parity, "parity_detail": parity_detail,
        "config": {"workload": "cohort_" + name, "samples": S, "contig_len": L, "depth": depth,
                   "aligned_bases_total": bases, "tool": "tools/bench_cohort.py", "sample_generation_s": gen_s},
        "gpu": gpu_info(),
        "cohort_ms": {"kernels": kern,
                      "phases_s": {"pileups": pile_s, "stack": build_s - pile_s, "cohort_build": build_s,
                                   "deletion_union": union_s, "records_text_pooled": text_s,
                                   "records_text_reference": text_ref_s,
                                   "note": "stack = Cohort's build (pileups + gathers + event decode) minus the "
                                           "pileups timed alone"},
                      "e2e_s": {"variants_vcf_paths": _stats(e2e["joint"]), "loop_variants_vcf_path": _stats(
                          e2e["loop"]), "note": "one process; each separate `kindel` call would also pay its own "
                                                "start-up, which this leaves out"},
                      "peak_device_gb": peak, "stacked_table_gb": 28 * S * co.layout.n_slots / 1e9},
    }


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workload", choices=sorted(WORKLOADS), action="append")
    ap.add_argument("--out", default=None, help="directory for one JSON file per workload")
    args = ap.parse_args(argv)
    from kindel_b200 import engine

    engine.require_cuda()
    with tempfile.TemporaryDirectory() as tmp:
        for name in args.workload or list(WORKLOADS):
            line = json.dumps(run_workload(name, tmp))
            print(line, flush=True)
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                with open(os.path.join(args.out, "h100_bench_n1_cohort_%s.json" % name), "w") as fh:
                    fh.write(line + "\n")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
