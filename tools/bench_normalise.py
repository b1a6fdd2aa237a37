"""Bench line of depth normalisation (`--normalise N`, K13; an extension): bench.py's single-GPU step over
BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds it), then K12 and K13 over two amplicon workloads with
seeded strands (synth.with_strands), each with synth.tiled_scheme's rows as a named BED (synth.named_scheme_bed) and
the cap N = 200:

  cfg4_amplicon  synth.amplicon_reads at cfg 4's size: 6.67 M reads over 5 Mb, 24 999 amplicons, ~133 reads per
                 (amplicon, strand)
  deep_30kb      synth.amplicon_reads over 30 kb at 5 000x: ~10^6 reads, 149 amplicons, ~3 300 reads per (amplicon,
                 strand), so most reads are over the cap

    python tools/bench_normalise.py [--steps K] [--warmup W]      # one JSON line on stdout

On top of bench.py's fields the line carries, per workload (`normalise_ms`):
  `ms`        K13 (kdl_normalise: its three launches K13c, K13s and K13m, into preallocated outputs), K12
              (kdl_amplicons_assign) and K0 + K1 (the pileup into a reused table) for scale, in 7 alternating rounds of
              20 launches; the reads, amplicons, dropped reads and K13's grid and scratch;
  `select_reads_s`  the host rebuild of the batch from the kept reads (bamio.select_reads), best of 3;
  `parity`    the keep bytes have the sha256 of oracle/py_noracle.py's keep_vectorised over oracle/py_aoracle.py's
              labels_of_batch, and the dropped count is theirs.
`e2e_normalise` times bam_to_consensus(path, primers=bed, normalise=200) against bam_to_consensus(path, primers=bed) on
a 10^6-read amplicon BAM, best of 3, alternating; `gpu` is the card's name and power limit, read in the same run.
Writes nothing into the tree."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from bench_amplicons import tiled_named_rows  # noqa: E402
from bench_fastq import alternate  # noqa: E402
from bench_variants_ref import gpu_info  # noqa: E402

WORKLOAD = "cfg4_5Mb_200x"
CAP = 200


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def normalise_workload(batch, rows, torch, dev):
    import ctypes as C

    from kindel_b200 import _ffi, bamio, engine, primers
    from kindel_b200 import synth
    from oracle import py_aoracle, py_noracle

    lib = _ffi.load()
    scheme = primers.read_scheme(synth.named_scheme_bed(rows).encode(), "scheme.bed")
    arrays = primers.amplicon_arrays(scheme, batch.contig_names, batch.contig_len)
    db = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    labels = engine.assign_amplicons(db, arrays)
    reverse = torch.from_numpy(batch.reverse).to(dev)
    keep, total, dropped = engine.normalise(labels, reverse, arrays.n_amplicons, CAP)
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    a, hold = engine._amplicons_on(arrays, dev)
    n, n_amp = int(batch.n_reads), arrays.n_amplicons
    words = int(lib.kdl_normalise_scratch_words(n, n_amp))
    scratch = torch.empty(max(words, 1), dtype=torch.int32, device=dev)
    lab_buf, keep_buf = torch.empty_like(labels), torch.empty_like(keep)
    tot_buf, drop_buf = torch.empty_like(total), torch.empty_like(dropped)

    def k12():
        lib.kdl_amplicons_assign(C.byref(db.struct), C.byref(a), lab_buf.data_ptr(), st)

    def k13():
        lib.kdl_normalise(labels.data_ptr(), reverse.data_ptr(), n, n_amp, CAP, scratch.data_ptr(), words,
                          keep_buf.data_ptr(), tot_buf.data_ptr(), drop_buf.data_ptr(), st)

    timing = alternate((("k0_k1_pileup", lambda: engine.pileup(db, check=False, table=table)), ("k12_assign", k12),
                        ("k13_normalise", k13)), torch)
    same = bool(torch.equal(keep_buf, keep) and torch.equal(tot_buf, total) and torch.equal(drop_buf, dropped)
                and torch.equal(lab_buf, labels))
    got = keep.cpu().numpy()
    n_drop = int(dropped.item())
    idx = np.flatnonzero(got)
    best = None
    for _ in range(3):
        t0 = time.perf_counter()
        bamio.select_reads(batch, idx)
        dt = time.perf_counter() - t0
        best = dt if best is None or dt < best else best
    timing.update(reads=n, amplicons=n_amp, cap=CAP, dropped=n_drop, kept=n - n_drop,
                  largest_group=int(total.max().item()) if n_amp else 0,
                  k13_grid=words // max(2 * n_amp, 1), k13_scratch_bytes=4 * words, select_reads_s=best,
                  note="k13_normalise: kdl_normalise (K13c + K13s + K13m) over preallocated outputs; k12_assign: "
                       "kdl_amplicons_assign; k0_k1_pileup: engine.pileup into a reused CountTable; select_reads_s: "
                       "bamio.select_reads(batch, kept), best of 3, host")
    print("normalise: timed %d reads, checking against the oracle" % n, file=sys.stderr, flush=True)
    want = py_noracle.keep_vectorised(py_aoracle.labels_of_batch(batch, tiled_named_rows(rows)), batch.reverse, CAP)
    detail = {"keep_sha256": sha(got), "oracle_keep_sha256": sha(want), "dropped": n_drop,
              "oracle_dropped": int((want == 0).sum())}
    detail["parity"] = bool(sha(got) == sha(want) and n_drop == detail["oracle_dropped"] and same)
    del hold
    return timing, detail


def e2e(rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub, rows = synth.amplicon_reads(4, 750_000, 200)  # 10^6 reads, as bench.py's host block
    sub = synth.with_strands(sub, 4)
    with tempfile.TemporaryDirectory() as tmp:
        path, bed = os.path.join(tmp, "amp.bam"), os.path.join(tmp, "scheme.bed")
        synth.write_simple_bam(path, sub)
        with open(bed, "w") as fh:
            fh.write(synth.named_scheme_bed(rows))
        on = lambda: K.bam_to_consensus(path, primers=bed, normalise=CAP)  # noqa: E731
        off = lambda: K.bam_to_consensus(path, primers=bed)  # noqa: E731
        on(), off()  # warm
        best = {"normalise": None, "primers": None}
        for _ in range(rounds):
            for key, fn in (("normalise", on), ("primers", off)):
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
    return {"consensus_normalise_s": best["normalise"], "consensus_primers_s": best["primers"],
            "reads": int(sub.n_reads), "amplicons": len(rows) // 2, "cap": CAP,
            "note": "bam_to_consensus(path, primers=bed, normalise=%d) vs bam_to_consensus(path, primers=bed), best of "
                    "%d, alternating" % (CAP, rounds)}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import engine, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = gpu_info()
    batch = bench.gen_reads(WORKLOAD)
    db = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    calls_buf = torch.empty(batch.n_slots, dtype=torch.uint8, device=dev)

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
    cfg = dict(reads=int(batch.n_reads), complex=int(batch.n_complex), aligned=int(batch.aligned_bases))
    del db, table, batch
    torch.cuda.empty_cache()
    print("step timed: %.4f ms" % (tm["total_ms"] / tm["reps"]), file=sys.stderr, flush=True)
    out = {}
    for name, (seed, length, depth) in (("cfg4_amplicon", (4, 5_000_000, 200)), ("deep_30kb", (5, 30_000, 5000))):
        amp, rows = synth.amplicon_reads(seed, length, depth)
        out[name] = normalise_workload(synth.with_strands(amp, seed), rows, torch, dev)
        del amp
        torch.cuda.empty_cache()
    print("timing bam_to_consensus with normalise", file=sys.stderr, flush=True)
    e2e_line = e2e()
    parity = all(v[1]["parity"] for v in out.values())
    ms_per_step = tm["total_ms"] / tm["reps"]
    line = {
        "metric": bench.METRIC, "value": cfg["aligned"] / (ms_per_step * 1e-3), "unit": bench.UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": parity, "parity_detail": {k: v[1] for k, v in out.items()},
        "config": {"workload": WORKLOAD, "reads_per_rank": cfg["reads"], "complex_reads_per_rank": cfg["complex"],
                   "aligned_bases_total": cfg["aligned"], "cap": CAP, "tool": "tools/bench_normalise.py",
                   "parity_oracle": "oracle/py_noracle.py (keep_vectorised over py_aoracle.labels_of_batch)"},
        "gpu": gpu, "normalise_ms": {k: v[0] for k, v in out.items()}, "e2e_normalise": e2e_line, "e2e": None,
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
