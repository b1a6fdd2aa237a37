"""Bench line of the per-base consensus qualities (an extension): BASELINE.json configs[3] (`cfg4_5Mb_200x`, as
bench.py builds it), bench.py's single-GPU step, then the qualities of its last table.

    python tools/bench_fastq.py [--steps K] [--warmup W]      # one JSON line on stdout

The timed step is bench.py's -- a fresh pileup into a reused CountTable (K0 + K1 + K1w) and the majority vote -- over
exactly K back-to-back steps with CUDA events.  On top of bench.py's fields the line carries:
  `qual_ms`      K2q (kdl_consensus_qual) against K2 (kdl_vote) over the last step's table and calls, alternating
                 for `rounds` rounds of `launches_per_timing` back-to-back launches;
  `assemble_ms`  K5 (kdl_assemble) against K5 + K5q (kdl_assemble_qual) over the same calls, alternating likewise;
  `e2e_qualities` bam_to_consensus(path, qualities=True) against qualities=False on a 10^6-read BAM of the workload's
                 shape (the file bench.py's host block times), best of 3 each, alternating;
  `parity`       the sha256 of the K2q bytes equals that of oracle/kindel_fqoracle.c over the C oracle's table and
                 vote, and the step's call bytes equal the C oracle's.
`e2e` is null: the host-buffer call (kdl_ctx_consensus) has no qualities.  Writes nothing into the tree."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload generator, step timer and clock sampler of the main bench)

WORKLOAD = "cfg4_5Mb_200x"


def alternate(named, torch, rounds=7, reps=20):
    """(name, fn) pairs timed in alternating rounds of `reps` launches: min / median / max ms per launch."""
    for _ in range(3):
        for _, fn in named:
            fn()
    torch.cuda.synchronize()
    ms = {name: [] for name, _ in named}
    for _ in range(rounds):
        for name, fn in named:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / reps)
    out = {"rounds": rounds, "launches_per_timing": reps}
    for name, v in ms.items():
        out[name] = {"min": min(v), "median": statistics.median(v), "max": max(v)}
    return out


def time_assemble(lib, calls, batch, torch):
    """K5 with and without K5q over the step's calls.  The inserted strings are host work resolved before either
    launch, so both variants are timed with an empty list of them."""
    dev = calls.device
    n = int(calls.shape[0])
    t_slot = torch.from_numpy(np.asarray(batch.contig_slot, dtype=np.int64)).to(dev)
    t_len = torch.from_numpy(np.asarray(batch.contig_len, dtype=np.int32)).to(dev)
    t_is = torch.zeros(1, dtype=torch.int64, device=dev)
    t_io = torch.zeros(2, dtype=torch.int32, device=dev)
    t_ib = torch.zeros(1, dtype=torch.uint8, device=dev)
    t_iq = torch.zeros(1, dtype=torch.uint8, device=dev)
    sums = torch.empty(int(lib.kdl_assemble_scratch_words(n)), dtype=torch.int32, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int32, device=dev)
    out = torch.empty(n + 16, dtype=torch.uint8, device=dev)
    qout = torch.empty(n + 16, dtype=torch.uint8, device=dev)
    qual = torch.zeros(n, dtype=torch.uint8, device=dev)
    st = int(torch.cuda.current_stream(dev).cuda_stream)

    def k5():
        lib.kdl_assemble(calls.data_ptr(), n, t_slot.data_ptr(), t_len.data_ptr(), batch.n_contigs, t_is.data_ptr(),
                         t_io.data_ptr(), t_ib.data_ptr(), 0, sums.data_ptr(), offsets.data_ptr(), out.data_ptr(), st)

    def k5q():
        k5()
        lib.kdl_assemble_qual(offsets.data_ptr(), qual.data_ptr(), n, t_is.data_ptr(), t_iq.data_ptr(), 0,
                              qout.data_ptr(), st)

    return alternate((("k5", k5), ("k5_k5q", k5q)), torch)


def e2e_qualities(path_rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub = synth.simple_reads(4, [750_000], 200)  # 10^6 reads, as bench.py's host block
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "slice.bam")
        synth.write_simple_bam(path, sub)
        K.bam_to_consensus(path, qualities=True)  # warm
        best = {"off": None, "on": None}
        for _ in range(path_rounds):
            for key, q in (("off", False), ("on", True)):
                t0 = time.perf_counter()
                res = K.bam_to_consensus(path, qualities=q)
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
        n_bases = sum(len(c.sequence) for c in res.consensuses)
        assert all(len(c.qualities) == len(c.sequence) for c in res.consensuses)
    return {"qualities_off_s": best["off"], "qualities_on_s": best["on"], "reads": int(sub.n_reads),
            "consensus_bases": n_bases, "note": "bam_to_consensus(path[, qualities=True]), best of %d, alternating"
            % path_rounds}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import _ffi, engine
    from oracle import coracle, fqoracle

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _ffi.load()
    sampler = bench.ClockSampler(0)
    sampler.start()
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

    sampler.wait_first_sample()
    launches0 = lib.kdl_launch_count()
    sampler.mark()
    tm = bench.time_steps(step, args.steps, args.warmup, torch, None, 1, dev)
    launches = lib.kdl_launch_count() - launches0
    clocks = sampler.stop()
    calls_dev = tm["out"]
    qual = engine.consensus_qual(table.t, calls_dev)
    q_host = qual.cpu().numpy()
    calls = calls_dev.cpu().numpy()
    vote_buf = torch.empty(n_slots, dtype=torch.uint8, device=dev)
    qual_ms = alternate((("k2_vote", lambda: engine.vote(table.t, 1, out=vote_buf)),
                         ("k2q_qual", lambda: engine.consensus_qual(table.t, calls_dev))), torch)
    k2q_bytes = n_slots * 18  # four int32 columns and the call byte in, one Q byte out per slot
    med = qual_ms["k2q_qual"]["median"]
    qual_ms.update(bytes_per_launch=k2q_bytes, k2q_gbs_at_median=k2q_bytes / (med * 1e-3) / 1e9)
    assemble_ms = time_assemble(lib, calls_dev, batch, torch)
    e2e_q = e2e_qualities()

    want_counts, _ = coracle.pileup(batch)
    want_calls = coracle.vote(want_counts, 1)
    want = hashlib.sha256(fqoracle.qual(want_counts, want_calls).tobytes()).hexdigest()
    got = hashlib.sha256(q_host.tobytes()).hexdigest()
    parity = got == want and np.array_equal(calls, want_calls)
    ms_per_step = tm["total_ms"] / tm["reps"]
    k1_bytes, k2_bytes = bench.algorithmic_bytes(batch)
    peak, peak_src = bench.measured_peak()
    achieved = k1_bytes / (tm["k1_ms"] * 1e-3) / 1e9
    launches_per_step = launches / (args.warmup + tm["reps"])
    hist = np.bincount(q_host, minlength=61)

    line = {
        "metric": bench.METRIC, "value": batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": bool(parity),
        "config": {"workload": WORKLOAD, "reads_per_rank": int(batch.n_reads),
                   "complex_reads_per_rank": int(batch.n_complex), "aligned_bases_total": int(batch.aligned_bases),
                   "tool": "tools/bench_fastq.py",
                   "parity_oracle": "oracle/kindel_fqoracle.c over oracle/kindel_oracle.c's table and vote"},
        "roofline": {"bound": "hbm", "kernel": "K0 tile index + K1 tile-owner pileup", "achieved": achieved,
                     "peak": peak, "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
                     "algorithmic_bytes_per_launch": k1_bytes, "kernel_ms": tm["k1_ms"]},
        "kernels_ms": {"k0_k1_pileup": tm["k1_ms"], "k2_vote_or_exchange": tm["k2_ms"],
                       "k2_vote_gbs": k2_bytes / (tm["k2_ms"] * 1e-3) / 1e9 if tm["k2_ms"] else None},
        "qualities": True, "qual_ms": qual_ms, "assemble_ms": assemble_ms, "e2e_qualities": e2e_q,
        "qual_sha256": got, "qual_q0_q20_q30_q60": [int(hist[0]), int(hist[20]), int(hist[30]), int(hist[60])],
        "e2e": None, "gpu_launches": int(round(launches_per_step * args.steps)),
        "gpu_launches_per_step": launches_per_step, "clocks": clocks,
        "gpu": {"name": torch.cuda.get_device_name(dev), "count": 1,
                "power_limit_w": clocks.get("power_limit_w") if clocks else None},
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
