"""Bench line of the IUPAC vote (an extension): BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds it) with
the step's vote replaced by the IUPAC vote at threshold T (kdl_vote_iupac).

    python tools/bench_iupac.py [--threshold T] [--steps K] [--warmup W]      # one JSON line on stdout

The timed step is bench.py's single-GPU step -- a fresh pileup into a reused CountTable (K0 + K1 + K1w) and the vote --
over exactly K back-to-back steps with CUDA events.  On top of bench.py's fields the line carries `iupac_threshold`,
`mixed_sites` (call bytes with bit 7 set: multi-base IUPAC codes) and `vote_ms`: the majority vote (kdl_vote) and the
IUPAC vote over the last step's table, `launches_per_timing` back-to-back launches per timing, the two alternating
for `rounds` rounds.  `parity`: the sha256 of the timed loop's call bytes equals that of oracle/kindel_ioracle.c's
vote over the C oracle's table.  `e2e` is null: the host-buffer call (kdl_ctx_consensus) has no IUPAC vote.
Writes nothing into the tree."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload generator, step timer and clock sampler of the main bench)

WORKLOAD = "cfg4_5Mb_200x"


def time_votes(counts, threshold, torch, rounds=7, reps=20):
    """The majority vote and the IUPAC vote over the same table, alternating: min / median / max ms per launch."""
    from kindel_b200 import engine

    buf = torch.empty(counts.shape[1], dtype=torch.uint8, device=counts.device)
    votes = (("majority", None), ("iupac", threshold))
    for _ in range(3):
        for _, t in votes:
            engine.vote(counts, 1, out=buf, iupac_threshold=t)
    torch.cuda.synchronize()
    ms = {name: [] for name, _ in votes}
    for _ in range(rounds):
        for name, t in votes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                engine.vote(counts, 1, out=buf, iupac_threshold=t)
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / reps)
    n_bytes = int(counts.shape[1]) * 29  # 7 int32 columns in, 1 call byte out per slot
    out = {"rounds": rounds, "launches_per_timing": reps, "bytes_per_launch": n_bytes}
    for name, v in ms.items():
        med = statistics.median(v)
        out[name] = {"min": min(v), "median": med, "max": max(v), "gbs_at_median": n_bytes / (med * 1e-3) / 1e9}
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--threshold", type=float, default=0.99)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)
    if not 0.0 <= args.threshold <= 1.0:
        ap.error("--threshold must lie in [0, 1]")

    import torch

    from kindel_b200 import _ffi, engine
    from oracle import coracle, ioracle

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
        out = engine.vote(table.t, 1, out=calls_buf, iupac_threshold=args.threshold)
        if timers:
            timers[2].record()
        return out

    sampler.wait_first_sample()
    launches0 = lib.kdl_launch_count()
    sampler.mark()
    tm = bench.time_steps(step, args.steps, args.warmup, torch, None, 1, dev)
    launches = lib.kdl_launch_count() - launches0
    clocks = sampler.stop()
    calls = tm["out"].cpu().numpy()
    vote_ms = time_votes(table.t, args.threshold, torch)

    want_counts, _ = coracle.pileup(batch)
    want = hashlib.sha256(ioracle.vote_iupac(want_counts, 1, args.threshold).tobytes()).hexdigest()
    got = hashlib.sha256(calls.tobytes()).hexdigest()
    ms_per_step = tm["total_ms"] / tm["reps"]
    k1_bytes, k2_bytes = bench.algorithmic_bytes(batch)
    peak, peak_src = bench.measured_peak()
    achieved = k1_bytes / (tm["k1_ms"] * 1e-3) / 1e9
    launches_per_step = launches / (args.warmup + tm["reps"])

    line = {
        "metric": bench.METRIC, "value": batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": got == want,
        "config": {"workload": WORKLOAD, "reads_per_rank": int(batch.n_reads),
                   "complex_reads_per_rank": int(batch.n_complex), "aligned_bases_total": int(batch.aligned_bases),
                   "tool": "tools/bench_iupac.py",
                   "parity_oracle": "oracle/kindel_ioracle.c over oracle/kindel_oracle.c's table"},
        "roofline": {"bound": "hbm", "kernel": "K0 tile index + K1 tile-owner pileup", "achieved": achieved,
                     "peak": peak, "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
                     "algorithmic_bytes_per_launch": k1_bytes, "kernel_ms": tm["k1_ms"]},
        "kernels_ms": {"k0_k1_pileup": tm["k1_ms"], "k2_vote_or_exchange": tm["k2_ms"],
                       "k2_vote_gbs": k2_bytes / (tm["k2_ms"] * 1e-3) / 1e9 if tm["k2_ms"] else None},
        "iupac_threshold": args.threshold, "mixed_sites": int(np.count_nonzero(calls & 0x80)), "vote_ms": vote_ms,
        "e2e": None, "gpu_launches": int(round(launches_per_step * args.steps)),
        "gpu_launches_per_step": launches_per_step, "clocks": clocks,
        "gpu": {"name": torch.cuda.get_device_name(dev), "count": 1,
                "power_limit_w": clocks.get("power_limit_w") if clocks else None},
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
