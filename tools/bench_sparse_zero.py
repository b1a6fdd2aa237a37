"""What zeroing columns 5..18 of a reused count table costs, and what the dirty-sector map saves: BASELINE.json
configs[3] (`cfg4_5Mb_200x`, as bench.py builds it) and its all-simple twin.

    python tools/bench_sparse_zero.py [--out DIR] [--steps K] [--warmup W] [--rounds R]   # one JSON line on stdout

Three measurements, each in a run of its own:
  profile      per-kernel device time of bench.py's single-GPU step (K0, K1, K1w, K1g, K2) with torch.profiler (CUDA
               activities), ms per step; the trace goes to DIR/sparse_zero_step.pt.trace.json.
  zero_stores  K0 + K1 of the all-simple batch into a reused table with columns 5..18 zeroed in full
               (kdl_pileup_range, KDL_PILEUP_ZERO_REST, no map) against not zeroed at all: what the stores of a full
               zeroing cost K1, without K1w.
  map_ab       the cfg4 pileup (K0 + K1 + K1w) into one reused table, full zeroing (kdl_pileup_range) against the
               map's (kdl_pileup_range_map), alternating rounds of K back-to-back pileups, min / median / max ms per
               pileup; `bytes_zeroed_per_step` from the map's popcount (32 bytes per set bit) against the full 56 bytes
               per slot.
Each timing is CUDA events around K launches; the rounds alternate so that drift hits both sides alike.  The line
also carries bench.py's fields for the timed step (`ms_per_step`, `value`, `kernels_ms`, `parity`: the sha256 of the
step's call bytes against the C oracle's), so tools/results_table.py lists it.  `gpu` holds the device's name and
power limit, read in the same run.  Writes nothing into the tree."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload generator, step timer and clock sampler of the main bench)

WORKLOAD = "cfg4_5Mb_200x"
KERNELS = (("tile_index_kernel", "K0"), ("pileup_tile_kernel", "K1"), ("pileup_window_kernel", "K1w"),
           ("pileup_events_kernel", "K1e"), ("pileup_general_kernel", "K1g"), ("zero_cols_kernel", "zero"),
           ("vote_kernel", "K2"))


def stats(v):
    return {"min": min(v), "median": statistics.median(v), "max": max(v)}


def alternate(variants, reps, rounds, torch):
    """variants: name -> (prepare, run).  Per round and variant: prepare() untimed, then `reps` run() between two
    CUDA events.  Returns name -> stats of ms per run."""
    for prepare, run in variants.values():  # warm-up of every variant
        prepare()
        for _ in range(3):
            run()
    torch.cuda.synchronize()
    ms = {name: [] for name in variants}
    for _ in range(rounds):
        for name, (prepare, run) in variants.items():
            prepare()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / reps)
    return {name: stats(v) for name, v in ms.items()}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="directory for the profiler trace (default: a temporary one)")
    ap.add_argument("--steps", type=int, default=20, help="steps profiled / pileups per timing")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args(argv)
    out_dir = args.out or tempfile.mkdtemp(prefix="kdl_sparse_zero_")
    os.makedirs(out_dir, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile

    from kindel_b200 import _ffi, engine
    from oracle import coracle

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _ffi.load()
    stream = lambda: int(torch.cuda.current_stream(dev).cuda_stream)  # noqa: E731
    sampler = bench.ClockSampler(0)
    sampler.start()

    # ---- profile of bench.py's step
    batch, _, _ = bench.make_workload(WORKLOAD)
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
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    trace = os.path.join(out_dir, "sparse_zero_step.pt.trace.json")
    prof.export_chrome_trace(trace)
    per = {}
    for e in prof.key_averages():
        for key, short in KERNELS:
            if key in e.key and e.device_time_total > 0:
                per[short] = per.get(short, 0.0) + e.device_time_total / 1e3 / args.steps
    want, _ = coracle.pileup(batch)
    parity = bool(np.array_equal(tm["out"].cpu().numpy(), coracle.vote(want, 1)))
    ms_per_step = tm["total_ms"] / tm["reps"]
    line = {"metric": bench.METRIC, "value": batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
            "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]), "parity": parity,
            "config": {"workload": WORKLOAD, "reads_per_rank": int(batch.n_reads),
                       "complex_reads_per_rank": int(batch.n_complex), "aligned_bases_total": int(batch.aligned_bases),
                       "tool": "tools/bench_sparse_zero.py", "rounds": args.rounds},
            "kernels_ms": {"k0_k1_pileup": tm["k1_ms"], "k2_vote_or_exchange": tm["k2_ms"]},
            "roofline": None, "e2e": None}
    line["profile_ms_per_step"] = per
    line["trace"] = os.path.basename(trace)  # (in --out)

    # ---- map A/B on the cfg4 table
    ev = db.tensors["_events"].data_ptr()
    flag = db.tensors["_flag"].data_ptr()
    fresh_zero = _ffi.KDL_PILEUP_FRESH_WEIGHTS | _ffi.KDL_PILEUP_ZERO_REST
    cptr = table.t.data_ptr()

    def full_zeroing():
        _ffi.check(lib.kdl_pileup_range(C.byref(db.struct), cptr, n_slots, 0, n_slots, fresh_zero, ev, flag,
                                        stream()), "kdl_pileup_range")

    def by_map():
        _ffi.check(lib.kdl_pileup_range_map(C.byref(db.struct), cptr, n_slots, 0, n_slots, fresh_zero,
                                            table.dirty_map.data_ptr(), ev, flag, stream()), "kdl_pileup_range_map")

    def map_valid():  # full zeroing marks nothing: every sector counts as dirty, one map pileup rebuilds the map
        table.dirty_map.fill_(-1)
        by_map()

    line["map_ab"] = alternate({"full_zeroing": (lambda: None, full_zeroing), "dirty_map": (map_valid, by_map)},
                               args.steps, args.rounds, torch)
    map_valid()
    torch.cuda.synchronize()
    words = table.dirty_map.cpu().numpy().view(np.uint32)
    set_bits = int(np.unpackbits(words.view(np.uint8)).sum())
    line["bytes_zeroed_per_step"] = {"dirty_map": set_bits * 32, "full_zeroing": 14 * 4 * int(n_slots),
                                     "sector_share": set_bits / (14 * 8 * (len(words) // 4))}
    line["parity_after_ab"] = bool(np.array_equal(table.t.cpu().numpy(), want))
    del db, table, want

    # ---- the stores of a full zeroing on the all-simple batch (no K1w)
    simple, _, _ = bench.make_workload("cfg4_5Mb_200x_simple")
    sdb = engine.upload(simple, dev)
    st = engine.CountTable(simple.n_slots, dev)
    sflag = torch.zeros(4, dtype=torch.int32, device=dev)

    def simple_pileup(flags):
        return lambda: _ffi.check(lib.kdl_pileup_range(C.byref(sdb.struct), st.t.data_ptr(), simple.n_slots, 0,
                                                       simple.n_slots, flags, None, sflag.data_ptr(), stream()),
                                  "kdl_pileup_range")

    line["zero_stores"] = alternate({"zero_rest_on": (lambda: None, simple_pileup(fresh_zero)),
                                     "zero_rest_off": (lambda: None, simple_pileup(_ffi.KDL_PILEUP_FRESH_WEIGHTS))},
                                    args.steps, args.rounds, torch)
    line["zero_stores"]["cost_ms_at_median"] = (line["zero_stores"]["zero_rest_on"]["median"] -
                                                line["zero_stores"]["zero_rest_off"]["median"])
    clocks = sampler.stop()
    line["clocks"] = clocks
    line["gpu"] = {"name": torch.cuda.get_device_name(dev),
                   "power_limit_w": clocks.get("power_limit_w") if clocks else None}
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
