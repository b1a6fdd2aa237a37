"""Bench line of the device selection of variant sites (K6, `variants --only-variants` and `--vcf`; an extension):
BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds it), bench.py's single-GPU step, then K6 over its last
table.

    python tools/bench_variants.py [--steps K] [--warmup W]      # one JSON line on stdout

The timed step is bench.py's -- a fresh pileup into a reused CountTable (K0 + K1 + K1w) and the majority vote -- over
exactly K back-to-back steps with CUDA events.  On top of bench.py's fields the line carries:
  `variant_ms`   K6's three launches (kdl_variant_count + kdl_variant_scatter) against K2 (kdl_vote) over the last
                 step's table, alternating for `rounds` rounds of `launches_per_timing` back-to-back launches, at
                 rel_threshold 0.01 and 0.2 (abs_threshold 1), with the number of sites at each;
  `e2e_variants` variants_from_run(run, only_variants=True) on a device run (K6, only the sites copied back) against
                 the previous host-copy path (the whole 19-column table copied back, a frame of every position, then
                 filtered), both after the same pileup of a 10^6-read BAM of the workload's shape, best of 3 each,
                 alternating; and `variants(path, only_variants=True)` end to end;
  `parity`       the sha256 of K6's site arrays equals that of the numpy helper's (kindel.variant_sites over the
                 host copy of the table) at both thresholds, the two e2e frames are equal, and the step's call bytes
                 equal the C oracle's.
`e2e` is null: the host-buffer call (kdl_ctx_consensus) has no variant output.  Writes nothing into the tree."""
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

import bench  # noqa: E402  (the workload generator, step timer and clock sampler of the main bench)
from bench_fastq import alternate  # noqa: E402  (the alternating CUDA-event timer of the qualities bench)

WORKLOAD = "cfg4_5Mb_200x"
THRESHOLDS = ((1, 0.01), (1, 0.2))


def _sha(sites) -> str:
    h = hashlib.sha256()
    for a in sites:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def host_copy_only_variants(run, abs_threshold=1, rel_threshold=0.01, absolute=False):
    """The previous `variants_from_run(..., only_variants=True)`: the whole table copied back, a frame of every
    position, then the variant rows kept."""
    import pandas as pd

    from kindel_b200 import kindel as K

    tab = run.counts.cpu().numpy()
    frames = []
    for c, chrom in enumerate(run.batch.contig_names):
        s, e = run.contig_slice(c)
        L = e - s - 1
        t = tab[[0, 1, 2, 3, 4, 5], s:s + L].astype(np.int64)
        depth, top, share, is_var = K.variant_alleles(t, abs_threshold, rel_threshold)
        value = np.where(is_var, t if absolute else np.round(share, 4), 0)
        df = pd.DataFrame({"chrom": [chrom] * L, "pos": np.arange(1, L + 1, dtype=np.int64), "depth": depth,
                           "consensus": np.where(depth > 0, np.array(list("ACGTN-"))[top], "N")})
        for k, a in enumerate(["A", "C", "G", "T", "N", "deletions"]):
            df[a] = value[k]
        frames.append(df[is_var.any(axis=0)])
    return pd.concat(frames, ignore_index=True)


def e2e_variants(rounds=3):
    import pandas as pd

    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub = synth.simple_reads(4, [750_000], 200)  # 10^6 reads, as bench.py's host block
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "slice.bam")
        synth.write_simple_bam(path, sub)
        run = K.pileup_run(path)[0]
        K.variants_from_run(run, only_variants=True)  # warm
        host_copy_only_variants(run)
        best = {"device": None, "host_copy": None, "e2e": None}
        for _ in range(rounds):
            for key, fn in (("device", lambda: K.variants_from_run(run, only_variants=True)),
                            ("host_copy", lambda: host_copy_only_variants(run)),
                            ("e2e", lambda: K.variants(path, only_variants=True))):
                t0 = time.perf_counter()
                df = fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
        dev, host = K.variants_from_run(run, only_variants=True), host_copy_only_variants(run)
        try:
            pd.testing.assert_frame_equal(dev, host)
            same = True
        except AssertionError:
            same = False
    return {"device_s": best["device"], "host_copy_s": best["host_copy"], "variants_path_s": best["e2e"],
            "rows": int(len(df)), "frames_equal": same, "reads": int(sub.n_reads),
            "note": "variants_from_run(run, only_variants=True) on a device run vs the host-copy path after the same "
                    "pileup, and variants(path, only_variants=True) end to end; best of %d, alternating" % rounds}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import _ffi, engine
    from kindel_b200 import kindel as K
    from oracle import coracle

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
    calls = tm["out"].cpu().numpy()

    # K6 over the last step's table, with every buffer allocated once
    t_slot = torch.from_numpy(np.asarray(batch.contig_slot, dtype=np.int64)).to(dev)
    t_len = torch.from_numpy(np.asarray(batch.contig_len, dtype=np.int32)).to(dev)
    sums = torch.empty(int(lib.kdl_variant_scratch_words(n_slots)), dtype=torch.int32, device=dev)
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    host_run = K.PileupRun.__new__(K.PileupRun)
    host_run.batch, host_run.counts, host_run._host_counts = batch, None, table.t.cpu().numpy()
    vote_buf = torch.empty(n_slots, dtype=torch.uint8, device=dev)
    variant_ms, parity_sites = {}, True
    for a, r in THRESHOLDS:
        sites = engine.variant_sites(table.t, batch.contig_slot, batch.contig_len, a, r)
        want = K.variant_sites(host_run, a, r)
        n = len(sites[0])
        parity_sites = parity_sites and _sha(sites) == _sha(want)
        o_slot = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        o_cnt = torch.empty((6, max(n, 1)), dtype=torch.int32, device=dev)
        o_mask = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        fl = engine.variant_abs_floor(a)

        def k6(a=fl, r=r, n=n, o_slot=o_slot, o_cnt=o_cnt, o_mask=o_mask):
            base = (table.t.data_ptr(), n_slots, t_slot.data_ptr(), t_len.data_ptr(), batch.n_contigs, a, r,
                    sums.data_ptr())
            lib.kdl_variant_count(*base, st)
            lib.kdl_variant_scatter(*base, n, o_slot.data_ptr(), o_cnt.data_ptr(), o_mask.data_ptr(), st)

        timing = alternate((("k2_vote", lambda: engine.vote(table.t, 1, out=vote_buf)), ("k6_variants", k6)), torch)
        k6_bytes = 2 * 24 * n_slots + n * 33  # columns 0-5 read by both passes, 33 B per site record
        timing.update(abs_threshold=a, rel_threshold=r, sites=n, sha256=_sha(sites), bytes_per_launch=k6_bytes,
                      k6_gbs_at_median=k6_bytes / (timing["k6_variants"]["median"] * 1e-3) / 1e9)
        variant_ms["rel_%g" % r] = timing
    e2e_v = e2e_variants()

    want_counts, _ = coracle.pileup(batch)
    want_calls = coracle.vote(want_counts, 1)
    parity = parity_sites and e2e_v["frames_equal"] and np.array_equal(calls, want_calls)
    ms_per_step = tm["total_ms"] / tm["reps"]
    k1_bytes, k2_bytes = bench.algorithmic_bytes(batch)
    peak, peak_src = bench.measured_peak()
    achieved = k1_bytes / (tm["k1_ms"] * 1e-3) / 1e9
    launches_per_step = launches / (args.warmup + tm["reps"])

    line = {
        "metric": bench.METRIC, "value": batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": bool(parity),
        "config": {"workload": WORKLOAD, "reads_per_rank": int(batch.n_reads),
                   "complex_reads_per_rank": int(batch.n_complex), "aligned_bases_total": int(batch.aligned_bases),
                   "tool": "tools/bench_variants.py",
                   "parity_oracle": "kindel.variant_sites (numpy) over the host copy of the table; the step's calls "
                                    "against oracle/kindel_oracle.c"},
        "roofline": {"bound": "hbm", "kernel": "K0 tile index + K1 tile-owner pileup", "achieved": achieved,
                     "peak": peak, "unit": "GB/s", "frac": achieved / peak, "peak_source": peak_src,
                     "algorithmic_bytes_per_launch": k1_bytes, "kernel_ms": tm["k1_ms"]},
        "kernels_ms": {"k0_k1_pileup": tm["k1_ms"], "k2_vote_or_exchange": tm["k2_ms"],
                       "k2_vote_gbs": k2_bytes / (tm["k2_ms"] * 1e-3) / 1e9 if tm["k2_ms"] else None},
        "variants": True, "variant_ms": variant_ms, "e2e_variants": e2e_v,
        "e2e": None, "gpu_launches": int(round(launches_per_step * args.steps)),
        "gpu_launches_per_step": launches_per_step, "clocks": clocks,
        "gpu": {"name": torch.cuda.get_device_name(dev), "count": 1,
                "power_limit_w": clocks.get("power_limit_w") if clocks else None},
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
