"""Bench line of the base-quality filter (an extension): BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds
it) with the seeded quality model of synth.qualities (~5 % of the bases below Q20, toward the 3' end), masked at
min_base_quality = 20.

    python tools/bench_quality.py [--steps K] [--warmup W]          # one JSON line on stdout

The timed step is bench.py's single-GPU step -- a fresh pileup into a reused CountTable (K0 + K1 + K1w + K1q) and the
vote -- over exactly K back-to-back steps with CUDA events.  On top of bench.py's fields the line carries a `quality`
block: the masked fraction, mask bytes per aligned base, K1q timed on its own (CUDA events, back-to-back launches into
a scratch copy of the table) and K0+K1 without it.  `parity`: the sha256 of the timed loop's call bytes equals that of
oracle/kindel_qoracle.c, which masks inside its own walk from the qualities (it never reads the engine's mask list).
`e2e`: kdl_ctx_consensus_masked from pinned host buffers, mask list included.  `host`: decode of a 10^6-read BGZF BAM
of the same shape with qualities from the same model, MAPQs / FLAGs from synth.mapq_flags, with the filters off and on.
Writes nothing into the tree."""
from __future__ import annotations

import argparse
import ctypes as C
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
MIN_BQ = 20
FILTERS = dict(min_base_quality=MIN_BQ, min_mapq=20, exclude_flags=0x900)


def host_decode(seed: int):
    """Decode of a 10^6-read BAM with qualities, MAPQs and FLAGs: filters off vs on (best of 3 each)."""
    import struct as S

    from kindel_b200 import bamio, synth

    sub = synth.simple_reads(4, [750_000], 200)
    qual = synth.qualities(seed, sub.seq_len)
    mapq, flag = synth.mapq_flags(seed + 1, sub.n_reads)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "slice.bam")
        synth.write_simple_bam(path, sub)
        # patch MAPQ, FLAG and QUAL into the uncompressed records and re-compress: write_simple_bam writes fixed ones
        raw = bamio.inflate_bam(path).copy()
        first = 12 + S.unpack_from("<i", raw, 4)[0]
        n_ref = S.unpack_from("<i", raw, first - 4)[0]
        off = first
        for _ in range(n_ref):
            off += 8 + S.unpack_from("<i", raw, off)[0]
        L = int(sub.seq_len[0])
        rec = raw[off:].reshape(sub.n_reads, -1)
        rec[:, 13] = mapq.astype(np.uint8)
        rec[:, 18:20] = flag.astype("<u2").view(np.uint8).reshape(-1, 2)
        rec[:, -L:] = qual.reshape(sub.n_reads, L)
        body = raw.tobytes()
        with open(path, "wb") as fh:
            for s in range(0, len(body), 65280):
                fh.write(bamio._bgzf_block(body[s:s + 65280], 1))
            fh.write(bamio._bgzf_block(b"", 1))

        def best(**kw):
            t = None
            for _ in range(3):
                t0 = time.perf_counter()
                b = bamio.read_bam(path, **kw)
                dt = time.perf_counter() - t0
                t = dt if t is None or dt < t else t
            return t, b

        t_off, b_off = best()
        t_on, b_on = best(**FILTERS)
    return {"bam_decode_s": t_off, "bam_decode_filtered_s": t_on, "reads": sub.n_reads,
            "kept_reads_filtered": b_on.n_reads, "masked_bases_filtered": b_on.n_masked,
            "filters": {k: (hex(v) if k == "exclude_flags" else v) for k, v in FILTERS.items()},
            "sample": "10^6 reads x 150 bp, BGZF level 1, C++ decoder with %d threads, best of 3" % bamio.decode_threads(),
            "cores": os.cpu_count()}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip the host decode timing")
    args = ap.parse_args(argv)

    import torch

    from kindel_b200 import _ffi, engine, synth
    from oracle import coracle, qoracle

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _ffi.load()
    sampler = bench.ClockSampler(0)
    sampler.start()
    plain = bench.gen_reads(WORKLOAD)
    batch, qual = synth.with_qualities(plain, 20, MIN_BQ)
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

    # K1q on its own, into a scratch copy of the table
    scratch = table.t.clone()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    stream = engine._stream_ptr(dev)
    _ffi.check(lib.kdl_unmask(C.byref(db.struct), C.byref(db.qmask), scratch.data_ptr(), n_slots, stream), "kdl_unmask")
    ev[0].record()
    for _ in range(args.steps):
        lib.kdl_unmask(C.byref(db.struct), C.byref(db.qmask), scratch.data_ptr(), n_slots, stream)
    ev[1].record()
    torch.cuda.synchronize()
    k1q_ms = ev[0].elapsed_time(ev[1]) / args.steps
    del scratch

    want_counts, _ = qoracle.pileup(plain, qual, MIN_BQ)
    want = hashlib.sha256(coracle.vote(want_counts, 1).tobytes()).hexdigest()
    got = hashlib.sha256(tm["out"].cpu().numpy().tobytes()).hexdigest()
    ms_per_step = tm["total_ms"] / tm["reps"]

    # e2e from pinned host buffers, the mask list included
    ctx = engine.HostContext(0)
    pin = {}
    for f in engine._FIELDS + engine._MASK_FIELDS:
        a = np.ascontiguousarray(getattr(batch, f))
        pin[f] = torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a).pin_memory() if a.size else None
    ptr = {f: (int(t.data_ptr()) if t is not None else None) for f, t in pin.items()}
    struct, qmask = engine.make_struct(batch, ptr), engine.make_qmask(batch, ptr)
    calls_np = torch.empty(n_slots, dtype=torch.uint8).pin_memory().numpy()
    rows = []
    for i in range(2 + 10):
        t0 = time.perf_counter()
        ctx.consensus(batch, 1, calls_out=calls_np, struct=struct, qmask=qmask)
        wall = (time.perf_counter() - t0) * 1e3
        t = ctx.last_timing()
        rows.append((t["h2d_ms"] + t["kernel_ms"] + t["d2h_ms"], wall, t))
    rows = rows[-10:]
    e2e_ms = statistics.mean(r[0] for r in rows)
    e2e = {"value": batch.aligned_bases / (e2e_ms * 1e-3), "unit": bench.UNIT, "ms_per_step": e2e_ms,
           "wall_ms_per_step": statistics.mean(r[1] for r in rows),
           "h2d_bytes_per_step": batch.input_bytes(), "d2h_bytes_per_step": int(n_slots) + 16,
           "breakdown_ms": {k: statistics.mean(r[2][k] for r in rows) for k in ("h2d_ms", "kernel_ms", "d2h_ms")},
           "parity": hashlib.sha256(calls_np.tobytes()).hexdigest() == want,
           "api": "kdl_ctx_consensus_masked (include/kindel_b200.h), pinned host buffers incl. the mask list"}
    ctx.close()

    line = {
        "metric": bench.METRIC, "value": batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT, "n_gpus": 1,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": got == want,
        "config": {"workload": WORKLOAD + "_q20", "reads_per_rank": int(batch.n_reads),
                   "complex_reads_per_rank": int(batch.n_complex), "aligned_bases_total": int(batch.aligned_bases),
                   "tool": "tools/bench_quality.py"},
        "kernels_ms": {"k0_k1_pileup": tm["k1_ms"], "k2_vote_or_exchange": tm["k2_ms"]},
        "quality": {"min_base_quality": MIN_BQ, "masked_bases": batch.n_masked, "masked_reads": batch.n_mask_reads,
                    "masked_fraction": batch.n_masked / batch.aligned_bases,
                    "mask_bytes_per_aligned_base": batch.mask_bytes() / batch.aligned_bases,
                    "k1q_ms": k1q_ms, "k0_k1_ms_without_k1q": tm["k1_ms"] - k1q_ms,
                    "k1q_share_of_k0_k1": k1q_ms / max(tm["k1_ms"] - k1q_ms, 1e-9),
                    "parity_oracle": "oracle/kindel_qoracle.c (masks inside its own walk, from the qualities)"},
        "e2e": e2e, "gpu_launches": int(round(launches / (args.warmup + tm["reps"]) * args.steps)),
        "clocks": clocks,
        "gpu": {"name": torch.cuda.get_device_name(dev), "count": 1,
                "power_limit_w": clocks.get("power_limit_w") if clocks else None},
    }
    if not args.no_host:
        line["host"] = host_decode(7)
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
