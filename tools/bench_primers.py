"""Bench line of amplicon primer masking (`--primers`, K9; an extension): bench.py's single-GPU step over
BASELINE.json configs[3] (`cfg4_5Mb_200x`, as bench.py builds it), then K9 and K1q over two workloads:

  cfg4       the step's batch with a synthetic tiled scheme (synth.tiled_scheme: 22-30 bp primers, one pair per
             ~200 bp, both rows of each pair); uniform read starts put only a fraction of the reads in a primer
  amplicon   synth.amplicon_reads at the same size: every read starts at a left primer or ends at a right one

    python tools/bench_primers.py [--steps K] [--warmup W]      # one JSON line on stdout

On top of bench.py's fields the line carries, per workload (`primers`):
  `ms`        K9 alone (kdl_primers_count + kdl_primers_apply over outputs allocated once: count, two scans, totals,
              scatter), K1q over the merged mask list, and K0 + K1 (the pileup into a reused table) for scale, in 7
              alternating rounds of 20 launches;
  masked reads and bases, and the bytes K9 reads (the batch's per-read words, the CIGARs of complex reads) and writes;
  `parity`    the masked run's table has the sha256 of oracle/py_poracle.py's (per-record rule, the C quality walk).
`e2e` times bam_to_consensus(path, primers=bed) against bam_to_consensus(path) on a 10^6-read BAM, best of 3,
alternating; `gpu` is the card's name and power limit, read in the same run.  Writes nothing into the tree."""
from __future__ import annotations

import argparse
import ctypes as C
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
from bench_fastq import alternate  # noqa: E402
from bench_variants_ref import gpu_info  # noqa: E402

WORKLOAD = "cfg4_5Mb_200x"
SCHEME_SEED = 1


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def primer_workload(batch, rows, torch, dev):
    from kindel_b200 import _ffi, engine, primers
    from oracle import py_poracle

    lib = _ffi.load()
    ps = primers.read_bed("".join("%s\t%d\t%d\n" % r for r in rows).encode(), "scheme.bed")
    arrays = primers.primer_arrays(ps, batch.contig_names, batch.contig_len)
    plain = engine.upload(batch, dev)
    table = engine.CountTable(batch.n_slots, dev)
    masked = engine.mask_primers(engine.upload(batch, dev), arrays)
    got = engine.pileup(masked)[0].cpu().numpy()
    st = int(torch.cuda.current_stream(dev).cuda_stream)
    t = {f: torch.from_numpy(np.ascontiguousarray(getattr(arrays, f))).to(dev)
         for f in ("contig_off", "start_sorted", "end_max", "end_sorted", "start_min")}
    p = engine.primers_struct(arrays, {f: int(x.data_ptr()) for f, x in t.items()})
    scratch = torch.empty(int(lib.kdl_primers_scratch_words(batch.n_reads)), dtype=torch.int32, device=dev)

    # K9 again over the masked batch (the same nibbles: N stays N) into outputs of the same size, with the decode's
    # mask list (none here) as its input
    assert batch.n_masked == 0
    q = masked.qmask
    out = [torch.empty(k, dtype=torch.int32, device=dev) for k in (q.n_reads, q.n_reads + 1, q.n_bases)]
    om = _ffi.KdlQmask(q.n_reads, q.n_bases, *(int(x.data_ptr()) for x in out))

    def k9():
        base = (C.byref(masked.struct), None, C.byref(p), scratch.data_ptr())
        lib.kdl_primers_count(*base, st)
        lib.kdl_primers_apply(*base, int(masked.tensors["seq4"].data_ptr()), C.byref(om), st)

    scratch_table = torch.zeros((_ffi.KDL_NCOL, batch.n_slots), dtype=torch.int32, device=dev)
    timing = alternate((("k0_k1_pileup", lambda: engine.pileup(plain, check=False, table=table)), ("k9_primers", k9),
                        ("k1q_unmask", lambda: lib.kdl_unmask(C.byref(masked.struct), C.byref(masked.qmask),
                                                              scratch_table.data_ptr(), batch.n_slots, st))), torch)
    again = engine.pileup(masked)[0].cpu().numpy()  # the batch the timed K9 launches rewrote, piled again
    n_pr, n_pb = masked.primer_masked
    cx_words = int(sum(2 + int(batch.cig_off[r + 1] - batch.cig_off[r]) for r in np.asarray(batch.complex_idx)))
    timing.update(reads=int(batch.n_reads), masked_reads=int(n_pr), masked_bases=int(n_pb), intervals=len(rows),
                  k9_bytes_read=int(2 * (12 * batch.n_reads + 4 * cx_words)),  # count and scatter each
                  k9_bytes_written=int(4 * (2 * n_pr + 1 + n_pb) + 4 * n_pb),  # the list; a word per masked base, at most
                  note="k9_primers: the two entry points over preallocated outputs, no read-back; k1q_unmask: kdl_unmask "
                       "of the merged list into a scratch table; k0_k1_pileup: engine.pileup into a reused CountTable")
    print("primers: timed %d reads, checking against the oracle" % batch.n_reads, file=sys.stderr, flush=True)
    masked_ref = py_poracle.masked_arrays(batch, rows)
    print("primers: the oracle's %d masked bases, its pileup" % int(masked_ref[0].sum()), file=sys.stderr, flush=True)
    want = py_poracle.pileup(batch, masked_ref)[0]
    return timing, {"table_sha256": sha(got), "oracle_sha256": sha(want),
                    "parity": bool(sha(got) == sha(want) == sha(again))}


def e2e(rounds=3):
    from kindel_b200 import kindel as K
    from kindel_b200 import synth

    sub = synth.simple_reads(4, [750_000], 200)  # 10^6 reads, as bench.py's host block
    rows = synth.tiled_scheme(SCHEME_SEED, sub.contig_names, sub.contig_len)
    with tempfile.TemporaryDirectory() as tmp:
        path, bed = os.path.join(tmp, "slice.bam"), os.path.join(tmp, "scheme.bed")
        synth.write_simple_bam(path, sub)
        with open(bed, "w") as fh:
            fh.write("".join("%s\t%d\t%d\n" % r for r in rows))
        K.bam_to_consensus(path, primers=bed), K.bam_to_consensus(path)  # warm
        best = {"primers": None, "plain": None}
        for _ in range(rounds):
            for key, fn in (("primers", lambda: K.bam_to_consensus(path, primers=bed)),
                            ("plain", lambda: K.bam_to_consensus(path))):
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                best[key] = dt if best[key] is None or dt < best[key] else best[key]
    return {"primers_s": best["primers"], "plain_s": best["plain"], "reads": int(sub.n_reads), "intervals": len(rows),
            "note": "bam_to_consensus(path, primers=bed) vs bam_to_consensus(path), best of %d, alternating" % rounds}


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
    del db, table
    out = {}
    rows = synth.tiled_scheme(SCHEME_SEED, batch.contig_names, batch.contig_len)
    print("step timed: %.4f ms" % (tm["total_ms"] / tm["reps"]), file=sys.stderr, flush=True)
    out["cfg4"] = primer_workload(batch, rows, torch, dev)
    del batch
    torch.cuda.empty_cache()
    amp, amp_rows = synth.amplicon_reads(4, 5_000_000, 200)
    out["amplicon"] = primer_workload(amp, amp_rows, torch, dev)
    aligned = int(amp.aligned_bases)
    del amp
    torch.cuda.empty_cache()
    print("timing bam_to_consensus", file=sys.stderr, flush=True)
    e2e_line = e2e()
    parity = all(v[1]["parity"] for v in out.values())
    ms_per_step = tm["total_ms"] / tm["reps"]
    cfg_batch = bench.gen_reads(WORKLOAD)  # (only its sizes, for the config block)
    line = {
        "metric": bench.METRIC, "value": cfg_batch.aligned_bases / (ms_per_step * 1e-3), "unit": bench.UNIT,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
        "dtype": "int32", "data": "synthetic", "steps_timed": tm["reps"], "step_ms": bench.quantiles(tm["step_ms"]),
        "parity": parity, "parity_detail": {k: v[1] for k, v in out.items()},
        "config": {"workload": WORKLOAD, "reads_per_rank": int(cfg_batch.n_reads),
                   "complex_reads_per_rank": int(cfg_batch.n_complex),
                   "aligned_bases_total": int(cfg_batch.aligned_bases), "amplicon_aligned_bases": aligned,
                   "scheme_seed": SCHEME_SEED, "tool": "tools/bench_primers.py",
                   "parity_oracle": "oracle/py_poracle.py (per-record primer rule) over oracle/kindel_qoracle.c"},
        "gpu": gpu, "primers_ms": {k: v[0] for k, v in out.items()}, "e2e_primers": e2e_line, "e2e": None,
    }
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
